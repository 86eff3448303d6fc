"""Build oracle/_ref/libref_knn.so: oracle/ref_knn_harness.cpp compiled against the reference's own nanoflann.hpp and
tinyply.hpp (include/external/), where the reference's sources are present.

  ref_knn_mean_dist   the reference's (approximate, eps = 10) neighbour query of compute_mean_neighbor_distances
  ref_write_ply       its PLY writer, write_ply_impl, through tinyply

Test and benchmark infrastructure only (git-ignored); a separate recipe from build_ref.py so that the existing
reference libraries and their stamps stay as they are.  load() returns the library through ctypes, or None."""
from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess
import sys

from .build_ref import CXX, OUT

HERE = os.path.dirname(os.path.abspath(__file__))
REF_EXT = "/root/reference/include/external"
HEADERS = [os.path.join(REF_EXT, "nanoflann.hpp"), os.path.join(REF_EXT, "tinyply.hpp")]
HARNESS = os.path.join(HERE, "ref_knn_harness.cpp")
SO = os.path.join(OUT, "libref_knn.so")
FLAGS = ["-O3", "-std=c++20", "-fPIC", "-fopenmp", "-shared"]


def build(verbose: bool = True) -> str | None:
    if not all(os.path.exists(h) for h in HEADERS):
        return None
    h = hashlib.sha256(" ".join(FLAGS).encode())
    for f in HEADERS + [HARNESS]:
        h.update(open(f, "rb").read())
    st = h.hexdigest()
    if os.path.exists(SO) and os.path.exists(SO + ".stamp") and open(SO + ".stamp").read() == st:
        return SO
    os.makedirs(OUT, exist_ok=True)
    if verbose:
        print("[build_ref_knn] ref_knn_harness.cpp", flush=True)
    p = subprocess.run([CXX] + FLAGS + ["-I", REF_EXT, HARNESS, "-o", SO], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-6000:])
        raise RuntimeError("oracle/ref_knn_harness.cpp failed to compile")
    with open(SO + ".stamp", "w") as f:
        f.write(st)
    return SO


def build_all(verbose: bool = True) -> None:
    build(verbose)


def load():
    """The built harness (ctypes), or None where it was not built."""
    if not os.path.exists(SO):
        return None
    lib = ctypes.CDLL(SO)
    lib.ref_knn_mean_dist.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.ref_write_ply.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p),
                                  ctypes.POINTER(ctypes.c_int), ctypes.c_char_p]
    return lib


def mean_dist(lib, points):
    """The reference's approximate mean neighbour distances of float32 points [N,3] (numpy)."""
    import numpy as np

    p = np.ascontiguousarray(points, np.float32)
    out = np.empty(p.shape[0], np.float32)
    lib.ref_knn_mean_dist(p.ctypes.data, p.shape[0], out.ctypes.data)
    return out


def write_ply(lib, path: str, groups: list, names: list) -> None:
    """groups: float32 arrays [rows, cols] in the order write_ply_impl adds them; names: all column names."""
    import numpy as np

    arrs = [np.ascontiguousarray(g, np.float32) for g in groups]
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    cols = (ctypes.c_int * len(arrs))(*[a.shape[1] for a in arrs])
    rc = lib.ref_write_ply(path.encode(), arrs[0].shape[0], len(arrs), ptrs, cols, "\n".join(names).encode())
    if rc != 0:
        raise RuntimeError(f"ref_write_ply failed ({rc})")


if __name__ == "__main__":
    print(build())
