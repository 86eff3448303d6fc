"""Build the REFERENCE's bilateral-grid kernels and its BilateralGrid component for the GPU box (SURVEY.md 8 f5).

  oracle/_ref/libbilagrid_ref.so      the reference's src/training/kernels/bilateral_grid_{forward,backward,tv}.cu,
                                      compiled unmodified from where they lie with the reference's flags
                                      (src/training/CMakeLists.txt:76: -O3 -use_fast_math) for plain sm_90, plus
                                      oracle/ref_bilagrid_binding.cpp: torch.ops.bilagrid_ref.*
  oracle/_ref/libref_bilagrid_b200.so the reference's src/training/components/bilateral_grid.cpp, unmodified, linked
                                      against THIS repository's drop-in library (include/kernels/bilateral_grid.cuh),
                                      plus oracle/ref_bilagrid_harness.cpp: torch.ops.bilagrid_component.*

Both outputs are git-ignored test infrastructure.  Runs only where the reference's sources are present; a separate
recipe from build_ref.py so that the existing reference libraries and their stamps stay as they are."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

from .build_ref import CUDA_INC, CXX, HOST_FLAGS, NVCC, OUT

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_TRAIN = "/root/reference/src/training"
KERNELS = [os.path.join(REF_TRAIN, "kernels", f) for f in
           ("bilateral_grid_forward.cu", "bilateral_grid_backward.cu", "bilateral_grid_tv.cu")]
REF_INC = "/root/reference/include"  # kernels/bilateral_grid.cuh (the reference's own header, for its kernels)
COMPONENT = os.path.join(REF_TRAIN, "components", "bilateral_grid.cpp")
BINDING = os.path.join(HERE, "ref_bilagrid_binding.cpp")
HARNESS = os.path.join(HERE, "ref_bilagrid_harness.cpp")


def kernels_available() -> bool:
    return os.path.exists(os.path.join(OUT, "libbilagrid_ref.so"))


def _stamp(files, extra="") -> str:
    h = hashlib.sha256(extra.encode())
    for f in files:
        h.update(open(f, "rb").read())
    return h.hexdigest()


def _fresh(so: str, st: str) -> bool:
    return os.path.exists(so) and os.path.exists(so + ".stamp") and open(so + ".stamp").read() == st


def _run(cmd, what):
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-6000:])
        raise RuntimeError(what)


def build_kernels(verbose: bool = True) -> str | None:
    if not all(os.path.exists(f) for f in KERNELS):
        return None
    from torch.utils import cpp_extension as ce

    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libbilagrid_ref.so")
    st = _stamp(KERNELS + [BINDING, os.path.join(REF_INC, "kernels", "bilateral_grid.cuh")])
    if _fresh(so, st):
        return so
    inc = []
    for i in [REF_INC] + ce.include_paths():
        inc += ["-I", i]
    nv = ["-O3", "-use_fast_math", "-std=c++20", "-Xcompiler", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-ccbin", CXX,
          "-gencode", "arch=compute_90,code=sm_90", "--expt-relaxed-constexpr", "-diag-suppress", "20012,20011,20014,177,550"]

    def compile_one(src):
        obj = os.path.join(OUT, "bg_" + os.path.basename(src).rsplit(".", 1)[0] + ".o")
        if verbose:
            print("[build_ref_bilagrid]", os.path.basename(src), flush=True)
        if src.endswith(".cpp"):
            cmd = [CXX, "-c", src, "-o", obj] + HOST_FLAGS + inc + ["-I", CUDA_INC]
        else:
            cmd = [NVCC, "-c", src, "-o", obj] + nv + inc
        _run(cmd, f"reference bilateral-grid source failed to compile: {src}")
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, KERNELS + [BINDING]))
    tl = ce.library_paths()[0]
    _run([NVCC, "-shared", "-o", so] + objs + ["-gencode", "arch=compute_90,code=sm_90", "-ccbin", CXX, "-L", tl, "-ltorch",
                                               "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda", "-Xlinker",
                                               "-rpath," + tl, "-Xlinker", "-Bsymbolic"],
         "linking oracle/_ref/libbilagrid_ref.so failed")
    for o in objs:
        os.remove(o)
    with open(so + ".stamp", "w") as f:
        f.write(st)
    return so


def build_component_harness(verbose: bool = True) -> str | None:
    if not os.path.exists(COMPONENT):
        return None
    from torch.utils import cpp_extension as ce

    lib_dir = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib")
    if not os.path.exists(os.path.join(lib_dir, "libgsplat_b200.so")):
        return None
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libref_bilagrid_b200.so")
    st = _stamp([COMPONENT, os.path.join(REF_TRAIN, "components", "bilateral_grid.hpp"), HARNESS,
                 os.path.join(ROOT, "include", "kernels", "bilateral_grid.cuh")])
    if _fresh(so, st):
        return so
    inc = []
    for i in [os.path.join(ROOT, "include"), os.path.join(REF_TRAIN, "components")] + ce.include_paths() + [CUDA_INC]:
        inc += ["-I", i]
    objs = []
    for src in (COMPONENT, HARNESS):
        obj = os.path.join(OUT, "bgc_" + os.path.basename(src).rsplit(".", 1)[0] + ".o")
        if verbose:
            print("[build_ref_bilagrid] component", os.path.basename(src), flush=True)
        _run([CXX, "-std=c++20", "-O2", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-c", src, "-o", obj] + inc,
             f"bilateral-grid harness source failed to compile: {src}")
        objs.append(obj)
    tl = ce.library_paths()[0]
    _run([CXX, "-shared", "-o", so] + objs + ["-L", lib_dir, "-lgsplat_b200", "-lgsb200", "-L", tl, "-ltorch",
                                              "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda", "-Wl,--no-undefined",
                                              "-Wl,-rpath,$ORIGIN/../../gaussian-splatting-cuda_b200/lib",
                                              "-Wl,-rpath," + tl],
         "linking oracle/_ref/libref_bilagrid_b200.so failed")
    for o in objs:
        os.remove(o)
    with open(so + ".stamp", "w") as f:
        f.write(st)
    return so


def build_all(verbose: bool = True) -> None:
    build_kernels(verbose)
    build_component_harness(verbose)


if __name__ == "__main__":
    build_all()
