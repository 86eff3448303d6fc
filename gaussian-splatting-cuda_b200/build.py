"""In-tree build of the CUDA backend (no GPU needed: nvcc cross-compiles sm_90a).

Artifacts (all under gaussian-splatting-cuda_b200/lib/, git-ignored):
  libgsb200.so           the C-ABI CUDA library (include/gsb200.h); no torch dependency
  libgsplat_b200.so      the libtorch shim exporting the reference's gsplat:: operator API
                         (include/gsplat/Ops.h), its fast_gs::rasterization API (include/fastgs/rasterization_api.h)
                         + a TORCH_LIBRARY binding used by tests/bench
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
SHIM = os.path.join(HERE, "shim")
LIB = os.path.join(HERE, "lib")
OBJ = os.path.join(HERE, "build")
INC = os.path.join(ROOT, "include")

NVCC = os.environ.get("GSB_NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr",
              "-ccbin", CXX]

# (source, extra flags).  -fmad=false where integer results (radii / tile bounds) depend on float
# rounding and must follow the reference's operation order (see the file headers).
CUDA_SOURCES = [
    ("gsb_projection.cu", ["-fmad=false"]),
    ("gsb_sh.cu", []),
    ("gsb_intersect.cu", ["-fmad=false"]),
    ("gsb_raster.cu", []),
    ("gsb_raster_rs.cu", []),
    ("gsb_misc.cu", []),
    ("gsb_fused.cu", ["-fmad=false"]),
    ("gsb_loss.cu", []),
    ("gsb_optim.cu", []),
    ("gsb_fastgs.cu", []),
    ("gsb_bilagrid.cu", []),
    ("gsb_mcmc.cu", []),
    ("gsb_adc.cu", []),
    ("gsb_sparsity.cu", []),
]
CUDA_HEADERS = ["gsb_common.cuh", "gsb_raster.cuh", "gsb_camera.cuh", "gsb_devsort.cuh", "gsb_sh.cuh", "gsb_projection.cuh", "gsb_ewa.cuh",
                "gsb_relocation.cuh", "gsb_select.cuh", "gsb_scan.cuh", "gsb_reduce.cuh"]
SHIM_SOURCES = ["Ops.cpp", "FusedOps.cpp", "FastGs.cpp", "BilateralGrid.cpp", "Mcmc.cpp", "Adc.cpp", "Sparsity.cpp", "torch_binding.cpp",
                "fastgs_binding.cpp"]


def _run(cmd: list[str], verbose: bool) -> str:
    if verbose:
        print(" ".join(cmd), flush=True)
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout)
        raise RuntimeError(f"build command failed ({p.returncode}): {' '.join(cmd)}")
    return p.stdout


def _stamp(paths: list[str], extra: str = "") -> str:
    h = hashlib.sha256(extra.encode())
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _needs(target: str, stamp: str) -> bool:
    sf = target + ".stamp"
    if not os.path.exists(target) or not os.path.exists(sf):
        return True
    return open(sf).read().strip() != stamp


def _mark(target: str, stamp: str) -> None:
    with open(target + ".stamp", "w") as f:
        f.write(stamp)


def build_cuda(verbose: bool = False, force: bool = False, ptxas_info: bool = False) -> str:
    os.makedirs(LIB, exist_ok=True)
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in CUDA_HEADERS] + [os.path.join(INC, "gsb200.h")]

    def compile_one(src_extra) -> tuple[str, str]:
        src, extra = src_extra
        sp = os.path.join(CSRC, src)
        op = os.path.join(OBJ, src.replace(".cu", ".o"))
        st = _stamp([sp] + hdrs, " ".join(NVCC_FLAGS + ARCH + extra))
        log = ""
        if force or _needs(op, st) or ptxas_info:
            cmd = [NVCC, "-c", sp, "-o", op] + NVCC_FLAGS + ARCH + extra + ["-I", INC]
            if ptxas_info:
                cmd += ["-Xptxas", "-v"]
            log = _run(cmd, verbose)
            _mark(op, st)
        return op, log

    # the translation units are independent: compile them side by side
    with ThreadPoolExecutor(max_workers=min(len(CUDA_SOURCES), os.cpu_count() or 1)) as ex:
        done = list(ex.map(compile_one, CUDA_SOURCES))
    objs = [op for op, _ in done]
    logs = [log for _, log in done if log]
    out = os.path.join(LIB, "libgsb200.so")
    st = _stamp(objs)
    if force or _needs(out, st):
        _run([NVCC, "-shared", "-o", out] + objs + ARCH + ["-Xcompiler", "-fPIC", "-ccbin", CXX], verbose)
        _mark(out, st)
    if ptxas_info:
        sys.stdout.write("\n".join(logs))
    return out


def build_shim(verbose: bool = False, force: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension as ce

    os.makedirs(LIB, exist_ok=True)
    os.makedirs(OBJ, exist_ok=True)
    tinc = ce.include_paths()
    tlib = ce.library_paths()[0]
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(NVCC)), "include")
    flags = ["-O2", "-std=c++17", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-Wall",
             "-Wno-unused-variable", "-DGSB_NO_GLM"]
    incs = []
    for i in [os.path.join(INC, "gsplat"), os.path.join(INC, "fastgs"), INC] + tinc + [cuda_inc]:
        incs += ["-I", i]
    hdrs = [os.path.join(INC, "gsb200.h")] + [os.path.join(INC, "gsplat", h) for h in ("Ops.h", "FusedOps.h", "Common.h", "Cameras.h")] + \
        [os.path.join(INC, "fastgs", "rasterization_api.h"), os.path.join(INC, "fastgs", "rasterization_ext.h"),
         os.path.join(SHIM, "SplatRows.h"),
         os.path.join(INC, "kernels", "bilateral_grid.cuh")]
    def compile_one(src: str) -> str:
        sp = os.path.join(SHIM, src)
        op = os.path.join(OBJ, "shim_" + src.replace(".cpp", ".o"))
        st = _stamp([sp] + hdrs, " ".join(flags) + torch.__version__)
        if force or _needs(op, st):
            _run([CXX, "-c", sp, "-o", op] + flags + incs, verbose)
            _mark(op, st)
        return op

    # each translation unit parses the torch headers (~20 s): compile them side by side
    with ThreadPoolExecutor(max_workers=min(len(SHIM_SOURCES), os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, SHIM_SOURCES))
    out = os.path.join(LIB, "libgsplat_b200.so")
    st = _stamp(objs + [os.path.join(LIB, "libgsb200.so")])
    if force or _needs(out, st):
        _run([CXX, "-shared", "-o", out] + objs +
             ["-L", LIB, "-lgsb200", "-L", tlib, "-ltorch", "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda",
              "-Wl,-rpath,$ORIGIN", "-Wl,-rpath," + tlib, "-Wl,-Bsymbolic", "-Wl,--no-as-needed"], verbose)
        _mark(out, st)
    return out


def build_all(verbose: bool = False, force: bool = False) -> dict:
    return {"cabi": build_cuda(verbose, force), "shim": build_shim(verbose, force)}


if __name__ == "__main__":
    v = "-q" not in sys.argv
    if "--ptxas" in sys.argv:
        build_cuda(verbose=v, force=True, ptxas_info=True)
    else:
        print(build_all(verbose=v, force="--force" in sys.argv))
