"""Build the REFERENCE's own gsplat CUDA library for the GPU box (checker + same-box baseline).

Compiles the reference's sources WHERE THEY LIE under /root/reference/gsplat (nothing is copied into
this repo), with the reference's own flags (-O3 --use_fast_math --expt-relaxed-constexpr,
gsplat/CMakeLists.txt:76) for plain sm_90, plus oracle/ref_binding.cpp, into
oracle/_ref/libgsplat_ref.so (git-ignored).

The reference's device math depends on GLM, which is not vendored in the reference tree and not
installed here; oracle/glm_shim/ provides the subset it uses (see glm_shim/glm/glm.hpp).

This does NOT run the reference's build system; it is a short explicit recipe (DESIGN.md "Oracle").
Runs only in the build container (needs /root/reference).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/gsplat"
OUT = os.path.join(HERE, "_ref")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CXX = "/usr/bin/g++"

CU = ["ProjectionUT3DGSFused.cu", "IntersectTile.cu", "SphericalHarmonicsCUDA.cu", "QuatToRotmatCUDA.cu",
      "RelocationCUDA.cu", "RasterizeToPixelsFromWorld3DGSFwd.cu", "RasterizeToPixelsFromWorld3DGSBwd.cu"]
CPP = ["Projection.cpp", "Intersect.cpp", "SphericalHarmonics.cpp", "QuatToRotmat.cpp", "Relocation.cpp",
       "Rasterization.cpp"]
# the training-step kernels next to the path (SURVEY.md 8 f2 / f3), compiled from where they lie as well
TRAIN_CU = ["/root/reference/src/training/kernels/ssim.cu"]
TRAIN_INC = ["/root/reference/fastgs/optimizer/include"]
EXTRA = ["ref_binding.cpp", "ref_train_binding.cu"]


# Host-only translation units (.cpp) go to the host compiler, as in the reference's own CMake build: through nvcc's
# device front end the torch headers cost minutes per file, through g++ seconds.
HOST_FLAGS = ["-O3", "-std=c++20", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1"]
CUDA_INC = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(NVCC))), "include")


def available() -> bool:
    return os.path.exists(os.path.join(OUT, "libgsplat_ref.so"))


# "precise": the same sources WITHOUT --use_fast_math, registered as torch.ops.gsplat_ref_precise.  The rolling-shutter
# pose interpolation calls sin() on angles of a few milliradians: sin.approx has an ABSOLUTE error of ~2^-21, i.e.
# 1e-4 relative there, and the unscented transform's -99 / +16.67 weights amplify that a hundredfold -- the fast-math
# build's rolling-shutter outputs carry ~0.1 px of noise.  The precise build is the noise-free statement of the same
# algorithm and is what the rolling-shutter parity tests compare against.
VARIANTS = {"fast": ("libgsplat_ref.so", "gsplat_ref", True), "precise": ("libgsplat_ref_precise.so", "gsplat_ref_precise", False)}


def _stamp() -> str:
    h = hashlib.sha256()
    for f in CU + CPP:
        h.update(open(os.path.join(REF, f), "rb").read())
    for f in TRAIN_CU + [os.path.join(TRAIN_INC[0], "adam_kernels.cuh")]:
        h.update(open(f, "rb").read())
    for root, _, files in os.walk(os.path.join(HERE, "glm_shim")):
        for f in sorted(files):
            h.update(open(os.path.join(root, f), "rb").read())
    for f in EXTRA:
        h.update(open(os.path.join(HERE, f), "rb").read())
    return h.hexdigest()


def build(verbose: bool = True, jobs: int = 7, variant: str = "fast") -> str | None:
    if not os.path.isdir(REF):
        return None
    from torch.utils import cpp_extension as ce

    so_name, ns, fast = VARIANTS[variant]
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, so_name)
    stamp_file = so + ".stamp"
    st = _stamp() + variant
    if os.path.exists(so) and os.path.exists(stamp_file) and open(stamp_file).read() == st:
        return so
    inc = []
    for i in [os.path.join(HERE, "glm_shim"), REF] + TRAIN_INC + ce.include_paths():
        inc += ["-I", i]
    common = ["-O3", "-std=c++20", "-Xcompiler", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-ccbin", CXX,
              "-gencode", "arch=compute_90,code=sm_90", "--expt-relaxed-constexpr", f"-DREF_NS={ns}",
              "-diag-suppress", "20012,20011,20014,177,550"] + (["--use_fast_math"] if fast else [])

    def compile_one(src: str):
        sp = src if os.path.isabs(src) else os.path.join(REF, src)
        obj = os.path.join(OUT, variant + "_" + os.path.basename(src).rsplit(".", 1)[0] + ".o")
        if sp.endswith(".cpp"):
            cmd = [CXX, "-c", sp, "-o", obj] + HOST_FLAGS + [f"-DREF_NS={ns}"] + inc + ["-I", CUDA_INC]
        else:
            cmd = [NVCC, "-c", sp, "-o", obj] + common + inc
        if verbose:
            print("[build_ref]", os.path.basename(src), flush=True)
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout[-6000:])
            raise RuntimeError(f"reference source failed to compile: {src}")
        return obj

    srcs = CU + CPP + ((TRAIN_CU + [os.path.join(HERE, f) for f in EXTRA]) if fast else [os.path.join(HERE, EXTRA[0])])
    with ThreadPoolExecutor(max_workers=jobs) as ex:
        objs = list(ex.map(compile_one, srcs))
    tl = ce.library_paths()[0]
    cmd = [NVCC, "-shared", "-o", so] + objs + ["-gencode", "arch=compute_90,code=sm_90", "-ccbin", CXX, "-L", tl,
                                                 "-ltorch", "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda",
                                                 "-Xlinker", "-rpath," + tl, "-Xlinker", "-Bsymbolic"]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-6000:])
        raise RuntimeError(f"linking oracle/_ref/{so_name} failed")
    for o in objs:
        os.remove(o)
    with open(stamp_file, "w") as f:
        f.write(st)
    return so


L3_SRC = "/root/reference/src/training/rasterization/rasterizer_autograd.cpp"


def build_l3_harness(verbose: bool = True) -> str | None:
    """The reference's rasterizer_autograd.cpp (unmodified) + oracle/ref_l3_harness.cpp linked against THIS repo's drop-in
    library: oracle/_ref/libref_l3_b200.so (tests/test_gpu_reference_l3.py executes it on the GPU)."""
    if not os.path.exists(L3_SRC):
        return None
    from torch.utils import cpp_extension as ce

    root = os.path.dirname(HERE)
    lib_dir = os.path.join(root, "gaussian-splatting-cuda_b200", "lib")
    shim = os.path.join(lib_dir, "libgsplat_b200.so")
    if not os.path.exists(shim):
        return None
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libref_l3_b200.so")
    h = hashlib.sha256()
    for f in (L3_SRC, os.path.join(HERE, "ref_l3_harness.cpp"), os.path.join(root, "include", "gsplat", "Ops.h")):
        h.update(open(f, "rb").read())
    st = h.hexdigest()
    if os.path.exists(so) and os.path.exists(so + ".stamp") and open(so + ".stamp").read() == st:
        return so
    inc = []
    for i in [os.path.join(root, "tests", "link_stubs"), os.path.join(root, "include", "gsplat"), os.path.join(root, "include"),
              "/root/reference/src/training"] + ce.include_paths() + ["/usr/local/cuda/include"]:
        inc += ["-I", i]
    objs = []
    for src in (L3_SRC, os.path.join(HERE, "ref_l3_harness.cpp")):
        obj = os.path.join(OUT, "l3_" + os.path.basename(src).rsplit(".", 1)[0] + ".o")
        if verbose:
            print("[build_ref] L3", os.path.basename(src), flush=True)
        p = subprocess.run([CXX, "-std=c++20", "-O2", "-fPIC", "-DGSB_NO_GLM", "-D_GLIBCXX_USE_CXX11_ABI=1", "-c", src, "-o",
                            obj] + inc, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout[-6000:])
            raise RuntimeError(f"L3 harness source failed to compile: {src}")
        objs.append(obj)
    tl = ce.library_paths()[0]
    p = subprocess.run([CXX, "-shared", "-o", so] + objs + ["-L", lib_dir, "-lgsplat_b200", "-lgsb200", "-L", tl, "-ltorch",
                        "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda", "-Wl,--no-undefined",
                        "-Wl,-rpath,$ORIGIN/../../gaussian-splatting-cuda_b200/lib", "-Wl,-rpath," + tl],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-6000:])
        raise RuntimeError("linking oracle/_ref/libref_l3_b200.so failed")
    for o in objs:
        os.remove(o)
    with open(so + ".stamp", "w") as f:
        f.write(st)
    return so


FAST_L3_SRC = "/root/reference/src/training/rasterization/fast_rasterizer_autograd.cpp"


def build_fastgs_l3_harness(verbose: bool = True) -> str | None:
    """The reference's fast_rasterizer_autograd.cpp (unmodified) + oracle/ref_fastgs_l3_harness.cpp linked against THIS
    repository's drop-in library: oracle/_ref/libref_fastgs_l3_b200.so (tests/test_gpu_fastgs.py executes it)."""
    if not os.path.exists(FAST_L3_SRC):
        return None
    from torch.utils import cpp_extension as ce

    root = os.path.dirname(HERE)
    lib_dir = os.path.join(root, "gaussian-splatting-cuda_b200", "lib")
    if not os.path.exists(os.path.join(lib_dir, "libgsplat_b200.so")):
        return None
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libref_fastgs_l3_b200.so")
    harness = os.path.join(HERE, "ref_fastgs_l3_harness.cpp")
    h = hashlib.sha256()
    for f in (FAST_L3_SRC, harness, os.path.join(root, "include", "fastgs", "rasterization_api.h")):
        h.update(open(f, "rb").read())
    st = h.hexdigest()
    if os.path.exists(so) and os.path.exists(so + ".stamp") and open(so + ".stamp").read() == st:
        return so
    inc = []
    for i in [os.path.join(root, "include", "fastgs"), "/root/reference/src/training"] + ce.include_paths() + ["/usr/local/cuda/include"]:
        inc += ["-I", i]
    objs = []
    for src in (FAST_L3_SRC, harness):
        obj = os.path.join(OUT, "fl3_" + os.path.basename(src).rsplit(".", 1)[0] + ".o")
        if verbose:
            print("[build_ref] fastgs L3", os.path.basename(src), flush=True)
        p = subprocess.run([CXX, "-std=c++20", "-O2", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-c", src, "-o", obj] + inc,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout[-6000:])
            raise RuntimeError(f"fastgs L3 harness source failed to compile: {src}")
        objs.append(obj)
    tl = ce.library_paths()[0]
    p = subprocess.run([CXX, "-shared", "-o", so] + objs + ["-L", lib_dir, "-lgsplat_b200", "-lgsb200", "-L", tl, "-ltorch",
                        "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda", "-Wl,--no-undefined",
                        "-Wl,-rpath,$ORIGIN/../../gaussian-splatting-cuda_b200/lib", "-Wl,-rpath," + tl],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-6000:])
        raise RuntimeError("linking oracle/_ref/libref_fastgs_l3_b200.so failed")
    for o in objs:
        os.remove(o)
    with open(so + ".stamp", "w") as f:
        f.write(st)
    return so


FASTGS = "/root/reference/fastgs"
FASTGS_CU = ["rasterization/src/forward.cu", "rasterization/src/backward.cu", "rasterization/src/rasterization_api.cu"]


def build_fastgs(verbose: bool = True, gencode: str = "arch=compute_90,code=sm_90", so_name: str = "libfastgs_ref.so") -> str | None:
    """The reference's fastgs rasterizer (SURVEY.md 8 f4), compiled unmodified from where it lies with its own flags
    (fastgs/CMakeLists.txt:58: -O3 --use_fast_math --expt-relaxed-constexpr), plus the product's
    shim/fastgs_binding.cpp compiled against the REFERENCE's rasterization_api.h: oracle/_ref/libfastgs_ref.so,
    torch.ops.fastgs_ref.*  (the pin of oracle/fastgs_oracle.c and of the H100 path; the same-box GPU baseline)."""
    if not os.path.isdir(FASTGS):
        return None
    from torch.utils import cpp_extension as ce

    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, so_name)
    binding = os.path.join(os.path.dirname(HERE), "gaussian-splatting-cuda_b200", "shim", "fastgs_binding.cpp")
    h = hashlib.sha256()
    for root, _, files in os.walk(os.path.join(FASTGS, "rasterization")):
        for f in sorted(files):
            h.update(open(os.path.join(root, f), "rb").read())
    h.update(open(binding, "rb").read())
    h.update(gencode.encode())
    st = h.hexdigest()
    if os.path.exists(so) and os.path.exists(so + ".stamp") and open(so + ".stamp").read() == st:
        return so
    inc = []
    for i in [os.path.join(FASTGS, "rasterization", "include"), os.path.join(FASTGS, "utils")] + ce.include_paths():
        inc += ["-I", i]
    common = ["-O3", "-std=c++20", "-Xcompiler", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-ccbin", CXX, "-gencode",
              gencode, "--expt-relaxed-constexpr", "--use_fast_math", "-DFGS_REFERENCE_LIBRARY",
              "-diag-suppress", "20012,186,221,177,550"]

    def compile_one(src: str):
        obj = os.path.join(OUT, "fgs_" + so_name + "_" + os.path.basename(src).rsplit(".", 1)[0] + ".o")
        if verbose:
            print("[build_ref] fastgs", os.path.basename(src), flush=True)
        if src.endswith(".cpp"):
            cmd = [CXX, "-c", src, "-o", obj] + HOST_FLAGS + ["-DFGS_REFERENCE_LIBRARY"] + inc + ["-I", CUDA_INC]
        else:
            cmd = [NVCC, "-c", src, "-o", obj] + common + inc
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout[-6000:])
            raise RuntimeError(f"reference fastgs source failed to compile: {src}")
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, [os.path.join(FASTGS, f) for f in FASTGS_CU] + [binding]))
    tl = ce.library_paths()[0]
    p = subprocess.run([NVCC, "-shared", "-o", so] + objs + ["-gencode", gencode, "-ccbin", CXX, "-L", tl,
                        "-ltorch", "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda", "-Xlinker", "-rpath," + tl,
                        "-Xlinker", "-Bsymbolic"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-6000:])
        raise RuntimeError(f"linking oracle/_ref/{so_name} failed")
    for o in objs:
        os.remove(o)
    with open(so + ".stamp", "w") as f:
        f.write(st)
    return so


def build_all(verbose: bool = True) -> None:
    """Every reference library.  The three kernel libraries are independent and each takes minutes of nvcc, so they
    compile side by side; the two caller harnesses link against this repository's shim and come after them."""
    with ThreadPoolExecutor(max_workers=3) as ex:
        for f in [ex.submit(build, verbose), ex.submit(build, verbose, variant="precise"), ex.submit(build_fastgs, verbose)]:
            f.result()
    with ThreadPoolExecutor(max_workers=2) as ex:
        for f in [ex.submit(build_l3_harness, verbose), ex.submit(build_fastgs_l3_harness, verbose)]:
            f.result()


if __name__ == "__main__":
    build_all()
