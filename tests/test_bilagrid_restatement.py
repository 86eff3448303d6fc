"""CPU: the float64 restatement of the bilateral grid (tests/bilagrid_restatement.py) against its own definition --
identity, finite differences of the slice and of the TV loss -- and the pieces of the feature that need no GPU: the
C ABI's new symbols and the learning-rate schedule."""
import os
import re

import numpy as np
import pytest
import torch

import bilagrid_restatement as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _img(h, w, seed, lo=-0.2, hi=1.2):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(h, w, 3, generator=g, dtype=torch.float64)).float().double()


def test_identity_grid_reproduces_clamped_input():
    img = _img(23, 40, 0)
    out = R.slice_fwd(R.identity_grids(1)[0], img)
    assert float((out - img.clamp(0, 1)).abs().max()) <= 1e-12


def _random_grid(L, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return R.identity_grids(1, W, H, L)[0] + 0.3 * torch.randn(12, L, H, W, generator=g, dtype=torch.float64)


@pytest.mark.parametrize("h,w,X,Y,L", [(23, 40, 16, 16, 8), (31, 29, 12, 9, 4)])
def test_slice_backward_matches_central_differences(h, w, X, Y, L):
    grid = _random_grid(L, Y, X, 1)
    # inputs inside (0, 1) and away from integer grid coordinates, so the slice is smooth around them
    img = _img(h, w, 2, 0.05, 0.95)
    c = R.coords(img, L, Y, X)
    fz = c["fz"]
    ok = (fz > 0.05) & (fz < 0.95)
    img = torch.where(ok[..., None], img, torch.full_like(img, 0.5))
    c = R.coords(img, L, Y, X)
    assert bool(((c["fz"] > 0.02) & (c["fz"] < 0.98)).all()), "test points must avoid integer gz"
    g = torch.Generator().manual_seed(3)
    v_out = torch.randn(h, w, 3, generator=g, dtype=torch.float64)
    v_grid, v_img = R.slice_bwd(grid, img, v_out)
    # The slice is quadratic in the input and linear in the grid inside a cell, so central differences are exact up to
    # rounding; the step stays inside the cell (|dz| < 0.05) and is large against the float32 coordinates' rounding.
    eps = 1e-3
    # directional derivatives along random directions, in the input and in the grid
    d_img = torch.randn(h, w, 3, generator=g, dtype=torch.float64).clamp(-2, 2)
    fd = ((R.slice_fwd(grid, img + eps * d_img) - R.slice_fwd(grid, img - eps * d_img)) * v_out).sum() / (2 * eps)
    assert abs(float(fd) - float((v_img * d_img).sum())) <= 1e-4 * max(1.0, abs(float(fd)))
    d_grid = torch.randn(12, L, Y, X, generator=g, dtype=torch.float64)
    fd = ((R.slice_fwd(grid + eps * d_grid, img) - R.slice_fwd(grid - eps * d_grid, img)) * v_out).sum() / (2 * eps)
    assert abs(float(fd) - float((v_grid * d_grid).sum())) <= 1e-9 * max(1.0, abs(float(fd)))


def test_slice_backward_masks_clamped_inputs():
    grid = _random_grid(8, 16, 16, 4)
    img = _img(9, 11, 5)
    _, v_img = R.slice_bwd(grid, img, torch.ones(9, 11, 3, dtype=torch.float64))
    outside = (img < 0) | (img > 1)
    assert bool(outside.any()) and float(v_img[outside].abs().max()) == 0.0


def test_tv_of_identity_is_zero_and_gradient_matches_finite_differences():
    assert float(R.tv_loss(R.identity_grids(3))) == 0.0
    g = torch.Generator().manual_seed(6)
    grids = torch.randn(2, 12, 4, 5, 3, generator=g, dtype=torch.float64)
    grad = R.tv_grad(grids)
    d = torch.randn(grids.shape, generator=g, dtype=torch.float64)
    eps = 1e-6
    fd = (R.tv_loss(grids + eps * d) - R.tv_loss(grids - eps * d)) / (2 * eps)
    assert abs(float(fd) - float((grad * d).sum())) <= 1e-8 * max(1.0, abs(float(fd)))
    # a direction of size 1 contributes nothing
    flat = torch.randn(1, 12, 1, 4, 4, generator=g, dtype=torch.float64)
    dx = torch.diff(flat, dim=4)
    dy = torch.diff(flat, dim=3)
    want = ((dx * dx).mean(dim=(2, 3, 4)).sum() + (dy * dy).mean(dim=(2, 3, 4)).sum()) / 12
    assert abs(float(R.tv_loss(flat)) - float(want)) <= 1e-15


def test_header_declares_bilateral_grid_entry_points():
    src = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    names = set(re.findall(r"GSB_API\s+[\w\s\*]+?\b(gsb_\w+)\s*\(", src))
    for n in ("gsb_bilagrid_slice_fwd", "gsb_bilagrid_slice_bwd", "gsb_bilagrid_tv", "gsb_bilagrid_tv_workspace"):
        assert n in names
    assert "GSB_LOSS_NO_CLAMP = 4" in src


def test_shim_exports_drop_in_bilateral_grid_api(pkg):
    import subprocess
    path = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib", "libgsplat_b200.so")
    if not os.path.exists(path):
        pkg.build()
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", path], capture_output=True, text=True).stdout
    for fn in ("slice_forward_cuda", "slice_backward_cuda", "tv_loss_forward_cuda", "tv_loss_backward_cuda"):
        assert f"gs::bilateral_grid::{fn}(" in out, fn
    assert "gsplat::photometric_loss_fused_unclamped(" in out


def test_cabi_rejects_degenerate_images(pkg):
    import ctypes
    lib = ctypes.CDLL(os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib", "libgsb200.so"))
    f = lib.gsb_bilagrid_slice_fwd
    f.restype = ctypes.c_int
    dummy = ctypes.c_void_p(16)
    # width 1: the grid coordinates would divide by zero (GSB_E_INVALID before any launch)
    assert f(16, 16, 8, 1, dummy, None, 1, 10, 0, dummy, dummy, None) == -1
    assert f(16, 16, 8, 1, dummy, None, 10, 1, 0, dummy, dummy, None) == -1
    assert f(0, 16, 8, 1, dummy, None, 10, 10, 0, dummy, dummy, None) == -1


def test_warmup_exponential_schedule():
    from importlib import import_module
    bil = import_module(pkg_name() + ".bilateral")
    s = bil.WarmupExponentialLR(2e-3, iterations=30000)
    lrs = [s.lr]
    for _ in range(1002):
        lrs.append(s.step())
    assert lrs[0] == 2e-3  # the first optimizer step runs at the initial rate
    assert np.isclose(lrs[1], 2e-3 * (0.01 + 0.99 / 1000))
    assert np.isclose(lrs[1000], 2e-3)
    assert np.isclose(lrs[1002], 2e-3 * (0.01 ** (1 / 30000)) ** 2)


def pkg_name():
    import __graft_entry__ as ge
    return ge.load_package().__name__


REF_COMPONENT = "/root/reference/src/training/components/bilateral_grid.cpp"


@pytest.mark.skipif(not os.path.exists(REF_COMPONENT), reason="reference tree not present")
def test_reference_bilateral_grid_component_links_against_backend(pkg, tmp_path):
    """The reference's BilateralGrid component compiles unmodified against include/kernels/bilateral_grid.cuh and links
    against libgsplat_b200.so with no undefined symbol."""
    import subprocess
    from torch.utils import cpp_extension as ce

    pkg.build()
    inc = []
    for i in [os.path.join(ROOT, "include")] + ce.include_paths() + ["/usr/local/cuda/include"]:
        inc += ["-I", i]
    obj = str(tmp_path / "bilateral_grid.o")
    subprocess.run(["/usr/bin/g++", "-std=c++20", "-O0", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=1", "-c", REF_COMPONENT,
                    "-o", obj] + inc, check=True)
    lib_dir = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib")
    tl = ce.library_paths()[0]
    so = str(tmp_path / "libcomponent.so")
    subprocess.run(["/usr/bin/g++", "-shared", "-o", so, obj, "-L", lib_dir, "-lgsplat_b200", "-lgsb200", "-L", tl,
                    "-ltorch", "-ltorch_cpu", "-lc10", "-ltorch_cuda", "-lc10_cuda", "-Wl,--no-undefined",
                    "-Wl,-rpath," + lib_dir, "-Wl,-rpath," + tl], check=True)
    out = subprocess.run(["nm", "-D", "--undefined-only", "-C", so], capture_output=True, text=True).stdout
    for fn in ("slice_forward_cuda", "slice_backward_cuda", "tv_loss_forward_cuda", "tv_loss_backward_cuda"):
        assert f"gs::bilateral_grid::{fn}" in out, fn
