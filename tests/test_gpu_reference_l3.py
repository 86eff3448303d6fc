"""GPU: the reference's OWN L3 code executes on the GPU through this repository's drop-in library.

oracle/_ref/libref_l3_b200.so = /root/reference/src/training/rasterization/rasterizer_autograd.cpp compiled unmodified
(SphericalHarmonicsFunction, fully_fused_projection_with_ut, GUTRasterizationFunction, forward and backward) + a
harness that strings them together as gs::training::rasterize does (oracle/ref_l3_harness.cpp), linked against
libgsplat_b200.so.  Its image and parameter gradients must equal those of the package's Python mirror of the same
sequence, which every other test uses: the boundary does not merely link, it runs."""
import os

import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, rel, to_dev

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle", "_ref", "libref_l3_b200.so")


@pytest.mark.parametrize("name", ["small_rot", "b30k"])
def test_reference_l3_autograd_runs_on_the_b200_backend(native, cuda_device, name):
    if not os.path.exists(SO):
        pytest.skip("oracle/_ref/libref_l3_b200.so not built (build() makes it where the reference's sources are present)")
    torch.ops.load_library(SO)
    sc = {"small_rot": lambda: scenes.scene_small(N=3000, width=200, height=120, view=1),
          "b30k": lambda: scenes.scene_b(N=30000, width=640, height=360, view=3, scale_mul=2.0)}[name]()
    W, H = sc["width"], sc["height"]
    t = to_dev(sc, cuda_device)
    names = ("means", "quats", "scales", "opacities", "sh_coeffs")
    g = torch.Generator(device=cuda_device).manual_seed(2)
    vr = torch.randn((1, H, W, 3), device=cuda_device, generator=g)
    va = torch.randn((1, H, W, 1), device=cuda_device, generator=g)
    res = {}
    for tag in ("reference_cpp", "python_mirror"):
        P = {k: t[k].clone().requires_grad_(True) for k in names}
        if tag == "reference_cpp":
            img, alpha, radii, flat = torch.ops.ref_l3_b200.render(P["means"], P["quats"], P["scales"], P["opacities"],
                                                                   P["sh_coeffs"], sc["sh_degree"], t["viewmats"], t["Ks"],
                                                                   W, H, t["background"])
            n = flat.shape[0]
        else:
            out = native.rasterize(P["means"], P["quats"], P["scales"], P["opacities"], P["sh_coeffs"], sc["sh_degree"],
                                   t["viewmats"], t["Ks"], W, H, bg_color=t["background"])
            img, alpha, n = out.render_colors, out.alpha.permute(1, 2, 0)[None], out.n_isects
        ((img * vr).sum() + (alpha * va).sum()).backward()
        res[tag] = (img.detach(), n, {k: P[k].grad for k in names})
    assert res["reference_cpp"][1] == res["python_mirror"][1] and res["python_mirror"][1] > 1000
    assert torch.equal(res["reference_cpp"][0], res["python_mirror"][0])  # same kernels, same inputs, same order
    for k in names:
        assert_grad_close(res["reference_cpp"][2][k], res["python_mirror"][2][k], k, sc["means"].shape[0], rel_tol=2e-5,
                          tag=f"reference C++ L3 vs Python mirror ({name})")
