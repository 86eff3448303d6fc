"""GPU: this backend against stored outputs of the REFERENCE'S OWN kernels, with nothing outside the repository.

tests/golden/ref_cuda_small.npz holds what the reference's gsplat kernels (built unmodified by oracle/build_ref.py)
computed on scenes.scene_small(N=1200, 160x96, SH degree 3, view=2) -- projection, tile intersection, blend forward and
backward -- and tests/golden/ref_fastgs_small.npz what its fastgs kernels computed on
scenes.fastgs_inputs(scenes.scene_small(N=1500, 176x112, SH degree 3, seed 13, view 2)); see the test_dump_* tests of
test_gpu_vs_reference.py and test_gpu_fastgs.py for how they are made.  Each stage is fed the reference's own inputs
from the file, so the comparisons are those of the live tests against the reference library, at the same tolerances."""
import importlib
import os

import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, rel

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "ref_cuda_small.npz"))


@pytest.fixture(scope="module")
def small(cuda_device):
    sc = scenes.scene_small(N=1200, width=160, height=96, sh_degree=3, view=2)
    return sc, {k: torch.from_numpy(v).to(cuda_device) for k, v in sc.items() if isinstance(v, np.ndarray)}


def _dev(gold, key, dev):
    return torch.from_numpy(gold[key]).to(dev)


def test_projection_vs_reference_golden(native, gold, small):
    sc, t = small
    radii, means2d, depths, conics, comp = native.projection_ut_3dgs_fused(
        t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], sc["width"], sc["height"],
        0.3, 0.01, 1e4, 0.0, calc_compensations=True)
    radii = radii.cpu().numpy()
    mism = int((radii != gold["radii"]).any(-1).sum())
    d = np.abs(radii.astype(np.int64) - gold["radii"].astype(np.int64))
    both = (radii > 0).all(-1) & (gold["radii"] > 0).all(-1)
    print(f"radii differ {mism}/{radii.shape[1]}, visible in both {int(both.sum())}")
    assert mism <= 3 and not ((d > 1) & both[..., None]).any()  # ceil()/cull borderline flips under fast-math vs IEEE
    assert both.sum() > 800
    assert rel(means2d.cpu().numpy()[both], gold["means2d"][both]) < 1e-4
    assert rel(depths.cpu().numpy()[both], gold["depths"][both]) < 1e-5
    assert rel(conics.cpu().numpy()[both], gold["conics"][both]) < 1e-3
    assert rel(comp.cpu().numpy()[both], gold["compensations"][both]) < 1e-4


def test_intersect_bit_exact_vs_reference_golden(native, gold, small, cuda_device):
    sc, _ = small
    tw, th = (sc["width"] + 15) // 16, (sc["height"] + 15) // 16
    tpg, ids, flat = native.intersect_tile(_dev(gold, "means2d", cuda_device), _dev(gold, "radii", cuda_device),
                                           _dev(gold, "depths", cuda_device), 1, 16, tw, th, True)
    assert np.array_equal(tpg.cpu().numpy(), gold["tiles_per_gauss"])
    assert np.array_equal(ids.cpu().numpy(), gold["isect_ids"])
    assert np.array_equal(flat.cpu().numpy(), gold["flatten_ids"])
    assert np.array_equal(native.intersect_offset(ids, 1, tw, th).cpu().numpy(), gold["tile_offsets"])


def _blend_args(gold, small, dev):
    sc, t = small
    return (t["means"], t["quats"], t["scales"], _dev(gold, "colors", dev), t["opacities"][None], t["background"], None,
            sc["width"], sc["height"], 16, t["viewmats"], t["Ks"], _dev(gold, "tile_offsets", dev),
            _dev(gold, "flatten_ids", dev))


def test_blend_forward_vs_reference_golden(native, gold, small, cuda_device):
    r, a, li = native.rasterize_to_pixels_from_world_3dgs_fwd(*_blend_args(gold, small, cuda_device))
    r, a, li = r.cpu().numpy(), a.cpu().numpy(), li.cpu().numpy()
    e = rel(r, gold["renders"])
    lm = float((li != gold["last_ids"]).mean())
    print(f"image rel_l2 vs reference kernels {e:.2e}; last_ids differ {lm:.2e}")
    assert e < 1e-4 and rel(a, gold["alphas"]) < 1e-4
    assert lm < 2e-3 and np.abs(r - gold["renders"]).max() < 2e-2


def test_blend_backward_vs_reference_golden(native, gold, small, cuda_device):
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*_blend_args(gold, small, cuda_device), _dev(gold, "alphas", cuda_device),
                                                       _dev(gold, "last_ids", cuda_device),
                                                       _dev(gold, "v_render_colors", cuda_device),
                                                       _dev(gold, "v_render_alphas", cuda_device))
    n = gold["v_means"].shape[0]
    for nm, got in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g):
        assert_grad_close(got.cpu().numpy().reshape(gold[nm].shape), gold[nm], nm, n, tag="blend bwd vs reference golden")


def test_fastgs_vs_reference_golden(native, cuda_device):
    fg = importlib.import_module(native.__name__ + ".fastgs")
    g = np.load(os.path.join(GOLDEN, "ref_fastgs_small.npz"))
    inp = scenes.fastgs_inputs(scenes.scene_small(N=1500, width=176, height=112, sh_degree=3, seed=13, view=2))
    names = ("means", "scales_raw", "rotations_raw", "opacities_raw", "sh0", "shN")
    P = {k: torch.from_numpy(inp[k]).to(cuda_device).requires_grad_(True) for k in names}
    w2c = torch.from_numpy(inp["w2c"]).to(cuda_device).requires_grad_(True)
    s = fg.FastGSSettings(cam_position=torch.from_numpy(inp["cam_position"]).to(cuda_device),
                          active_sh_bases=inp["active_sh_bases"], width=inp["width"], height=inp["height"],
                          focal_x=inp["fx"], focal_y=inp["fy"], center_x=inp["cx"], center_y=inp["cy"],
                          near_plane=inp["near_plane"], far_plane=inp["far_plane"])
    n = inp["means"].shape[0]
    dens = torch.zeros((2, n), device=cuda_device)
    image, alpha = fg.fast_rasterize(fg.default_backend(), P["means"], P["scales_raw"], P["rotations_raw"],
                                     P["opacities_raw"], P["sh0"], P["shN"], w2c, s, densification_info=dens)
    ((image * _dev(g, "grad_image", cuda_device)).sum() + (alpha * _dev(g, "grad_alpha", cuda_device)).sum()).backward()
    torch.cuda.synchronize()
    img = image.detach().cpu().numpy()
    e, ea = rel(img, g["image"]), rel(alpha.detach().cpu().numpy(), g["alpha"])
    d = np.abs(img - g["image"])
    print(f"fastgs image rel_l2 vs reference kernels {e:.2e}, alpha {ea:.2e}, max |d| {float(d.max()):.2e}")
    assert e < 1e-4 and ea < 1e-4
    assert float((d > 1e-3).mean()) < 1e-3 and float(d.max()) < 2e-2
    for k in names:
        got = P[k].grad if P[k].grad is not None else torch.zeros_like(P[k])
        assert_grad_close(got.cpu().numpy().reshape(g["grad_" + k].shape), g["grad_" + k], k, n,
                          tag="fastgs vs reference golden")
    assert rel(w2c.grad[:3].cpu().numpy(), g["grad_w2c"][:3]) < 1e-3
    dn = dens.cpu().numpy()
    assert np.array_equal(dn[0], g["densification_info"][0])
    assert rel(dn[1], g["densification_info"][1]) < 1e-3
