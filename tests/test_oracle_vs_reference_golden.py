"""CPU: pin the oracle on the rows the reference's tests do not cover (UT projection, from-world
blend forward / backward) against outputs of the REFERENCE'S OWN CUDA KERNELS.

tests/golden/ref_cuda_small.npz was produced on the GPU by tests/test_gpu_vs_reference.py::
test_dump_reference_golden from oracle/_ref/libgsplat_ref.so, i.e. /root/reference/gsplat/*.cu compiled
unmodified with the reference's flags (oracle/build_ref.py).  Scene: scenes.scene_small(N=1200, 160x96,
SH deg 3, view=2), colours / cotangents from numpy default_rng(11)."""
import os

import numpy as np
import pytest

import scenes

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cuda_small.npz")


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.fixture(scope="module")
def gold():
    return np.load(G)


@pytest.fixture(scope="module")
def sc():
    return scenes.scene_small(N=1200, width=160, height=96, sh_degree=3, view=2)


def test_projection_vs_reference_cuda(orc, gold, sc):
    radii, means2d, depths, conics, comp = orc.projection_ut(
        sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"], sc["Ks"], sc["width"], sc["height"],
        0.3, 0.01, 1e4, 0.0, calc_compensations=True)
    mism = int((radii != gold["radii"]).any(-1).sum())
    assert mism <= 2, mism  # ceil()/cull borderline under fast-math vs IEEE
    both = (radii > 0).all(-1) & (gold["radii"] > 0).all(-1)
    assert both.sum() > 800
    assert rel(means2d[both], gold["means2d"][both]) < 1e-4
    assert rel(depths[both], gold["depths"][both]) < 1e-5
    assert rel(conics[both], gold["conics"][both]) < 1e-3
    assert rel(comp[both], gold["compensations"][both]) < 1e-4


def test_intersect_vs_reference_cuda(orc, gold, sc):
    tw, th = (sc["width"] + 15) // 16, (sc["height"] + 15) // 16
    tpg, ids, flat = orc.isect_tiles(gold["means2d"], gold["radii"], gold["depths"], 1, 16, tw, th, True)
    assert np.array_equal(tpg, gold["tiles_per_gauss"])
    assert np.array_equal(ids, gold["isect_ids"])
    assert np.array_equal(flat, gold["flatten_ids"])
    assert np.array_equal(orc.isect_offsets(ids, 1, tw, th), gold["tile_offsets"])


def test_blend_forward_vs_reference_cuda(orc, gold, sc):
    r, a, li = orc.raster_fwd(sc["means"], sc["quats"], sc["scales"], gold["colors"], sc["opacities"][None],
                              sc["background"], None, sc["width"], sc["height"], 16, sc["viewmats"], sc["Ks"],
                              gold["tile_offsets"], gold["flatten_ids"])
    assert rel(r, gold["renders"]) < 1e-4      # north_star: RGB within 1e-4 relative
    assert rel(a, gold["alphas"]) < 1e-4
    assert (li != gold["last_ids"]).mean() < 2e-3
    assert np.abs(r - gold["renders"]).max() < 2e-2


def test_blend_backward_vs_reference_cuda(orc, gold, sc):
    g = orc.raster_bwd(sc["means"], sc["quats"], sc["scales"], gold["colors"], sc["opacities"][None], sc["background"],
                       None, sc["width"], sc["height"], 16, sc["viewmats"], sc["Ks"], gold["tile_offsets"],
                       gold["flatten_ids"], gold["alphas"], gold["last_ids"], gold["v_render_colors"],
                       gold["v_render_alphas"], precision="f64")
    for nm, got in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g):
        e = rel(got.reshape(gold[nm].shape), gold[nm])
        assert e < 1e-3, (nm, e)   # north_star: gradients within 1e-3 relative
