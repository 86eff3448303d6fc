"""GPU: the planned intersect path at the inputs that take its rarely-used branches, bit-exact against the CPU oracle.

  * Depth-sort pass skipping.  The depth order is a stable LSD radix sort that skips every 8-bit pass whose digit is
    the same for all Gaussians with tiles.  Random depths skip only pass 3; the fixtures of tests/isect_fixtures.py skip
    all four, pass 0 only, passes 0, 1 and 3, or pass 1 only (tests/test_isect_skip_patterns.py checks that they do).
    Inactive Gaussians (zero radii, boxes clamped to zero tiles) are interleaved with depths that differ in every byte.
  * Whole paths on a scene with one Gaussian in view and on a wall of Gaussians at one depth, where the order of
    equal-depth Gaussians decides the image.
  * Windowed placement: more than 36 864 (camera, tile) pairs, so the histogram and placement run per window of tiles.
  * A capacity below the true intersection count: the lists and every blend range are clipped to it.
"""
import numpy as np
import pytest
import torch

import isect_fixtures as fx
import scenes
from parity import assert_grad_close, rel, to_dev

pytestmark = pytest.mark.gpu
W, H = 1280, 720


def _check_intersect(native, orc, dev, m2d, radii, depths, C, tile_size, tw, th):
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    tpg, ids, flat = native.intersect_tile(d(m2d), d(radii), d(depths), C, tile_size, tw, th, True)
    off = native.intersect_offset(ids, C, tw, th)
    tpg_ref, ids_ref, flat_ref = orc.isect_tiles(m2d, radii, depths, C, tile_size, tw, th)
    off_ref = orc.isect_offsets(ids_ref, C, tw, th)
    assert np.array_equal(tpg.cpu().numpy(), tpg_ref)
    assert np.array_equal(ids.cpu().numpy(), ids_ref)
    assert np.array_equal(flat.cpu().numpy(), flat_ref)
    assert np.array_equal(off.cpu().numpy(), off_ref)
    return tpg_ref, ids_ref


def _cases():
    out = [("skip_all", 1, 1)]  # one Gaussian: every fixture skips all four passes, so one case is enough
    for N in (1, 3000, 200_000):
        for C in (1, 3):
            if (N, C) != (1, 1):
                out += [(name, N, C) for name in sorted(fx.DEPTHS)]
    return out


@pytest.mark.parametrize("name,N,C", _cases())
def test_intersect_tile_skip_patterns_equal_oracle(native, orc, cuda_device, name, N, C):
    m2d, radii, depths, active = fx.intersect_inputs(name, C, N, W, H, seed=N + C)
    pattern = fx.skip_pattern(depths, active)
    want = (0, 1, 2, 3) if C * N == 1 else fx.DEPTHS[name][1]
    tpg, ids = _check_intersect(native, orc, cuda_device, m2d, radii, depths, C, 16, W // 16, H // 16)
    print(f"[{name} N={N} C={C}] skipped passes {pattern}, {int(active.sum())} Gaussians with tiles, "
          f"{len(ids)} intersections")
    assert pattern == want
    assert np.array_equal(tpg > 0, active)


def test_intersect_tile_back_to_back_patterns(native, orc, cuda_device):
    """Consecutive calls in one process reuse the caching allocator's blocks for the plan workspace: a sort that read
    the previous call's permutation instead of its own would give a wrong tie order here."""
    C, N = 3, 20_000
    for i, name in enumerate(("skip_3", "skip_all", "skip_0", "skip_013", "skip_1", "skip_all")):
        m2d, radii, depths, active = fx.intersect_inputs(name, C, N, W, H, seed=100 + i)
        pattern = fx.skip_pattern(depths, active)
        print(f"call {i}: [{name}] skipped passes {pattern}")
        assert pattern == fx.DEPTHS[name][1]
        _check_intersect(native, orc, cuda_device, m2d, radii, depths, C, 16, W // 16, H // 16)


@pytest.mark.parametrize("name", ["skip_3", "skip_all"])
def test_intersect_tile_size_4_windowed(native, orc, cuda_device, name):
    """Tile size 4 at 1024x768: 49 152 tiles, two windows of the histogram and placement."""
    Wi, Hi, ts = 1024, 768, 4
    tw, th = Wi // ts, Hi // ts
    m2d, radii, depths, active = fx.intersect_inputs(name, 1, 60_000, Wi, Hi, tile_size=ts, seed=5, max_radius=10)
    _, ids = _check_intersect(native, orc, cuda_device, m2d, radii, depths, 1, ts, tw, th)
    windows = -(-tw * th // fx.WINDOW_TILES)
    tiles = ids >> 32
    print(f"[{name}] {tw * th} tiles in {windows} windows, {len(ids)} intersections, "
          f"{int((tiles >= fx.WINDOW_TILES).sum())} past the first window, skipped passes {fx.skip_pattern(depths, active)}")
    assert tw * th > fx.WINDOW_TILES and windows == 2
    assert (tiles >= fx.WINDOW_TILES).sum() > 1000
    assert fx.skip_pattern(depths, active) == fx.DEPTHS[name][1]


# ------------------------------------------------------------------------------------------
# whole paths on the one-visible and wall scenes
# ------------------------------------------------------------------------------------------
SCENES = {"one_visible": scenes.scene_one_visible, "wall": scenes.scene_wall}


def _pattern_of(orc, m2d, radii, depths, sc):
    W_, H_ = sc["width"], sc["height"]
    tpg, _, _ = orc.isect_tiles(m2d, radii, depths, 1, 16, (W_ + 15) // 16, (H_ + 15) // 16)
    return fx.skip_pattern(depths, tpg > 0), int((tpg > 0).sum())


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_fused_vs_oracle_pipeline(native, orc, cuda_device, scene):
    from test_gpu_fused import raw_leaves
    sc = SCENES[scene]()
    Wi, Hi, N = sc["width"], sc["height"], sc["means"].shape[0]
    rng = np.random.default_rng(8)
    vrc = rng.standard_normal((1, Hi, Wi, 3)).astype(np.float32)
    vra = rng.standard_normal((1, Hi, Wi, 1)).astype(np.float32)
    ref = orc.render_pipeline(sc, "f32", True, vrc, vra)
    t = to_dev(sc, cuda_device)
    P = raw_leaves(native, t, None)
    o = native.rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                               sc["sh_degree"], t["viewmats"], t["Ks"], Wi, Hi, bg_color=t["background"])
    ((o.render_colors * torch.from_numpy(vrc).to(cuda_device)).sum() +
     (o.alpha * torch.from_numpy(vra).to(cuda_device)).sum()).backward()
    pattern, n_act = _pattern_of(orc, o.means2d.detach().cpu().numpy(), o.radii.cpu().numpy(),
                                 o.depths.detach().cpu().numpy(), sc)
    e = rel(o.render_colors.detach().cpu().numpy(), ref["renders"])
    print(f"[{scene}] fused: {n_act} Gaussians with tiles, skipped passes {pattern}, "
          f"{int(o.n_isects.item())} intersections (oracle {len(ref['flatten_ids'])}), image rel_l2 {e:.2e}")
    assert pattern == (0, 1, 2, 3)
    assert abs(int(o.n_isects.item()) - len(ref["flatten_ids"])) <= 8
    assert e < 1e-4
    op = sc["opacities"].astype(np.float64)
    want = {"means": ref["v_means"] + ref["v_dirs"][0], "sh0": ref["v_sh_coeffs"][:, :1], "shN": ref["v_sh_coeffs"][:, 1:],
            "scaling_raw": ref["v_scales"] * sc["scales"], "rotation_raw": ref["v_quats"],
            "opacity_raw": (ref["v_opacities"][0] * op * (1 - op))[:, None]}
    for k, w in want.items():
        assert_grad_close(P[k].grad, w, k, N, tag=f"{scene} fused vs CPU oracle")


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_fastgs_vs_oracle(native, orc, cuda_device, scene):
    from oracle import fastgs_oracle as fgo
    from test_gpu_fastgs import PARAMS, _fg, _weights, grads_close, image_close, run
    sc = SCENES[scene]()
    r, m2d, d, _, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"],
                                        sc["Ks"], sc["width"], sc["height"], 0.3, 0.01, 1e4, 0.0)
    pattern, n_act = _pattern_of(orc, m2d, r, d, sc)
    inp = scenes.fastgs_inputs(sc)
    gi, ga = _weights(inp, cuda_device, 4)
    fg = _fg(native)
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga)
    o = fgo.render(**inp, grad_image=gi.cpu().numpy(), grad_alpha=ga.cpu().numpy(), precision="f64")
    print(f"[{scene}] fastgs: {o['n_instances']} instances, {n_act} Gaussians with tiles, skipped passes {pattern}")
    assert pattern == (0, 1, 2, 3) and o["n_instances"] > 0
    oracle = dict(image=torch.from_numpy(o["image"]).to(cuda_device), alpha=torch.from_numpy(o["alpha"]).to(cuda_device),
                  grads={k: o["grad_" + k] for k in PARAMS})
    image_close(mine, oracle, f"{scene} fastgs vs f64 oracle")
    grads_close(mine, oracle, inp["means"].shape[0], f"{scene} fastgs vs f64 oracle")


# ------------------------------------------------------------------------------------------
# clipped capacity
# ------------------------------------------------------------------------------------------
def test_fused_clipped_capacity_equals_oracle_on_clipped_lists(native, orc, cuda_device):
    """isect_capacity below the true count: the first `cap` list entries are the exact run's, n_isects still reports
    the true count, and the image is the blend of every tile's range clipped to `cap`."""
    from test_gpu_fused import raw_leaves
    sc = scenes.scene_b(N=20000, width=640, height=360, view=2, scale_mul=2.0)
    Wi, Hi = sc["width"], sc["height"]
    tw, th = (Wi + 15) // 16, (Hi + 15) // 16
    t = to_dev(sc, cuda_device)
    P = raw_leaves(native, t, None, requires_grad=False)
    fwd = torch.ops.gsplat_b200.rasterize_from_world_fused_fwd

    def call(capacity):
        o = fwd(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"], 3, 1.0,
                t["viewmats"], t["Ks"], Wi, Hi, 0.3, 0.01, 1e4, 0.0, t["background"], 0, None, None, None, capacity, False)
        torch.cuda.synchronize()
        return dict(img=o[0].cpu().numpy(), off=o[6].cpu().numpy(), flat=o[7].cpu().numpy(), n=int(o[9].item()))

    exact = call(0)
    n = exact["n"]
    assert len(exact["flat"]) == n and exact["off"][-1] == n
    counts = np.diff(exact["off"])
    t_cut = int(np.argmax(np.where((exact["off"][:-1] > n // 4) & (exact["off"][:-1] < 3 * n // 4), counts, 0)))
    cap = int(exact["off"][t_cut] + counts[t_cut] // 2)  # halfway through the longest list in the middle half
    assert exact["off"][t_cut] < cap < exact["off"][t_cut + 1]
    clipped = call(cap)
    print(f"{n} intersections, capacity {cap}: cuts tile {t_cut} ({counts[t_cut]} entries) at {cap - exact['off'][t_cut]}")
    assert clipped["n"] == n
    assert len(clipped["flat"]) == cap
    assert np.array_equal(clipped["flat"], exact["flat"][:cap])
    assert np.array_equal(clipped["off"], exact["off"])
    ref = orc.render_pipeline(sc, "f32")
    off_cap = np.minimum(exact["off"][:-1], cap).reshape(1, th, tw)
    img, _, _ = orc.raster_fwd(sc["means"], sc["quats"], sc["scales"], ref["colors"], sc["opacities"][None],
                               sc["background"], None, Wi, Hi, 16, sc["viewmats"], sc["Ks"], off_cap, clipped["flat"])
    e_clip, e_full = rel(clipped["img"], img), rel(clipped["img"], exact["img"])
    print(f"image vs oracle on the clipped lists rel_l2 {e_clip:.2e}; vs the unclipped image {e_full:.2e}")
    assert e_clip < 1e-4
    assert e_full > 1e-2  # the clipping is visible: the comparison above is not the unclipped image again
