"""GPU: parity of the sm_90a path (through the gsplat:: shim -> C ABI) against the CPU oracle and
the committed golden vectors.  Tolerances follow BASELINE.json's north_star: integer / index
results bit-exact, rendered RGB within 1e-4 relative, gradients within 1e-3 relative.

"Relative" is the relative L2 error over the whole tensor (||a-b|| / ||b||): the blend is only
piecewise continuous (alpha < 1/255 cut, T <= 1e-4 stop, ceil() of radii), so a handful of
element-wise outliers at decision boundaries are inherent to any float implementation -- the tests
additionally bound the FRACTION of pixels / Gaussians that may differ by more than the tolerance.
"""
import math
import os

import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, rel, to_dev

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ------------------------------------------------------------------------------------------
# a5/a6: tile intersection -- bit-exact against the reference's torch oracle golden vectors
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["c3", "c1"])
def test_intersect_bit_exact_vs_golden(native, cuda_device, name):
    g = np.load(os.path.join(G, f"torch_impl_isect_{name}.npz"))
    C = g["means2d"].shape[0]
    tw, th, ts = int(g["tile_width"]), int(g["tile_height"]), int(g["tile_size"])
    m2d = torch.from_numpy(g["means2d"]).to(cuda_device)
    rad = torch.from_numpy(g["radii"]).to(cuda_device)
    dep = torch.from_numpy(g["depths"]).to(cuda_device)
    tpg, ids, flat = native.intersect_tile(m2d, rad, dep, C, ts, tw, th, True)
    assert tpg.dtype == torch.int32 and ids.dtype == torch.int64 and flat.dtype == torch.int32
    assert np.array_equal(tpg.cpu().numpy(), g["tiles_per_gauss"])
    assert np.array_equal(ids.cpu().numpy(), g["isect_ids"])
    assert np.array_equal(flat.cpu().numpy(), g["flatten_ids"])
    # unsorted emission order == oracle emission order
    _, ids_u, flat_u = native.intersect_tile(m2d, rad, dep, C, ts, tw, th, False)
    assert np.array_equal(np.sort(ids_u.cpu().numpy()), g["isect_ids"])


def test_intersect_offsets_and_empty(native, orc, cuda_device):
    g = np.load(os.path.join(G, "torch_impl_isect_c3.npz"))
    C, tw, th = 3, int(g["tile_width"]), int(g["tile_height"])
    ids = torch.from_numpy(g["isect_ids"]).to(cuda_device)
    off = native.intersect_offset(ids, C, tw, th)
    assert off.shape == (C, th, tw) and off.dtype == torch.int32
    assert np.array_equal(off.cpu().numpy(), orc.isect_offsets(g["isect_ids"], C, tw, th))
    # no intersections at all: everything zero (IntersectTile.cu:268-271)
    z = torch.zeros(1, 50, 2, device=cuda_device)
    tpg, ids0, flat0 = native.intersect_tile(z, torch.zeros(1, 50, 2, dtype=torch.int32, device=cuda_device),
                                             torch.ones(1, 50, device=cuda_device), 1, 16, 4, 4, True)
    assert ids0.numel() == 0 and flat0.numel() == 0 and int(tpg.sum()) == 0
    assert int(native.intersect_offset(ids0, 1, 4, 4).abs().sum()) == 0


# ------------------------------------------------------------------------------------------
# a3/a4: spherical harmonics
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3, 4])
def test_sh_vs_golden(native, cuda_device, deg):
    g = np.load(os.path.join(G, "torch_impl_sh.npz"))
    dirs = torch.from_numpy(g["dirs"]).to(cuda_device)
    coeffs = torch.from_numpy(g["coeffs"]).to(cuda_device)
    vcol = torch.from_numpy(g["v_colors"]).to(cuda_device)
    col = native.spherical_harmonics_fwd(deg, dirs, coeffs, None)
    np.testing.assert_allclose(col.cpu().numpy(), g[f"colors_deg{deg}"], rtol=1e-4, atol=1e-4)
    v_coeffs, v_dirs = native.spherical_harmonics_bwd(25, deg, dirs, coeffs, None, vcol, True)
    np.testing.assert_allclose(v_coeffs.cpu().numpy(), g[f"v_coeffs_deg{deg}"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(v_dirs.cpu().numpy(), g[f"v_dirs_deg{deg}"], rtol=1e-4, atol=2e-4)


@pytest.mark.parametrize("K,deg", [(16, 3), (16, 1), (4, 1), (9, 2), (1, 0)])
def test_sh_masks_vs_oracle(native, orc, cuda_device, K, deg):
    rng = np.random.default_rng(5)
    n = 1500
    dirs = rng.standard_normal((n, 3)).astype(np.float32)
    coeffs = rng.standard_normal((n, K, 3)).astype(np.float32)
    vcol = rng.standard_normal((n, 3)).astype(np.float32)
    masks = rng.random(n) > 0.3
    d, c, v, m = (torch.from_numpy(x).to(cuda_device) for x in (dirs, coeffs, vcol, masks))
    col = native.spherical_harmonics_fwd(deg, d, c, m).cpu().numpy()
    ref = orc.sh_fwd(deg, dirs, coeffs, masks)
    np.testing.assert_allclose(col[masks], ref[masks], rtol=1e-4, atol=1e-4)
    v_coeffs, v_dirs = native.spherical_harmonics_bwd(K, deg, d, c, m, v, True)
    rc, rd = orc.sh_bwd(deg, dirs, coeffs, masks, vcol)
    np.testing.assert_allclose(v_coeffs.cpu().numpy(), rc, rtol=1e-4, atol=1e-4)  # incl. zeros for masked / inactive
    np.testing.assert_allclose(v_dirs.cpu().numpy(), rd, rtol=1e-4, atol=2e-4)
    v_coeffs2, v_dirs2 = native.spherical_harmonics_bwd(K, deg, d, c, m, v, False)
    assert v_dirs2 is None and torch.equal(v_coeffs2, v_coeffs)


# ------------------------------------------------------------------------------------------
# a1: UT projection
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["a", "small_rot", "b20k"])
def test_projection_vs_oracle(native, orc, cuda_device, scene):
    sc = {"a": lambda: scenes.scene_a(), "small_rot": lambda: scenes.scene_small(N=5000, view=3),
          "b20k": lambda: scenes.scene_b(N=20000, view=2)}[scene]()
    t = to_dev(sc, cuda_device)
    radii, means2d, depths, conics, comp = native.projection_ut_3dgs_fused(
        t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], sc["width"], sc["height"],
        0.3, 0.01, 1e4, 0.0, calc_compensations=True)
    r_ref, m_ref, d_ref, c_ref, comp_ref = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"],
                                                            sc["viewmats"], sc["Ks"], sc["width"], sc["height"], 0.3,
                                                            0.01, 1e4, 0.0, calc_compensations=True)
    radii = radii.cpu().numpy()
    assert radii.dtype == np.int32 and radii.shape == r_ref.shape
    mism = int((radii != r_ref).any(-1).sum())
    # same operation order as the oracle: only ceil()/cull borderline flips (libm vs CUDA logf/sinf) may differ
    assert mism <= max(2, radii.shape[1] // 2000), mism
    both = ((radii > 0).all(-1) & (r_ref > 0).all(-1))
    assert both.sum() > 0.5 * radii.shape[1]
    np.testing.assert_allclose(means2d.cpu().numpy()[both], m_ref[both], rtol=1e-5, atol=2e-3)
    np.testing.assert_allclose(depths.cpu().numpy()[both], d_ref[both], rtol=1e-5, atol=1e-5)
    assert rel(conics.cpu().numpy()[both], c_ref[both]) < 1e-4
    np.testing.assert_allclose(comp.cpu().numpy()[both], comp_ref[both], rtol=1e-4, atol=1e-5)
    # without opacities / compensations
    r2, _, _, _, comp2 = native.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], None, t["viewmats"],
                                                         t["Ks"], sc["width"], sc["height"], 0.3, 0.01, 1e4, 0.0)
    r2_ref = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], None, sc["viewmats"], sc["Ks"], sc["width"],
                               sc["height"], 0.3, 0.01, 1e4, 0.0)[0]
    assert comp2 is None
    assert int((r2.cpu().numpy() != r2_ref).any(-1).sum()) <= max(2, radii.shape[1] // 2000)


def test_projection_accepts_offset_views(native, cuda_device):
    """Contiguous views with a 4- / 12-byte storage offset (means[1:], opacities[1:] ...) are valid inputs of the
    reference op (CHECK_INPUT only tests contiguity); the TMA staging path needs 16-byte aligned bases and must
    not be taken for them."""
    sc = scenes.scene_b(N=3001, width=640, height=360, view=1, scale_mul=3.0)
    t = to_dev(sc, cuda_device)
    args = lambda sl: (t["means"][sl], t["quats"][sl], t["scales"][sl], t["opacities"][sl], t["viewmats"], t["Ks"],
                       sc["width"], sc["height"], 0.3, 0.01, 1e4, 0.0)
    whole = native.projection_ut_3dgs_fused(*args(slice(None)))
    view = native.projection_ut_3dgs_fused(*args(slice(1, None)))  # 3000 rows starting 12 / 16 / 4 bytes in
    assert t["means"][1:].data_ptr() % 16 != 0 and t["means"][1:].is_contiguous()
    torch.cuda.synchronize()
    vis = (whole[0][:, 1:] > 0).all(-1)
    assert torch.equal(view[0], whole[0][:, 1:])
    assert torch.equal(view[1][vis], whole[1][:, 1:][vis]) and torch.equal(view[2][vis], whole[2][:, 1:][vis])
    assert torch.equal(view[3][vis], whole[3][:, 1:][vis]) and int(vis.sum()) > 500


# ------------------------------------------------------------------------------------------
# a7/a8: blend forward / backward, fed with the ORACLE's isect lists and colours
# ------------------------------------------------------------------------------------------
def _blend_case(name):
    if name == "a":
        return scenes.scene_a(background=False)
    if name == "small_rot":
        return scenes.scene_small(N=3000, width=200, height=120, view=1)
    if name == "b30k":
        return scenes.scene_b(N=30000, width=640, height=360, view=3, scale_mul=2.0)
    if name == "one_visible":  # the intersect stage's depth sort skips all four passes (tests/isect_fixtures.py)
        return scenes.scene_one_visible()
    if name == "wall":  # the same, and every tile's order is decided by the ties of equal depths
        return scenes.scene_wall()
    raise KeyError(name)


@pytest.mark.parametrize("name", ["a", "small_rot", "b30k"])
def test_blend_fwd_bwd_vs_oracle(native, orc, cuda_device, name):
    sc = _blend_case(name)
    W, H = sc["width"], sc["height"]
    rng = np.random.default_rng(2)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    ref = orc.render_pipeline(sc, "f32", True, vrc, vra)
    ref64 = orc.render_pipeline(sc, "f64", True, vrc, vra)
    t = to_dev(sc, cuda_device)
    colors = torch.from_numpy(ref["colors"]).to(cuda_device)
    off = torch.from_numpy(ref["tile_offsets"]).to(cuda_device)
    flat = torch.from_numpy(ref["flatten_ids"]).to(cuda_device)
    bg = t.get("background")
    renders, alphas, last_ids = native.rasterize_to_pixels_from_world_3dgs_fwd(
        t["means"], t["quats"], t["scales"], colors, t["opacities"][None], bg, None, W, H, 16, t["viewmats"], t["Ks"],
        off, flat)
    r, a, li = renders.cpu().numpy(), alphas.cpu().numpy(), last_ids.cpu().numpy()
    assert r.shape == (1, H, W, 3) and a.shape == (1, H, W, 1) and li.dtype == np.int32
    e_img, e_alpha = rel(r, ref["renders"]), rel(a, ref["alphas"])
    noise = rel(ref["renders"], ref64["renders"]) if np.array_equal(ref["flatten_ids"], ref64["flatten_ids"]) else 0
    print(f"[{name}] rel_l2 image {e_img:.2e} alpha {e_alpha:.2e} (oracle f32-vs-f64 noise {noise:.2e}); "
          f"last_ids mismatches {(li != ref['last_ids']).mean():.2e}")
    assert e_img < 1e-4 and e_alpha < 1e-4
    assert np.abs(r - ref["renders"]).max() < 2e-2           # a 1/255-cut flip moves a pixel by <= alpha*colour
    assert (np.abs(r - ref["renders"]).max(-1) > 1e-4).mean() < 2e-3
    assert (li != ref["last_ids"]).mean() < 2e-3

    g = native.rasterize_to_pixels_from_world_3dgs_bwd(
        t["means"], t["quats"], t["scales"], colors, t["opacities"][None], bg, None, W, H, 16, t["viewmats"], t["Ks"],
        off, flat, torch.from_numpy(ref["alphas"]).to(cuda_device), torch.from_numpy(ref["last_ids"]).to(cuda_device),
        torch.from_numpy(vrc).to(cuda_device), torch.from_numpy(vra).to(cuda_device))
    names = ("v_means", "v_quats", "v_scales", "v_colors", "v_opacities")
    n_g = sc["means"].shape[0]
    for nm, gt in zip(names, g):
        got = gt.cpu().numpy().reshape(ref64[nm].shape)
        n32 = rel(ref[nm], ref64[nm])
        # whole-tensor 1e-3 AND per-Gaussian bounds (tests/parity.py)
        assert_grad_close(got, ref64[nm], nm, n_g, tag=f"{name} vs f64 oracle; f32 oracle itself {n32:.1e}")
        # untouched Gaussians get exact zeros
        untouched = np.abs(ref64[nm]).reshape(n_g, -1).sum(-1) == 0
        assert np.all(got.reshape(n_g, -1)[untouched] == 0)


def test_blend_masks_no_background_and_ragged_image(native, orc, cuda_device):
    sc = scenes.scene_small(N=1500, width=150, height=70, view=5)  # neither dimension a multiple of 16
    sc["background"] = None
    W, H = sc["width"], sc["height"]
    ref = orc.render_pipeline(sc, "f32")
    t = to_dev(sc, cuda_device)
    tw, th = (W + 15) // 16, (H + 15) // 16
    masks = np.ones((1, th, tw), bool)
    masks[0, 1, 2] = False
    masks[0, 0, 0] = False
    colors = torch.from_numpy(ref["colors"]).to(cuda_device)
    off = torch.from_numpy(ref["tile_offsets"]).to(cuda_device)
    flat = torch.from_numpy(ref["flatten_ids"]).to(cuda_device)
    rm, am, lm = orc.raster_fwd(sc["means"], sc["quats"], sc["scales"], ref["colors"], sc["opacities"][None], None, masks,
                                W, H, 16, sc["viewmats"], sc["Ks"], ref["tile_offsets"], ref["flatten_ids"])
    renders = torch.full((1, H, W, 3), -7.0, device=cuda_device)
    r, a, li = native.rasterize_to_pixels_from_world_3dgs_fwd(
        t["means"], t["quats"], t["scales"], colors, t["opacities"][None], None, torch.from_numpy(masks).to(cuda_device),
        W, H, 16, t["viewmats"], t["Ks"], off, flat)
    keep = np.repeat(np.repeat(masks[0], 16, 0), 16, 1)[:H, :W]
    assert rel(r.cpu().numpy()[0][keep], rm[0][keep]) < 1e-4
    assert np.all(r.cpu().numpy()[0][~keep] == 0)  # masked tiles: background (none -> 0) only
    assert rel(a.cpu().numpy()[0][keep], am[0][keep]) < 1e-4
    # backward ignores masked tiles
    rng = np.random.default_rng(3)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    gref = orc.raster_bwd(sc["means"], sc["quats"], sc["scales"], ref["colors"], sc["opacities"][None], None, masks, W, H,
                          16, sc["viewmats"], sc["Ks"], ref["tile_offsets"], ref["flatten_ids"], am, lm, vrc, vra,
                          precision="f64")
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(
        t["means"], t["quats"], t["scales"], colors, t["opacities"][None], None, torch.from_numpy(masks).to(cuda_device),
        W, H, 16, t["viewmats"], t["Ks"], off, flat, torch.from_numpy(am).to(cuda_device),
        torch.from_numpy(lm).to(cuda_device), torch.from_numpy(vrc).to(cuda_device), torch.from_numpy(vra).to(cuda_device))
    for nm, got, want in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g, gref):
        assert_grad_close(got.cpu().numpy().reshape(want.shape), want, nm, sc["means"].shape[0], tag="masked tiles")


def test_blend_empty_inputs(native, cuda_device):
    dev = cuda_device
    W, H = 64, 48
    vm = torch.eye(4, device=dev)[None]
    K = torch.tensor([[[50.0, 0, 32], [0, 50.0, 24], [0, 0, 1]]], device=dev)
    means = torch.zeros(5, 3, device=dev); means[:, 2] = 3
    quats = torch.tensor([[1.0, 0, 0, 0]], device=dev).repeat(5, 1)
    scales = torch.full((5, 3), 0.1, device=dev)
    colors = torch.rand(1, 5, 3, device=dev)
    opac = torch.full((1, 5), 0.5, device=dev)
    off = torch.zeros(1, 3, 4, dtype=torch.int32, device=dev)
    flat = torch.zeros(0, dtype=torch.int32, device=dev)
    bg = torch.tensor([[0.1, 0.2, 0.3]], device=dev)
    r, a, li = native.rasterize_to_pixels_from_world_3dgs_fwd(means, quats, scales, colors, opac, bg, None, W, H, 16, vm,
                                                              K, off, flat)
    assert torch.allclose(r, bg.view(1, 1, 1, 3).expand(1, H, W, 3)) and float(a.abs().max()) == 0 and int(li.abs().max()) == 0
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(means, quats, scales, colors, opac, bg, None, W, H, 16, vm, K, off,
                                                       flat, a, li, torch.ones_like(r), torch.ones_like(a))
    assert all(float(x.abs().max()) == 0 for x in g)


# ------------------------------------------------------------------------------------------
# whole path through the L3 mirror (autograd), against the oracle pipeline
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small_rot", "a", "b30k", "one_visible", "wall"])
def test_pipeline_autograd_vs_oracle(native, orc, cuda_device, name):
    """Whole L3 path (SH -> intersect -> blend and the autograd chain back to every parameter) against the oracle
    pipeline.  Both sides are given the SAME projection outputs (the oracle's): a radius that flips at a ceil()
    boundary between two float implementations changes the intersection lists and makes an element-wise comparison
    meaningless -- that effect is counted separately in test_projection_vs_oracle -- so the test asserts on every run."""
    sc = _blend_case(name)
    W, H = sc["width"], sc["height"]
    rng = np.random.default_rng(4)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    ref = orc.render_pipeline(sc, "f32", True, vrc, vra)
    ref64 = orc.render_pipeline(sc, "f64", False)
    same64 = np.array_equal(ref64["flatten_ids"], ref["flatten_ids"])
    if same64:
        orc.backward_pipeline(sc, ref64, vrc, vra, "f64")
    t = to_dev(sc, cuda_device)
    vis = (ref["radii"] > 0).all(-1)
    proj = (torch.from_numpy(ref["radii"]).to(cuda_device),
            torch.from_numpy(np.where(vis[..., None], ref["means2d"], 0).astype(np.float32)).to(cuda_device),
            torch.from_numpy(np.where(vis, ref["depths"], 0).astype(np.float32)).to(cuda_device))
    leaves = {k: t[k].clone().requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh_coeffs")}
    out = native.rasterize(leaves["means"], leaves["quats"], leaves["scales"], leaves["opacities"], leaves["sh_coeffs"],
                           sc["sh_degree"], t["viewmats"], t["Ks"], W, H, bg_color=t.get("background"), projection=proj)
    assert out.n_isects == len(ref["flatten_ids"])
    loss = (out.render_colors * torch.from_numpy(vrc).to(cuda_device)).sum() + \
           (out.alpha.permute(1, 2, 0)[None] * torch.from_numpy(vra).to(cuda_device)).sum()
    loss.backward()
    assert rel(out.render_colors.detach().cpu().numpy(), ref["renders"]) < 1e-4
    truth = ref64 if same64 else ref  # float64 arithmetic on the same lists when the f64 projection agrees
    n_g = sc["means"].shape[0]
    want = {"means": truth["v_means"] + truth["v_dirs"][0], "quats": truth["v_quats"], "scales": truth["v_scales"],
            "opacities": truth["v_opacities"][0], "sh_coeffs": truth["v_sh_coeffs"]}
    for k, w in want.items():
        assert_grad_close(leaves[k].grad, w, k, n_g, tag=f"pipeline {name} vs {'f64' if same64 else 'f32'} oracle")


def test_host_staged_steps_match_sequential_steps(native, cuda_device):
    """The three-stream host pipeline (hoststream.py) returns, for every step, exactly what a blocking
    copy-in / step / copy-out sequence returns: same loss, same image, same gradients (bit for bit -- the
    kernels and their inputs are the same; only the copies overlap)."""
    from gsplat_b200 import hoststream
    sc = _blend_case("small_rot")
    W, H = sc["width"], sc["height"]
    names = ("means", "quats", "scales", "opacities", "sh_coeffs")
    host = {k: torch.from_numpy(np.ascontiguousarray(sc[k])).pin_memory()
            for k in names + ("viewmats", "Ks", "background")}
    host["target"] = torch.from_numpy(np.random.default_rng(9).random((1, H, W, 3), dtype=np.float32)).pin_memory()

    def step(Pd):
        for k in names:
            Pd[k].grad = None
        out = native.rasterize(Pd["means"], Pd["quats"], Pd["scales"], Pd["opacities"], Pd["sh_coeffs"],
                               sc["sh_degree"], Pd["viewmats"], Pd["Ks"], W, H, bg_color=Pd["background"])
        loss = (out.render_colors - Pd["target"]).abs().mean()
        loss.backward()
        return loss, out.render_colors

    Pd = {k: host[k].to(cuda_device).requires_grad_(k in names) for k in host}
    loss, img = step(Pd)
    want = {k: Pd[k].grad.cpu() for k in names}
    staged = hoststream.HostStagedSteps(cuda_device, host, names, step)
    losses = staged.run(5)
    assert len(losses) == 5
    # blend gradients are accumulated with float atomics: equal up to summation order
    want_loss = float(loss.item())
    assert all(abs(l - want_loss) <= 1e-6 * abs(want_loss) for l in losses)
    for slot in (0, 1):
        assert torch.equal(staged.host_img[slot], img.detach().cpu())
        for k in names:
            assert rel(staged.host_grads[slot][k].numpy(), want[k].numpy()) < 1e-5
    assert staged.h2d_bytes == sum(t.numel() * t.element_size() for t in host.values())


# ------------------------------------------------------------------------------------------
# multi-GPU exchange step (SURVEY.md 8e): multi-view SH backward and the deferred L3 path
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,deg", [(16, 3), (16, 1), (16, 0), (25, 4), (9, 2)])
def test_sh_bwd_views_equals_sum_of_single_view_backwards(native, orc, cuda_device, K, deg):
    rng = np.random.default_rng(21)
    M, V = 5003, 3
    means = rng.standard_normal((M, 3)).astype(np.float32) * 3
    campos = rng.standard_normal((V, 3)).astype(np.float32) * 6
    coeffs = rng.standard_normal((M, K, 3)).astype(np.float32)
    vc = rng.standard_normal((V, M, 3)).astype(np.float32)
    vc[rng.random((V, M)) < 0.5] = 0.0  # not blended in that view
    vm0 = rng.standard_normal((M, 3)).astype(np.float32)
    want_c = np.zeros_like(coeffs, dtype=np.float64)
    want_m = vm0.astype(np.float64)
    for v in range(V):
        a, b = orc.sh_bwd(deg, means - campos[v], coeffs, None, vc[v], True, precision="f64")
        want_c += a
        want_m += b
    d = lambda x: torch.from_numpy(x).to(cuda_device)
    v_means = d(vm0.copy())
    got_c = native.default_backend().spherical_harmonics_bwd_views(deg, d(means), d(campos), d(coeffs), d(vc), v_means)
    assert rel(got_c.cpu().numpy(), want_c) < 1e-5
    assert rel(v_means.cpu().numpy(), want_m) < 1e-5
    # also against the product's own single-view op (same arithmetic per view, sums in a different order)
    acc = torch.zeros_like(got_c)
    for v in range(V):
        a, _ = native.spherical_harmonics_bwd(K, deg, d(means - campos[v]), d(coeffs), None, d(vc[v]), True)
        acc += a
    assert rel(got_c.cpu().numpy(), acc.cpu().numpy()) < 1e-6


def test_deferred_sh_exchange_single_rank_equals_plain_backward(native, cuda_device):
    """rasterize(..., sh_exchange=...) + exchange_gradients_compact at world size 1 == the plain autograd path."""
    from gsplat_b200 import multiview as mv
    sc = _blend_case("small_rot")
    W, H = sc["width"], sc["height"]
    names = ("means", "quats", "scales", "opacities", "sh_coeffs")
    t = to_dev(sc, cuda_device)
    target = torch.rand((1, H, W, 3), device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(3))

    def run(deferred):
        P = {k: t[k].clone().requires_grad_(True) for k in names}
        out = native.rasterize(P["means"], P["quats"], P["scales"], P["opacities"], P["sh_coeffs"], sc["sh_degree"],
                               t["viewmats"], t["Ks"], W, H, bg_color=t.get("background"), sh_exchange=deferred)
        (out.render_colors - target).abs().mean().backward()
        if deferred is not None:
            assert P["sh_coeffs"].grad is None and deferred.v_colors.shape == (P["means"].shape[0], 3)
            mv.exchange_gradients_compact(P, deferred)
        return {k: P[k].grad.cpu().numpy() for k in names}

    plain = run(None)
    compact = run(native.DeferredSHBackward())
    for k in names:
        assert rel(compact[k], plain[k]) < 2e-5, k


# ------------------------------------------------------------------------------------------
# link-surface ops
# ------------------------------------------------------------------------------------------
def test_strategy_helpers_vs_oracle(native, orc, cuda_device):
    rng = np.random.default_rng(6)
    n = 4097
    q = rng.standard_normal((n, 4)).astype(np.float32)
    R = native.quats_to_rotmats(torch.from_numpy(q).to(cuda_device)).cpu().numpy()
    np.testing.assert_allclose(R, orc.quat_to_rotmat(q), rtol=1e-5, atol=1e-5)
    # relocation (tests/test_gsplat_ops.cpp:19-63 recipe: binomial table, ratios in [1, n_max])
    n_max = 8
    binoms = np.zeros((n_max, n_max), np.float32)
    for i in range(n_max):
        for k in range(i + 1):
            binoms[i, k] = math.comb(i, k)
    op = (rng.random(n) * 0.8 + 0.1).astype(np.float32)
    sc = (rng.random((n, 3)) * 0.1 + 0.01).astype(np.float32)
    ratios = rng.integers(1, n_max + 1, n).astype(np.int32)
    no, ns = native.relocation(*(torch.from_numpy(x).to(cuda_device) for x in (op, sc, ratios, binoms)), n_max)
    ro, rs = orc.relocation(op, sc, ratios, binoms, n_max)
    np.testing.assert_allclose(no.cpu().numpy(), ro, rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(ns.cpu().numpy(), rs, rtol=2e-4, atol=1e-6)
    assert np.all(no.cpu().numpy() <= op + 1e-6) and np.all(no.cpu().numpy() > 0)
    # add_noise
    raw_op = rng.standard_normal(n).astype(np.float32) * 3
    raw_sc = np.log(sc)
    noise = rng.standard_normal((n, 3)).astype(np.float32)
    means = rng.standard_normal((n, 3)).astype(np.float32)
    m_dev = torch.from_numpy(means.copy()).to(cuda_device)
    native.add_noise(*(torch.from_numpy(x).to(cuda_device) for x in (raw_op, raw_sc, q, noise)), m_dev, 0.5)
    np.testing.assert_allclose(m_dev.cpu().numpy(), orc.add_noise(raw_op, raw_sc, q, noise, means, 0.5), rtol=1e-5,
                               atol=1e-6)


def test_unsupported_configurations_fail_loudly(native, cuda_device):
    sc = scenes.scene_small(N=64)
    t = to_dev(sc, cuda_device)
    with pytest.raises(RuntimeError, match="not supported"):  # orthographic: rejected by the reference too
        native.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"],
                                        sc["width"], sc["height"], camera_model=native.ORTHO)
    with pytest.raises(RuntimeError, match="CUDA"):
        native.quats_to_rotmats(torch.randn(4, 4))


# ------------------------------------------------------------------------------------------
# a2: distorted camera models (OpenCV pinhole with radial/tangential/thin-prism, OpenCV fisheye)
# ------------------------------------------------------------------------------------------
DISTORTED = {
    "opencv": dict(camera_model=0, radial=np.array([[-0.12, 0.05, 0.002, 0.01, -0.003, 0.0005]], np.float32),
                   tangential=np.array([[0.002, -0.001]], np.float32),
                   thin_prism=np.array([[0.001, 0.0002, -0.0005, 0.0001]], np.float32)),
    "fisheye": dict(camera_model=2, radial=np.array([[0.03, -0.004, 0.0007, -0.0001]], np.float32), tangential=None,
                    thin_prism=None),
}


@pytest.mark.parametrize("model", ["opencv", "fisheye"])
def test_distorted_camera_whole_path_vs_oracle(native, orc, cuda_device, model):
    cfg = DISTORTED[model]
    sc = scenes.scene_small(N=2500, width=208, height=128, view=2)
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    okw = dict(camera_model=cfg["camera_model"], radial=cfg["radial"], tangential=cfg["tangential"],
               thin_prism=cfg["thin_prism"])
    dev = lambda a: None if a is None else torch.from_numpy(a).to(cuda_device)
    nkw = dict(camera_model=cfg["camera_model"], radial_coeffs=dev(cfg["radial"]), tangential_coeffs=dev(cfg["tangential"]),
               thin_prism_coeffs=dev(cfg["thin_prism"]))
    t = to_dev(sc, cuda_device)
    # projection
    r_ref, m_ref, d_ref, c_ref, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"],
                                                      sc["viewmats"], sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **okw)
    radii, means2d, depths, conics, _ = native.projection_ut_3dgs_fused(
        t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **nkw)
    mism = int((radii.cpu().numpy() != r_ref).any(-1).sum())
    assert mism <= 3, mism
    both = (radii.cpu().numpy() > 0).all(-1) & (r_ref > 0).all(-1)
    assert both.sum() > 1000
    assert rel(means2d.cpu().numpy()[both], m_ref[both]) < 1e-4
    # blend forward / backward on the oracle's lists
    tpg, ids, flat = orc.isect_tiles(m_ref, r_ref, d_ref, 1, 16, tw, th)
    off = orc.isect_offsets(ids, 1, tw, th)
    rng = np.random.default_rng(21)
    colors = rng.random((1, sc["means"].shape[0], 3), dtype=np.float32)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    img, alp, li = orc.raster_fwd(sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None],
                                  sc["background"], None, W, H, 16, sc["viewmats"], sc["Ks"], off, flat, **okw)
    fa = (t["means"], t["quats"], t["scales"], torch.from_numpy(colors).to(cuda_device), t["opacities"][None],
          t["background"], None, W, H, 16, t["viewmats"], t["Ks"], torch.from_numpy(off).to(cuda_device),
          torch.from_numpy(flat).to(cuda_device))
    r, a, l = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **nkw)
    e = rel(r.cpu().numpy(), img)
    print(f"[{model}] image rel_l2 {e:.2e}, last_ids differ {(l.cpu().numpy() != li).mean():.2e}")
    assert e < 1e-4 and rel(a.cpu().numpy(), alp) < 1e-4
    assert (l.cpu().numpy() != li).mean() < 3e-3
    g_ref = orc.raster_bwd(sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None], sc["background"], None,
                           W, H, 16, sc["viewmats"], sc["Ks"], off, flat, alp, li, vrc, vra, precision="f64", **okw)
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, torch.from_numpy(alp).to(cuda_device),
                                                       torch.from_numpy(li).to(cuda_device),
                                                       torch.from_numpy(vrc).to(cuda_device),
                                                       torch.from_numpy(vra).to(cuda_device), **nkw)
    for nm, got, want in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g, g_ref):
        assert_grad_close(got.cpu().numpy().reshape(want.shape), want, nm, sc["means"].shape[0],
                          tag=f"{model} vs f64 oracle")
