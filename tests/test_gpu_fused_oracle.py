"""GPU: rasterize_fused -- the raw-parameter path every training step runs (csrc/gsb_fused.cu front and back around
the intersect and blend kernels) -- against the float64 restatement of fused_restatement.py, in the configurations
training and the viewer put it in: partial SH degrees on K = 16 storage, a scaling modifier, unnormalised quaternions,
clamped colours, a camera inside the cloud, distorted lenses and no background.

The other fused tests compare the kernels with the unfused CUDA path, which shares the projection, the blend and the
SH basis with them and applies the scaling modifier in Python; here nothing on the reference side is CUDA.  Each case
prints the float32 oracle's own distance from float64 beside the kernel's."""
import numpy as np
import pytest
import torch

import fused_restatement as fr
import scenes
from parity import rel
from test_gpu_blend_wide import assert_close_as_f32

pytestmark = pytest.mark.gpu
C0 = 0.2820947917738781  # SH basis of degree 0
NEAR = 0.01  # the operators' default near plane
N, W, H = 3000, 200, 120

BASE = dict(deg=3, K=16, modifier=1.0, unit=True, clamp=False, inside=False, camera="pinhole", bg=True)
CASES = {
    # each SH layout once at the baseline: degrees 0..2 on K = 16 storage are what training runs before its last step up
    "sh0_k1": dict(deg=0, K=1), "sh0_k16": dict(deg=0, K=16), "sh1_k16": dict(deg=1, K=16),
    "sh2_k16": dict(deg=2, K=16), "sh3_k16": dict(), "sh4_k25": dict(deg=4, K=25), "sh2_k25": dict(deg=2, K=25),
    # the viewer's scaling modifier, with the unit and the stored (unnormalised) quaternions
    "mod0.5": dict(modifier=0.5), "mod1.7": dict(modifier=1.7), "unnorm": dict(unit=False),
    "unnorm_mod0.5": dict(unit=False, modifier=0.5), "unnorm_mod1.7": dict(unit=False, modifier=1.7),
    # colours below -0.5 in at least one channel
    "clamp": dict(clamp=True), "clamp_sh1_unnorm_mod0.5": dict(clamp=True, deg=1, unit=False, modifier=0.5),
    # the camera inside the cloud: Gaussians behind it and at its near plane
    "inside_mod0.5": dict(inside=True, unit=False, modifier=0.5),
    "inside_mod1.7": dict(inside=True, unit=False, modifier=1.7),
    "opencv": dict(camera="opencv"), "fisheye": dict(camera="fisheye"), "no_background": dict(bg=False),
}


@pytest.fixture(scope="module")
def threads(orc):
    orc.set_threads(orc.max_threads())


def _scene(cfg, seed):
    """A scene dict (activated parameters, scenes.py's layout) with K coefficients per Gaussian."""
    if cfg["inside"]:
        sc = scenes.scene_small(N=N, width=W, height=H, sh_degree=cfg["deg"], seed=seed)
        sc["viewmats"] = scenes.look_at((0.2, 0.1, 2.9), (0.6, 0.0, 4.0))[None]
        # 2 % of the Gaussians within 2 x near_plane of the camera, half of them in front of it and inside the frustum
        # (those at depth 0.01 .. 0.017 project, with radii of tens of pixels); small, so that they do not hide the rest
        rng = np.random.default_rng(seed + 1)
        idx = rng.choice(N, N // 50, replace=False)
        z = rng.uniform(-0.017, 0.017, len(idx))
        pc = np.stack([z * rng.uniform(-0.5, 0.5, len(idx)), z * rng.uniform(-0.3, 0.3, len(idx)), z], -1)
        V = sc["viewmats"][0].astype(np.float64)
        sc["means"][idx] = ((pc - V[:3, 3]) @ V[:3, :3]).astype(np.float32)
        sc["scales"][idx] = rng.uniform(0.0005, 0.003, (len(idx), 3)).astype(np.float32)
    else:
        sc = scenes.scene_small(N=N, width=W, height=H, sh_degree=cfg["deg"], seed=seed, view=1)
    rng = np.random.default_rng(seed + 2)
    sc["sh_coeffs"] = ((rng.random((N, cfg["K"], 3)) - 0.5) * 0.3).astype(np.float32)
    if cfg["clamp"]:
        # 22 % of the Gaussians get one channel well below -0.5 whatever the view-dependent terms add
        idx = rng.choice(N, N // 5 + N // 50, replace=False)
        sc["sh_coeffs"][idx, 0, rng.integers(0, 3, len(idx))] = ((-0.5 - rng.uniform(0.3, 0.8, len(idx))) / C0)
    if not cfg["bg"]:
        sc["background"] = None
    return sc


def _raw(sc, cfg, seed):
    rng = np.random.default_rng(seed + 3)
    q = sc["quats"] if cfg["unit"] else sc["quats"] * rng.uniform(0.3, 3.0, (N, 1)).astype(np.float32)
    o = sc["opacities"].astype(np.float64)
    return dict(means=sc["means"], sh0=np.ascontiguousarray(sc["sh_coeffs"][:, :1]),
                shN=np.ascontiguousarray(sc["sh_coeffs"][:, 1:]), scaling_raw=np.log(sc["scales"]),
                rotation_raw=q.astype(np.float32), opacity_raw=np.log(o / (1 - o)).astype(np.float32)[:, None])


def _camera(name, dev):
    if name == "pinhole":
        return {}, {}
    from test_gpu_parity import DISTORTED
    c = DISTORTED[name]
    d = lambda a: None if a is None else torch.from_numpy(a).to(dev)
    return (dict(camera_model=c["camera_model"], radial=c["radial"], tangential=c["tangential"],
                 thin_prism=c["thin_prism"]),
            dict(camera_model=c["camera_model"], radial_coeffs=d(c["radial"]), tangential_coeffs=d(c["tangential"]),
                 thin_prism_coeffs=d(c["thin_prism"])))


def _image_close(got, want, w32, tag):
    """[1,H,W,C] against the float64 forward.  A pixel where a Gaussian's alpha >= 1/255 cut or a radius flips between
    float32 and float64 moves by up to about 1e-3: at most max(10, twice the float32 oracle's count) pixels may move by
    more than 1e-4.  Over the other pixels the relative L2 error stays below the larger of 1e-5 and twice the float32
    oracle's; the second is larger only with the camera in the cloud, where a Gaussian's float32 camera-space depth
    near the near plane carries a relative rounding error of ~1e-5."""
    d, d32 = (np.abs(x - want).max(-1)[0] for x in (got, w32))
    flip, flip32 = d > 1e-4, d32 > 1e-4
    bulk = lambda x, f: float(np.linalg.norm((x - want)[0][~f]) / np.linalg.norm(want))
    e, e32 = bulk(got, flip), bulk(w32, flip32)
    print(f"[{tag}] vs f64: rel_l2 {rel(got, want):.2e} (f32 oracle {rel(w32, want):.2e}); {int(flip.sum())} pixels off by "
          f"> 1e-4 (f32 oracle {int(flip32.sum())}), the largest {float(d.max()):.1e}; rel_l2 of the others {e:.2e} "
          f"(f32 oracle {e32:.2e})")
    assert e < max(1e-5, 2.0 * e32)
    assert flip.sum() <= max(10, 2 * flip32.sum()) and d.max() < 2e-2


@pytest.mark.parametrize("case", list(CASES))
def test_fused_vs_f64_restatement(native, orc, cuda_device, threads, case):
    cfg = dict(BASE, **CASES[case])
    seed = sorted(CASES).index(case) * 10 + 100
    sc = _scene(cfg, seed)
    raw = _raw(sc, cfg, seed)
    deg, mod, nb = cfg["deg"], cfg["modifier"], (cfg["deg"] + 1) ** 2
    okw, nkw = _camera(cfg["camera"], cuda_device)
    rng = np.random.default_rng(seed + 4)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    args = (raw, deg, sc["viewmats"], sc["Ks"], W, H, sc["background"], vrc, vra, mod)
    o64, want = fr.render_raw(orc, *args, precision="f64", **okw)
    o32, w32 = fr.render_raw(orc, *args, precision="f32", **okw)

    if cfg["inside"]:
        V = sc["viewmats"][0].astype(np.float64)
        zc = sc["means"] @ V[:3, :3].T + V[:3, 3]
        behind, near = float((zc[:, 2] < 0).mean()), float((np.linalg.norm(zc, axis=-1) < 2 * NEAR).mean())
        near_vis = int((o64["masks"][0] & (np.linalg.norm(zc, axis=-1) < 2 * NEAR)).sum())
        print(f"[{case}] behind the camera {behind:.1%}, within 2 x near_plane {near:.1%} ({near_vis} of them visible)")
        assert behind >= 0.10 and near >= 0.01 and near_vis >= 3
    vis64 = o64["masks"][0]
    clamped = (o64["sh_colors"][0] + 0.5 < 0).any(-1)
    frac = float(clamped[vis64].mean())
    print(f"[{case}] {int(vis64.sum())} of {N} visible, {frac:.1%} of them with a clamped channel")
    if cfg["clamp"]:
        assert 0.15 <= frac <= 0.30

    t = {k: torch.from_numpy(v).to(cuda_device) for k, v in sc.items() if isinstance(v, np.ndarray)}
    P = {k: torch.from_numpy(v).to(cuda_device).requires_grad_(True) for k, v in raw.items()}
    o = native.rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                               deg, t["viewmats"], t["Ks"], W, H, bg_color=t.get("background"), scaling_modifier=mod,
                               **nkw)
    ((o.render_colors * torch.from_numpy(vrc).to(cuda_device)).sum() +
     (o.alpha * torch.from_numpy(vra).to(cuda_device)).sum()).backward()
    torch.cuda.synchronize()

    # projection: only borderline ceil() / cull flips between float32 and float64.  Tile counts differ where a radius
    # flipped or a centre sits within rounding of a tile edge.  The float32 oracle flips up to 2 of the 3000 radii and
    # 3 tile counts in these cases (printed), so the bound is 0.2 % of the Gaussians rather than max(2, N / 2000).
    radii, m2d, depths = (x.detach().cpu().numpy() for x in (o.radii, o.means2d, o.depths))
    tw, th = (W + 15) // 16, (H + 15) // 16
    tpg, _, flat = orc.isect_tiles(m2d, radii, depths, 1, 16, tw, th)
    mism, mism32 = (int((r != o64["radii"]).any(-1).sum()) for r in (radii, o32["radii"]))
    tpg_off, tpg_off32 = (int((t_ != o64["tiles_per_gauss"]).sum()) for t_ in (tpg, o32["tiles_per_gauss"]))
    n_is = int(o.n_isects.item())
    print(f"[{case}] vs f64: radii differ for {mism} Gaussians (f32 oracle {mism32}), tile counts for {tpg_off} "
          f"(f32 oracle {tpg_off32}); {n_is} intersections (f64 {len(o64['flatten_ids'])}, f32 oracle "
          f"{len(o32['flatten_ids'])})")
    assert mism <= max(4, N // 500) and tpg_off <= max(4, N // 500)
    # the intersect stage's count on the kernel's own projection, exactly
    assert n_is == len(flat)

    _image_close(o.render_colors.detach().cpu().numpy(), o64["renders"], o32["renders"], f"{case} image")
    _image_close(o.alpha.detach().cpu().numpy(), o64["alphas"], o32["alphas"], f"{case} alpha")

    culled = ~(radii[0] > 0).all(-1)
    for k in fr.RAW:
        g = P[k].grad
        assert g is not None or raw[k].size == 0, k  # shN [N,0,3] at K = 1 gets no gradient
        got = np.zeros_like(raw[k]) if g is None else g.cpu().numpy()
        assert_close_as_f32(got, want[k], w32[k], k, N, case)
        # culled Gaussians get exact zeros, and so do the SH rows the active degree does not read
        assert not np.any(got[culled]), k
    if cfg["K"] > nb:
        assert not np.any(P["shN"].grad.cpu().numpy()[:, nb - 1:])
    if cfg["inside"]:
        assert culled.sum() >= 0.10 * N
