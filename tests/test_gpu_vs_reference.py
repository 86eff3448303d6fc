"""GPU: the sm_90a path and the CPU oracle against the REFERENCE's own CUDA kernels
(oracle/_ref/libgsplat_ref.so = /root/reference/gsplat/*.cu compiled unmodified with the reference's
flags; GLM provided by oracle/glm_shim).  This is the pin for the rows the reference's own tests
do not cover: UT projection and from-world blend forward / backward (SURVEY.md 8c).

Where the reference library was not built (build() makes it where the reference's sources are present),
the CPU oracle stands in for it: tests/test_oracle_vs_reference_golden.py pins the oracle to stored outputs of
those kernels, and test_gpu_vs_reference_golden.py compares this library with the stored outputs directly.  The rolling-shutter tests
here need the reference's precise build and skip without it; test_gpu_rolling_shutter.py checks that mode against the
float64 oracle and the stored outputs of the precise build everywhere."""
import os

import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, rel, to_dev

pytestmark = pytest.mark.gpu


class OracleBackend:
    """The operators of the reference computed by the CPU oracle (oracle/gut_oracle.c) on the inputs' values, returned
    on the inputs' device: the same call sites as an OpsBackend.  Global shutter only."""

    def __init__(self, orc):
        self.orc = orc

    @staticmethod
    def _np(t):
        return None if t is None else t.detach().cpu().numpy()

    @staticmethod
    def _dev(a, like):
        return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(like.device)

    def projection_ut_3dgs_fused(self, means, quats, scales, opacities, viewmats0, Ks, image_width, image_height,
                                 eps2d=0.3, near_plane=0.01, far_plane=1e10, radius_clip=0.0, calc_compensations=False,
                                 camera_model=0, ut_params=None, viewmats1=None, rs_type=0, radial_coeffs=None,
                                 tangential_coeffs=None, thin_prism_coeffs=None):
        assert viewmats1 is None and ut_params is None, "the oracle stand-in covers the global shutter, default UT"
        n = self._np
        out = self.orc.projection_ut(n(means), n(quats), n(scales), n(opacities), n(viewmats0), n(Ks), image_width,
                                     image_height, eps2d, near_plane, far_plane, radius_clip, calc_compensations,
                                     camera_model, radial=n(radial_coeffs), tangential=n(tangential_coeffs),
                                     thin_prism=n(thin_prism_coeffs))
        return tuple(self._dev(a, means) for a in out)

    def spherical_harmonics_fwd(self, degrees_to_use, dirs, coeffs, masks=None):
        return self._dev(self.orc.sh_fwd(degrees_to_use, self._np(dirs), self._np(coeffs), self._np(masks)), dirs)

    def spherical_harmonics_bwd(self, K, degrees_to_use, dirs, coeffs, masks, v_colors, compute_v_dirs=True):
        vc, vd = self.orc.sh_bwd(degrees_to_use, self._np(dirs), self._np(coeffs), self._np(masks), self._np(v_colors),
                                 compute_v_dirs)
        return self._dev(vc, dirs), self._dev(vd, dirs)

    def intersect_tile(self, means2d, radii, depths, C, tile_size, tile_width, tile_height, sort=True):
        out = self.orc.isect_tiles(self._np(means2d), self._np(radii), self._np(depths), C, tile_size, tile_width,
                                   tile_height, sort)
        return tuple(self._dev(a, means2d) for a in out)

    def intersect_offset(self, isect_ids, C, tile_width, tile_height):
        return self._dev(self.orc.isect_offsets(self._np(isect_ids), C, tile_width, tile_height), isect_ids)

    def _blend_args(self, means, quats, scales, colors, opacities, backgrounds, masks, image_width, image_height,
                    tile_size, viewmats0, Ks, tile_offsets, flatten_ids):
        n = self._np
        return (n(means), n(quats), n(scales), n(colors), n(opacities), n(backgrounds), n(masks), image_width,
                image_height, tile_size, n(viewmats0), n(Ks), n(tile_offsets), n(flatten_ids))

    def rasterize_to_pixels_from_world_3dgs_fwd(self, *a, camera_model=0, viewmats1=None, rs_type=0, radial_coeffs=None,
                                                tangential_coeffs=None, thin_prism_coeffs=None):
        assert viewmats1 is None, "the oracle stand-in covers the global shutter"
        out = self.orc.raster_fwd(*self._blend_args(*a), camera_model=camera_model, radial=self._np(radial_coeffs),
                                  tangential=self._np(tangential_coeffs), thin_prism=self._np(thin_prism_coeffs))
        return tuple(self._dev(x, a[0]) for x in out)

    def rasterize_to_pixels_from_world_3dgs_bwd(self, *a, camera_model=0, viewmats1=None, rs_type=0, radial_coeffs=None,
                                                tangential_coeffs=None, thin_prism_coeffs=None):
        assert viewmats1 is None, "the oracle stand-in covers the global shutter"
        n = self._np
        out = self.orc.raster_bwd(*self._blend_args(*a[:14]), *(n(x) for x in a[14:18]), camera_model=camera_model,
                                  precision="f64", radial=n(radial_coeffs), tangential=n(tangential_coeffs),
                                  thin_prism=n(thin_prism_coeffs))
        return tuple(self._dev(x.astype(np.float32), a[0]) for x in out)


@pytest.fixture(scope="module")
def ref(native, orc):
    from oracle import ref_ops
    if not ref_ops.available():
        return OracleBackend(orc)
    return ref_ops.backend(native)


@pytest.fixture(scope="module")
def ref_precise(native):
    """The reference's kernels compiled without --use_fast_math (oracle/build_ref.py VARIANTS)."""
    from oracle import ref_ops
    if not ref_ops.precise_available():
        pytest.skip("oracle/_ref/libgsplat_ref_precise.so not built")
    return ref_ops.backend_precise(native)


def _scene(name):
    return {"a": lambda: scenes.scene_a(background=False),
            "small_rot": lambda: scenes.scene_small(N=3000, width=200, height=120, view=1),
            "b30k": lambda: scenes.scene_b(N=30000, width=640, height=360, view=3, scale_mul=2.0),
            "b200k": lambda: scenes.scene_b(N=200000, view=5)}[name]()


@pytest.mark.parametrize("name", ["a", "small_rot", "b30k", "b200k"])
def test_projection_reference_vs_b200_and_oracle(native, ref, orc, cuda_device, name):
    sc = _scene(name)
    t = to_dev(sc, cuda_device)
    args = (t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], sc["width"], sc["height"],
            0.3, 0.01, 1e4, 0.0)
    r_ref, m_ref, d_ref, c_ref, _ = ref.projection_ut_3dgs_fused(*args)
    r_new, m_new, d_new, c_new, _ = native.projection_ut_3dgs_fused(*args)
    r_ref, r_new = r_ref.cpu().numpy(), r_new.cpu().numpy()
    N = r_ref.shape[1]
    mism = int((r_ref != r_new).any(-1).sum())
    r_orc = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"], sc["Ks"],
                              sc["width"], sc["height"], 0.3, 0.01, 1e4, 0.0)[0]
    mism_orc = int((r_ref != r_orc).any(-1).sum())
    print(f"[{name}] radii: reference vs b200 {mism}/{N} differ, reference vs oracle {mism_orc}/{N}")
    # ceil()/cull borderline flips only (fast-math vs IEEE arithmetic): a few per 10^4
    assert mism <= max(3, N // 1000) and mism_orc <= max(3, N // 1000)
    # every flipped radius is a +-1 step or a cull decision at the boundary
    d = np.abs(r_ref.astype(np.int64) - r_new.astype(np.int64))
    bad = (d > 1) & (r_ref > 0) & (r_new > 0)
    assert not bad.any()
    both = (r_ref > 0).all(-1) & (r_new > 0).all(-1)
    em = rel(m_new.cpu().numpy()[both], m_ref.cpu().numpy()[both])
    ed = rel(d_new.cpu().numpy()[both], d_ref.cpu().numpy()[both])
    ec = rel(c_new.cpu().numpy()[both], c_ref.cpu().numpy()[both])
    am = float(np.abs(m_new.cpu().numpy()[both] - m_ref.cpu().numpy()[both]).max())
    print(f"[{name}] rel_l2 b200 vs reference: means2d {em:.2e} (max abs {am:.2e} px) depths {ed:.2e} conics {ec:.2e}")
    # the UT sums seven points with weights (-99, 16.67 x 6): ~100x rounding amplification, and the
    # reference is built with --use_fast_math; north_star asks for 1e-4 relative on K1 outputs
    assert em < 1e-4 and ed < 1e-5 and ec < 1e-3


@pytest.mark.parametrize("name", ["small_rot", "b30k"])
def test_intersect_bit_exact_vs_reference(native, ref, cuda_device, name):
    sc = _scene(name)
    t = to_dev(sc, cuda_device)
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    radii, means2d, depths, _, _ = ref.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"],
                                                                t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0)
    # culled rows of means2d / depths are uninitialised in the reference: both libraries see the same bytes
    a = ref.intersect_tile(means2d, radii, depths, 1, 16, tw, th, True)
    b = native.intersect_tile(means2d, radii, depths, 1, 16, tw, th, True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert torch.equal(ref.intersect_offset(a[1], 1, tw, th), native.intersect_offset(b[1], 1, tw, th))


@pytest.mark.parametrize("name", ["a", "small_rot", "b30k"])
def test_blend_reference_vs_b200_and_oracle(native, ref, orc, cuda_device, name):
    sc = _scene(name)
    W, H = sc["width"], sc["height"]
    rng = np.random.default_rng(2)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    o32 = orc.render_pipeline(sc, "f32", True, vrc, vra)
    o64 = orc.render_pipeline(sc, "f64", True, vrc, vra)
    t = to_dev(sc, cuda_device)
    colors = torch.from_numpy(o32["colors"]).to(cuda_device)
    off = torch.from_numpy(o32["tile_offsets"]).to(cuda_device)
    flat = torch.from_numpy(o32["flatten_ids"]).to(cuda_device)
    bg = t.get("background")
    fa = (t["means"], t["quats"], t["scales"], colors, t["opacities"][None], bg, None, W, H, 16, t["viewmats"], t["Ks"],
          off, flat)
    r_ref, a_ref, l_ref = ref.rasterize_to_pixels_from_world_3dgs_fwd(*fa)
    r_new, a_new, l_new = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa)
    e_new = rel(r_new.cpu().numpy(), r_ref.cpu().numpy())
    e_orc = rel(o32["renders"], r_ref.cpu().numpy())
    e_ref64 = rel(r_ref.cpu().numpy(), o64["renders"])
    e_new64 = rel(r_new.cpu().numpy(), o64["renders"])
    lm = float((l_new != l_ref).float().mean())
    print(f"[{name}] image rel_l2: b200 vs reference {e_new:.2e}; oracle(f32) vs reference {e_orc:.2e}; "
          f"reference vs f64 truth {e_ref64:.2e}; b200 vs f64 truth {e_new64:.2e}; last_ids differ {lm:.2e}")
    assert e_new < 1e-4 and e_orc < 1e-4
    assert rel(a_new.cpu().numpy(), a_ref.cpu().numpy()) < 1e-4
    assert lm < 2e-3
    # backward, both fed with the REFERENCE's forward outputs
    vr, va = torch.from_numpy(vrc).to(cuda_device), torch.from_numpy(vra).to(cuda_device)
    g_ref = ref.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a_ref, l_ref, vr, va)
    g_new = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a_ref, l_ref, vr, va)
    g_orc = orc.raster_bwd(sc["means"], sc["quats"], sc["scales"], o32["colors"], sc["opacities"][None],
                           sc.get("background"), None, W, H, 16, sc["viewmats"], sc["Ks"], o32["tile_offsets"],
                           o32["flatten_ids"], a_ref.cpu().numpy(), l_ref.cpu().numpy(), vrc, vra, precision="f64")
    n_g = sc["means"].shape[0]
    for nm, gr, gn, go in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g_ref, g_new, g_orc):
        gr, gn = gr.cpu().numpy(), gn.cpu().numpy()
        e2, e3 = rel(go.reshape(gr.shape), gr), rel(gn, go.reshape(gr.shape))
        print(f"[{name}] {nm}: oracle(f64) vs reference {e2:.2e}; b200 vs oracle(f64) {e3:.2e}")
        assert e2 < 1e-3, (nm, e2)
        assert_grad_close(gn, gr, nm, n_g, tag=f"{name} b200 vs reference kernels")


def test_whole_path_autograd_reference_vs_b200(native, ref, cuda_device):
    """Same L3 call sequence, two backends: image and parameter gradients.  Both are handed the REFERENCE's
    projection outputs (as test_intersect_bit_exact_vs_reference does), so the intersection lists are identical by
    construction and the comparison asserts on every run; the few radii that flip between the two projections are
    counted in test_projection_reference_vs_b200_and_oracle."""
    sc = _scene("b30k")
    W, H = sc["width"], sc["height"]
    t = to_dev(sc, cuda_device)
    rng = np.random.default_rng(9)
    target = torch.from_numpy(rng.random((1, H, W, 3), dtype=np.float32)).to(cuda_device)
    radii, means2d, depths, _, _ = ref.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"],
                                                                t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0)
    vis = (radii > 0).all(-1)
    proj = (radii, torch.where(vis[..., None], means2d, torch.zeros_like(means2d)),
            torch.where(vis, depths, torch.zeros_like(depths)))
    res = {}
    for tag, be in (("ref", ref), ("new", None)):
        P = {k: t[k].clone().requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh_coeffs")}
        out = native.rasterize(P["means"], P["quats"], P["scales"], P["opacities"], P["sh_coeffs"], sc["sh_degree"],
                               t["viewmats"], t["Ks"], W, H, bg_color=t["background"], backend=be, projection=proj)
        ((out.render_colors - target) ** 2).mean().backward()
        res[tag] = (out, {k: v.grad.detach() for k, v in P.items()})
    assert res["ref"][0].n_isects == res["new"][0].n_isects and res["new"][0].n_isects > 100_000
    e_img = rel(res["new"][0].render_colors.detach(), res["ref"][0].render_colors.detach())
    print(f"[whole path] image rel_l2 {e_img:.2e}")
    assert e_img < 1e-4
    for k in res["ref"][1]:
        assert_grad_close(res["new"][1][k], res["ref"][1][k], k, sc["means"].shape[0], tag="whole path b200 vs reference")


def test_dump_reference_golden(native, cuda_device, tmp_path):
    """Writes ref_cuda_small.npz (into $GSB_GOLDEN_OUT, else a temporary directory): outputs of the reference's own kernels on a small scene.
    The file is committed as tests/golden/ref_cuda_small.npz and pins the CPU oracle in the
    no-GPU suite (tests/test_oracle_vs_reference_golden.py)."""
    from oracle import ref_ops
    if not ref_ops.available():
        pytest.skip("oracle/_ref/libgsplat_ref.so not built (build() makes it where the reference's sources are present)")
    ref = ref_ops.backend(native)
    sc = scenes.scene_small(N=1200, width=160, height=96, sh_degree=3, view=2)
    t = to_dev(sc, cuda_device)
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    radii, means2d, depths, conics, comp = ref.projection_ut_3dgs_fused(
        t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0,
        calc_compensations=True)
    vis = (radii > 0).all(-1)
    means2d = torch.where(vis[..., None], means2d, torch.zeros_like(means2d))
    depths = torch.where(vis, depths, torch.zeros_like(depths))
    conics = torch.where(vis[..., None], conics, torch.zeros_like(conics))
    rng = np.random.default_rng(11)
    colors = torch.from_numpy(rng.random((1, sc["means"].shape[0], 3), dtype=np.float32)).to(cuda_device)
    tpg, ids, flat = ref.intersect_tile(means2d, radii, depths, 1, 16, tw, th, True)
    off = ref.intersect_offset(ids, 1, tw, th)
    fa = (t["means"], t["quats"], t["scales"], colors, t["opacities"][None], t["background"], None, W, H, 16,
          t["viewmats"], t["Ks"], off, flat)
    r, a, li = ref.rasterize_to_pixels_from_world_3dgs_fwd(*fa)
    vrc = torch.from_numpy(rng.standard_normal((1, H, W, 3)).astype(np.float32)).to(cuda_device)
    vra = torch.from_numpy(rng.standard_normal((1, H, W, 1)).astype(np.float32)).to(cuda_device)
    g = ref.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a, li, vrc, vra)
    out = os.environ.get("GSB_GOLDEN_OUT") or str(tmp_path)
    os.makedirs(out, exist_ok=True)
    np.savez_compressed(
        os.path.join(out, "ref_cuda_small.npz"), radii=radii.cpu().numpy(), means2d=means2d.cpu().numpy(),
        depths=depths.cpu().numpy(), conics=conics.cpu().numpy(), compensations=comp.cpu().numpy(),
        colors=colors.cpu().numpy(), tiles_per_gauss=tpg.cpu().numpy(), isect_ids=ids.cpu().numpy(),
        flatten_ids=flat.cpu().numpy(), tile_offsets=off.cpu().numpy(), renders=r.cpu().numpy(), alphas=a.cpu().numpy(),
        last_ids=li.cpu().numpy(), v_render_colors=vrc.cpu().numpy(), v_render_alphas=vra.cpu().numpy(),
        v_means=g[0].cpu().numpy(), v_quats=g[1].cpu().numpy(), v_scales=g[2].cpu().numpy(),
        v_colors=g[3].cpu().numpy(), v_opacities=g[4].cpu().numpy())


DISTORTED = {
    "opencv": dict(camera_model=0, radial=np.array([[-0.12, 0.05, 0.002, 0.01, -0.003, 0.0005]], np.float32),
                   tangential=np.array([[0.002, -0.001]], np.float32),
                   thin_prism=np.array([[0.001, 0.0002, -0.0005, 0.0001]], np.float32)),
    "fisheye": dict(camera_model=2, radial=np.array([[0.03, -0.004, 0.0007, -0.0001]], np.float32), tangential=None,
                    thin_prism=None),
}


@pytest.mark.parametrize("model", ["opencv", "fisheye"])
def test_distorted_cameras_reference_vs_b200(native, ref, cuda_device, model):
    """OpenCV pinhole with all 6+2+4 distortion coefficients (the only distorted pinhole layout whose reads
    are in bounds in the reference, SURVEY.md section 7) and the 4-coefficient fisheye."""
    cfg = DISTORTED[model]
    sc = scenes.scene_small(N=3000, width=208, height=128, view=2)
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    dev = lambda a: None if a is None else torch.from_numpy(a).to(cuda_device)
    kw = dict(camera_model=cfg["camera_model"], radial_coeffs=dev(cfg["radial"]), tangential_coeffs=dev(cfg["tangential"]),
              thin_prism_coeffs=dev(cfg["thin_prism"]))
    t = to_dev(sc, cuda_device)
    pa = (t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0)
    r_ref, m_ref, d_ref, c_ref, _ = ref.projection_ut_3dgs_fused(*pa, **kw)
    r_new, m_new, d_new, c_new, _ = native.projection_ut_3dgs_fused(*pa, **kw)
    mism = int((r_ref != r_new).any(-1).sum())
    both = ((r_ref > 0).all(-1) & (r_new > 0).all(-1)).cpu().numpy()
    em = rel(m_new.cpu().numpy()[both], m_ref.cpu().numpy()[both])
    print(f"[{model}] radii differ {mism}/{r_ref.shape[1]}, means2d rel {em:.2e}, visible {both.sum()}")
    assert mism <= 4 and em < 1e-4 and both.sum() > 1000
    vis = (r_ref > 0).all(-1)
    m2 = torch.where(vis[..., None], m_ref, torch.zeros_like(m_ref))
    dp = torch.where(vis, d_ref, torch.zeros_like(d_ref))
    _, ids, flat = ref.intersect_tile(m2, r_ref, dp, 1, 16, tw, th, True)
    off = ref.intersect_offset(ids, 1, tw, th)
    rng = np.random.default_rng(5)
    colors = torch.from_numpy(rng.random((1, sc["means"].shape[0], 3), dtype=np.float32)).to(cuda_device)
    fa = (t["means"], t["quats"], t["scales"], colors, t["opacities"][None], t["background"], None, W, H, 16,
          t["viewmats"], t["Ks"], off, flat)
    rr, ar, lr = ref.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **kw)
    rn, an, ln = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **kw)
    e = rel(rn.cpu().numpy(), rr.cpu().numpy())
    print(f"[{model}] image rel_l2 b200 vs reference {e:.2e}; last_ids differ {float((ln != lr).float().mean()):.2e}")
    assert e < 1e-4 and rel(an.cpu().numpy(), ar.cpu().numpy()) < 1e-4
    vr = torch.from_numpy(rng.standard_normal((1, H, W, 3)).astype(np.float32)).to(cuda_device)
    va = torch.from_numpy(rng.standard_normal((1, H, W, 1)).astype(np.float32)).to(cuda_device)
    g_ref = ref.rasterize_to_pixels_from_world_3dgs_bwd(*fa, ar, lr, vr, va, **kw)
    g_new = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, ar, lr, vr, va, **kw)
    for nm, a, b in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g_new, g_ref):
        assert_grad_close(a, b, nm, sc["means"].shape[0], tag=f"{model} b200 vs reference kernels")


# ------------------------------------------------------------------------------------------
# a2: rolling shutter (Cameras.cuh:268-413) -- per-pixel camera poses; here against the reference's kernels (the float64
# oracle and the stored reference outputs: test_gpu_rolling_shutter.py)
# ------------------------------------------------------------------------------------------
RS_IDS = ["top_to_bottom", "left_to_right", "bottom_to_top", "right_to_left"]


def _rolling_inputs(sc, cuda_device, rs_type):
    """End-of-frame pose = the start pose turned by 2.5 degrees and moved by a few centimetres."""
    t = to_dev(sc, cuda_device)
    ang = np.deg2rad(2.5)
    dR = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], np.float64)
    V0 = sc["viewmats"][0].astype(np.float64)
    V1 = V0.copy()
    V1[:3, :3] = dR @ V0[:3, :3]
    V1[:3, 3] = dR @ V0[:3, 3] + np.array([0.04, -0.02, 0.03])
    vm1 = torch.from_numpy(V1[None].astype(np.float32)).to(cuda_device)
    return t, dict(viewmats1=vm1, rs_type=rs_type)


@pytest.mark.parametrize("rs_type", [0, 1, 2, 3], ids=RS_IDS)
def test_rolling_shutter_projection_reference_vs_b200(native, ref, ref_precise, cuda_device, rs_type):
    """Oracle: the reference's projection kernel built WITHOUT --use_fast_math.  Under fast-math the pose interpolation
    evaluates sin() of milliradian angles with sin.approx (absolute error 2^-21: 1e-5..1e-4 relative there) separately
    for each sigma point, and the unscented transform's weights (-99, +16.67) amplify the differences a hundredfold:
    the fast build's rolling-shutter outputs are noisy at the 0.1 px level (printed below as the floor).  The product
    kernel uses the accurate sinf and has to agree with the precise build."""
    sc = scenes.scene_small(N=3000, width=208, height=128, view=2)
    W, H = sc["width"], sc["height"]
    t, kw = _rolling_inputs(sc, cuda_device, rs_type)
    pa = (t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0)
    r_ref, m_ref, d_ref, c_ref, _ = ref_precise.projection_ut_3dgs_fused(*pa, **kw)
    r_fast, m_fast, _, _, _ = ref.projection_ut_3dgs_fused(*pa, **kw)
    r_new, m_new, d_new, c_new, _ = native.projection_ut_3dgs_fused(*pa, **kw)
    mism = int((r_ref != r_new).any(-1).sum())
    both = ((r_ref > 0).all(-1) & (r_new > 0).all(-1))
    dm = (m_new - m_ref)[both].abs().max(-1).values
    ok = dm <= 0.02
    em = rel(m_new[both][ok].cpu().numpy(), m_ref[both][ok].cpu().numpy())
    ed = rel(d_new[both].cpu().numpy(), d_ref[both].cpu().numpy())
    ec = rel(c_new[both][ok].cpu().numpy(), c_ref[both][ok].cpu().numpy())
    off = float((~ok).float().mean())
    # the rolling projection really differs from the global one (the test would be vacuous otherwise)
    _, m_glob, _, _, _ = ref_precise.projection_ut_3dgs_fused(*pa)
    moved = float((m_glob - m_ref)[both].abs().max(-1).values.median())
    bf = ((r_ref > 0).all(-1) & (r_fast > 0).all(-1))
    floor_fast = float(((m_fast - m_ref)[bf].abs().max(-1).values > 0.02).float().mean())
    print(f"[rs {rs_type}] vs precise reference: radii differ {mism}/{r_ref.shape[1]}, means2d rel {em:.2e}, depths rel "
          f"{ed:.2e}, conics rel {ec:.2e}, visible {int(both.sum())}, off by > 0.02 px: {off:.2e} (max {float(dm.max()):.3f} "
          f"px); median shift vs global shutter {moved:.2f} px; the reference's own fast-math build vs its precise build: "
          f"{floor_fast:.2e} off by > 0.02 px, radii differ {int((r_ref != r_fast).any(-1).sum())}")
    assert int(both.sum()) > 1000 and moved > 1.0
    # a sigma point whose row estimate sits exactly on a floor() boundary may settle one row apart (amplified by the UT
    # weights): a handful of Gaussians at most, an order of magnitude fewer than the reference's own fast-math build
    # differs from its precise build by.
    assert mism <= 20 and off < 5e-3 and em < 5e-5 and ed < 1e-6 and ec < 1e-3
    assert mism * 10 <= int((r_ref != r_fast).any(-1).sum())  # an order of magnitude inside the reference's own noise


@pytest.mark.parametrize("rs_type", [0, 1, 2, 3], ids=RS_IDS)
def test_rolling_shutter_blend_reference_vs_b200(native, ref_precise, cuda_device, rs_type):
    ref = ref_precise  # see the projection test: per-pixel poses through sin.approx are the fast build's noise
    sc = scenes.scene_small(N=3000, width=208, height=128, view=2)
    W, H = sc["width"], sc["height"]
    tw, th = (W + 15) // 16, (H + 15) // 16
    t, kw = _rolling_inputs(sc, cuda_device, rs_type)
    pa = (t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0)
    r_ref, m_ref, d_ref, c_ref, _ = ref.projection_ut_3dgs_fused(*pa, **kw)
    vis = (r_ref > 0).all(-1)
    m2 = torch.where(vis[..., None], m_ref, torch.zeros_like(m_ref))
    dp = torch.where(vis, d_ref, torch.zeros_like(d_ref))
    _, ids, flat = ref.intersect_tile(m2, r_ref, dp, 1, 16, tw, th, True)
    off = ref.intersect_offset(ids, 1, tw, th)
    rng = np.random.default_rng(5 + rs_type)
    colors = torch.from_numpy(rng.random((1, sc["means"].shape[0], 3), dtype=np.float32)).to(cuda_device)
    fa = (t["means"], t["quats"], t["scales"], colors, t["opacities"][None], t["background"], None, W, H, 16,
          t["viewmats"], t["Ks"], off, flat)
    rr, ar, lr = ref.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **kw)
    rn, an, ln = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **kw)
    e = rel(rn.cpu().numpy(), rr.cpu().numpy())
    lm = float((ln != lr).float().mean())
    print(f"[rs {rs_type}] image rel_l2 b200 vs reference {e:.2e}; last_ids differ {lm:.2e}")
    assert e < 1e-4 and rel(an.cpu().numpy(), ar.cpu().numpy()) < 1e-4 and lm < 3e-3
    vr = torch.from_numpy(rng.standard_normal((1, H, W, 3)).astype(np.float32)).to(cuda_device)
    va = torch.from_numpy(rng.standard_normal((1, H, W, 1)).astype(np.float32)).to(cuda_device)
    g_ref = ref.rasterize_to_pixels_from_world_3dgs_bwd(*fa, ar, lr, vr, va, **kw)
    g_new = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, ar, lr, vr, va, **kw)
    for nm, a, b in zip(("v_means", "v_quats", "v_scales", "v_colors", "v_opacities"), g_new, g_ref):
        assert_grad_close(a, b, nm, sc["means"].shape[0], tag=f"rolling shutter {rs_type} b200 vs reference kernels")
