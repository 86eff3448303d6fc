"""CPU: the depth render modes (RenderMode D / ED / RGB_D / RGB_ED) without a GPU.

* The C ABI's channel-count and render-mode entry points validate their arguments before any launch.
* The mode plumbing of rasterize(render_mode=...) -- the blend's channels, the background it gets, ED's division,
  the clamp and which outputs exist -- through an oracle-backed stand-in OpsBackend.  The stand-in blends 1 and 4
  channels with the 3-channel float oracle, one channel at a time (the blend is independent per channel: see
  tests/test_gpu_render_modes.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import scenes
from test_cabi_validation import NULL, PTR, E_INVALID, E_UNSUPPORTED, E_WORKSPACE, SHUTTER_ROLLING, camera, lib  # noqa: F401
from test_cabi_validation import _buf

u32, u64, sz, i32, f32 = C.c_uint32, C.c_uint64, C.c_size_t, C.c_int32, C.c_float
MODES = ("RGB", "D", "ED", "RGB_D", "RGB_ED")
WS = C.c_void_p((_buf.ctypes.data + 255) & ~255)


def test_channel_entry_points_are_exported(lib):
    for n in ("gsb_raster_fwd_nc", "gsb_raster_bwd_nc", "gsb_fused_front_mode", "gsb_raster_fwd_recs_nc",
              "gsb_raster_bwd_recs_nc", "gsb_fused_back_mode"):
        assert hasattr(lib, n), n


def _fwd_nc(lib, channels, cam=None, means=PTR, ws_bytes=None, n_isects=10):
    cam = cam if cam is not None else camera()
    ws = sz(ws_bytes if ws_bytes is not None else lib.gsb_raster_fwd_workspace(u32(8)))
    return lib.gsb_raster_fwd_nc(u32(1), u32(8), u64(n_isects), u32(channels), means, PTR, PTR, PTR, PTR, NULL, NULL,
                                 u32(64), u32(64), u32(16), C.byref(cam), PTR, PTR, PTR, PTR, PTR, WS, ws, NULL)


def _bwd_nc(lib, channels, cam=None, means=PTR):
    cam = cam if cam is not None else camera()
    return lib.gsb_raster_bwd_nc(u32(1), u32(8), u64(10), u32(channels), means, PTR, PTR, PTR, PTR, NULL, NULL, u32(64),
                                 u32(64), u32(16), C.byref(cam), PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR,
                                 WS, sz(64), NULL)


@pytest.mark.parametrize("channels", [0, 2, 5, 16])
def test_operator_entry_points_reject_channel_counts(lib, channels):
    assert _fwd_nc(lib, channels) == E_UNSUPPORTED
    assert _bwd_nc(lib, channels) == E_UNSUPPORTED


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_operator_entry_points_validate_like_the_rgb_ones(lib, channels):
    assert lib.gsb_raster_fwd_nc(u32(1), u32(8), u64(10), u32(channels), PTR, PTR, PTR, PTR, PTR, NULL, NULL, u32(64),
                                 u32(64), u32(16), NULL, PTR, PTR, PTR, PTR, PTR, WS, sz(1 << 20), NULL) == E_INVALID
    assert _fwd_nc(lib, channels, means=NULL) == E_INVALID
    assert _fwd_nc(lib, channels, ws_bytes=64) == E_WORKSPACE
    assert _fwd_nc(lib, channels, cam=camera(model=1)) == E_UNSUPPORTED  # orthographic
    assert _bwd_nc(lib, channels) == E_WORKSPACE                         # 64-byte workspace for 8 Gaussians
    # a rolling shutter blends three channels only
    rs = camera(shutter=SHUTTER_ROLLING, viewmats1=PTR.value)
    want = E_WORKSPACE if channels == 3 else E_UNSUPPORTED
    assert _fwd_nc(lib, channels, cam=rs, ws_bytes=64) == want
    assert _bwd_nc(lib, channels, cam=rs) == want


def test_fused_mode_entry_points_validate(lib):
    cam = camera()
    for mode in (-1, 5, 9):  # POINT_CLOUD (5) is not a blend
        assert lib.gsb_fused_front_mode(PTR, C.byref(cam), u32(64), u32(64), f32(0.3), f32(0.01), f32(1e4), f32(0.0),
                                        i32(1), i32(mode), PTR, PTR, PTR, WS, sz(1 << 20), NULL) == E_UNSUPPORTED
        assert lib.gsb_fused_back_mode(PTR, C.byref(cam), u32(64), u32(64), i32(mode), PTR, WS, sz(1 << 20), PTR, PTR,
                                       PTR, PTR, PTR, PTR, NULL) == E_UNSUPPORTED
    for mode in range(5):  # valid mode, no splats
        assert lib.gsb_fused_front_mode(NULL, C.byref(cam), u32(64), u32(64), f32(0.3), f32(0.01), f32(1e4), f32(0.0),
                                        i32(1), i32(mode), PTR, PTR, PTR, WS, sz(1 << 20), NULL) == E_INVALID
        assert lib.gsb_fused_back_mode(NULL, C.byref(cam), u32(64), u32(64), i32(mode), PTR, WS, sz(1 << 20), PTR, PTR,
                                       PTR, PTR, PTR, PTR, NULL) == E_INVALID

    def fwd(channels, depths=PTR, cam_=cam):
        return lib.gsb_raster_fwd_recs_nc(u32(8), u32(16), u32(channels), WS, sz(64), depths, NULL, NULL, u32(64),
                                          u32(64), C.byref(cam_), PTR, PTR, PTR, PTR, PTR, NULL)

    def bwd(channels, depths=PTR, cam_=cam):
        return lib.gsb_raster_bwd_recs_nc(u32(8), u32(16), u32(channels), WS, sz(64), depths, NULL, NULL, u32(64),
                                          u32(64), C.byref(cam_), PTR, PTR, PTR, PTR, PTR, PTR, NULL)

    for f in (fwd, bwd):
        assert f(2) == E_UNSUPPORTED and f(5) == E_UNSUPPORTED
        assert f(4, depths=NULL) == E_INVALID  # the fourth channel is read from the front's depths
        assert f(1, depths=NULL) == E_WORKSPACE and f(4) == E_WORKSPACE and f(3) == E_WORKSPACE
        assert f(1, cam_=camera(shutter=SHUTTER_ROLLING, viewmats1=PTR.value)) == E_UNSUPPORTED


# ---------------------------------------------------------------------------------------------
# the Python mirror's mode plumbing, on an oracle-backed stand-in backend
# ---------------------------------------------------------------------------------------------
def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _pad3(x):
    return np.ascontiguousarray(np.concatenate([x, np.zeros(x.shape[:-1] + (2,), x.dtype)], -1))


@pytest.fixture(scope="module")
def oracle_backend(pkg, orc):
    class OracleOps(pkg.OpsBackend):
        """The operators rasterize() calls, computed by the float oracle on CPU tensors.  The blend at 1 or 4 channels
        runs the 3-channel oracle once per group of channels; the backgrounds it was given are recorded."""

        def __init__(self):
            super().__init__(lambda: None)
            self.backgrounds = []

        def projection_ut_3dgs_fused(self, means, quats, scales, opacities, viewmats0, Ks, width, height, eps2d=0.3,
                                     near_plane=0.01, far_plane=1e10, radius_clip=0.0, calc_compensations=False,
                                     camera_model=0, **_):
            r = orc.projection_ut(_np(means), _np(quats), _np(scales), _np(opacities), _np(viewmats0), _np(Ks), width,
                                  height, eps2d, near_plane, far_plane, radius_clip, camera_model=camera_model)
            return tuple(torch.from_numpy(x) for x in r[:4]) + (None,)

        def spherical_harmonics_fwd(self, degrees_to_use, dirs, coeffs, masks=None):
            return torch.from_numpy(orc.sh_fwd(degrees_to_use, _np(dirs), _np(coeffs), _np(masks)))

        def spherical_harmonics_bwd(self, K, degrees_to_use, dirs, coeffs, masks, v_colors, compute_v_dirs=True):
            vc, vd = orc.sh_bwd(degrees_to_use, _np(dirs), _np(coeffs), _np(masks), _np(v_colors), compute_v_dirs)
            return torch.from_numpy(vc), (torch.from_numpy(vd) if compute_v_dirs else None)

        def intersect_tile(self, means2d, radii, depths, C_, tile_size, tile_width, tile_height, sort=True):
            return tuple(torch.from_numpy(x) for x in orc.isect_tiles(_np(means2d), _np(radii), _np(depths), C_,
                                                                      tile_size, tile_width, tile_height, sort))

        def intersect_offset(self, isect_ids, C_, tile_width, tile_height):
            return torch.from_numpy(orc.isect_offsets(_np(isect_ids), C_, tile_width, tile_height))

        @staticmethod
        def _groups(x):
            """[..., NC] -> the 3-channel oracle calls' inputs: channels 0..2, then (c3, 0, 0); NC = 1: (c0, 0, 0)."""
            nc = x.shape[-1]
            if nc == 3:
                return [x]
            return ([x[..., :3]] if nc == 4 else []) + [_pad3(x[..., -1:])]

        def rasterize_to_pixels_from_world_3dgs_fwd(self, means, quats, scales, colors, opacities, backgrounds, masks,
                                                    image_width, image_height, tile_size, viewmats0, Ks, tile_offsets,
                                                    flatten_ids, **_):
            self.backgrounds.append(_np(backgrounds))
            c = _np(colors)
            bgs = [None] * 2 if backgrounds is None else self._groups(_np(backgrounds))
            outs = [orc.raster_fwd(_np(means), _np(quats), _np(scales), np.ascontiguousarray(cg), _np(opacities), bg,
                                   _np(masks), image_width, image_height, tile_size, _np(viewmats0), _np(Ks),
                                   _np(tile_offsets), _np(flatten_ids)) for cg, bg in zip(self._groups(c), bgs)]
            nc = c.shape[-1]
            renders = outs[0][0] if nc == 3 else (outs[0][0][..., :1] if nc == 1 else
                                                  np.concatenate([outs[0][0], outs[1][0][..., :1]], -1))
            return torch.from_numpy(np.ascontiguousarray(renders)), torch.from_numpy(outs[0][1]), \
                torch.from_numpy(outs[0][2])

        def rasterize_to_pixels_from_world_3dgs_bwd(self, means, quats, scales, colors, opacities, backgrounds, masks,
                                                    image_width, image_height, tile_size, viewmats0, Ks, tile_offsets,
                                                    flatten_ids, render_alphas, last_ids, v_render_colors,
                                                    v_render_alphas, **_):
            c, v, va = _np(colors), _np(v_render_colors), _np(v_render_alphas)
            nc = c.shape[-1]
            bgs = [None] * 2 if backgrounds is None else self._groups(_np(backgrounds))
            vas = [va] if nc != 4 else [va, np.zeros_like(va)]
            sums, v_colors = None, []
            for cg, bg, vg, vag in zip(self._groups(c), bgs, self._groups(v), vas):
                g = orc.raster_bwd(_np(means), _np(quats), _np(scales), np.ascontiguousarray(cg), _np(opacities), bg,
                                   _np(masks), image_width, image_height, tile_size, _np(viewmats0), _np(Ks),
                                   _np(tile_offsets), _np(flatten_ids), _np(render_alphas), _np(last_ids),
                                   np.ascontiguousarray(vg), vag)
                sums = list(g) if sums is None else [s + x for s, x in zip(sums, g)]
                v_colors.append(g[3])
            vc = v_colors[0][..., :1] if nc == 1 else (v_colors[0] if nc == 3 else
                                                       np.concatenate([v_colors[0], v_colors[1][..., :1]], -1))
            f = lambda x: torch.from_numpy(np.asarray(x, np.float32))
            return f(sums[0]), f(sums[1]), f(sums[2]), f(vc), f(sums[4])

    return OracleOps()


@pytest.fixture(scope="module")
def scene():
    sc = scenes.scene_small(N=400, width=64, height=48, view=1)
    t = {k: (torch.from_numpy(np.ascontiguousarray(v)) if isinstance(v, np.ndarray) else v) for k, v in sc.items()}
    return sc, t


def _render(pkg, be, t, mode, bg=True, grad=False):
    P = {k: t[k].clone().requires_grad_(grad) for k in ("means", "quats", "scales", "opacities", "sh_coeffs")}
    o = pkg.rasterize(P["means"], P["quats"], P["scales"], P["opacities"], P["sh_coeffs"], t["sh_degree"],
                      t["viewmats"], t["Ks"], t["width"], t["height"], bg_color=t["background"] if bg else None,
                      backend=be, render_mode=mode)
    return o, P


@pytest.mark.parametrize("with_bg", [True, False])
def test_rasterize_modes_plumbing(pkg, oracle_backend, scene, with_bg):
    _sc, t = scene
    W, H = t["width"], t["height"]
    out = {}
    for mode in MODES:
        oracle_backend.backgrounds.clear()
        o, _ = _render(pkg, oracle_backend, t, mode, bg=with_bg)
        nc = pkg.RENDER_MODES[mode]
        assert o.render_colors.shape == (1, H, W, nc)
        assert o.alpha.shape == (1, H, W)
        assert (o.image is None) == (mode in ("D", "ED"))
        assert (o.depth is None) == (mode == "RGB")
        if o.image is not None:
            assert o.image.shape == (3, H, W) and float(o.image.min()) >= 0 and float(o.image.max()) <= 1
        if o.depth is not None:
            assert o.depth.shape == (1, H, W)
        # the background the blend got (rasterizer.cpp:276-298)
        bg = oracle_backend.backgrounds[0]
        if not with_bg:
            assert bg is None
        elif mode == "RGB":
            assert np.array_equal(bg, _np(t["background"]))
        elif nc == 1:
            assert bg.shape == (1, 1) and not bg.any()
        else:
            assert np.array_equal(bg, np.concatenate([_np(t["background"]), [[0.0]]], -1))
        out[mode] = o
    rgb, d, ed, rgbd, rgbed = (out[m] for m in MODES)
    for m in MODES[1:]:
        assert torch.equal(out[m].alpha, rgb.alpha)
    assert torch.equal(rgbd.image, rgb.image) and torch.equal(rgbed.image, rgb.image)
    assert torch.equal(rgbd.depth, d.depth) and torch.equal(rgbed.depth, ed.depth)
    assert torch.equal(d.depth, d.render_colors[0].permute(2, 0, 1))
    acc_alpha = rgb.alpha.permute(1, 2, 0)[None]  # [1,H,W,1]
    assert torch.equal(ed.depth, (d.render_colors / acc_alpha.clamp_min(1e-10))[0].permute(2, 0, 1))
    assert float(d.depth.max()) > 0  # the depth of a visible Gaussian is its camera-space z


def test_depth_gradient_reaches_geometry_not_colour(pkg, oracle_backend, scene):
    _sc, t = scene
    o, P = _render(pkg, oracle_backend, t, "D", grad=True)
    (o.depth * torch.randn_like(o.depth)).sum().backward()
    for k in ("means", "quats", "scales", "opacities"):
        assert P[k].grad is not None and torch.count_nonzero(P[k].grad) > 0, k
    assert P["sh_coeffs"].grad is None or torch.count_nonzero(P["sh_coeffs"].grad) == 0


@pytest.mark.parametrize("mode", ["rgb", "DEPTH", "POINT_CLOUD", "RGB-D", ""])
def test_unknown_render_mode_raises(pkg, scene, mode):
    _sc, t = scene
    with pytest.raises(ValueError, match="Invalid render mode"):
        pkg.rasterize(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"], t["sh_degree"],
                      t["viewmats"], t["Ks"], t["width"], t["height"], render_mode=mode)
    raw = pkg.raw_from_activated(t["means"], t["quats"], t["scales"], t["opacities"], t["sh_coeffs"])
    with pytest.raises(ValueError, match="Invalid render mode"):
        pkg.rasterize_fused(raw["means"], raw["sh0"], raw["shN"], raw["scaling_raw"], raw["rotation_raw"],
                            raw["opacity_raw"], t["sh_degree"], t["viewmats"], t["Ks"], t["width"], t["height"],
                            render_mode=mode)


@pytest.mark.parametrize("mode", ["ED", "RGB_ED"])
def test_expected_depth_gradient_is_the_chain_rule(pkg, orc, oracle_backend, scene, mode):
    """ED = acc / max(alpha, 1e-10): the mirror's gradients are the blend backward's at the cotangents
    v_acc = v_ed / max(alpha, 1e-10),  v_alpha -= v_ed acc / alpha^2  (alpha > 1e-10), computed here in float64."""
    sc, t = scene
    W, H = t["width"], t["height"]
    o, P = _render(pkg, oracle_backend, t, mode, grad=True)
    g = torch.Generator().manual_seed(3)
    v_ed, v_al = torch.randn((1, H, W), generator=g), torch.randn((1, H, W), generator=g)
    loss = (o.depth * v_ed).sum() + (o.alpha * v_al).sum()
    if mode == "RGB_ED":
        v_im = torch.randn((3, H, W), generator=g)
        loss = loss + (o.image * v_im).sum()
    loss.backward()
    renders, alphas = _np(o.render_colors), _np(o.alpha.permute(1, 2, 0)[None])
    acc, al = renders[..., -1:].astype(np.float64), alphas.astype(np.float64)
    v_acc = _np(v_ed)[..., None] / np.maximum(al, 1e-10)
    v_alpha = _np(v_al)[..., None] - _np(v_ed)[..., None] * acc / np.maximum(al, 1e-10) ** 2 * (al > 1e-10)
    vrc = v_acc
    if mode == "RGB_ED":
        img = renders[0, ..., :3]
        vrc = np.concatenate([(_np(v_im).transpose(1, 2, 0) * ((img >= 0) & (img <= 1)))[None], v_acc], -1)
    # the same blend call the mirror made: its colours and projection (the stand-in is deterministic)
    with torch.no_grad():
        radii, means2d, depths, _, _ = oracle_backend.projection_ut_3dgs_fused(
            t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 10000.0, 0.0)
        tw, th = (W + 15) // 16, (H + 15) // 16
        _, ids, flat = oracle_backend.intersect_tile(means2d, radii, depths, 1, 16, tw, th)
        off = oracle_backend.intersect_offset(ids, 1, tw, th)
    colors = depths[..., None]
    if mode == "RGB_ED":
        ref = orc.render_pipeline(sc, "f32")
        colors = torch.cat([torch.from_numpy(ref["colors"]), colors], -1)
    bg = pkg._mode_background(mode, t["background"])
    f32 = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32))
    _r, a, li = oracle_backend.rasterize_to_pixels_from_world_3dgs_fwd(
        t["means"], t["quats"], t["scales"], colors, t["opacities"][None], bg, None, W, H, 16, t["viewmats"], t["Ks"],
        off, flat)
    gk = oracle_backend.rasterize_to_pixels_from_world_3dgs_bwd(
        t["means"], t["quats"], t["scales"], colors, t["opacities"][None], bg, None, W, H, 16, t["viewmats"], t["Ks"],
        off, flat, a, li, f32(vrc), f32(v_alpha))
    for key, want in (("quats", gk[1]), ("scales", gk[2]), ("opacities", gk[4][0])) + \
            ((("means", gk[0]),) if mode == "ED" else ()):  # RGB_ED: the SH direction gradient reaches the means too
        got = P[key].grad
        e = float(torch.linalg.norm(got - want.reshape(got.shape)) / torch.linalg.norm(want))
        assert e < 1e-4, (key, e)
