"""GPU: the rolling-shutter path (gsb_raster_rs.cu, project_rolling in gsb_projection.cuh) against the float64 CPU oracle.

A rolling-shutter camera gives every image row (or column) its own pose between viewmats0 and viewmats1.  The library
runs such cameras through kernels of their own: a 64-byte record per Gaussian, one thread per pixel, records staged
256 at a time, a per-warp skip of the slots behind the warp's newest contributor, a 16-slot moment row reduced with the
pre-swapped butterfly (lanes 16..31, the odd pixel rows of a warp, hold their slots swapped), and a finalize kernel.
The cases:
  a. the projection, four directions x three camera models;
  b. blend forward and backward on the oracle's lists, on a ragged image dense enough that many tiles hold more than
     256 and more than 512 records, with and without a background and with tile masks;
  c. a wide-angle fisheye whose corners lie beyond its maximum angle: those pixels have no ray;
  d. a sentinel scene checked per Gaussian: even and odd rows of a warp, each of a tile's eight warps, tile boundaries,
     the ragged edges, and one pixel under a stack of 320 faint Gaussians whose list crosses a 256-record batch;
  e. a static camera through the rolling-shutter kernels against the global-shutter kernels at a large image;
  f. the reversed direction with swapped poses;
  g. empty inputs;
  h. the library against stored outputs of the reference's kernels (tests/golden/ref_rolling_small.npz), which
     test_dump_reference_rolling_golden writes where the reference's build without --use_fast_math exists.
Each oracle comparison prints the float32 oracle's own error beside the GPU's and bounds the GPU by it."""
import math
import os

import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, grad_metrics, rel, to_dev
from test_gpu_blend_wide import (SENTINEL_TOL_FLOOR, _edge_classes, assert_untouched_near_zero, per_gauss_ratio, shape,
                                 tiles)
from test_oracle_rolling_shutter import (CAMERAS, G, GOLDEN_CASES, GRADS, RS_IDS, RS_TYPES, end_pose, golden_colors,
                                         golden_cotangents, golden_end_pose, golden_scene)

pytestmark = pytest.mark.gpu

RS_BATCH = 256  # gsb_raster_rs.cu kRsThreads: records staged per batch
# Whole-tensor bound of a gradient on the dense scenes.  One Gaussian whose pixel flips at the 1/255 cut can carry
# 1e-3 of a tensor's norm there (v_quats, measured on an H100: 1.03e-3 against the float64 oracle, and the float32
# oracle itself up to 1.1e-3), so the bound is 2e-3 or twice the float32 oracle's, whichever is larger; the
# per-Gaussian fraction is the check that matters (test_gpu_blend_wide.assert_close_as_f32).
GRAD_REL_TOL = 2e-3


def assert_close_as_f32(got, want, w32, name, n_g, tag):
    n32 = grad_metrics(w32, want, n_g)
    assert_grad_close(got, want, name, n_g, rel_tol=max(GRAD_REL_TOL, 2.0 * n32["rel"]),
                      frac_tol=max(2e-3, 2.0 * n32["frac_bad"]),
                      tag=f"{tag} vs f64 oracle; f32 oracle itself {n32['rel']:.1e}, {n32['n_bad']} Gaussians off by > 0.01")


@pytest.fixture(scope="module", autouse=True)
def _oracle_threads(orc):
    orc.set_threads(orc.max_threads())
    yield
    orc.set_threads(1)


def native_kwargs(cam, dev, viewmats1=None, rs_type=None):
    """The oracle's camera keywords (CAMERAS) as the library's, plus the end pose and the direction."""
    c = CAMERAS[cam] if isinstance(cam, str) else cam
    d = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    kw = dict(camera_model=c["camera_model"], radial_coeffs=d(c.get("radial")), tangential_coeffs=d(c.get("tangential")),
              thin_prism_coeffs=d(c.get("thin_prism")))
    if viewmats1 is not None:
        kw.update(viewmats1=d(viewmats1), rs_type=rs_type)
    return kw


def oracle_kwargs(cam, viewmats1=None, rs_type=None):
    c = dict(CAMERAS[cam]) if isinstance(cam, str) else dict(cam)
    if viewmats1 is not None:
        c.update(viewmats1=viewmats1, rs_type=rs_type)
    return c


def oracle_lists(orc, sc, okw):
    W, H = sc["width"], sc["height"]
    tw, th = tiles(W, H)
    radii, m2d, depths, _, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"],
                                                 sc["viewmats"], sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **okw)
    _, ids, flat = orc.isect_tiles(m2d, radii, depths, 1, 16, tw, th)
    return orc.isect_offsets(ids, 1, tw, th), flat


def tile_counts(off, n_isects):
    start = np.asarray(off, np.int64).ravel()
    return np.append(start[1:], n_isects) - start


# ------------------------------------------------------------------------------------------
# a. projection
# ------------------------------------------------------------------------------------------
PROJ_SCENE = dict(N=3000, width=210, height=125, view=2)  # 210 % 16 = 2, 125 % 16 = 13


@pytest.mark.parametrize("cam", list(CAMERAS))
@pytest.mark.parametrize("rs_type", RS_TYPES, ids=RS_IDS)
def test_rolling_projection_vs_f64_oracle(native, orc, cuda_device, rs_type, cam):
    """Radii, means2d, depths and conics against the float64 oracle.  A sigma point whose row estimate lies on a
    floor() boundary may settle one row apart between float32 and float64 (the ten fixed-point steps do not contract
    there): the Gaussians that move by more than 0.02 px and the radii that differ are bounded by twice the float32
    oracle's count (and 5 / 0.2 %), the rest must agree to 1e-4."""
    sc = scenes.scene_small(**PROJ_SCENE)
    W, H = sc["width"], sc["height"]
    V1 = end_pose(sc["viewmats"])
    t = to_dev(sc, cuda_device)
    okw = oracle_kwargs(cam, V1, rs_type)
    pa = (sc["means"], sc["quats"], sc["scales"], sc["opacities"], sc["viewmats"], sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0)
    o64 = orc.projection_ut(*pa, precision="f64", **okw)
    o32 = orc.projection_ut(*pa, precision="f32", **okw)
    glob = orc.projection_ut(*pa, precision="f64", **CAMERAS[cam])
    out = native.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W,
                                          H, 0.3, 0.01, 1e4, 0.0, **native_kwargs(cam, cuda_device, V1, rs_type))
    out = [x.cpu().numpy() for x in out[:4]]
    n_g = sc["means"].shape[0]

    def errors(r, m, d, c):
        mism = int((r != o64[0]).any(-1).sum())
        both = (r > 0).all(-1) & (o64[0] > 0).all(-1)
        ok = both & (np.abs(m - o64[1]).max(-1) <= 0.02)
        return dict(mism=mism, both=int(both.sum()), off=int((both & ~ok).sum()), m=rel(m[ok], o64[1][ok]),
                    d=rel(d[both], o64[2][both]), c=rel(c[ok], o64[3][ok]))

    e, e32 = errors(*out), errors(*o32[:4])
    vis = (glob[0] > 0).all(-1) & (o64[0] > 0).all(-1)
    moved = float(np.median(np.abs(o64[1][vis] - glob[1][vis]).max(-1)))
    print(f"[{cam} {RS_IDS[rs_type]}] GPU vs f64 oracle: radii differ {e['mism']} (f32 oracle {e32['mism']}), visible "
          f"{e['both']} of {n_g}, off by > 0.02 px {e['off']} (f32 oracle {e32['off']}); means2d rel {e['m']:.2e} (f32 "
          f"oracle {e32['m']:.2e}), depths {e['d']:.2e} ({e32['d']:.2e}), conics {e['c']:.2e} ({e32['c']:.2e}); median "
          f"shift from the global shutter {moved:.2f} px")
    assert moved > 1.0  # the motion is not a no-op
    assert e["both"] > n_g // 2
    assert e["mism"] <= max(5, 2 * e32["mism"]) and e["off"] <= max(2e-3 * n_g, 2 * e32["off"])
    assert e["m"] < 1e-4 and e["d"] < 1e-5 and e["c"] < 1e-3


# ------------------------------------------------------------------------------------------
# b. blend on the oracle's lists, dense and ragged
# ------------------------------------------------------------------------------------------
DENSE_SCENE = dict(N=10000, width=300, height=195, view=2, sh_degree=0)  # 300 % 16 = 12, 195 % 16 = 3
# tiles with more than 256 / 512 records, measured with orc.isect_tiles on every camera and direction: 76..85 / 50..58
MIN_TILES_OVER_256, MIN_TILES_OVER_512 = 60, 40


def blend_vs_oracle(native, orc, dev, tag, sc, colors, off, flat, bg, masks, vrc, vra, okw, nkw):
    """Blend forward and backward on the GPU against the oracle on the same lists: image, alpha and last_ids against
    the float64 forward, gradients against the float64 backward given the float32 oracle's alpha and last_ids, each
    beside the float32 oracle's own error (test_gpu_blend_wide's bounds)."""
    W, H = sc["width"], sc["height"]
    oa = (sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None], bg, masks, W, H, 16, sc["viewmats"],
          sc["Ks"], off, flat)
    r32, a32, l32 = orc.raster_fwd(*oa, precision="f32", **okw)
    r64, a64, l64 = orc.raster_fwd(*oa, precision="f64", **okw)
    t = to_dev(sc, dev)
    d = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    na = (t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], d(bg), d(masks), W, H, 16,
          t["viewmats"], t["Ks"], d(off), d(flat))
    r, a, li = (x.cpu().numpy() for x in native.rasterize_to_pixels_from_world_3dgs_fwd(*na, **nkw))
    keep = np.ones((H, W), bool)
    if masks is not None:
        keep = np.repeat(np.repeat(masks[0], 16, 0), 16, 1)[:H, :W]
        want_bg = np.zeros(3, np.float32) if bg is None else np.asarray(bg, np.float32).reshape(3)
        assert np.all(r[0][~keep] == want_bg)  # masked tiles: the background and nothing else
    e_img, e_alpha = rel(r[0][keep], r64[0][keep]), rel(a[0][keep], a64[0][keep])
    n_img, n_alpha = rel(r32[0][keep], r64[0][keep]), rel(a32[0][keep], a64[0][keep])
    li_bad = float((li[0][keep] != l64[0][keep]).mean())
    d_img = np.abs(r[0][keep] - r64[0][keep]).max(-1)
    print(f"[{tag}] vs f64 oracle: image rel_l2 {e_img:.2e} (f32 oracle {n_img:.2e}), alpha {e_alpha:.2e} (f32 oracle "
          f"{n_alpha:.2e}), last_ids differ {li_bad:.2e} (f32 oracle {float((l32[0][keep] != l64[0][keep]).mean()):.2e}), "
          f"max |d image| {float(d_img.max()):.2e}")
    assert e_img < 1e-4 and e_alpha < 1e-4
    assert float(d_img.max()) < 2e-2  # a 1/255-cut flip moves a pixel by <= alpha * colour
    assert (d_img > 1e-4).mean() < 2e-3
    assert li_bad < 2e-3
    ga = (a32, l32, vrc, vra)
    g64 = orc.raster_bwd(*oa, *ga, precision="f64", **okw)
    g32 = orc.raster_bwd(*oa, *ga, precision="f32", **okw)
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*na, *(d(x) for x in ga), **nkw)
    n_g = sc["means"].shape[0]
    for nm, got, want, w32 in zip(GRADS, g, g64, g32):
        got = got.cpu().numpy().reshape(want.shape)
        assert_close_as_f32(got, want, w32, nm, n_g, tag)
        assert_untouched_near_zero(got, want, w32, nm, n_g, tag)
    return r, a, li


@pytest.fixture(scope="module")
def dense():
    sc = scenes.scene_small(**DENSE_SCENE)
    W, H = sc["width"], sc["height"]
    rng = np.random.default_rng(4)
    colors = rng.random((1, sc["means"].shape[0], 3), dtype=np.float32)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    return dict(sc=sc, colors=colors, vrc=vrc, vra=vra, V1=end_pose(sc["viewmats"]))


def _dense_case(native, orc, dev, dense, cam, rs_type, background=True, masks=None):
    sc, V1 = dense["sc"], dense["V1"]
    W, H = sc["width"], sc["height"]
    assert W % 16 and H % 16
    okw = oracle_kwargs(cam, V1, rs_type)
    off, flat = oracle_lists(orc, sc, okw)
    n = tile_counts(off, len(flat))
    if masks is not None:
        n = n * masks.ravel()
    tag = f"{cam} {RS_IDS[rs_type]}{'' if background else ', no background'}{', tile masks' if masks is not None else ''}"
    print(f"[{tag}] {W}x{H}, {len(flat)} intersections; tiles over {RS_BATCH} records: {int((n > RS_BATCH).sum())}, over "
          f"{2 * RS_BATCH}: {int((n > 2 * RS_BATCH).sum())}, longest list {int(n.max())}")
    # the staging loop and the cross-batch skip run past their first and second batch in many tiles
    assert (n > RS_BATCH).sum() >= MIN_TILES_OVER_256 * (0.5 if masks is not None else 1)
    assert (n > 2 * RS_BATCH).sum() >= MIN_TILES_OVER_512 * (0.5 if masks is not None else 1)
    bg = sc["background"] if background else None
    return blend_vs_oracle(native, orc, dev, tag, sc, dense["colors"], off, flat, bg, masks, dense["vrc"], dense["vra"],
                           okw, native_kwargs(cam, dev, V1, rs_type))


@pytest.mark.parametrize("cam", list(CAMERAS))
@pytest.mark.parametrize("rs_type", RS_TYPES, ids=RS_IDS)
def test_rolling_blend_dense_vs_f64_oracle(native, orc, cuda_device, dense, rs_type, cam):
    _dense_case(native, orc, cuda_device, dense, cam, rs_type)


def test_rolling_blend_no_background_vs_f64_oracle(native, orc, cuda_device, dense):
    _dense_case(native, orc, cuda_device, dense, "opencv", 2, background=False)


def test_rolling_blend_tile_masks_vs_f64_oracle(native, orc, cuda_device, dense):
    """A checkerboard of masked tiles: every other tile renders the background and walks nothing."""
    sc = dense["sc"]
    tw, th = tiles(sc["width"], sc["height"])
    masks = ((np.arange(th)[:, None] + np.arange(tw)[None, :]) % 2 == 0)[None]
    _dense_case(native, orc, cuda_device, dense, "pinhole", 1, masks=masks)


# ------------------------------------------------------------------------------------------
# c. pixels without a ray
# ------------------------------------------------------------------------------------------
WIDE_FISHEYE = dict(camera_model=2, radial=np.array([[-0.08, 0.0, 0.0, 0.0]], np.float32))


def fisheye_invalid_pixels(W, H, fx, fy, cx, cy, k1, band=1e-4):
    """Pixel centres whose fisheye angle (theta (1 + k1 theta^2) = |normalised point|, by Newton in float64) reaches the
    model's maximum angle (Cameras.cuh:830-885: the first root of the derivative, capped by the image's farthest
    corner), and those within `band` of it, where float32 and float64 may disagree."""
    r = math.hypot(max(W - cx, cx), max(H - cy, cy))
    max_angle = min(math.sqrt(-1.0 / (3.0 * k1)), max(r / fx, r / fy))
    ys, xs = np.mgrid[0:H, 0:W]
    delta = np.hypot((xs + 0.5 - cx) / fx, (ys + 0.5 - cy) / fy)
    th = delta.copy()
    for _ in range(50):
        th -= (th * (1 + k1 * th * th) - delta) / (1 + 3 * k1 * th * th)
    return th >= max_angle, np.abs(th - max_angle) < band


def test_rolling_fisheye_pixels_beyond_the_max_angle(native, orc, cuda_device):
    """A wide-angle fisheye (f = 100 px on a 200x120 image, k1 = -0.08) whose corners lie beyond the maximum angle.
    Those pixels have no ray: they render the background with alpha 0 and, given cotangents there only, the backward
    gives exact zeros.  The rest of the image is compared with the float64 oracle."""
    sc = scenes.scene_small(N=6000, width=200, height=120, sh_degree=0)
    W, H = sc["width"], sc["height"]
    f, cx, cy = 100.0, W / 2.0, H / 2.0
    sc["Ks"] = np.array([[[f, 0, cx], [0, f, cy], [0, 0, 1]]], np.float32)
    # Gaussians all over the field of view, corners included: directions of uniformly drawn pixels under the
    # equidistant approximation theta = |pixel - centre| / f, at distances 2..4
    rng = np.random.default_rng(6)
    u, v = rng.uniform(-cx, cx, 6000), rng.uniform(-cy, cy, 6000)
    th_ = np.hypot(u, v) / f
    dist = rng.uniform(2.0, 4.0, 6000)
    sc["means"] = (np.stack([np.sin(th_) * u, np.sin(th_) * v, np.cos(th_) * np.hypot(u, v)], -1)
                   / np.hypot(u, v)[:, None] * dist[:, None]).astype(np.float32)
    V1 = end_pose(sc["viewmats"])
    rs_type = 1
    okw = oracle_kwargs(WIDE_FISHEYE, V1, rs_type)
    nkw = native_kwargs(WIDE_FISHEYE, cuda_device, V1, rs_type)
    off, flat = oracle_lists(orc, sc, okw)
    invalid, border = fisheye_invalid_pixels(W, H, f, f, cx, cy, float(WIDE_FISHEYE["radial"][0, 0]))
    tw, th = tiles(W, H)
    listed = np.repeat(np.repeat((tile_counts(off, len(flat)) > 0).reshape(th, tw), 16, 0), 16, 1)[:H, :W]
    sure = invalid & ~border
    print(f"[wide fisheye] {int(sure.sum())} pixels beyond the max angle, {int((sure & listed).sum())} of them in tiles "
          f"with records; {int(border.sum())} within 1e-4 rad of it left out")
    assert (sure & listed).sum() >= 500
    colors = rng.random((1, sc["means"].shape[0], 3), dtype=np.float32)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    r, a, li = blend_vs_oracle(native, orc, cuda_device, "wide fisheye", sc, colors, off, flat, sc["background"], None,
                               vrc, vra, okw, nkw)
    assert np.all(r[0][sure] == sc["background"][0]) and np.all(a[0][sure] == 0)
    assert float(a[0][~invalid & ~border & listed].mean()) > 0.3  # the valid pixels do render the scene
    t = to_dev(sc, cuda_device)
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(cuda_device)
    only = sure[None, :, :, None]
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(
        t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], t["background"], None, W, H, 16,
        t["viewmats"], t["Ks"], d(off), d(flat), d(a), d(li), d(vrc * only), d(vra * only), **nkw)
    for nm, x in zip(GRADS, g):
        assert not x.any(), nm


# ------------------------------------------------------------------------------------------
# d. sentinel scene: the pixel classes of the rolling-shutter kernels, checked per Gaussian
# ------------------------------------------------------------------------------------------
# A CTA of 256 threads covers a 16x16 tile, thread (x, y) at lane 16 (y % 2) + x of warp y // 2: a warp is two pixel
# rows, the even row in lanes 0..15 and the odd row in lanes 16..31 (the half whose moment slots are pre-swapped).
# Each class: tile-local pixel box [x0, x1) x [y0, y1) its footprint must stay in, optional ranges of its centre,
# ranges of its two standard deviations in pixels, the range of its in-plane rotation.
def _rs_classes(W, H):
    c = {
        # centred on their row: the rows one pixel away stay outside the footprint
        "even-row": dict(box=(0, 16, 6, 7), sig=(0.6, 1.5, 0.15, 0.22), rot=0.0, centred=True),
        "odd-row": dict(box=(0, 16, 9, 10), sig=(0.6, 1.5, 0.15, 0.22), rot=0.0, centred=True),
        "tile-boundary-x": dict(box=(8, 24, 0, 16), cx=(15.6, 16.4), sig=(0.5, 1.2, 0.5, 1.5)),
        "tile-boundary-y": dict(box=(0, 16, 8, 24), cy=(15.6, 16.4), sig=(0.5, 1.5, 0.5, 1.2)),
    }
    for w in range(8):
        # centred between the warp's two rows: both rows' centres (0.5 px away) inside the footprint, the neighbouring
        # rows' (1.5 px away) outside
        c[f"warp{w}"] = dict(box=(0, 16, 2 * w, 2 * w + 2), sig=(0.5, 1.5, 0.2, 0.3), rot=0.0, centred=True)
    return c


SENTINEL_F = 500.0
STACK = 320  # faint Gaussians on one pixel: more than one 256-record batch, and T = 0.98^320 > 1e-4


def rs_pose(tau, V1):
    """World -> camera of the start pose (identity) interpolated towards V1 (a turn about one axis and a move): GLM's
    slerp from the identity quaternion turns by tau x the angle about the same axis."""
    from scipy.spatial.transform import Rotation
    rv = Rotation.from_matrix(V1[0, :3, :3].astype(np.float64)).as_rotvec()
    return Rotation.from_rotvec(tau * rv).as_matrix(), tau * V1[0, :3, 3].astype(np.float64)


def frame_time(rs_type, u, v, W, H):
    return [math.floor(v) / (H - 1), math.floor(u) / (W - 1), (H - math.ceil(v)) / (H - 1),
            (W - math.ceil(u)) / (W - 1)][rs_type]


def rs_sentinel_scene(W, H, rs_type, V1, seed=5):
    """Small non-overlapping Gaussians, each placed so that under the rolling-shutter camera its footprint falls in one
    class of pixel: its centre is put on the ray of the wanted image point cast from the pose of that point's read-out
    time.  Every other tile of every other tile row (except the last two) holds one class; the last tile column, row
    and the corner hold the ragged-edge classes; one tile further in holds the stack on its pixel (12, 12)."""
    tw, th = tiles(W, H)
    rng = np.random.default_rng(seed)
    reg = _rs_classes(W, H)
    classes = dict(reg, **_edge_classes(W, H))
    names = list(reg)
    slots = [((tx, ty), names[(tx // 2 + 5 * (ty // 2)) % len(names)]) for ty in range(0, th - 2, 2)
             for tx in range(0, tw - 2, 2)]
    slots += [((tw - 1, ty), "last-col-inside" if (ty // 2) % 2 == 0 else "last-col-edge") for ty in range(0, th - 2, 2)]
    slots += [((tx, th - 1), "last-row-inside" if (tx // 2) % 2 == 0 else "last-row-edge") for tx in range(0, tw - 2, 2)]
    slots += [((tw - 1, th - 1), "corner-edge")]
    f, cxK, cyK = SENTINEL_F, W / 2.0, H / 2.0

    def place(u, v, z):
        R, t = rs_pose(frame_time(rs_type, u, v, W, H), V1)
        pc = np.array([(u - cxK) * z / f, (v - cyK) * z / f, z])
        return R.T @ (pc - t), R

    means, quats, scales, opac, boxes, labels = [], [], [], [], [], []
    for (tx, ty), name in slots:
        c = classes[name]
        x0, x1, y0, y1 = c["box"]
        sa_lo, sa_hi, sb_lo, sb_hi = c["sig"]
        rot = c.get("rot", math.pi)
        o = 0.5 + 0.4 * rng.random()
        k = math.sqrt(2.0 * math.log(255.0 * o))  # Mahalanobis radius of alpha = 1/255
        centred = c.get("centred", False)
        for _ in range(1000):
            sa, sb = rng.uniform(sa_lo, sa_hi), rng.uniform(sb_lo, sb_hi)
            th_ = rng.uniform(-rot, rot)
            cs, sn = math.cos(th_), math.sin(th_)
            hx = k * math.sqrt((sa * cs) ** 2 + (sb * sn) ** 2) + 0.35
            hy = k * math.sqrt((sa * sn) ** 2 + (sb * cs) ** 2) + 0.35
            lox, hix = max(x0 + hx, c.get("cx", (-1e9, 1e9))[0]), min(x1 - hx, c.get("cx", (-1e9, 1e9))[1])
            loy, hiy = max(y0 + hy, c.get("cy", (-1e9, 1e9))[0]), min(y1 - hy, c.get("cy", (-1e9, 1e9))[1])
            if lox <= hix and (centred or loy <= hiy):
                break
        else:
            raise AssertionError(f"sentinel class {name} cannot be placed")
        u = 16 * tx + rng.uniform(lox, hix)
        v = 16 * ty + (0.5 * (y0 + y1) if centred else rng.uniform(loy, hiy))
        z = 4.0
        m, R = place(u, v, z)
        # the footprint's axes in the image are the camera's x and y turned by th_: in the world, R^T of those
        qc = np.array([math.cos(th_ / 2), 0.0, 0.0, math.sin(th_ / 2)])
        from scipy.spatial.transform import Rotation
        qw = (Rotation.from_matrix(R.T) * Rotation.from_quat([qc[1], qc[2], qc[3], qc[0]])).as_quat()
        means.append(m)
        quats.append([qw[3], qw[0], qw[1], qw[2]])
        scales.append([sa * z / f, sb * z / f, 0.5 * min(sa, sb) * z / f])
        opac.append(o)
        boxes.append((16 * tx + x0, 16 * tx + x1, 16 * ty + y0, 16 * ty + y1))
        labels.append(name)
    sx, sy = 16 * (tw - 3) + 12, 16 * (th - 3) + 12
    for i in range(STACK):  # nearest first in the list: the depths spread over [3, 4)
        z = 3.0 + i / STACK
        m, _ = place(sx + 0.5, sy + 0.5, z)
        means.append(m)
        quats.append([1.0, 0.0, 0.0, 0.0])
        scales.append([0.3 * z / f] * 3)
        opac.append(0.02)
        boxes.append((sx, sx + 1, sy, sy + 1))
        labels.append("stack")
    n = len(means)
    sh = ((rng.random((n, 1, 3)) - 0.5) * 1.2).astype(np.float32)
    sc = dict(means=np.array(means, np.float32), quats=np.array(quats, np.float32), scales=np.array(scales, np.float32),
              opacities=np.array(opac, np.float32), sh_coeffs=sh, sh_degree=0, viewmats=np.eye(4, dtype=np.float32)[None],
              Ks=np.array([[[f, 0, cxK], [0, f, cyK], [0, 0, 1]]], np.float32), width=W, height=H, tile_size=16,
              background=rng.random((1, 3), dtype=np.float32))
    return sc, np.array(boxes, np.int64), labels


SENTINEL_SHAPE = (16 * 16 - 5, 16 * 12 - 7)  # 251 x 185: 16 x 12 tiles, W % 16 = 11, H % 16 = 9


@pytest.mark.parametrize("rs_type", RS_TYPES, ids=RS_IDS)
def test_rolling_sentinel_scene_per_gaussian_vs_f64_oracle(native, orc, cuda_device, rs_type):
    W, H = SENTINEL_SHAPE
    V1 = end_pose(np.eye(4, dtype=np.float32)[None], deg=1.0, shift=(0.01, 0.005, 0.0))
    sc, boxes, labels = rs_sentinel_scene(W, H, rs_type, V1)
    rs = dict(viewmats1=V1, rs_type=rs_type)
    n_g = sc["means"].shape[0]
    lab = np.array(labels)
    ref = orc.render_pipeline(sc, "f32", **rs)
    colors, off, flat, bg = ref["colors"], ref["tile_offsets"], ref["flatten_ids"], sc["background"]
    oa = (sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None], bg, None, W, H, 16, sc["viewmats"],
          sc["Ks"], off, flat)
    r64, a64, l64 = orc.raster_fwd(*oa, precision="f64", **rs)
    # the scene is what it claims: every sentinel is visible, alone on its pixels, and inside its box
    owner = np.where(a64[0, ..., 0] > 0, flat[l64[0]], -1)
    ys, xs = np.nonzero(owner >= 0)
    ids = owner[ys, xs]
    single = lab != "stack"
    assert set(np.nonzero(single)[0]) <= set(np.unique(ids)), "a sentinel has no footprint"
    assert np.all((xs >= boxes[ids, 0]) & (xs < boxes[ids, 1]) & (ys >= boxes[ids, 2]) & (ys < boxes[ids, 3]))
    one = single[ids]
    own_alpha = a64[0, ys, xs, 0][one]
    assert np.allclose(r64[0, ys[one], xs[one]], colors[0, ids[one]] * own_alpha[:, None] + (1 - own_alpha[:, None]) * bg,
                       atol=1e-5)
    for g in np.nonzero(lab == "even-row")[0]:
        assert set(ys[ids == g] % 2) == {0}
    for g in np.nonzero(lab == "odd-row")[0]:
        assert set(ys[ids == g] % 2) == {1}
    for w in range(8):
        for g in np.nonzero(lab == f"warp{w}")[0]:
            assert set(ys[ids == g] % 16) == {2 * w, 2 * w + 1}, (w, set(ys[ids == g] % 16))
    for g in np.nonzero(lab == "tile-boundary-x")[0]:
        assert {15, 0} <= set(xs[ids == g] % 16)
    for g in np.nonzero(lab == "tile-boundary-y")[0]:
        assert {15, 0} <= set(ys[ids == g] % 16)
    # the stack: one pixel, one list crossing a batch, every stacked Gaussian blended (T stays above 1e-4)
    stack = np.nonzero(~single)[0]
    sx, sy = boxes[stack[0], 0], boxes[stack[0], 2]
    tw, _ = tiles(W, H)
    tid = (sy // 16) * tw + sx // 16
    n_list = tile_counts(off, len(flat))[tid]
    assert n_list > RS_BATCH and l64[0, sy, sx] - off.ravel()[tid] >= RS_BATCH and 1 - a64[0, sy, sx, 0] > 1e-3
    print(f"[sentinel {RS_IDS[rs_type]}] {n_g} Gaussians ({STACK} stacked on pixel ({sx}, {sy}), whose tile lists "
          f"{n_list}), {len(flat)} intersections; classes: "
          + ", ".join(f"{c} {int((lab == c).sum())}" for c in sorted(set(labels))))

    rng = np.random.default_rng(11)
    vrc = (0.1 * rng.standard_normal((1, H, W, 3))).astype(np.float32)
    vra = (0.5 + rng.random((1, H, W, 1))).astype(np.float32)  # keeps dL/dalpha one-signed (test_gpu_blend_wide)
    t = to_dev(sc, cuda_device)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    nkw = dict(viewmats1=d(V1), rs_type=rs_type)
    na = (t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], t["background"], None, W, H, 16,
          t["viewmats"], t["Ks"], d(off), d(flat))
    r, a, li = (x.cpu().numpy() for x in native.rasterize_to_pixels_from_world_3dgs_fwd(*na, **nkw))
    e_img, e_a = rel(r, r64), rel(a, a64)
    print(f"[sentinel {RS_IDS[rs_type]}] image rel_l2 {e_img:.2e} (f32 oracle {rel(ref['renders'], r64):.2e}), alpha "
          f"{e_a:.2e} (f32 oracle {rel(ref['alphas'], a64):.2e}), last_ids differ at {int((li != l64).sum())} pixels")
    assert e_img < 1e-5 and e_a < 1e-4 and np.array_equal(li, ref["last_ids"])
    ga = (ref["alphas"], ref["last_ids"], vrc, vra)
    g64 = orc.raster_bwd(*oa, *ga, precision="f64", **rs)
    g32 = orc.raster_bwd(*oa, *ga, precision="f32", **rs)
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*na, *(d(x) for x in ga), **nkw)
    for nm, got, want, w32 in zip(GRADS, g, g64, g32):
        got = got.cpu().numpy().reshape(want.shape)
        noise = per_gauss_ratio(w32, want, n_g)
        tol = min(1e-2, max(SENTINEL_TOL_FLOOR, 10.0 * float(noise.max())))
        mine = per_gauss_ratio(got, want, n_g)
        worst = int(mine.argmax())
        m = grad_metrics(got, want, n_g, per_gauss_tol=tol)
        print(f"[sentinel {RS_IDS[rs_type]}] {nm}: rel_l2 {m['rel']:.2e} (f32 oracle {rel(w32, want):.2e}); worst "
              f"Gaussian {worst} ({labels[worst]}) at {mine[worst]:.2e} of its bound, f32 oracle's worst "
              f"{noise.max():.2e}; tolerance {tol:.1e}, over it: {m['n_bad']}")
        assert m["n_bad"] == 0, (nm, [(int(i), labels[i], float(mine[i])) for i in np.argsort(-mine)[:8]])
        assert m["rel"] < 1e-3 and m["max_abs"] < 5e-2, (nm, m)


# ------------------------------------------------------------------------------------------
# e. a static camera: the rolling-shutter kernels against the global-shutter ones
# ------------------------------------------------------------------------------------------
def test_static_rolling_shutter_equals_global_kernels(native, cuda_device):
    """viewmats1 = viewmats0 with a rolling direction sends the blend through gsb_raster_rs.cu on a camera that does not
    move: the image and gradients must match the quadratic-form kernels of gsb_raster.cu, an independent implementation,
    on the same lists, at an image of at least 32 x SMs tiles, where the float64 oracle would be slow."""
    dev = cuda_device
    W, H = shape("wide")
    sc = scenes.scene_b(width=W, height=H, N=40000, view=3, scale_mul=2.0)
    t = to_dev(sc, dev)
    tw, th = tiles(W, H)
    assert tw * th >= 32 * torch.cuda.get_device_properties(0).multi_processor_count
    radii, m2d, depths, _, _ = native.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"],
                                                               t["viewmats"], t["Ks"], W, H)
    _, ids, flat = native.intersect_tile(m2d, radii, depths, 1, 16, tw, th, True)
    off = native.intersect_offset(ids, 1, tw, th)
    n = tile_counts(off.cpu().numpy(), len(flat))
    assert (n > RS_BATCH).sum() >= 100, int((n > RS_BATCH).sum())
    n_g = sc["means"].shape[0]
    gen = torch.Generator(device=dev).manual_seed(3)
    colors = torch.rand((1, n_g, 3), device=dev, generator=gen)
    vc = torch.randn((1, H, W, 3), device=dev, generator=gen)
    va = torch.randn((1, H, W, 1), device=dev, generator=gen)
    fa = (t["means"], t["quats"], t["scales"], colors, t["opacities"][None], t["background"], None, W, H, 16,
          t["viewmats"], t["Ks"], off, flat)
    r0, a0, l0 = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa)
    g0 = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a0, l0, vc, va)
    print(f"[static] {W}x{H}, {len(flat)} intersections, {int((n > RS_BATCH).sum())} tiles over {RS_BATCH} records")
    for rs_type in RS_TYPES:
        kw = dict(viewmats1=t["viewmats"].clone(), rs_type=rs_type)
        r1, a1, l1 = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **kw)
        d_img = (r1 - r0).abs().amax(-1)
        lm = float((l1 != l0).float().mean())
        tag = f"static {RS_IDS[rs_type]} vs global kernels"
        print(f"[{tag}] image rel_l2 {rel(r1, r0):.2e}, alpha {rel(a1, a0):.2e}, last_ids differ {lm:.2e}, "
              f"max |d image| {float(d_img.max()):.2e}")
        assert rel(r1, r0) < 5e-5 and rel(a1, a0) < 1e-5 and lm < 1e-3
        assert float(d_img.max()) < 2e-2 and float((d_img > 1e-4).float().mean()) < 1e-3
        g1 = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a0, l0, vc, va, **kw)
        for nm, x, y in zip(GRADS, g1, g0):
            assert_grad_close(x, y, nm, n_g, rel_tol=GRAD_REL_TOL, tag=tag)


# ------------------------------------------------------------------------------------------
# f. reversal symmetry
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", [(0, 2), (1, 3)], ids=["vertical", "horizontal"])
def test_reversed_direction_with_swapped_poses_on_the_gpu(native, orc, cuda_device, dense, pair):
    """Top-to-bottom from A to B and bottom-to-top from B to A read every pixel centre at the same pose (likewise for
    the two horizontal directions): the GPU must give the same image and gradients, to float32 rounding."""
    sc, V1 = dense["sc"], dense["V1"]
    W, H = sc["width"], sc["height"]
    a_t, b_t = pair
    off, flat = oracle_lists(orc, sc, oracle_kwargs("pinhole", V1, a_t))
    t = to_dev(sc, cuda_device)
    d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(cuda_device)
    A, B = t["viewmats"], d(V1)
    colors, vc, va = d(dense["colors"]), d(dense["vrc"]), d(dense["vra"])

    def run(v0, v1, rs_type, alphas=None, last=None):
        fa = (t["means"], t["quats"], t["scales"], colors, t["opacities"][None], t["background"], None, W, H, 16, v0,
              t["Ks"], d(off), d(flat))
        out = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa, viewmats1=v1, rs_type=rs_type)
        a_, l_ = (out[1], out[2]) if alphas is None else (alphas, last)
        return out, native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a_, l_, vc, va, viewmats1=v1, rs_type=rs_type)

    (r1, a1, l1), g1 = run(A, B, a_t)
    (r2, a2, l2), g2 = run(B, A, b_t, a1, l1)
    (rg, _, _), _ = run(A, None, 4)
    lm = float((l1 != l2).float().mean())
    tag = f"{RS_IDS[a_t]} (A, B) vs {RS_IDS[b_t]} (B, A)"
    print(f"[{tag}] image rel_l2 {rel(r2, r1):.2e}, alpha {rel(a2, a1):.2e}, last_ids differ {lm:.2e}; the global "
          f"shutter differs by {rel(rg, r1):.2e}")
    assert rel(rg, r1) > 1e-2  # the motion matters
    assert rel(r2, r1) < 5e-5 and rel(a2, a1) < 1e-5 and lm < 1e-3
    for nm, x, y in zip(GRADS, g2, g1):
        assert_grad_close(x, y, nm, sc["means"].shape[0], rel_tol=GRAD_REL_TOL, tag=tag)


# ------------------------------------------------------------------------------------------
# g. empty inputs
# ------------------------------------------------------------------------------------------
def _edge_run(native, dev, sc, masks=None):
    W, H = sc["width"], sc["height"]
    tw, th = tiles(W, H)
    t = to_dev(sc, dev)
    kw = dict(viewmats1=torch.from_numpy(end_pose(sc["viewmats"])).to(dev), rs_type=0)
    if sc["means"].shape[0]:
        radii, m2d, depths, _, _ = native.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"],
                                                                   t["viewmats"], t["Ks"], W, H, **kw)
        _, ids, flat = native.intersect_tile(m2d, radii, depths, 1, 16, tw, th, True)
        off = native.intersect_offset(ids, 1, tw, th)
    else:
        off = torch.zeros((1, th, tw), dtype=torch.int32, device=dev)
        flat = torch.zeros((0,), dtype=torch.int32, device=dev)
    n_g = sc["means"].shape[0]
    colors = torch.rand((1, n_g, 3), device=dev)
    mk = None if masks is None else torch.from_numpy(masks).to(dev)
    fa = (t["means"], t["quats"], t["scales"], colors, t["opacities"][None], t["background"], mk, W, H, 16,
          t["viewmats"], t["Ks"], off, flat)
    r, a, li = native.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **kw)
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a, li, torch.randn((1, H, W, 3), device=dev),
                                                       torch.randn((1, H, W, 1), device=dev), **kw)
    torch.cuda.synchronize()
    assert torch.all(r == t["background"].reshape(1, 1, 1, 3))
    for nm, x in zip(GRADS, g):
        assert x.shape[0] in (n_g, 1) and not x.any(), nm
    return len(flat), a


def test_rolling_edges_empty_lists_masks_and_no_gaussians(native, cuda_device):
    """With a rolling shutter: every Gaussian behind the camera (n_isects = 0), every tile masked, and N = 0.  The
    forward gives the background, the backward exact zeros, and neither raises."""
    sc = scenes.scene_small(N=500, width=90, height=70, view=None, sh_degree=0)
    behind = dict(sc, means=sc["means"] * np.array([1, 1, -1], np.float32))
    n, a = _edge_run(native, cuda_device, behind)
    assert n == 0 and not a.any()
    tw, th = tiles(sc["width"], sc["height"])
    n, _ = _edge_run(native, cuda_device, sc, masks=np.zeros((1, th, tw), bool))
    assert n > 1000
    empty = dict(sc, means=sc["means"][:0], quats=sc["quats"][:0], scales=sc["scales"][:0], opacities=sc["opacities"][:0])
    n, a = _edge_run(native, cuda_device, empty)
    assert n == 0 and not a.any()


# ------------------------------------------------------------------------------------------
# h. the reference's kernels, stored; and the dump that stores them
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(GOLDEN_CASES)), ids=[f"{c}-{RS_IDS[r]}" for c, r in GOLDEN_CASES])
def test_library_matches_reference_rolling_golden(native, cuda_device, case):
    gold = np.load(G)
    cam, rs_type = GOLDEN_CASES[case]
    p = f"c{case}_"
    sc = golden_scene()
    W, H = sc["width"], sc["height"]
    V1 = golden_end_pose(sc)
    t = to_dev(sc, cuda_device)
    nkw = native_kwargs(cam, cuda_device, V1, rs_type)
    out = native.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W,
                                          H, 0.3, 0.01, 1e4, 0.0, **nkw)
    radii, m2d, depths, conics = (x.cpu().numpy() for x in out[:4])
    g_r = gold[p + "radii"]
    mism = int((radii != g_r).any(-1).sum())
    both = (radii > 0).all(-1) & (g_r > 0).all(-1)
    ok = both & (np.abs(m2d - gold[p + "means2d"]).max(-1) <= 0.02)
    tag = f"{cam} {RS_IDS[rs_type]} vs stored reference"
    print(f"[{tag}] radii differ {mism}, visible {int(both.sum())}, off by > 0.02 px {int((both & ~ok).sum())}; "
          f"means2d rel {rel(m2d[ok], gold[p + 'means2d'][ok]):.2e}")
    assert both.sum() > 180 and mism <= 3 and (both & ~ok).sum() <= 3
    assert rel(m2d[ok], gold[p + "means2d"][ok]) < 5e-5 and rel(depths[both], gold[p + "depths"][both]) < 1e-6
    assert rel(conics[ok], gold[p + "conics"][ok]) < 1e-3
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    fa = (t["means"], t["quats"], t["scales"], d(golden_colors(sc)), t["opacities"][None], t["background"], None, W, H,
          16, t["viewmats"], t["Ks"], d(gold[p + "tile_offsets"]), d(gold[p + "flatten_ids"]))
    r, a, li = (x.cpu().numpy() for x in native.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **nkw))
    lm = float((li != gold[p + "last_ids"]).mean())
    print(f"[{tag}] image rel_l2 {rel(r, gold[p + 'renders']):.2e}, last_ids differ {lm:.2e}")
    assert rel(r, gold[p + "renders"]) < 1e-4 and rel(a, gold[p + "alphas"]) < 1e-4 and lm < 2e-3
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*fa, d(gold[p + "alphas"]), d(gold[p + "last_ids"]),
                                                       d(gold["v_render_colors"]), d(gold["v_render_alphas"]), **nkw)
    for nm, x in zip(GRADS, g):
        assert_grad_close(x.cpu().numpy().reshape(gold[p + nm].shape), gold[p + nm], nm, sc["means"].shape[0], tag=tag)


def test_dump_reference_rolling_golden(native, cuda_device, tmp_path):
    """Writes ref_rolling_small.npz (into $GSB_GOLDEN_OUT, else a temporary directory): the rolling-shutter outputs of
    the reference's kernels built without --use_fast_math, for the cases of GOLDEN_CASES on a small ragged scene.  The
    file is committed as tests/golden/ref_rolling_small.npz and pins the oracle in the no-GPU suite
    (tests/test_oracle_rolling_shutter.py) and this library in test_library_matches_reference_rolling_golden."""
    from oracle import ref_ops
    if not ref_ops.precise_available():
        pytest.skip("oracle/_ref/libgsplat_ref_precise.so not built (build() makes it where the reference's sources are "
                    "present)")
    ref = ref_ops.backend_precise(native)
    sc = golden_scene()
    W, H = sc["width"], sc["height"]
    tw, th = tiles(W, H)
    t = to_dev(sc, cuda_device)
    V1 = golden_end_pose(sc)
    vrc, vra = golden_cotangents(sc)
    colors = golden_colors(sc)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    arrays = dict(v_render_colors=vrc, v_render_alphas=vra, colors=colors, viewmats1=V1)
    for case, (cam, rs_type) in enumerate(GOLDEN_CASES):
        kw = native_kwargs(cam, cuda_device, V1, rs_type)
        radii, m2d, depths, conics, _ = ref.projection_ut_3dgs_fused(
            t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **kw)
        vis = (radii > 0).all(-1)
        m2d = torch.where(vis[..., None], m2d, torch.zeros_like(m2d))
        depths = torch.where(vis, depths, torch.zeros_like(depths))
        conics = torch.where(vis[..., None], conics, torch.zeros_like(conics))
        _, ids, flat = ref.intersect_tile(m2d, radii, depths, 1, 16, tw, th, True)
        off = ref.intersect_offset(ids, 1, tw, th)
        fa = (t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], t["background"], None, W, H, 16,
              t["viewmats"], t["Ks"], off, flat)
        r, a, li = ref.rasterize_to_pixels_from_world_3dgs_fwd(*fa, **kw)
        g = ref.rasterize_to_pixels_from_world_3dgs_bwd(*fa, a, li, d(vrc), d(vra), **kw)
        p = f"c{case}_"
        for k, v in dict(radii=radii, means2d=m2d, depths=depths, conics=conics, tile_offsets=off, flatten_ids=flat,
                         renders=r, alphas=a, last_ids=li, **dict(zip(GRADS, g))).items():
            arrays[p + k] = v.cpu().numpy()
    out = os.environ.get("GSB_GOLDEN_OUT") or str(tmp_path)
    os.makedirs(out, exist_ok=True)
    np.savez_compressed(os.path.join(out, "ref_rolling_small.npz"), **arrays)
