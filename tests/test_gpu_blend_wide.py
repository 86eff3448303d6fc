"""GPU: the blend backward's four-pixel ("wide") variant against the float64 CPU oracle.

The from-world and EWA blend backward runs in one of two shapes (gsb_raster.cu:733-760, launch_bwd_kernel): four
pixels per thread in 64-thread CTAs, where a warp covers an 8x16 half tile, when the image has at least
SMs x (resident 64-thread CTAs per SM) tiles; else two pixels per thread in 128-thread CTAs.  Every training-sized
image takes the wide variant.  The tests here pick image sizes that force one variant or the other whatever the
occupancy query returns, and check the wide one against an exact reference:
  * the operator path with and without a background, with tile masks, and with distorted cameras (the
    general-camera instantiation, whose pixels each have their own x);
  * a sparse "sentinel" scene whose Gaussians each cover one class of pixel of the 8x16 layout, checked per
    Gaussian with no allowance for outliers;
  * the wide variant against the two-pixel one on the same pixels, through a tile-aligned crop;
  * the fastgs (EWA) and fused paths.
"""
import math
import re

import numpy as np
import pytest
import torch

import scenes
from parity import assert_grad_close, grad_metrics, rel, to_dev
from test_gpu_parity import DISTORTED

pytestmark = pytest.mark.gpu

GRADS = ("v_means", "v_quats", "v_scales", "v_colors", "v_opacities")
MAX_CTAS_PER_SM = 32  # the most resident CTAs an sm_90 multiprocessor can hold, whatever their size
# Dense enough that many tiles walk more records than the wide backward's ring holds (see batches_walked).
WIDE_SCENE = dict(N=40000, view=3, scale_mul=2.0)
BWD_WIDE_BATCH, BWD_RING = 64, 3  # gsb_raster.cu raster_bwd_kernel<.., 4>: one record per thread, three stages


# ------------------------------------------------------------------------------------------
# shapes that force each backward variant
# ------------------------------------------------------------------------------------------
def sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def shape(kind: str):
    """(W, H) of an image whose tile count forces the backward variant `kind`.  launch_bwd_kernel
    (gsb_raster.cu:733-760) runs four pixels per thread from SMs x (resident CTAs per SM) tiles on: at least
    32 x SMs tiles takes that branch for any occupancy, fewer than SMs tiles never does.  Both shapes have ragged
    edges with different remainders (W % 16 = 12, H % 16 = 3): the last tile column leaves part of the right warp
    half outside the image, and in the last tile row only each thread's first pixel row is inside."""
    sms = sm_count()
    n = math.isqrt(MAX_CTAS_PER_SM * sms - 1) + 2 if kind == "wide" else math.isqrt(sms - 1)
    return 16 * n - 4, 16 * n - 13


def tiles(W, H):
    return (W + 15) // 16, (H + 15) // 16


def check_tiles(kind, W, H):
    tw, th = tiles(W, H)
    sms = sm_count()
    print(f"[{kind}] {W}x{H}: {tw}x{th} = {tw * th} tiles on {sms} SMs")
    if kind == "wide":
        assert tw * th >= MAX_CTAS_PER_SM * sms  # gsb_raster.cu:733-760: four pixels per thread
    else:
        assert tw * th < sms  # gsb_raster.cu:733-760: two pixels per thread
    assert W % 16 and H % 16 and W % 16 != H % 16


_BWD_NAME = re.compile(r"raster_bwd_kernel<(\w+), (\w+), (\d+)>")


def bwd_kernels(fn):
    """Template arguments (general camera, EWA, pixels per thread) of every raster_bwd_kernel that `fn` launches,
    from a torch.profiler CUDA trace; None where kernel tracing is unavailable."""
    from torch.profiler import ProfilerActivity, profile
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
    except Exception as e:  # no CUPTI on this machine
        print(f"kernel tracing unavailable: {e}")
        return None
    if not any("kernel" in n for n in names):
        print("kernel tracing returned no kernels")
        return None
    return {m.groups() for n in names for m in [_BWD_NAME.search(n)] if m}


@pytest.fixture(scope="module", autouse=True)
def _oracle_threads(orc):
    orc.set_threads(orc.max_threads())
    yield
    orc.set_threads(1)


@pytest.fixture(scope="module")
def wide(orc, cuda_device):
    """A 1080p-like slab at the wide shape: the oracle's lists and colours, and seeded cotangents."""
    W, H = shape("wide")
    sc = scenes.scene_b(width=W, height=H, **WIDE_SCENE)
    rng = np.random.default_rng(2)
    vrc = rng.standard_normal((1, H, W, 3)).astype(np.float32)
    vra = rng.standard_normal((1, H, W, 1)).astype(np.float32)
    ref = orc.render_pipeline(sc, "f32")
    n_max = int(np.diff(np.append(ref["tile_offsets"].ravel(), len(ref["flatten_ids"]))).max())
    nb = batches_walked(ref["tile_offsets"], len(ref["flatten_ids"]), ref["last_ids"], W, H)
    n_reuse = int((nb > BWD_RING).sum())
    print(f"[wide scene] {W}x{H}, {sc['means'].shape[0]} Gaussians, {len(ref['flatten_ids'])} intersections, "
          f"longest tile list {n_max}, mean alpha {float(ref['alphas'].mean()):.3f}; the wide backward walks up to "
          f"{int(nb.max())} batches of {BWD_WIDE_BATCH} records, more than its {BWD_RING} ring stages in {n_reuse} tiles")
    # the ring's stage reuse (wait on the stage's release, refill, phase parity) must run, and run in many tiles
    assert n_reuse >= 100, n_reuse
    return dict(sc=sc, ref=ref, vrc=vrc, vra=vra, W=W, H=H)


def batches_walked(tile_offsets, n_isects, last_ids, W, H, batch=BWD_WIDE_BATCH):
    """Per tile, the batches of `batch` records the backward walks: from the tile's first record up to its newest
    contributor, max(last_ids) over the tile capped at the tile's last record (gsb_raster.cu:537-543)."""
    tw, th = tiles(W, H)
    newest = np.full((th * 16, tw * 16), -1, np.int64)
    newest[:H, :W] = np.asarray(last_ids).reshape(H, W)
    newest = newest.reshape(th, 16, tw, 16).max(axis=(1, 3)).ravel()
    start = np.asarray(tile_offsets, np.int64).ravel()
    end = np.append(start[1:], n_isects)
    total = np.maximum(np.minimum(newest, end - 1) - start + 1, 0)
    return (total + batch - 1) // batch


@pytest.mark.parametrize("kind", ["wide", "small"])
def test_shapes_select_the_backward_variant(native, cuda_device, kind):
    W, H = shape(kind)
    check_tiles(kind, W, H)
    sc = scenes.scene_small(N=400, width=W, height=H, view=1)
    t = to_dev(sc, cuda_device)
    kpix = "4" if kind == "wide" else "2"
    for model, general in (("pinhole", "false"), ("opencv", "true")):
        cam = {}
        if model == "opencv":
            cfg = DISTORTED["opencv"]
            cam = dict(camera_model=cfg["camera_model"], radial_coeffs=torch.from_numpy(cfg["radial"]).to(cuda_device),
                       tangential_coeffs=torch.from_numpy(cfg["tangential"]).to(cuda_device),
                       thin_prism_coeffs=torch.from_numpy(cfg["thin_prism"]).to(cuda_device))

        def step():
            leaves = {k: t[k].clone().requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh_coeffs")}
            out = native.rasterize(leaves["means"], leaves["quats"], leaves["scales"], leaves["opacities"],
                                   leaves["sh_coeffs"], sc["sh_degree"], t["viewmats"], t["Ks"], W, H,
                                   bg_color=t["background"], **cam)
            out.render_colors.sum().backward()

        launched = bwd_kernels(step)
        if launched is None:
            print(f"[{kind} {model}] launched kernel not confirmed")
            continue
        print(f"[{kind} {model}] raster_bwd_kernel launches: {sorted(launched)}")
        assert launched == {(general, "false", kpix)}


# ------------------------------------------------------------------------------------------
# operator path at the wide shape vs the float64 oracle, on the oracle's lists and colours
# ------------------------------------------------------------------------------------------
def _oracle_args(sc, colors, bg, masks, off, flat):
    W, H = sc["width"], sc["height"]
    return (sc["means"], sc["quats"], sc["scales"], colors, sc["opacities"][None], bg, masks, W, H, 16,
            sc["viewmats"], sc["Ks"], off, flat)


def _blend_vs_oracle(native, orc, dev, tag, sc, colors, off, flat, bg, masks, vrc, vra, okw=None, nkw=None):
    """Blend forward and backward on the GPU against the oracle on the same lists: the image, alpha and last_ids
    against the float64 forward (the float32 oracle's distance from it printed beside), the gradients against the
    float64 backward given the float32 oracle's alpha and last_ids (both sides get the same ones)."""
    okw, nkw = okw or {}, nkw or {}
    W, H = sc["width"], sc["height"]
    oa = _oracle_args(sc, colors, bg, masks, off, flat)
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
    print(f"[{tag}] vs f64 oracle: image rel_l2 {e_img:.2e} (f32 oracle {n_img:.2e}), alpha {e_alpha:.2e} "
          f"(f32 oracle {n_alpha:.2e}), last_ids differ {li_bad:.2e} (f32 oracle "
          f"{float((l32[0][keep] != l64[0][keep]).mean()):.2e}), max |d image| {float(d_img.max()):.2e}")
    assert e_img < 1e-4 and e_alpha < 1e-4
    assert float(d_img.max()) < 2e-2  # a 1/255-cut flip moves a pixel by <= alpha * colour
    assert (d_img > 1e-4).mean() < 2e-3
    assert li_bad < 2e-3
    nb = batches_walked(off, len(flat), l32, W, H)
    if masks is not None:
        nb = nb * masks.ravel()  # a masked tile walks nothing
    print(f"[{tag}] tiles whose backward walks more than {BWD_RING} batches: {int((nb > BWD_RING).sum())}")
    assert (nb > BWD_RING).sum() >= 100

    ga = (a32, l32, vrc, vra)
    g64 = orc.raster_bwd(*oa, *ga, precision="f64", **okw)
    g32 = orc.raster_bwd(*oa, *ga, precision="f32", **okw)
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*na, *(d(x) for x in ga), **nkw)
    n_g = sc["means"].shape[0]
    for nm, got, want, w32 in zip(GRADS, g, g64, g32):
        got = got.cpu().numpy().reshape(want.shape)
        assert_close_as_f32(got, want, w32, nm, n_g, tag)
        assert_untouched_near_zero(got, want, w32, nm, n_g, tag)


def assert_untouched_near_zero(got, want, w32, name, n_g, tag):
    """A Gaussian the float64 oracle gives no contribution gets none on the GPU either, except where one of its pixels
    sits at the alpha >= 1/255 cut and float32 rounding lets it through: there may be at most twice as many such
    Gaussians as the float32 oracle has (and 2), each with a gradient below 1e-3 of the RMS Gaussian gradient (one
    such Gaussian measured in the opencv case, at 6e-6 of the RMS, and the float32 oracle has the same one)."""
    g, w, s = (np.abs(np.asarray(x, np.float64)).reshape(n_g, -1).sum(-1) for x in (got, want, w32))
    untouched = w == 0
    rms = float(np.sqrt(np.mean(w[~untouched] ** 2)))
    n_gpu, n_32 = int((g[untouched] > 0).sum()), int((s[untouched] > 0).sum())
    worst = float(g[untouched].max() / rms) if untouched.any() else 0.0
    print(f"[{tag}] {name}: of {int(untouched.sum())} Gaussians without a contribution, {n_gpu} get a gradient "
          f"(f32 oracle {n_32}), the largest {worst:.1e} of the RMS")
    assert n_gpu <= max(2, 2 * n_32) and worst < 1e-3, (name, n_gpu, n_32, worst)


def assert_close_as_f32(got, want, w32, name, n_g, tag):
    """parity.assert_grad_close against the float64 oracle.  The fraction of Gaussians off by more than 1 % may reach
    twice what the float32 oracle shows on the same inputs (each one a pixel whose 1/255 or saturation decision
    flips between float32 and float64), and never less than the default 2e-3.

    This is NOT a per-Gaussian check: on these dense scenes the float32 oracle itself has a few tenths of a percent
    of Gaussians off by more than 1 %, so a bug confined to a few dozen Gaussians (one pixel class, one warp half,
    one ragged tile) can pass here.  test_sentinel_scene_per_gaussian_vs_f64_oracle is the check that allows no
    outlier; these cases bound the whole tensor and the bulk of the Gaussians."""
    n32 = grad_metrics(w32, want, n_g)
    frac_tol = max(2e-3, 2.0 * n32["frac_bad"])
    assert_grad_close(got, want, name, n_g, frac_tol=frac_tol,
                      tag=f"{tag} vs f64 oracle; f32 oracle itself {n32['rel']:.1e}, {n32['n_bad']} Gaussians off by > 0.01")


@pytest.mark.parametrize("background", [True, False], ids=["background", "no_background"])
def test_wide_blend_vs_f64_oracle(native, orc, cuda_device, wide, background):
    sc, ref = dict(wide["sc"]), wide["ref"]
    check_tiles("wide", sc["width"], sc["height"])
    bg = sc["background"] if background else None
    sc["background"] = bg
    _blend_vs_oracle(native, orc, cuda_device, f"wide, {'with' if background else 'no'} background", sc, ref["colors"],
                     ref["tile_offsets"], ref["flatten_ids"], bg, None, wide["vrc"], wide["vra"])


def tile_masks(tw, th, seed=8):
    """Masked tiles: the ragged corner, one whole tile row, a ragged tile of the last column and of the last row,
    and scattered single tiles."""
    m = np.ones((1, th, tw), bool)
    m[0, th - 1, tw - 1] = False
    m[0, th // 2, :] = False
    m[0, th // 3, tw - 1] = False
    m[0, th - 1, tw // 3] = False
    rng = np.random.default_rng(seed)
    m.reshape(-1)[rng.choice(tw * th, max(8, tw * th // 100), replace=False)] = False
    return m


def test_wide_blend_tile_masks_vs_f64_oracle(native, orc, cuda_device, wide):
    sc, ref = wide["sc"], wide["ref"]
    tw, th = tiles(wide["W"], wide["H"])
    masks = tile_masks(tw, th)
    print(f"[wide, tile masks] {int((~masks).sum())} of {tw * th} tiles masked")
    _blend_vs_oracle(native, orc, cuda_device, "wide, tile masks", sc, ref["colors"], ref["tile_offsets"],
                     ref["flatten_ids"], sc["background"], masks, wide["vrc"], wide["vra"])


def _camera_kwargs(model, dev):
    cfg = DISTORTED[model]
    okw = dict(camera_model=cfg["camera_model"], radial=cfg["radial"], tangential=cfg["tangential"],
               thin_prism=cfg["thin_prism"])
    d = lambda a: None if a is None else torch.from_numpy(a).to(dev)
    nkw = dict(camera_model=cfg["camera_model"], radial_coeffs=d(cfg["radial"]), tangential_coeffs=d(cfg["tangential"]),
               thin_prism_coeffs=d(cfg["thin_prism"]))
    return okw, nkw


@pytest.mark.parametrize("model", ["opencv", "fisheye"])
def test_wide_distorted_camera_vs_f64_oracle(native, orc, cuda_device, wide, model):
    """The general-camera backward, raster_bwd_kernel<true, false, 4>: every pixel has its own unprojected x and
    the warp's cull box is reduced over 16 rows of unprojected pixels."""
    sc = wide["sc"]
    W, H = sc["width"], sc["height"]
    tw, th = tiles(W, H)
    okw, nkw = _camera_kwargs(model, cuda_device)
    t = to_dev(sc, cuda_device)
    r_ref, m_ref, d_ref, _, _ = orc.projection_ut(sc["means"], sc["quats"], sc["scales"], sc["opacities"],
                                                  sc["viewmats"], sc["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **okw)
    radii, means2d, _, _, _ = native.projection_ut_3dgs_fused(
        t["means"], t["quats"], t["scales"], t["opacities"], t["viewmats"], t["Ks"], W, H, 0.3, 0.01, 1e4, 0.0, **nkw)
    n_g = sc["means"].shape[0]
    mism = int((radii.cpu().numpy() != r_ref).any(-1).sum())
    both = (radii.cpu().numpy() > 0).all(-1) & (r_ref > 0).all(-1)
    e_m2d = rel(means2d.cpu().numpy()[both], m_ref[both])
    print(f"[wide {model}] projection: radii differ for {mism} of {n_g}, means2d rel_l2 {e_m2d:.2e}")
    assert mism <= max(3, n_g // 2000) and both.sum() > n_g // 2 and e_m2d < 1e-4
    _, ids, flat = orc.isect_tiles(m_ref, r_ref, d_ref, 1, 16, tw, th)
    off = orc.isect_offsets(ids, 1, tw, th)
    colors = np.random.default_rng(21).random((1, n_g, 3), dtype=np.float32)
    _blend_vs_oracle(native, orc, cuda_device, f"wide {model}", sc, colors, off, flat, sc["background"], None,
                     wide["vrc"], wide["vra"], okw, nkw)


# ------------------------------------------------------------------------------------------
# sentinel scene: every pixel class of the 8x16 warp layout, checked per Gaussian
# ------------------------------------------------------------------------------------------
# Each class: the tile-local pixel box [x0, x1) x [y0, y1) its footprint must stay in, the range of its centre
# (tile-local pixel coordinates, pixel centres at k + 0.5; None = anywhere the box allows), the ranges of its two
# standard deviations in pixels and of its in-plane rotation.  Boxes reach at most 8 pixels into the next tile,
# which the layout leaves empty, so no two footprints overlap.
REGULAR = {
    "rows0-3": dict(box=(0, 16, 0, 4), sig=(0.6, 1.2, 0.28, 0.38), rot=0.2),
    "rows4-7": dict(box=(0, 16, 4, 8), sig=(0.6, 1.2, 0.28, 0.38), rot=0.2),
    "rows8-11": dict(box=(0, 16, 8, 12), sig=(0.6, 1.2, 0.28, 0.38), rot=0.2),
    "rows12-15": dict(box=(0, 16, 12, 16), sig=(0.6, 1.2, 0.28, 0.38), rot=0.2),
    "left-half": dict(box=(0, 8, 0, 16), sig=(0.4, 0.9, 0.4, 1.6), rot=0.2),
    "right-half": dict(box=(8, 16, 0, 16), sig=(0.4, 0.9, 0.4, 1.6), rot=0.2),
    "warp-boundary": dict(box=(2, 14, 0, 16), cx=(7.6, 8.4), sig=(0.5, 1.2, 0.5, 1.5)),
    "tile-boundary-x": dict(box=(8, 24, 0, 16), cx=(15.6, 16.4), sig=(0.5, 1.2, 0.5, 1.5)),
    "tile-boundary-y": dict(box=(0, 16, 8, 24), cy=(15.6, 16.4), sig=(0.5, 1.5, 0.5, 1.2)),
    "thin-rows8-15": dict(box=(0, 16, 8, 16), sig=(1.5, 2.2, 0.3, 0.55), rot=0.35),
}


def _edge_classes(W, H):
    rx, ry = W % 16, H % 16
    return {
        "last-col-inside": dict(box=(0, rx, 0, 16), sig=(0.3, 0.8, 0.3, 1.2)),
        "last-col-edge": dict(box=(rx - 6, 24, 0, 16), cx=(rx - 0.4, rx + 0.4), sig=(0.5, 1.0, 0.5, 1.2)),
        "last-row-inside": dict(box=(0, 16, 0, ry), sig=(0.3, 1.2, 0.25, 0.32), rot=0.0),
        "last-row-edge": dict(box=(0, 16, ry - 3, 24), cy=(ry - 0.4, ry + 0.4), sig=(0.5, 1.2, 0.5, 0.8)),
        "corner-edge": dict(box=(rx - 6, 24, ry - 3, 24), cx=(rx - 0.4, rx + 0.4), cy=(ry - 0.4, ry + 0.4),
                            sig=(0.5, 0.9, 0.5, 0.8)),
    }


def sentinel_scene(W, H, seed=5, f=500.0):
    """Small non-overlapping Gaussians on an identity view, each placed (through a known K) so that its footprint
    -- the pixels where alpha >= 1/255 -- falls in one class of pixel of the tile.  Every other tile of every
    other tile row (except the last two) holds one regular class; the last tile column, the last tile row and the
    corner tile hold the ragged-edge classes.  The layout depends only on the tile grid."""
    tw, th = tiles(W, H)
    rng = np.random.default_rng(seed)
    classes = dict(REGULAR, **_edge_classes(W, H))
    reg = list(REGULAR)
    slots = [((tx, ty), reg[(tx // 2 + 3 * (ty // 2)) % len(reg)]) for ty in range(0, th - 2, 2)
             for tx in range(0, tw - 2, 2)]
    slots += [((tw - 1, ty), "last-col-inside" if (ty // 2) % 2 == 0 else "last-col-edge") for ty in range(0, th - 2, 2)]
    slots += [((tx, th - 1), "last-row-inside" if (tx // 2) % 2 == 0 else "last-row-edge") for tx in range(0, tw - 2, 2)]
    slots += [((tw - 1, th - 1), "corner-edge")]
    Z = 4.0
    cxK, cyK = W / 2.0, H / 2.0
    n = len(slots)
    means = np.zeros((n, 3), np.float64)
    quats = np.zeros((n, 4), np.float64)
    scales = np.zeros((n, 3), np.float64)
    opac = (0.5 + 0.4 * rng.random(n)).astype(np.float32)
    boxes, labels = np.zeros((n, 4), np.int64), []
    for i, ((tx, ty), name) in enumerate(slots):
        c = classes[name]
        x0, x1, y0, y1 = c["box"]
        sa_lo, sa_hi, sb_lo, sb_hi = c["sig"]
        rot = c.get("rot", math.pi)
        k = math.sqrt(2.0 * math.log(255.0 * float(opac[i])))  # Mahalanobis radius of alpha = 1/255
        for _ in range(1000):
            sa, sb = rng.uniform(sa_lo, sa_hi), rng.uniform(sb_lo, sb_hi)
            th_ = rng.uniform(-rot, rot)
            cs, sn = math.cos(th_), math.sin(th_)
            hx = k * math.sqrt((sa * cs) ** 2 + (sb * sn) ** 2) + 0.35  # half extents of the footprint + margin
            hy = k * math.sqrt((sa * sn) ** 2 + (sb * cs) ** 2) + 0.35
            lox, hix = max(x0 + hx, c.get("cx", (-1e9, 1e9))[0]), min(x1 - hx, c.get("cx", (-1e9, 1e9))[1])
            loy, hiy = max(y0 + hy, c.get("cy", (-1e9, 1e9))[0]), min(y1 - hy, c.get("cy", (-1e9, 1e9))[1])
            if lox <= hix and loy <= hiy:
                break
        else:
            raise AssertionError(f"sentinel class {name} cannot be placed")
        u = 16 * tx + rng.uniform(lox, hix)
        v = 16 * ty + rng.uniform(loy, hiy)
        means[i] = ((u - cxK) * Z / f, (v - cyK) * Z / f, Z)
        quats[i] = (math.cos(th_ / 2), 0.0, 0.0, math.sin(th_ / 2))
        scales[i] = (sa * Z / f, sb * Z / f, 0.5 * min(sa, sb) * Z / f)
        boxes[i] = (16 * tx + x0, 16 * tx + x1, 16 * ty + y0, 16 * ty + y1)
        labels.append(name)
    sh = ((rng.random((n, 1, 3)) - 0.5) * 1.2).astype(np.float32)
    sc = dict(means=means.astype(np.float32), quats=quats.astype(np.float32), scales=scales.astype(np.float32),
              opacities=opac, sh_coeffs=sh, sh_degree=0, viewmats=np.eye(4, dtype=np.float32)[None],
              Ks=np.array([[[f, 0, cxK], [0, f, cyK], [0, 0, 1]]], np.float32), width=W, height=H, tile_size=16,
              background=rng.random((1, 3), dtype=np.float32))
    return sc, boxes, labels


def per_gauss_ratio(got, want, n_gauss, floor_frac=1e-2):
    """Each Gaussian's error over the bound of parity.grad_metrics: a Gaussian counts as bad there exactly when its
    ratio exceeds per_gauss_tol."""
    g = np.asarray(got, np.float64).reshape(n_gauss, -1)
    w = np.asarray(want, np.float64).reshape(n_gauss, -1)
    err, ref = np.linalg.norm(g - w, axis=1), np.linalg.norm(w, axis=1)
    rms = float(np.sqrt(np.mean(ref[ref > 0] ** 2))) if (ref > 0).any() else 0.0
    return err / np.maximum(ref + floor_frac * rms, 1e-300)


SENTINEL_TOL_FLOOR = 1e-4  # per-Gaussian tolerance never below this; 10x the f32 oracle's worst Gaussian above it


@pytest.mark.parametrize("kind", ["wide", "small"])
def test_sentinel_scene_per_gaussian_vs_f64_oracle(native, orc, cuda_device, kind):
    W, H = shape(kind)
    check_tiles(kind, W, H)
    sc, boxes, labels = sentinel_scene(W, H)
    n_g = sc["means"].shape[0]
    ref = orc.render_pipeline(sc, "f32")
    colors, off, flat, bg = ref["colors"], ref["tile_offsets"], ref["flatten_ids"], sc["background"]
    oa = _oracle_args(sc, colors, bg, None, off, flat)
    r64, a64, l64 = orc.raster_fwd(*oa, precision="f64")
    # the scene is what it claims: every sentinel is visible, alone on its pixels, and inside its box
    owner = np.where(a64[0, ..., 0] > 0, flat[l64[0]], -1)
    ys, xs = np.nonzero(owner >= 0)
    ids = owner[ys, xs]
    assert np.array_equal(np.unique(ids), np.arange(n_g)), "a sentinel has no footprint"
    assert np.all((xs >= boxes[ids, 0]) & (xs < boxes[ids, 1]) & (ys >= boxes[ids, 2]) & (ys < boxes[ids, 3]))
    # one contributor per pixel: the oracle composites exactly alpha of the owner's colour over the background
    own_alpha = a64[0, ys, xs, 0]
    assert np.allclose(r64[0, ys, xs], colors[0, ids] * own_alpha[:, None] + (1 - own_alpha[:, None]) * bg, atol=1e-5)
    lab = np.array(labels)
    for name in ("warp-boundary", "tile-boundary-x"):
        for g in np.nonzero(lab == name)[0]:
            cols = xs[ids == g] % 16
            assert {7, 8} <= set(cols) if name == "warp-boundary" else {15, 0} <= set(cols)
    for g in np.nonzero(lab == "tile-boundary-y")[0]:
        assert {15, 0} <= set(ys[ids == g] % 16)
    print(f"[sentinel {kind}] {n_g} Gaussians, {len(flat)} intersections, {len(ids)} covered pixels; classes: "
          + ", ".join(f"{c} {int((lab == c).sum())}" for c in sorted(set(labels))))

    # dL/d(alpha) = (colour - background) . v_colour + v_alpha on a pixel with one contributor: an alpha cotangent in
    # [0.5, 1.5] keeps it positive, so a Gaussian's opacity gradient is not a sum that cancels to near zero, where
    # float32 rounding alone would exceed a tight relative bound
    rng = np.random.default_rng(11)
    vrc = (0.1 * rng.standard_normal((1, H, W, 3))).astype(np.float32)
    vra = (0.5 + rng.random((1, H, W, 1))).astype(np.float32)
    t = to_dev(sc, cuda_device)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    na = (t["means"], t["quats"], t["scales"], d(colors), t["opacities"][None], t["background"], None, W, H, 16,
          t["viewmats"], t["Ks"], d(off), d(flat))
    r, a, li = (x.cpu().numpy() for x in native.rasterize_to_pixels_from_world_3dgs_fwd(*na))
    e_img, e_a = rel(r, r64), rel(a, a64)
    print(f"[sentinel {kind}] image rel_l2 {e_img:.2e} (f32 oracle {rel(ref['renders'], r64):.2e}), alpha {e_a:.2e} "
          f"(f32 oracle {rel(ref['alphas'], a64):.2e}), last_ids differ at {int((li != l64).sum())} pixels")
    assert e_img < 1e-5 and e_a < 1e-4 and np.array_equal(li, ref["last_ids"])

    ga = (ref["alphas"], ref["last_ids"], vrc, vra)
    g64 = orc.raster_bwd(*oa, *ga, precision="f64")
    g32 = orc.raster_bwd(*oa, *ga, precision="f32")
    g = native.rasterize_to_pixels_from_world_3dgs_bwd(*na, *(d(x) for x in ga))
    for nm, got, want, w32 in zip(GRADS, g, g64, g32):
        got = got.cpu().numpy().reshape(want.shape)
        noise = per_gauss_ratio(w32, want, n_g)
        tol = min(1e-2, max(SENTINEL_TOL_FLOOR, 10.0 * float(noise.max())))
        mine = per_gauss_ratio(got, want, n_g)
        worst = int(mine.argmax())
        m = grad_metrics(got, want, n_g, per_gauss_tol=tol)
        print(f"[sentinel {kind}] {nm}: rel_l2 {m['rel']:.2e} (f32 oracle {rel(w32, want):.2e}); worst Gaussian "
              f"{worst} ({labels[worst]}) at {mine[worst]:.2e} of its bound, f32 oracle's worst {noise.max():.2e}; "
              f"tolerance {tol:.1e}, over it: {m['n_bad']}")
        assert m["n_bad"] == 0, (nm, [(int(i), labels[i], float(mine[i])) for i in np.argsort(-mine)[:8]])
        assert m["rel"] < 1e-3 and m["max_abs"] < 5e-2, (nm, m)


# ------------------------------------------------------------------------------------------
# the wide variant against the two-pixel one on the same pixels
# ------------------------------------------------------------------------------------------
def crop_lists(off, flat, tw, th, tx0, ty0, cw, ch):
    """tile_offsets / flatten_ids of the window of tiles [tx0, tx0+cw) x [ty0, ty0+ch), cut out of the whole
    image's lists and re-based.  A window row is one contiguous run of the whole image's flatten_ids."""
    off = off.reshape(th, tw).astype(np.int64)
    assert np.all(np.diff(off.ravel()) >= 0)
    ends = np.append(off.ravel()[1:], len(flat)).reshape(th, tw)
    coff, pieces, pos = [], [], 0
    for row in range(ty0, ty0 + ch):
        s, e = off[row, tx0], ends[row, tx0 + cw - 1]
        coff.append(off[row, tx0:tx0 + cw] - s + pos)
        pieces.append(flat[s:e])
        pos += e - s
    return np.stack(coff)[None].astype(np.int32), np.concatenate(pieces).astype(np.int32)


WINDOW_MAX_BAD = 5  # Gaussians of a window's lists allowed over the per-Gaussian bound of 1e-3


@pytest.mark.parametrize("window,model", [("interior", "pinhole"), ("corner", "pinhole"), ("corner", "opencv")])
def test_wide_equals_small_on_a_window(native, cuda_device, window, model):
    """The same pixels through both variants: the backward of the whole wide image, with cotangents that are zero
    outside a tile-aligned window, against forward and backward of the window alone, which has fewer tiles than
    SMs and takes two pixels per thread.  The window's lists are cut out of the whole image's and its principal
    point is shifted by the window's offset, so both sides blend the same records in the same order; they differ
    by the summation order of the gradients and the rounding of the shifted projected centres."""
    dev = cuda_device
    W, H = shape("wide")
    check_tiles("wide", W, H)
    tw, th = tiles(W, H)
    cw = ch = math.isqrt(sm_count() - 1)
    tx0, ty0 = (tw // 3, th // 3) if window == "interior" else (tw - cw, th - ch)
    cW, cH = min(16 * cw, W - 16 * tx0), min(16 * ch, H - 16 * ty0)
    assert tiles(cW, cH) == (cw, ch) and cw * ch < sm_count()  # gsb_raster.cu:733-760: two pixels per thread
    sc = scenes.scene_b(width=W, height=H, **WIDE_SCENE)
    t = to_dev(sc, dev)
    nkw = _camera_kwargs(model, dev)[1] if model != "pinhole" else {}
    radii, m2d, depths, _, _ = native.projection_ut_3dgs_fused(t["means"], t["quats"], t["scales"], t["opacities"],
                                                               t["viewmats"], t["Ks"], W, H, **nkw)
    _, ids, flat = native.intersect_tile(m2d, radii, depths, 1, 16, tw, th, True)
    off = native.intersect_offset(ids, 1, tw, th)
    coff, cflat = crop_lists(off.cpu().numpy(), flat.cpu().numpy(), tw, th, tx0, ty0, cw, ch)
    n_g = sc["means"].shape[0]
    g = torch.Generator(device=dev).manual_seed(5)
    colors = torch.rand((1, n_g, 3), device=dev, generator=g)
    bg = t["background"]
    Kc = t["Ks"].clone()
    Kc[0, 0, 2] -= 16 * tx0
    Kc[0, 1, 2] -= 16 * ty0

    def fwd(Wi, Hi, K, o, fl):
        return native.rasterize_to_pixels_from_world_3dgs_fwd(t["means"], t["quats"], t["scales"], colors,
                                                              t["opacities"][None], bg, None, Wi, Hi, 16, t["viewmats"],
                                                              K, o, fl, **nkw)

    def bwd(Wi, Hi, K, o, fl, a, li, vc, va):
        return native.rasterize_to_pixels_from_world_3dgs_bwd(t["means"], t["quats"], t["scales"], colors,
                                                              t["opacities"][None], bg, None, Wi, Hi, 16, t["viewmats"],
                                                              K, o, fl, a, li, vc, va, **nkw)

    r, a, li = fwd(W, H, t["Ks"], off, flat)
    coff_d, cflat_d = torch.from_numpy(coff).to(dev), torch.from_numpy(cflat).to(dev)
    rc, ac, lc = fwd(cW, cH, Kc, coff_d, cflat_d)
    ys, xs = slice(16 * ty0, 16 * ty0 + cH), slice(16 * tx0, 16 * tx0 + cW)
    e_img, e_a = rel(rc, r[:, ys, xs]), rel(ac, a[:, ys, xs])
    # A pixel whose 1/255 or saturation decision flips with the rounding of the shifted centres blends a different
    # set of Gaussians on the two sides: it gets no cotangent, so both backward passes skip it.
    a_w = a[:, ys, xs].squeeze(-1)
    same_last = cflat_d[lc.long()] == flat[li[:, ys, xs].long()]  # the same Gaussian blended last
    same = (ac.squeeze(-1) - a_w).abs().le(1e-6) & (same_last | (a_w == 0))
    n_flip = int((~same).sum())
    vc = torch.zeros((1, H, W, 3), device=dev)
    va = torch.zeros((1, H, W, 1), device=dev)
    vc[:, ys, xs] = torch.randn((1, cH, cW, 3), device=dev, generator=g) * same[..., None]
    va[:, ys, xs] = torch.randn((1, cH, cW, 1), device=dev, generator=g) * same[..., None]
    g_wide = bwd(W, H, t["Ks"], off, flat, a, li, vc, va)
    g_small = bwd(cW, cH, Kc, coff_d, cflat_d, ac, lc, vc[:, ys, xs].contiguous(), va[:, ys, xs].contiguous())
    tag = f"{window} window {cW}x{cH} at tile ({tx0}, {ty0}), {model}"
    print(f"[{tag}] {len(cflat)} intersections; window vs whole image: image rel_l2 {e_img:.2e}, alpha {e_a:.2e}, "
          f"{n_flip} of {cW * cH} pixels with a flipped decision")
    assert e_img < 1e-4 and e_a < 1e-5 and n_flip < 1e-3 * cW * cH
    nb = batches_walked(off.cpu().numpy(), len(flat), li.cpu().numpy(), W, H).reshape(th, tw)[ty0:ty0 + ch, tx0:tx0 + cw]
    print(f"[{tag}] window tiles whose wide backward walks more than {BWD_RING} batches: {int((nb > BWD_RING).sum())}")
    if window == "interior":  # the scene is dense there; the corner window covers the ragged edges instead
        assert (nb > BWD_RING).sum() >= 10
    # Only Gaussians on the window's lists can receive gradient: every other one gets exact zeros on both sides.
    touched = torch.zeros(n_g, dtype=torch.bool, device=dev)
    touched[cflat_d.long()] = True
    n_touch = int(touched.sum())
    assert n_touch > 100, n_touch
    # Measured on an H100 80GB HBM3 (400 W limit): rel_l2 <= 4.7e-5 and max |err| / max |ref| <= 5.8e-5 per tensor,
    # at most 3 Gaussians off by more than 1e-3 relative, of the 900 to 2600 on a window's lists.  The bounds: 10x
    # tighter per tensor and per Gaussian than the oracle comparisons, and at most WINDOW_MAX_BAD Gaussians over 1e-3.
    for nm, gw, gs in zip(GRADS, g_wide, g_small):
        gw, gs = gw.reshape(n_g, -1), gs.reshape(n_g, -1)
        m = assert_grad_close(gw[touched], gs[touched], nm, n_touch, rel_tol=1e-4, per_gauss_tol=1e-3, frac_tol=1.0,
                              max_tol=2e-4, tag=f"{tag}: wide vs small, over the {n_touch} Gaussians that touch it")
        assert m["n_bad"] <= WINDOW_MAX_BAD, (nm, m)
        assert not gw[~touched].any() and not gs[~touched].any()


# ------------------------------------------------------------------------------------------
# fastgs (EWA) and fused paths at the wide shape
# ------------------------------------------------------------------------------------------
def test_fastgs_wide_vs_f64_oracle(native, cuda_device):
    """raster_bwd_kernel<false, true, 4>: the EWA blend backward against the float64 CPU restatement."""
    from oracle import fastgs_oracle as fgo
    from test_gpu_fastgs import PARAMS, _fg, _weights, grads_close, image_close, run
    fg = _fg(native)
    W, H = shape("wide")
    check_tiles("wide", W, H)
    inp = scenes.fastgs_inputs(scenes.scene_b(width=W, height=H, **WIDE_SCENE))
    gi, ga = _weights(inp, cuda_device, 12)
    mine = run(fg, fg.default_backend(), inp, cuda_device, gi, ga)

    def oracle(precision):
        o = fgo.render(**inp, grad_image=gi.cpu().numpy(), grad_alpha=ga.cpu().numpy(), precision=precision)
        return dict(image=torch.from_numpy(o["image"]).to(cuda_device), alpha=torch.from_numpy(o["alpha"]).to(cuda_device),
                    grads={k: torch.from_numpy(o["grad_" + k]).to(cuda_device) for k in PARAMS},
                    n=o["n_instances"])

    o64, o32 = oracle("f64"), oracle("f32")
    n = inp["means"].shape[0]
    print(f"[fastgs wide] {o64['n']} instances; f32 oracle vs f64: image {rel(o32['image'], o64['image']):.2e}, "
          + ", ".join(f"{k} {rel(o32['grads'][k], o64['grads'][k]):.1e}" for k in PARAMS))
    image_close(mine, o64, "fastgs wide vs f64 oracle")
    grads_close(mine, o64, n, "fastgs wide vs f64 oracle")


def test_fused_wide_capacity_vs_f64_oracle(native, orc, cuda_device, wide):
    """rasterize_fused with a preset intersection capacity (closed tile offsets, gsb_raster_bwd_recs) at the wide
    shape, against the float64 oracle pipeline, chained to the raw parameters by hand."""
    from test_gpu_fused import raw_leaves
    sc, W, H = wide["sc"], wide["W"], wide["H"]
    check_tiles("wide", W, H)
    vrc, vra = wide["vrc"], wide["vra"]
    ref64 = orc.render_pipeline(sc, "f64", True, vrc, vra)
    ref32 = orc.backward_pipeline(sc, dict(wide["ref"]), vrc, vra, "f32")
    t = to_dev(sc, cuda_device)
    P = raw_leaves(native, t, None)
    cap = int(len(ref64["flatten_ids"]) * 1.25) + 64
    o = native.rasterize_fused(P["means"], P["sh0"], P["shN"], P["scaling_raw"], P["rotation_raw"], P["opacity_raw"],
                               sc["sh_degree"], t["viewmats"], t["Ks"], W, H, bg_color=t["background"], isect_capacity=cap)
    n_is = int(o.n_isects.item())
    assert o.capacity == cap and n_is <= cap
    # a radius that flips at a ceil() boundary between float32 and float64 moves a few intersections
    assert abs(n_is - len(ref64["flatten_ids"])) <= max(8, len(ref64["flatten_ids"]) // 2000), (n_is, len(ref64["flatten_ids"]))
    ((o.render_colors * torch.from_numpy(vrc).to(cuda_device)).sum() +
     (o.alpha * torch.from_numpy(vra).to(cuda_device)).sum()).backward()
    e_img = rel(o.render_colors.detach().cpu().numpy(), ref64["renders"])
    print(f"[fused wide] {n_is} intersections (f64 oracle {len(ref64['flatten_ids'])}); image rel_l2 vs f64 {e_img:.2e} "
          f"(f32 oracle {rel(ref32['renders'], ref64['renders']):.2e})")
    assert e_img < 1e-4
    op = sc["opacities"].astype(np.float64)
    n_g = sc["means"].shape[0]

    def raw(r):
        return {"means": r["v_means"] + r["v_dirs"][0], "sh0": r["v_sh_coeffs"][:, :1], "shN": r["v_sh_coeffs"][:, 1:],
                "scaling_raw": r["v_scales"] * sc["scales"], "rotation_raw": r["v_quats"],
                "opacity_raw": (r["v_opacities"][0] * op * (1 - op))[:, None]}

    want, w32 = raw(ref64), raw(ref32)
    for k, w in want.items():
        assert_close_as_f32(P[k].grad.cpu().numpy(), w, w32[k], k, n_g, "fused wide")
