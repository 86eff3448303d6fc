"""ctypes front-end of the CPU oracle (oracle/gut_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py.  The product package never
imports this module.

All functions take / return numpy arrays (float32 / int32 / int64 as in the
reference's tensors, gsplat/Ops.h:12-165).  `precision` selects the float32
restatement ("f32") or the same algorithm in float64 ("f64", noise-floor truth).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS: dict[str, C.CDLL] = {}

PINHOLE, ORTHO, FISHEYE = 0, 1, 2
# gsplat/Common.h ShutterType
ROLLING_TOP_TO_BOTTOM, ROLLING_LEFT_TO_RIGHT, ROLLING_BOTTOM_TO_TOP, ROLLING_RIGHT_TO_LEFT, GLOBAL = 0, 1, 2, 3, 4


class OrcUTParams(C.Structure):
    _fields_ = [
        ("alpha", C.c_float),
        ("beta", C.c_float),
        ("kappa", C.c_float),
        ("in_image_margin_factor", C.c_float),
        ("require_all_sigma_points_valid", C.c_int32),
    ]


@dataclass
class UTParams:
    """gsplat/Cameras.h:27-44 defaults."""

    alpha: float = 0.1
    beta: float = 2.0
    kappa: float = 0.0
    in_image_margin_factor: float = 0.1
    require_all_sigma_points_valid: bool = True

    def c(self) -> OrcUTParams:
        return OrcUTParams(self.alpha, self.beta, self.kappa, self.in_image_margin_factor,
                           1 if self.require_all_sigma_points_valid else 0)


def build(force: bool = False) -> None:
    """Compile the two oracle libraries with the committed Makefile."""
    need = force or not all(
        os.path.exists(os.path.join(_HERE, f"libgut_oracle_{p}.so")) for p in ("f32", "f64", "f64s"))
    src = os.path.join(_HERE, "gut_oracle.c")
    if not need:
        need = any(os.path.getmtime(os.path.join(_HERE, f"libgut_oracle_{p}.so")) < os.path.getmtime(src)
                   for p in ("f32", "f64", "f64s"))
    if need:
        subprocess.run(["make", "-C", _HERE, "-s", "-B"], check=True)


def lib(precision: str = "f32") -> C.CDLL:
    if precision not in _LIBS:
        path = os.path.join(_HERE, f"libgut_oracle_{precision}.so")
        if not os.path.exists(path):
            build()
        _LIBS[precision] = C.CDLL(path)
        _LIBS[precision].orc_isect_count.restype = C.c_int64
    return _LIBS[precision]


def set_threads(n: int) -> None:
    for p in ("f32", "f64"):
        lib(p).orc_set_threads(C.c_int(n))


def max_threads() -> int:
    """Host threads this process may actually use: min(online CPUs, affinity, cgroup CPU quota)."""
    n = int(lib("f32").orc_max_threads())
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except (AttributeError, OSError):
        pass
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, int(np.ceil(int(quota) / int(period)))))
    except (OSError, ValueError):
        pass
    return max(1, n)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a, ty=C.c_float):
    return None if a is None else a.ctypes.data_as(C.POINTER(ty))


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"oracle {what} failed with code {rc} (1 = unsupported configuration)")


def _dist(radial, tangential, thin_prism, Cn):
    """(pointer, floats-per-camera) triples for the optional distortion coefficient arrays."""
    out, keep = [], []
    for a in (radial, tangential, thin_prism):
        if a is None:
            out += [None, C.c_int(0)]
        else:
            a = np.ascontiguousarray(a, dtype=np.float32).reshape(Cn, -1)
            keep.append(a)
            out += [_ptr(a), C.c_int(a.shape[1])]
    return out, keep


def projection_ut(means, quats, scales, opacities, viewmats, Ks, width, height, eps2d=0.3,
                  near_plane=0.01, far_plane=1e10, radius_clip=0.0, calc_compensations=False,
                  camera_model=PINHOLE, ut: UTParams | None = None, precision="f32", radial=None, tangential=None,
                  thin_prism=None, viewmats1=None, rs_type=GLOBAL):
    """gsplat::projection_ut_3dgs_fused (Ops.h:69-98). Returns radii, means2d, depths, conics,
    compensations (or None). Rows with radii == 0 hold zeros here (garbage in the reference).
    viewmats1: end-of-frame poses of a rolling shutter of type rs_type (None: the start poses)."""
    means, quats, scales = _f32(means), _f32(quats), _f32(scales)
    opacities = _f32(opacities)
    viewmats, Ks, viewmats1 = _f32(viewmats), _f32(Ks), _f32(viewmats1)
    Cn, N = viewmats.shape[0], means.shape[0]
    radii = np.zeros((Cn, N, 2), np.int32)
    means2d = np.zeros((Cn, N, 2), np.float32)
    depths = np.zeros((Cn, N), np.float32)
    conics = np.zeros((Cn, N, 3), np.float32)
    comp = np.zeros((Cn, N), np.float32) if calc_compensations else None
    ut = ut or UTParams()
    dist, _keep = _dist(radial, tangential, thin_prism, Cn)
    rc = lib(precision).orc_projection_ut(
        C.c_uint32(Cn), C.c_uint32(N), _ptr(means), _ptr(quats), _ptr(scales), _ptr(opacities),
        _ptr(viewmats), _ptr(viewmats1), _ptr(Ks), C.c_uint32(width), C.c_uint32(height),
        C.c_float(eps2d), C.c_float(near_plane), C.c_float(far_plane), C.c_float(radius_clip),
        C.c_int(camera_model), ut.c(), C.c_int(rs_type), *dist,
        _ptr(radii, C.c_int32), _ptr(means2d), _ptr(depths), _ptr(conics), _ptr(comp))
    _check(rc, "projection_ut")
    return radii, means2d, depths, conics, comp


def sh_fwd(degree, dirs, coeffs, masks=None, precision="f32"):
    dirs, coeffs = _f32(dirs), _f32(coeffs)
    n, K = dirs.reshape(-1, 3).shape[0], coeffs.shape[-2]
    colors = np.zeros_like(dirs)
    m = None if masks is None else np.ascontiguousarray(masks, dtype=np.uint8)
    rc = lib(precision).orc_sh_fwd(C.c_uint32(n), C.c_uint32(K), C.c_uint32(degree), _ptr(dirs),
                                   _ptr(coeffs), _ptr(m, C.c_uint8), _ptr(colors))
    _check(rc, "sh_fwd")
    return colors


def sh_bwd(degree, dirs, coeffs, masks, v_colors, compute_v_dirs=True, precision="f32"):
    dirs, coeffs, v_colors = _f32(dirs), _f32(coeffs), _f32(v_colors)
    n, K = dirs.reshape(-1, 3).shape[0], coeffs.shape[-2]
    v_coeffs = np.zeros_like(coeffs)
    v_dirs = np.zeros_like(dirs) if compute_v_dirs else None
    m = None if masks is None else np.ascontiguousarray(masks, dtype=np.uint8)
    rc = lib(precision).orc_sh_bwd(C.c_uint32(n), C.c_uint32(K), C.c_uint32(degree), _ptr(dirs),
                                   _ptr(coeffs), _ptr(m, C.c_uint8), _ptr(v_colors),
                                   _ptr(v_coeffs), _ptr(v_dirs))
    _check(rc, "sh_bwd")
    return v_coeffs, v_dirs


def isect_tiles(means2d, radii, depths, Cn, tile_size, tile_width, tile_height, sort=True):
    """gsplat::intersect_tile (Ops.h:28-38): tiles_per_gauss [C,N] i32, isect_ids [I] i64,
    flatten_ids [I] i32."""
    means2d = _f32(means2d)
    radii = np.ascontiguousarray(radii, dtype=np.int32)
    depths = _f32(depths)
    N = means2d.shape[1]
    L = lib("f32")
    tpg = np.zeros((Cn, N), np.int32)
    n_isects = int(L.orc_isect_count(C.c_uint32(Cn), C.c_uint32(N), _ptr(means2d),
                                     _ptr(radii, C.c_int32), C.c_uint32(tile_size),
                                     C.c_uint32(tile_width), C.c_uint32(tile_height),
                                     _ptr(tpg, C.c_int32)))
    ids = np.zeros((n_isects,), np.int64)
    flat = np.zeros((n_isects,), np.int32)
    rc = L.orc_isect_emit_sort(C.c_uint32(Cn), C.c_uint32(N), _ptr(means2d), _ptr(radii, C.c_int32),
                               _ptr(depths), C.c_uint32(tile_size), C.c_uint32(tile_width),
                               C.c_uint32(tile_height), C.c_int(1 if sort else 0),
                               C.c_int64(n_isects), _ptr(ids, C.c_int64), _ptr(flat, C.c_int32))
    _check(rc, "isect_emit_sort")
    return tpg, ids, flat


def isect_offsets(isect_ids, Cn, tile_width, tile_height):
    ids = np.ascontiguousarray(isect_ids, dtype=np.int64)
    off = np.zeros((Cn, tile_height, tile_width), np.int32)
    rc = lib("f32").orc_isect_offsets(C.c_int64(ids.shape[0]), _ptr(ids, C.c_int64), C.c_uint32(Cn),
                                      C.c_uint32(tile_width), C.c_uint32(tile_height),
                                      _ptr(off, C.c_int32))
    _check(rc, "isect_offsets")
    return off


def raster_fwd(means, quats, scales, colors, opacities, backgrounds, masks, width, height,
               tile_size, viewmats, Ks, tile_offsets, flatten_ids, camera_model=PINHOLE,
               precision="f32", radial=None, tangential=None, thin_prism=None, viewmats1=None, rs_type=GLOBAL):
    """gsplat::rasterize_to_pixels_from_world_3dgs_fwd (Ops.h:100-129)."""
    means, quats, scales = _f32(means), _f32(quats), _f32(scales)
    colors, opacities = _f32(colors), _f32(opacities)
    bg = _f32(backgrounds) if backgrounds is not None and np.size(backgrounds) else None
    m = None if masks is None else np.ascontiguousarray(masks, dtype=np.uint8)
    viewmats, Ks, viewmats1 = _f32(viewmats), _f32(Ks), _f32(viewmats1)
    toff = np.ascontiguousarray(tile_offsets, dtype=np.int32)
    flat = np.ascontiguousarray(flatten_ids, dtype=np.int32)
    Cn, N = viewmats.shape[0], means.shape[0]
    renders = np.zeros((Cn, height, width, 3), np.float32)
    alphas = np.zeros((Cn, height, width, 1), np.float32)
    last_ids = np.zeros((Cn, height, width), np.int32)
    rc = lib(precision).orc_raster_fwd(
        C.c_uint32(Cn), C.c_uint32(N), C.c_int64(flat.shape[0]), _ptr(means), _ptr(quats),
        _ptr(scales), _ptr(colors), _ptr(opacities), _ptr(bg), _ptr(m, C.c_uint8),
        C.c_uint32(width), C.c_uint32(height), C.c_uint32(tile_size), _ptr(viewmats), _ptr(viewmats1),
        _ptr(Ks), C.c_int(camera_model), C.c_int(rs_type), *_dist(radial, tangential, thin_prism, Cn)[0],
        _ptr(toff, C.c_int32), _ptr(flat, C.c_int32), _ptr(renders), _ptr(alphas), _ptr(last_ids, C.c_int32))
    _check(rc, "raster_fwd")
    return renders, alphas, last_ids


def raster_bwd(means, quats, scales, colors, opacities, backgrounds, masks, width, height,
               tile_size, viewmats, Ks, tile_offsets, flatten_ids, render_alphas, last_ids,
               v_render_colors, v_render_alphas, camera_model=PINHOLE, precision="f32", radial=None, tangential=None,
               thin_prism=None, viewmats1=None, rs_type=GLOBAL):
    """gsplat::rasterize_to_pixels_from_world_3dgs_bwd (Ops.h:131-165); float64 gradients."""
    means, quats, scales = _f32(means), _f32(quats), _f32(scales)
    colors, opacities = _f32(colors), _f32(opacities)
    bg = _f32(backgrounds) if backgrounds is not None and np.size(backgrounds) else None
    m = None if masks is None else np.ascontiguousarray(masks, dtype=np.uint8)
    viewmats, Ks, viewmats1 = _f32(viewmats), _f32(Ks), _f32(viewmats1)
    toff = np.ascontiguousarray(tile_offsets, dtype=np.int32)
    flat = np.ascontiguousarray(flatten_ids, dtype=np.int32)
    ra, li = _f32(render_alphas), np.ascontiguousarray(last_ids, dtype=np.int32)
    vrc, vra = _f32(v_render_colors), _f32(v_render_alphas)
    Cn, N = viewmats.shape[0], means.shape[0]
    v_means = np.zeros((N, 3), np.float64)
    v_quats = np.zeros((N, 4), np.float64)
    v_scales = np.zeros((N, 3), np.float64)
    v_colors = np.zeros(colors.shape, np.float64)
    v_opac = np.zeros(opacities.shape, np.float64)
    D = C.c_double
    rc = lib(precision).orc_raster_bwd(
        C.c_uint32(Cn), C.c_uint32(N), C.c_int64(flat.shape[0]), _ptr(means), _ptr(quats),
        _ptr(scales), _ptr(colors), _ptr(opacities), _ptr(bg), _ptr(m, C.c_uint8),
        C.c_uint32(width), C.c_uint32(height), C.c_uint32(tile_size), _ptr(viewmats), _ptr(viewmats1),
        _ptr(Ks), C.c_int(camera_model), C.c_int(rs_type), *_dist(radial, tangential, thin_prism, Cn)[0],
        _ptr(toff, C.c_int32), _ptr(flat, C.c_int32), _ptr(ra),
        _ptr(li, C.c_int32), _ptr(vrc), _ptr(vra), _ptr(v_means, D), _ptr(v_quats, D),
        _ptr(v_scales, D), _ptr(v_colors, D), _ptr(v_opac, D))
    _check(rc, "raster_bwd")
    return v_means, v_quats, v_scales, v_colors, v_opac


def quat_to_rotmat(quats, precision="f32"):
    quats = _f32(quats)
    out = np.zeros((quats.shape[0], 3, 3), np.float32)
    _check(lib(precision).orc_quat_to_rotmat(C.c_uint32(quats.shape[0]), _ptr(quats), _ptr(out)),
           "quat_to_rotmat")
    return out


def relocation(opacities, scales, ratios, binoms, n_max, precision="f32"):
    opacities, scales, binoms = _f32(opacities), _f32(scales), _f32(binoms)
    ratios = np.ascontiguousarray(ratios, dtype=np.int32)
    no, ns = np.zeros_like(opacities), np.zeros_like(scales)
    _check(lib(precision).orc_relocation(C.c_uint32(opacities.shape[0]), _ptr(opacities), _ptr(scales),
                                         _ptr(ratios, C.c_int32), _ptr(binoms), C.c_int(n_max),
                                         _ptr(no), _ptr(ns)), "relocation")
    return no, ns


def add_noise(raw_opacities, raw_scales, raw_quats, noise, means, current_lr, precision="f32"):
    means = _f32(means).copy()
    a, b, c, d = _f32(raw_opacities), _f32(raw_scales), _f32(raw_quats), _f32(noise)
    _check(lib(precision).orc_add_noise(C.c_uint32(means.shape[0]), _ptr(a), _ptr(b), _ptr(c), _ptr(d),
                                        _ptr(means), C.c_float(current_lr)), "add_noise")
    return means


# ---------------------------------------------------------------------------------------------
# Whole-path convenience: what gs::training::rasterize does around the ops
# (src/training/rasterization/rasterizer.cpp:46-437), restated with numpy.
# ---------------------------------------------------------------------------------------------

def render_pipeline(scene: dict, precision="f32", with_bwd=False, v_render_colors=None,
                    v_render_alphas=None, viewmats1=None, rs_type=GLOBAL):
    """Run projection -> SH -> intersect -> blend (and optionally the backward chain through
    blend bwd and SH bwd) on a scene dict made by tests/scenes.py. C == 1.  viewmats1 / rs_type: a rolling
    shutter's end-of-frame pose and direction (the SH directions use the start pose's camera centre)."""
    rs = dict(viewmats1=viewmats1, rs_type=rs_type)
    W, H, ts = scene["width"], scene["height"], scene.get("tile_size", 16)
    tw, th = (W + ts - 1) // ts, (H + ts - 1) // ts
    means, quats, scales, opac = scene["means"], scene["quats"], scene["scales"], scene["opacities"]
    viewmats, Ks, sh = scene["viewmats"], scene["Ks"], scene["sh_coeffs"]
    deg = scene["sh_degree"]
    out = {}
    radii, means2d, depths, conics, _ = projection_ut(
        means, quats, scales, opac, viewmats, Ks, W, H, eps2d=0.3, near_plane=0.01,
        far_plane=1e4, radius_clip=0.0, precision=precision, **rs)
    out.update(radii=radii, means2d=means2d, depths=depths, conics=conics)
    campos = np.linalg.inv(viewmats.astype(np.float64))[:, :3, 3].astype(np.float32)  # rasterizer.cpp:250-251
    dirs = means[None, :, :] - campos[:, None, :]
    masks = (radii > 0).all(-1)
    colors = sh_fwd(deg, dirs, np.broadcast_to(sh[None], (1,) + sh.shape), masks, precision=precision)
    colors_act = np.maximum(colors + 0.5, 0.0).astype(np.float32)  # rasterizer.cpp:266
    colors_act[~masks] = 0.0
    out.update(dirs=dirs, masks=masks, sh_colors=colors, colors=colors_act)
    tpg, ids, flat = isect_tiles(means2d, radii, depths, 1, ts, tw, th, True)
    off = isect_offsets(ids, 1, tw, th)
    out.update(tiles_per_gauss=tpg, isect_ids=ids, flatten_ids=flat, tile_offsets=off)
    bg = scene.get("background")
    renders, alphas, last_ids = raster_fwd(means, quats, scales, colors_act, opac[None], bg, None, W, H,
                                           ts, viewmats, Ks, off, flat, precision=precision, **rs)
    out.update(renders=renders, alphas=alphas, last_ids=last_ids)
    if with_bwd:
        backward_pipeline(scene, out, v_render_colors, v_render_alphas, precision, **rs)
    return out


def backward_pipeline(scene: dict, out: dict, v_render_colors, v_render_alphas, precision="f32", viewmats1=None,
                      rs_type=GLOBAL):
    """Backward chain of render_pipeline's forward `out` (blend bwd -> clamp -> SH bwd); adds the
    gradients to `out` in place and returns it."""
    W, H, ts = scene["width"], scene["height"], scene.get("tile_size", 16)
    means, quats, scales, opac = scene["means"], scene["quats"], scene["scales"], scene["opacities"]
    sh, deg = scene["sh_coeffs"], scene["sh_degree"]
    g = raster_bwd(means, quats, scales, out["colors"], opac[None], scene.get("background"), None, W, H, ts,
                   scene["viewmats"], scene["Ks"], out["tile_offsets"], out["flatten_ids"], out["alphas"],
                   out["last_ids"], v_render_colors, v_render_alphas, precision=precision, viewmats1=viewmats1,
                   rs_type=rs_type)
    out.update(v_means=g[0], v_quats=g[1], v_scales=g[2], v_colors=g[3], v_opacities=g[4])
    # clamp_min(+0.5) backward, then SH backward (rasterizer_autograd.cpp:84-132)
    v_sh_colors = (g[3] * ((out["sh_colors"] + 0.5) > 0)).astype(np.float32)
    v_coeffs, v_dirs = sh_bwd(deg, out["dirs"], np.broadcast_to(sh[None], (1,) + sh.shape), out["masks"],
                              v_sh_colors, True, precision=precision)
    out.update(v_sh_coeffs=v_coeffs[0], v_dirs=v_dirs)
    return out
