"""gaussian-splatting-cuda_b200: H100-native (sm_90a) 3DGUT rasterizer hot path.

Python host-side mirror used by the tests and bench.py.  The product is the C-ABI CUDA library
(lib/libgsb200.so, include/gsb200.h) and the libtorch shim exporting the reference's
`gsplat::` operator API (lib/libgsplat_b200.so, include/gsplat/Ops.h); this module only loads the
shim and re-states, in Python, the thin L3 caller the reference keeps in
src/training/rasterization/{rasterizer,rasterizer_autograd}.cpp so the whole path can be driven
and differentiated from Python.  There is no CPU / eager fallback: if the native library is
missing or cannot be loaded every entry point raises.

The directory name contains '-' (it is the reference's name + "_b200"), so import it with
`__graft_entry__.load_package()` or tests/conftest.py, which register it as `gsplat_b200`.
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.join(_HERE, "lib")
SHIM_PATH = os.path.join(LIB_DIR, "libgsplat_b200.so")
CABI_PATH = os.path.join(LIB_DIR, "libgsb200.so")

PINHOLE, ORTHO, FISHEYE = 0, 1, 2  # gsplat::CameraModelType
SHUTTER_GLOBAL = 4                 # ShutterType::GLOBAL

_loaded = False


class NativeLibraryError(RuntimeError):
    pass


def build(verbose: bool = False, force: bool = False) -> dict:
    """Compile libgsb200.so and libgsplat_b200.so in-tree (nvcc cross-compiles; no GPU needed)."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("_gsb_build", os.path.join(_HERE, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build_all(verbose=verbose, force=force)


def load() -> None:
    """Load the native shim (registers torch.ops.gsplat_b200.*).  Raises if it is not built."""
    global _loaded
    if _loaded:
        return
    for p in (CABI_PATH, SHIM_PATH):
        if not os.path.exists(p):
            raise NativeLibraryError(
                f"{p} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback for the CUDA backend)")
    torch.ops.load_library(SHIM_PATH)
    _loaded = True


@dataclass
class UTParams:
    """UnscentedTransformParameters defaults (gsplat/Cameras.h:27-44)."""
    alpha: float = 0.1
    beta: float = 2.0
    kappa: float = 0.0
    in_image_margin_factor: float = 0.1
    require_all_sigma_points_valid: bool = True


class OpsBackend:
    """The eleven gsplat:: operators (gsplat/Ops.h) of one native library, by the reference's
    names and argument order.  `namespace` is a torch.ops namespace registered by a TORCH_LIBRARY
    binding with the flattened signatures of shim/torch_binding.cpp.  The product backend is
    `default_backend()`; tests build a second one over the reference's own kernels
    (oracle/ref_ops.py) to compare the two through identical call sites."""

    def __init__(self, namespace_getter):
        self._get = namespace_getter

    @property
    def ns(self):
        return self._get()

    def projection_ut_3dgs_fused(self, means, quats, scales, opacities, viewmats0, Ks, image_width, image_height,
                                 eps2d=0.3, near_plane=0.01, far_plane=1e10, radius_clip=0.0,
                                 calc_compensations=False, camera_model=PINHOLE, ut_params: UTParams | None = None,
                                 viewmats1=None, rs_type=SHUTTER_GLOBAL, radial_coeffs=None, tangential_coeffs=None,
                                 thin_prism_coeffs=None):
        ut = ut_params or UTParams()
        r = self.ns.projection_ut_3dgs_fused(
            means, quats, scales, opacities, viewmats0, viewmats1, Ks, image_width, image_height, eps2d, near_plane,
            far_plane, radius_clip, calc_compensations, camera_model, ut.alpha, ut.beta, ut.kappa,
            ut.in_image_margin_factor, ut.require_all_sigma_points_valid, rs_type, radial_coeffs, tangential_coeffs,
            thin_prism_coeffs)
        comp = r[4] if r[4].numel() else None
        return r[0], r[1], r[2], r[3], comp

    def spherical_harmonics_fwd(self, degrees_to_use, dirs, coeffs, masks=None):
        return self.ns.spherical_harmonics_fwd(degrees_to_use, dirs, coeffs, masks)

    def spherical_harmonics_bwd(self, K, degrees_to_use, dirs, coeffs, masks, v_colors, compute_v_dirs=True):
        v_coeffs, v_dirs = self.ns.spherical_harmonics_bwd(K, degrees_to_use, dirs, coeffs, masks, v_colors,
                                                           compute_v_dirs)
        return v_coeffs, (v_dirs if compute_v_dirs else None)

    def spherical_harmonics_bwd_views(self, degrees_to_use, means, campos, coeffs, v_colors, v_means):
        """Extension (multi-GPU exchange step, include/gsb200.h gsb_sh_bwd_views): SH backward of V views at
        once from their gathered colour gradients; returns v_coeffs, accumulates into v_means."""
        return self.ns.spherical_harmonics_bwd_views(degrees_to_use, means, campos, coeffs, v_colors, v_means)

    def spherical_harmonics_bwd_views_peer(self, degrees_to_use, means, coeffs, view_addrs, v_means):
        """The same with the gather inside the kernel (gsb_sh_bwd_views_peer): `view_addrs` are the device addresses
        of the V ranks' symmetric-memory blocks [M*3 colour gradients | 3 camera position]."""
        return self.ns.spherical_harmonics_bwd_views_peer(degrees_to_use, means, coeffs, list(view_addrs), v_means)

    def intersect_tile(self, means2d, radii, depths, C, tile_size, tile_width, tile_height, sort=True):
        return self.ns.intersect_tile(means2d, radii, depths, C, tile_size, tile_width, tile_height, sort)

    def intersect_offset(self, isect_ids, C, tile_width, tile_height):
        return self.ns.intersect_offset(isect_ids, C, tile_width, tile_height)

    def rasterize_to_pixels_from_world_3dgs_fwd(self, means, quats, scales, colors, opacities, backgrounds, masks,
                                                image_width, image_height, tile_size, viewmats0, Ks, tile_offsets,
                                                flatten_ids, camera_model=PINHOLE, viewmats1=None,
                                                rs_type=SHUTTER_GLOBAL, radial_coeffs=None, tangential_coeffs=None,
                                                thin_prism_coeffs=None):
        return self.ns.rasterize_to_pixels_from_world_3dgs_fwd(
            means, quats, scales, colors, opacities, backgrounds, masks, image_width, image_height, tile_size,
            viewmats0, viewmats1, Ks, camera_model, rs_type, radial_coeffs, tangential_coeffs, thin_prism_coeffs,
            tile_offsets, flatten_ids)

    def rasterize_to_pixels_from_world_3dgs_bwd(self, means, quats, scales, colors, opacities, backgrounds, masks,
                                                image_width, image_height, tile_size, viewmats0, Ks, tile_offsets,
                                                flatten_ids, render_alphas, last_ids, v_render_colors,
                                                v_render_alphas, camera_model=PINHOLE, viewmats1=None,
                                                rs_type=SHUTTER_GLOBAL, radial_coeffs=None, tangential_coeffs=None,
                                                thin_prism_coeffs=None):
        return self.ns.rasterize_to_pixels_from_world_3dgs_bwd(
            means, quats, scales, colors, opacities, backgrounds, masks, image_width, image_height, tile_size,
            viewmats0, viewmats1, Ks, camera_model, rs_type, radial_coeffs, tangential_coeffs, thin_prism_coeffs,
            tile_offsets, flatten_ids, render_alphas, last_ids, v_render_colors, v_render_alphas)

    def quats_to_rotmats(self, quats):
        return self.ns.quats_to_rotmats(quats)

    def relocation(self, opacities, scales, ratios, binoms, n_max):
        return self.ns.relocation(opacities, scales, ratios, binoms, n_max)

    def add_noise(self, raw_opacities, raw_scales, raw_quats, noise, means, current_lr):
        self.ns.add_noise(raw_opacities, raw_scales, raw_quats, noise, means, current_lr)


def _product_ns():
    load()
    return torch.ops.gsplat_b200


_DEFAULT = OpsBackend(_product_ns)


def default_backend() -> OpsBackend:
    return _DEFAULT


def ops():
    return _product_ns()


# module-level aliases of the product backend (same names as gsplat/Ops.h)
projection_ut_3dgs_fused = _DEFAULT.projection_ut_3dgs_fused
spherical_harmonics_fwd = _DEFAULT.spherical_harmonics_fwd
spherical_harmonics_bwd = _DEFAULT.spherical_harmonics_bwd
intersect_tile = _DEFAULT.intersect_tile
intersect_offset = _DEFAULT.intersect_offset
rasterize_to_pixels_from_world_3dgs_fwd = _DEFAULT.rasterize_to_pixels_from_world_3dgs_fwd
rasterize_to_pixels_from_world_3dgs_bwd = _DEFAULT.rasterize_to_pixels_from_world_3dgs_bwd
quats_to_rotmats = _DEFAULT.quats_to_rotmats
relocation = _DEFAULT.relocation
add_noise = _DEFAULT.add_noise


# ---------------------------------------------------------------------------------------------
# L3 mirror: what gs::training::rasterize does around the ops (rasterizer.cpp:46-437,
# rasterizer_autograd.cpp:12-391).  Activated parameters in, image + gradients out.
# ---------------------------------------------------------------------------------------------

class SphericalHarmonicsFunction(torch.autograd.Function):
    """rasterizer_autograd.cpp:12-132."""

    @staticmethod
    def forward(ctx, backend: OpsBackend, sh_degree: int, dirs, coeffs, masks):
        dirs = dirs.contiguous()
        coeffs = coeffs.contiguous()
        colors = backend.spherical_harmonics_fwd(sh_degree, dirs.reshape(-1, 3),
                                                 coeffs.reshape(-1, coeffs.shape[-2], 3),
                                                 masks.reshape(-1).contiguous())
        ctx.save_for_backward(dirs, coeffs, masks)
        ctx.sh_degree = sh_degree
        ctx.backend = backend
        return colors.reshape(dirs.shape)

    @staticmethod
    def backward(ctx, v_colors):
        dirs, coeffs, masks = ctx.saved_tensors
        K = coeffs.shape[-2]
        v_coeffs, v_dirs = ctx.backend.spherical_harmonics_bwd(
            K, ctx.sh_degree, dirs.reshape(-1, 3), coeffs.reshape(-1, K, 3), masks.reshape(-1).contiguous(),
            v_colors.contiguous().reshape(-1, 3), ctx.needs_input_grad[2])
        return (None, None, v_dirs.reshape(dirs.shape) if v_dirs is not None else None,
                v_coeffs.reshape(coeffs.shape) if ctx.needs_input_grad[3] else None, None)


class DeferredSHBackward:
    """Filled by rasterize(..., sh_exchange=...) during backward(): the view's colour gradient as the SH
    backward would receive it (12 B/Gaussian), instead of the expanded 192 B/Gaussian coefficient gradient.
    multiview.exchange_gradients_compact() gathers these over the ranks and expands all views at once."""

    def __init__(self):
        self.v_colors = None  # [N, 3], zero where the Gaussian was masked / not blended
        self.campos = None    # [3] camera position of this rank's view
        self.sh_degree = None


class DeferredSphericalHarmonicsFunction(torch.autograd.Function):
    """Same forward as SphericalHarmonicsFunction; the backward only records v_colors (see DeferredSHBackward)
    and lets no gradient flow to coeffs / dirs -- the exchange step supplies both, summed over all views."""

    @staticmethod
    def forward(ctx, backend: OpsBackend, sh_degree: int, dirs, coeffs, masks, sink: DeferredSHBackward):
        colors = backend.spherical_harmonics_fwd(sh_degree, dirs.contiguous().reshape(-1, 3),
                                                 coeffs.contiguous().reshape(-1, coeffs.shape[-2], 3),
                                                 masks.reshape(-1).contiguous())
        ctx.save_for_backward(masks)
        ctx.sink = sink
        return colors.reshape(dirs.shape)

    @staticmethod
    def backward(ctx, v_colors):
        (masks,) = ctx.saved_tensors
        ctx.sink.v_colors = (v_colors.reshape(-1, 3) * masks.reshape(-1, 1)).contiguous()
        return None, None, None, None, None, None


class GUTRasterizationFunction(torch.autograd.Function):
    """rasterizer_autograd.cpp:267-391."""

    @staticmethod
    def forward(ctx, backend: OpsBackend, means, quats, scales, colors, opacities, bg, viewmat, K, isect_offsets,
                flatten_ids, width, height, tile_size, camera=None):
        camera = camera or {}
        renders, alphas, last_ids = backend.rasterize_to_pixels_from_world_3dgs_fwd(
            means.contiguous(), quats.contiguous(), scales.contiguous(), colors.contiguous(),
            opacities.contiguous(), bg, None, width, height, tile_size, viewmat.contiguous(), K.contiguous(),
            isect_offsets.contiguous(), flatten_ids.contiguous(), **camera)
        ctx.camera = camera
        ctx.save_for_backward(means, quats, scales, colors, opacities, bg if bg is not None else torch.empty(0),
                              viewmat, K, isect_offsets, flatten_ids, alphas, last_ids)
        ctx.dims = (width, height, tile_size, bg is not None)
        ctx.backend = backend
        return renders, alphas

    @staticmethod
    def backward(ctx, v_render_colors, v_render_alphas):
        (means, quats, scales, colors, opacities, bg, viewmat, K, isect_offsets, flatten_ids, alphas,
         last_ids) = ctx.saved_tensors
        width, height, tile_size, has_bg = ctx.dims
        g = ctx.backend.rasterize_to_pixels_from_world_3dgs_bwd(
            means, quats, scales, colors, opacities, bg if has_bg else None, None, width, height, tile_size, viewmat,
            K, isect_offsets, flatten_ids, alphas, last_ids, v_render_colors.contiguous(),
            v_render_alphas.contiguous(), **ctx.camera)
        v_bg = None
        if has_bg and ctx.needs_input_grad[6]:
            v_bg = (v_render_colors * (1.0 - alphas)).sum(dim=(-3, -2))
        return None, g[0], g[1], g[2], g[3], g[4], v_bg, None, None, None, None, None, None, None, None


# gs::training::RenderMode (rasterizer.hpp:25-31) by the names stringToRenderMode accepts, and the blend's channel count
RENDER_MODES = {"RGB": 3, "D": 1, "ED": 1, "RGB_D": 4, "RGB_ED": 4}
_RENDER_MODE_IDS = {"RGB": 0, "D": 1, "ED": 2, "RGB_D": 3, "RGB_ED": 4}  # gsplat::RenderMode (FusedOps.h)


def _check_render_mode(mode: str) -> str:
    if mode not in RENDER_MODES:  # stringToRenderMode (rasterizer.hpp:45-57)
        raise ValueError(f"Invalid render mode: {mode}")
    return mode


def _mode_background(mode: str, bg_color):
    """The blend's background in a render mode (rasterizer.cpp:276-298)."""
    if mode == "RGB" or bg_color is None:
        return bg_color
    zero = torch.zeros((1, 1), dtype=bg_color.dtype, device=bg_color.device)
    return zero if RENDER_MODES[mode] == 1 else torch.cat([bg_color, zero], -1)


def _split_render(mode: str, renders, alphas):
    """(image [1,H,W,3] or None, depth [1,H,W,1] or None) of the blend's output (rasterizer.cpp:367-395)."""
    if mode == "RGB":
        return renders, None
    image = None if RENDER_MODES[mode] == 1 else renders[..., :-1]
    depth = renders if RENDER_MODES[mode] == 1 else renders[..., -1:]
    if mode in ("ED", "RGB_ED"):
        depth = depth / alphas.clamp_min(1e-10)
    return image, depth


@dataclass
class RenderOutput:
    image: torch.Tensor | None   # [3, H, W], clamped to [0, 1] (rasterizer.cpp:401); None in D / ED
    alpha: torch.Tensor          # [1, H, W]
    render_colors: torch.Tensor  # [1, H, W, C] unclamped blend output (what the loss gradient flows through), C of the mode
    radii: torch.Tensor          # [N]
    depths: torch.Tensor         # [N]
    means2d: torch.Tensor        # [1, N, 2]
    n_isects: int
    visibility: torch.Tensor     # [N] bool (radii > 0), rasterizer.cpp:419
    depth: torch.Tensor | None = None  # [1, H, W] accumulated (D, RGB_D) or expected (ED, RGB_ED) depth; None in RGB

    @property
    def n_visible(self) -> int:  # host sync; kept out of the render path
        return int(self.visibility.sum().item())


def rasterize(means, quats, scales, opacities, sh_coeffs, sh_degree, viewmat, K, width, height, bg_color=None,
              scaling_modifier=1.0, tile_size=16, eps2d=0.3, near_plane=0.01, far_plane=10000.0,
              radius_clip=0.0, backend: OpsBackend | None = None, camera_model=PINHOLE, radial_coeffs=None,
              tangential_coeffs=None, thin_prism_coeffs=None,
              sh_exchange: DeferredSHBackward | None = None, projection=None, render_mode: str = "RGB") -> RenderOutput:
    """gs::training::rasterize, C == 1 (rasterizer.cpp:46-437).

    Inputs are the ACTIVATED parameters (get_means/get_rotation/get_scaling/get_opacity/get_shs of
    SplatData): means [N,3], unit quats [N,4] (w,x,y,z), scales [N,3] > 0, opacities [N] in (0,1),
    sh_coeffs [N,K,3]; viewmat [1,4,4], K [1,3,3]; bg_color [1,3] or None.  Distortion coefficients as the
    reference's Camera supplies them (rasterizer.cpp:183-206); camera_model PINHOLE or FISHEYE.
    `projection` = (radii, means2d, depths) replaces the projection step (the op is not differentiable, Ops.h:67):
    parity tests feed two backends the SAME projection so that their intersection lists are identical.
    render_mode: "RGB", "D", "ED", "RGB_D" or "RGB_ED" (RenderMode).  The depth modes blend the projection's
    camera-space depths as one more channel (rasterizer.cpp:272-298); the depth is not differentiable (Ops.h:67), so a
    depth loss reaches the Gaussians through the blend weights only.
    """
    _check_render_mode(render_mode)
    be = backend or _DEFAULT
    camera = dict(camera_model=camera_model, radial_coeffs=radial_coeffs, tangential_coeffs=tangential_coeffs,
                  thin_prism_coeffs=thin_prism_coeffs)
    scaled = scales * scaling_modifier if scaling_modifier != 1.0 else scales
    with torch.no_grad():  # "none differentiable" (Ops.h:67)
        if projection is not None:
            radii, means2d, depths = projection
        else:
            radii, means2d, depths, _conics, _ = be.projection_ut_3dgs_fused(
                means.detach().contiguous(), quats.detach().contiguous(), scaled.detach().contiguous(),
                opacities.detach().contiguous(), viewmat, K, width, height, eps2d, near_plane, far_plane,
                radius_clip, **camera)
        # rasterizer.cpp:250-251 (torch::inverse).  inv_ex is the same LU inverse without the host-side
        # singularity check, i.e. without a device->host sync in the middle of the step.
        campos = torch.linalg.inv_ex(viewmat).inverse[:, :3, 3]
        masks = (radii > 0).all(-1)                                      # :257
    dirs = means.unsqueeze(0) - campos.unsqueeze(1)                      # :254
    if sh_exchange is not None:  # multi-GPU step: the SH backward happens in the exchange (multiview.py)
        sh_exchange.campos, sh_exchange.sh_degree = campos[0], sh_degree
        colors = DeferredSphericalHarmonicsFunction.apply(be, sh_degree, dirs, sh_coeffs.unsqueeze(0), masks,
                                                          sh_exchange)
    else:
        colors = SphericalHarmonicsFunction.apply(be, sh_degree, dirs, sh_coeffs.unsqueeze(0), masks)
    colors = torch.clamp_min(colors + 0.5, 0.0)                          # :266
    tile_w = (width + tile_size - 1) // tile_size
    tile_h = (height + tile_size - 1) // tile_size
    with torch.no_grad():
        _tpg, isect_ids, flatten_ids = be.intersect_tile(means2d, radii, depths, 1, tile_size, tile_w, tile_h, True)
        offsets = be.intersect_offset(isect_ids, 1, tile_w, tile_h)
    if render_mode != "RGB":
        depth_col = depths.unsqueeze(-1)                                 # [1, N, 1], no gradient
        colors = depth_col if RENDER_MODES[render_mode] == 1 else torch.cat([colors, depth_col], -1)
        bg_color = _mode_background(render_mode, bg_color)
    renders, alphas = GUTRasterizationFunction.apply(be, means, quats, scaled, colors, opacities.unsqueeze(0),
                                                     bg_color, viewmat, K, offsets, flatten_ids, width, height,
                                                     tile_size, camera)
    image, depth = _split_render(render_mode, renders, alphas)
    return RenderOutput(
        image=None if image is None else torch.clamp(image[0].permute(2, 0, 1), 0.0, 1.0),
        alpha=alphas[0].permute(2, 0, 1), render_colors=renders, radii=radii[0].max(-1).values, depths=depths[0],
        means2d=means2d, n_isects=int(flatten_ids.shape[0]), visibility=masks[0],
        depth=None if depth is None else depth[0].permute(2, 0, 1))


# ---------------------------------------------------------------------------------------------
# SURVEY.md 8(f1): the extended operator over the RAW SplatData tensors (include/gsplat/FusedOps.h).
# ---------------------------------------------------------------------------------------------

class _FusedGUTFunction(torch.autograd.Function):
    """rasterize_from_world_fused_fwd / _bwd as one autograd node: raw parameters in, image out."""

    @staticmethod
    def forward(ctx, means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, viewmat, K, bg, cfg, mode):
        sh_degree, scaling_modifier, width, height, eps2d, near, far, clip, camera, capacity = cfg
        needs_bwd = any(t.requires_grad for t in (means, sh0, shN, scaling_raw, rotation_raw, opacity_raw))
        args = (means.detach().contiguous(), sh0.detach().contiguous(), shN.detach().contiguous(),
                scaling_raw.detach().contiguous(), rotation_raw.detach().contiguous(), opacity_raw.detach().contiguous())
        cam = (camera.get("camera_model", PINHOLE), camera.get("radial_coeffs"), camera.get("tangential_coeffs"),
               camera.get("thin_prism_coeffs"))
        fwd_args = (*args, sh_degree, scaling_modifier, viewmat.contiguous(), K.contiguous(), width, height, eps2d, near,
                    far, clip, bg, cam[0], cam[1], cam[2], cam[3], capacity, needs_bwd)
        if mode == "RGB":
            out = _product_ns().rasterize_from_world_fused_fwd(*fwd_args)
        else:
            out = _product_ns().rasterize_from_world_fused_fwd_mode(*fwd_args, _RENDER_MODE_IDS[mode])
        renders, alphas, radii, means2d, depths, last_ids, tile_offsets, flatten_ids, workspace, n_isects = out
        if mode == "RGB":
            ctx.save_for_backward(*args, viewmat, K, bg if bg is not None else torch.empty(0), radii, tile_offsets,
                                  flatten_ids, workspace, alphas, last_ids)
        else:
            ctx.save_for_backward(*args, viewmat, K, bg if bg is not None else torch.empty(0), radii, tile_offsets,
                                  flatten_ids, workspace, alphas, last_ids, depths)
        ctx.mode = mode
        ctx.cfg = (sh_degree, scaling_modifier, width, height, cam, bg is not None)
        ctx.mark_non_differentiable(radii, means2d, depths, n_isects)
        return renders, alphas, radii, means2d, depths, n_isects

    @staticmethod
    def backward(ctx, v_renders, v_alphas, *_):
        (means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, viewmat, K, bg, radii, tile_offsets, flatten_ids,
         workspace, alphas, last_ids) = ctx.saved_tensors[:15]
        sh_degree, scaling_modifier, width, height, cam, has_bg = ctx.cfg
        if v_alphas is None:
            v_alphas = torch.zeros_like(alphas)
        bwd_args = (means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, sh_degree, scaling_modifier, viewmat, K,
                    width, height, bg if has_bg else None, cam[0], cam[1], cam[2], cam[3], radii, tile_offsets,
                    flatten_ids, workspace, alphas, last_ids, v_renders.contiguous(), v_alphas.contiguous())
        if ctx.mode == "RGB":
            g = _product_ns().rasterize_from_world_fused_bwd(*bwd_args)
        else:
            g = _product_ns().rasterize_from_world_fused_bwd_mode(*bwd_args, ctx.saved_tensors[15],
                                                                  _RENDER_MODE_IDS[ctx.mode])
        v_bg = None
        if has_bg and ctx.needs_input_grad[8]:
            v_bg = (v_renders * (1.0 - alphas)).sum(dim=(-3, -2))
        return g[0], g[1], (g[2] if g[2].numel() else None), g[3], g[4], g[5], None, None, v_bg, None, None


@dataclass
class FusedRenderOutput:
    render_colors: torch.Tensor  # [1, H, W, C], C = RENDER_MODES[render_mode]
    alpha: torch.Tensor          # [1, H, W, 1]
    radii: torch.Tensor          # [1, N, 2] int32
    means2d: torch.Tensor        # [1, N, 2]
    depths: torch.Tensor         # [1, N]
    n_isects: torch.Tensor       # [1] int64 on the device
    capacity: int                # 0: flatten_ids was sized exactly (one host read-back)
    render_mode: str = "RGB"

    @property
    def image(self):             # [3, H, W] clamped (rasterizer.cpp:401); None in D / ED
        if self.render_mode == "RGB":
            return torch.clamp(self.render_colors[0].permute(2, 0, 1), 0.0, 1.0)
        image, _ = _split_render(self.render_mode, self.render_colors, self.alpha)
        return None if image is None else torch.clamp(image[0].permute(2, 0, 1), 0.0, 1.0)

    @property
    def depth(self):             # [1, H, W] as RenderOutput.depth; None in RGB
        _, depth = _split_render(self.render_mode, self.render_colors, self.alpha)
        return None if depth is None else depth[0].permute(2, 0, 1)


def rasterize_fused(means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, sh_degree, viewmat, K, width, height,
                    bg_color=None, scaling_modifier=1.0, eps2d=0.3, near_plane=0.01, far_plane=10000.0, radius_clip=0.0,
                    camera_model=PINHOLE, radial_coeffs=None, tangential_coeffs=None, thin_prism_coeffs=None,
                    isect_capacity: int = 0, render_mode: str = "RGB") -> FusedRenderOutput:
    """gs::training::rasterize for RenderMode::RGB on the RAW SplatData tensors (what Trainer holds as parameters,
    include/core/splat_data.hpp:104-109): means [N,3], sh0 [N,1,3], shN [N,K-1,3], log-scales [N,3], unnormalised
    quaternions [N,4], logit opacities [N,1].  Same image and the same parameter gradients as

        rasterize(means, normalize(rotation), exp(scaling), sigmoid(opacity), cat(sh0, shN), ...)

    through autograd, in two kernels plus the intersect / blend kernels, with no torch glue.  isect_capacity > 0
    removes the one host read-back (compare `n_isects` with the capacity afterwards).  render_mode as in rasterize():
    bg_color stays [1,3]; the depth modes build the blend's background from it as rasterizer.cpp:276-298 does."""
    _check_render_mode(render_mode)
    load()
    camera = dict(camera_model=camera_model, radial_coeffs=radial_coeffs, tangential_coeffs=tangential_coeffs,
                  thin_prism_coeffs=thin_prism_coeffs)
    cfg = (int(sh_degree), float(scaling_modifier), int(width), int(height), float(eps2d), float(near_plane),
           float(far_plane), float(radius_clip), camera, int(isect_capacity))
    renders, alphas, radii, means2d, depths, n_isects = _FusedGUTFunction.apply(
        means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, viewmat, K, _mode_background(render_mode, bg_color),
        cfg, render_mode)
    return FusedRenderOutput(renders, alphas, radii, means2d, depths, n_isects, int(isect_capacity), render_mode)


def raw_from_activated(means, quats, scales, opacities, sh_coeffs):
    """Test / bench helper: the raw SplatData tensors whose activations give the arguments (inverse of
    splat_data.cpp:267-286): log-scales, the quaternion itself, logit opacities [N,1], sh split into sh0 / shN."""
    op = opacities.clamp(1e-6, 1 - 1e-6)
    return dict(means=means.clone(), sh0=sh_coeffs[:, :1, :].contiguous(), shN=sh_coeffs[:, 1:, :].contiguous(),
                scaling_raw=torch.log(scales), rotation_raw=quats.clone(),
                opacity_raw=torch.log(op / (1 - op)).unsqueeze(-1))


def rasterize_from_raw(raw: dict, sh_degree, viewmat, K, width, height, bg_color=None, scaling_modifier=1.0,
                       backend: OpsBackend | None = None, **kw) -> RenderOutput:
    """The reference's own sequence on raw tensors: activations (splat_data.cpp:267-286) with torch, then rasterize().
    The unfused counterpart of rasterize_fused(), used as its parity oracle and as the same-call-site baseline."""
    means = raw["means"]
    opac = torch.sigmoid(raw["opacity_raw"]).squeeze(-1)
    quats = torch.nn.functional.normalize(raw["rotation_raw"], dim=-1)
    scales = torch.exp(raw["scaling_raw"])
    shs = torch.cat([raw["sh0"], raw["shN"]], dim=1)
    return rasterize(means, quats, scales, opac, shs, sh_degree, viewmat, K, width, height, bg_color=bg_color,
                     scaling_modifier=scaling_modifier, backend=backend, **kw)
