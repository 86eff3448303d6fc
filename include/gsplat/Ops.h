// Ops.h -- the reference's operator API (namespace gsplat), served by the CUDA backend of this library.
//
// Signature-for-signature the eleven free functions of /root/reference/gsplat/Ops.h:12-165, which is
// everything src/training, src/rendering and the strategies reference (SURVEY.md section 8b).  Each
// function validates like the reference (CHECK_INPUT -> c10::Error), allocates its outputs with the
// torch caching allocator on the inputs' device, and forwards raw pointers to the C ABI in
// include/gsb200.h on at::cuda::getCurrentCUDAStream().  Implementation: shim/Ops.cpp.
#pragma once

#include <ATen/core/Tensor.h>

#include <tuple>

#include "Cameras.h"
#include "Common.h"

namespace gsplat {

    // ---- spherical harmonics (a3/a4) --------------------------------------------------------
    // colors[..., 3] for dirs[..., 3] (not normalised), coeffs[..., K, 3], optional bool masks[...]
    at::Tensor spherical_harmonics_fwd(
        const uint32_t degrees_to_use,
        const at::Tensor dirs,
        const at::Tensor coeffs,
        const at::optional<at::Tensor> masks);

    // (v_coeffs[..., K, 3], v_dirs[..., 3] or undefined)
    std::tuple<at::Tensor, at::Tensor> spherical_harmonics_bwd(
        const uint32_t K,
        const uint32_t degrees_to_use,
        const at::Tensor dirs,
        const at::Tensor coeffs,
        const at::optional<at::Tensor> masks,
        const at::Tensor v_colors,
        bool compute_v_dirs);

    // ---- tile intersection (a5/a6) ----------------------------------------------------------
    // (tiles_per_gauss[C, N] int32, isect_ids[I] int64, flatten_ids[I] int32)
    std::tuple<at::Tensor, at::Tensor, at::Tensor> intersect_tile(
        const at::Tensor means2d,                    // [C, N, 2]
        const at::Tensor radii,                      // [C, N, 2] int32
        const at::Tensor depths,                     // [C, N]
        const at::optional<at::Tensor> camera_ids,   // packed mode only (unsupported, as in the callers)
        const at::optional<at::Tensor> gaussian_ids, // packed mode only
        const uint32_t C,
        const uint32_t tile_size,
        const uint32_t tile_width,
        const uint32_t tile_height,
        const bool sort);

    // offsets[C, tile_height, tile_width] int32
    at::Tensor intersect_offset(
        const at::Tensor isect_ids,
        const uint32_t C,
        const uint32_t tile_width,
        const uint32_t tile_height);

    // ---- strategy helpers ---------------------------------------------------------------------
    at::Tensor quats_to_rotmats(const at::Tensor quats); // [N, 4] -> [N, 3, 3]

    // MCMC relocation, eq. (9) of "3D Gaussian Splatting as Markov Chain Monte Carlo"
    std::tuple<at::Tensor, at::Tensor> relocation(
        at::Tensor opacities, // [N]
        at::Tensor scales,    // [N, 3]
        at::Tensor ratios,    // [N] int32
        at::Tensor binoms,    // [n_max, n_max]
        const int n_max);

    // means += lr * sigmoid-gate(opacity) * Sigma * noise, in place
    void add_noise(
        at::Tensor raw_opacities, // [N]
        at::Tensor raw_scales,    // [N, 3]
        at::Tensor raw_quats,     // [N, 4]
        at::Tensor noise,         // [N, 3]
        at::Tensor means,         // [N, 3]
        const float current_lr);

    // ---- unscented-transform projection (a1), not differentiable ----------------------------------
    // (radii[C, N, 2] int32, means2d[C, N, 2], depths[C, N], conics[C, N, 3], compensations[C, N] or undefined)
    std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor>
    projection_ut_3dgs_fused(
        const at::Tensor means,                   // [N, 3]
        const at::Tensor quats,                   // [N, 4]
        const at::Tensor scales,                  // [N, 3]
        const at::optional<at::Tensor> opacities, // [N]
        const at::Tensor viewmats0,               // [C, 4, 4]
        const at::optional<at::Tensor> viewmats1, // [C, 4, 4] rolling shutter end pose
        const at::Tensor Ks,                      // [C, 3, 3]
        const uint32_t image_width,
        const uint32_t image_height,
        const float eps2d,
        const float near_plane,
        const float far_plane,
        const float radius_clip,
        const bool calc_compensations,
        const CameraModelType camera_model,
        const UnscentedTransformParameters ut_params,
        ShutterType rs_type,
        const at::optional<at::Tensor> radial_coeffs,
        const at::optional<at::Tensor> tangential_coeffs,
        const at::optional<at::Tensor> thin_prism_coeffs);

    // ---- from-world rasterization (a7/a8) ------------------------------------------------------------
    // (renders[C, H, W, 3], alphas[C, H, W, 1], last_ids[C, H, W] int32)
    std::tuple<at::Tensor, at::Tensor, at::Tensor>
    rasterize_to_pixels_from_world_3dgs_fwd(
        const at::Tensor means,                     // [N, 3]
        const at::Tensor quats,                     // [N, 4]
        const at::Tensor scales,                    // [N, 3]
        const at::Tensor colors,                    // [C, N, 3]
        const at::Tensor opacities,                 // [C, N]
        const at::optional<at::Tensor> backgrounds, // [C, 3]
        const at::optional<at::Tensor> masks,       // [C, tile_height, tile_width] bool
        const uint32_t image_width,
        const uint32_t image_height,
        const uint32_t tile_size,
        const at::Tensor viewmats0,
        const at::optional<at::Tensor> viewmats1,
        const at::Tensor Ks,
        const CameraModelType camera_model,
        const UnscentedTransformParameters ut_params,
        ShutterType rs_type,
        const at::optional<at::Tensor> radial_coeffs,
        const at::optional<at::Tensor> tangential_coeffs,
        const at::optional<at::Tensor> thin_prism_coeffs,
        const at::Tensor tile_offsets, // [C, tile_height, tile_width] int32
        const at::Tensor flatten_ids); // [I] int32

    // (v_means[N, 3], v_quats[N, 4], v_scales[N, 3], v_colors[C, N, 3], v_opacities[C, N])
    std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor>
    rasterize_to_pixels_from_world_3dgs_bwd(
        const at::Tensor means,
        const at::Tensor quats,
        const at::Tensor scales,
        const at::Tensor colors,
        const at::Tensor opacities,
        const at::optional<at::Tensor> backgrounds,
        const at::optional<at::Tensor> masks,
        const uint32_t image_width,
        const uint32_t image_height,
        const uint32_t tile_size,
        const at::Tensor viewmats0,
        const at::optional<at::Tensor> viewmats1,
        const at::Tensor Ks,
        const CameraModelType camera_model,
        const UnscentedTransformParameters ut_params,
        ShutterType rs_type,
        const at::optional<at::Tensor> radial_coeffs,
        const at::optional<at::Tensor> tangential_coeffs,
        const at::optional<at::Tensor> thin_prism_coeffs,
        const at::Tensor tile_offsets,
        const at::Tensor flatten_ids,
        const at::Tensor render_alphas,   // [C, H, W, 1] forward output
        const at::Tensor last_ids,        // [C, H, W] forward output
        const at::Tensor v_render_colors, // [C, H, W, 3]
        const at::Tensor v_render_alphas); // [C, H, W, 1]

} // namespace gsplat
