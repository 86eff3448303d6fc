// FusedOps.h -- EXTENDED operators of the CUDA backend (SURVEY.md 8 f1): the hot path over the RAW SplatData
// tensors, with the L3 glue of the reference's caller folded in.  Not part of the reference's gsplat/Ops.h; the
// eleven operators of Ops.h stay available and unchanged.  What a maintainer replaces with one call each:
//
//   forward   src/core/splat_data.cpp:267-286 (get_means / get_opacity / get_rotation / get_scaling / get_shs:
//             exp, sigmoid, normalize, cat) + src/training/rasterization/rasterizer.cpp:250-266 (inverse(viewmat),
//             dirs, masks, spherical harmonics, clamp_min(+0.5)) + projection_ut_3dgs_fused + intersect_tile +
//             intersect_offset + rasterize_to_pixels_from_world_3dgs_fwd
//   backward  rasterize_to_pixels_from_world_3dgs_bwd + spherical_harmonics_bwd + the autograd backward of all of
//             the above, down to the gradients of the raw parameter tensors
//
// C == 1 (one camera per call, like the reference's kernels), tile size 16, global shutter; RGB, or a depth render
// mode through the RenderMode overloads.
#pragma once

#include <ATen/core/Tensor.h>
#include <c10/util/Optional.h>

#include <tuple>
#include <vector>

#include "Cameras.h"
#include "Common.h"

namespace gsplat {

struct FusedForwardResult {
    at::Tensor renders;      // [1,H,W,3]  (unclamped, background composited)
    at::Tensor alphas;       // [1,H,W,1]
    at::Tensor radii;        // [1,N,2] int32, 0 = culled
    at::Tensor means2d;      // [1,N,2]
    at::Tensor depths;       // [1,N]
    // context for the backward (opaque to callers)
    at::Tensor last_ids;     // [1,H,W] int32
    at::Tensor tile_offsets; // [th*tw + 1] int32, closed: the last entry is n_isects
    at::Tensor flatten_ids;  // [capacity] int32
    at::Tensor workspace;    // bytes: blend records + gradient moments
    at::Tensor n_isects;     // [1] int64 on the device (compare with flatten_ids.size(0) when a capacity was given)
};

// isect_capacity > 0: flatten_ids is allocated with that many entries and NOTHING in the call synchronises with
// the host (the whole step can be captured in a CUDA graph); intersections beyond the capacity are dropped, so the
// caller compares n_isects with the capacity afterwards.  isect_capacity <= 0: the call reads the count back once
// and allocates exactly, like gsplat::intersect_tile.
FusedForwardResult rasterize_from_world_fused_fwd(
    const at::Tensor means,        // [N,3]
    const at::Tensor sh0,          // [N,1,3]
    const at::Tensor shN,          // [N,K-1,3]
    const at::Tensor scaling_raw,  // [N,3]
    const at::Tensor rotation_raw, // [N,4]
    const at::Tensor opacity_raw,  // [N,1] or [N]
    const uint32_t sh_degree, const float scaling_modifier,
    const at::Tensor viewmat,      // [1,4,4]
    const at::Tensor K,            // [1,3,3]
    const uint32_t image_width, const uint32_t image_height, const float eps2d, const float near_plane,
    const float far_plane, const float radius_clip, const at::optional<at::Tensor> backgrounds, // [1,3]
    const CameraModelType camera_model, const UnscentedTransformParameters ut_params,
    const at::optional<at::Tensor> radial_coeffs, const at::optional<at::Tensor> tangential_coeffs,
    const at::optional<at::Tensor> thin_prism_coeffs, const int64_t isect_capacity, const bool prepare_backward);

// gradients of (means, sh0, shN, scaling_raw, rotation_raw, opacity_raw), shaped like the inputs
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> rasterize_from_world_fused_bwd(
    const at::Tensor means, const at::Tensor sh0, const at::Tensor shN, const at::Tensor scaling_raw,
    const at::Tensor rotation_raw, const at::Tensor opacity_raw, const uint32_t sh_degree, const float scaling_modifier,
    const at::Tensor viewmat, const at::Tensor K, const uint32_t image_width, const uint32_t image_height,
    const at::optional<at::Tensor> backgrounds, const CameraModelType camera_model,
    const UnscentedTransformParameters ut_params, const at::optional<at::Tensor> radial_coeffs,
    const at::optional<at::Tensor> tangential_coeffs, const at::optional<at::Tensor> thin_prism_coeffs,
    const at::Tensor radii, const at::Tensor tile_offsets, const at::Tensor flatten_ids, at::Tensor workspace,
    const at::Tensor render_alphas, const at::Tensor last_ids, const at::Tensor v_render_colors,
    const at::Tensor v_render_alphas);

// Render modes (gs::training::RenderMode, rasterizer.hpp:25-31; POINT_CLOUD is not a blend and has no value here).
enum class RenderMode { RGB = 0, D = 1, ED = 2, RGB_D = 3, RGB_ED = 4 };

// The same two operators in a render mode: the blend runs at 1 channel (D, ED: the camera-space depth), 3 (RGB) or 4
// (RGB_D, RGB_ED: SH colour + depth).  renders / v_render_colors are [1,H,W,channels]; backgrounds [1,channels] as
// rasterizer.cpp:272-298 builds them (zeros [1,1] for D / ED, cat(bg, 0) for RGB_D / RGB_ED).  The depth is not
// differentiable (Ops.h:67): its colour-gradient column is dropped, and D / ED give sh0 / shN gradients of zero; a depth
// loss still reaches means, rotation, scaling and opacity through the blend weights.  ED's division by alpha and the
// image / depth split stay with the caller (rasterizer.cpp:367-420).  render_mode = RGB is the overload above.
FusedForwardResult rasterize_from_world_fused_fwd(
    const at::Tensor means, const at::Tensor sh0, const at::Tensor shN, const at::Tensor scaling_raw,
    const at::Tensor rotation_raw, const at::Tensor opacity_raw, const uint32_t sh_degree, const float scaling_modifier,
    const at::Tensor viewmat, const at::Tensor K, const uint32_t image_width, const uint32_t image_height,
    const float eps2d, const float near_plane, const float far_plane, const float radius_clip,
    const at::optional<at::Tensor> backgrounds, const CameraModelType camera_model,
    const UnscentedTransformParameters ut_params, const at::optional<at::Tensor> radial_coeffs,
    const at::optional<at::Tensor> tangential_coeffs, const at::optional<at::Tensor> thin_prism_coeffs,
    const int64_t isect_capacity, const bool prepare_backward, const RenderMode render_mode);

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> rasterize_from_world_fused_bwd(
    const at::Tensor means, const at::Tensor sh0, const at::Tensor shN, const at::Tensor scaling_raw,
    const at::Tensor rotation_raw, const at::Tensor opacity_raw, const uint32_t sh_degree, const float scaling_modifier,
    const at::Tensor viewmat, const at::Tensor K, const uint32_t image_width, const uint32_t image_height,
    const at::optional<at::Tensor> backgrounds, const CameraModelType camera_model,
    const UnscentedTransformParameters ut_params, const at::optional<at::Tensor> radial_coeffs,
    const at::optional<at::Tensor> tangential_coeffs, const at::optional<at::Tensor> thin_prism_coeffs,
    const at::Tensor radii, const at::Tensor tile_offsets, const at::Tensor flatten_ids, at::Tensor workspace,
    const at::Tensor render_alphas, const at::Tensor last_ids, const at::Tensor v_render_colors,
    const at::Tensor v_render_alphas,
    const at::Tensor depths, // the forward's FusedForwardResult::depths; read by RGB_D / RGB_ED only
    const RenderMode render_mode);

// SURVEY.md 8 (f2): loss = (1 - lambda) * l1(clamp(render, 0, 1), target) + lambda * (1 - fused_ssim(.., "valid")) of
// src/training/trainer.cpp:103-126 and, when `compute_grad`, dLoss/d(renders) in the same kernel.
// renders [1,H,W,3] (the from-world blend's output) or [3,H,W] (the fastgs image), target [3,H,W] / [1,3,H,W] (the
// reference's layout) or [1,H,W,3].
// Returns (stats = device float[3]: loss, l1 mean, ssim mean;  v_renders shaped like renders, or an undefined tensor).
std::tuple<at::Tensor, at::Tensor> photometric_loss_fused(const at::Tensor renders, const at::Tensor target,
                                                          const float lambda_dssim, const bool compute_grad);

// SURVEY.md 8 (f5): the same loss on an image used as it is -- no clamp, no clamp mask -- as the reference computes it
// on the output of the bilateral grid (trainer.cpp:662-665 -> 103-126).
std::tuple<at::Tensor, at::Tensor> photometric_loss_fused_unclamped(const at::Tensor renders, const at::Tensor target,
                                                                    const float lambda_dssim, const bool compute_grad);

// SURVEY.md 8 (f3): one Adam step over all parameter groups in one launch (fastgs/optimizer/include/adam_kernels.cuh:13-36,
// src/training/optimizers/fused_adam.cpp:22-95).  step_counts are the per-group counts AFTER the increment.
void fused_adam_step(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &grads,
                     const std::vector<at::Tensor> &exp_avg, const std::vector<at::Tensor> &exp_avg_sq,
                     const std::vector<double> &lr, const double beta1, const double beta2, const double eps,
                     const std::vector<int64_t> &step_counts);

// The same step with (lr, 1/(1-beta1^t), 1/sqrt(1-beta2^t), enabled) per group in a DEVICE tensor [n_groups,4]: nothing
// step-dependent is baked into the launch, so the iteration can be replayed from a CUDA graph.
void fused_adam_step_dynamic(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &grads,
                             const std::vector<at::Tensor> &exp_avg, const std::vector<at::Tensor> &exp_avg_sq,
                             const at::Tensor dynamic_scalars, const double beta1, const double beta2, const double eps);

// SURVEY.md 8 (f6): the MCMC strategy (src/training/strategies/mcmc.cpp) over the raw SplatData tensors, in place.
// `params` are (means, sh0, shN, scaling_raw, rotation_raw, opacity_raw); exp_avg / exp_avg_sq their Adam moments in the
// same order, or empty lists.  No operator reads a device value on the host.
//
// (dead_indices [N] int32, ascending in the first n_dead entries; n_dead [1] int32 on the device; weights [N]:
// sigmoid(opacity_raw) where alive, 0 where dead) -- the dead mask of relocate_gs (mcmc.cpp:119-121).
std::tuple<at::Tensor, at::Tensor, at::Tensor> mcmc_dead(const at::Tensor opacity_raw, const at::Tensor rotation_raw,
                                                         const float min_opacity);
// n_samples indices [n_samples] int32 drawn with replacement in proportion to weights (sigmoid(weights) when
// weights_are_logits); only the first *n_samples_dev are drawn when it is given.  Uniforms from torch's default CUDA
// generator (seeded by torch.manual_seed, graph-capturable) unless `uniforms` (float64) is given.
at::Tensor mcmc_sample(const at::Tensor weights, const int64_t n_samples, const c10::optional<at::Tensor> n_samples_dev,
                       const c10::optional<at::Tensor> uniforms, const bool weights_are_logits);
// relocate_gs (mcmc.cpp:140-187) after the draw: sample j moves onto dead_indices[j], j < *n_dead
void mcmc_relocate(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &exp_avg,
                   const std::vector<at::Tensor> &exp_avg_sq, const at::Tensor samples, const at::Tensor dead_indices,
                   const at::Tensor n_dead, const at::Tensor binoms, const float min_opacity);
// add_new_gs (mcmc.cpp:213-344) after the draw: sample j is appended as row n_rows + j of storage that holds the rows
void mcmc_grow(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &exp_avg,
               const std::vector<at::Tensor> &exp_avg_sq, const int64_t n_rows, const at::Tensor samples,
               const at::Tensor binoms, const float min_opacity);
// inject_noise (mcmc.cpp:349-367) with the rate lr[0] * lr_scale read on the device
void mcmc_add_noise(const at::Tensor raw_opacities, const at::Tensor raw_scales, const at::Tensor raw_quats,
                    const at::Tensor noise, at::Tensor means, const at::Tensor lr, const float lr_scale);
// trainer.cpp:132-158: gradients added into v_scaling / v_opacity; returns (scale loss, opacity loss) on the device
at::Tensor mcmc_regularize(const at::Tensor scaling_raw, const at::Tensor opacity_raw, const float scale_reg,
                           const float opacity_reg, c10::optional<at::Tensor> v_scaling,
                           c10::optional<at::Tensor> v_opacity);

// Adaptive density control, the default strategy (src/training/strategies/default_strategy.cpp:164-290).  A refine is
// adc_classify then adc_apply; between them the caller reads counts back once (the output size and the shape of
// torch::randn({2, n_split, 3})).
//
// grow_gs and prune_gs classified per row: (counts [8] int32 on the device -- duplicated, split, pruned, final rows,
// kept rest rows, kept duplicate copies, kept split rows, 0 -- and the workspace that adc_apply reads).  An undefined or
// empty densification_info means no row is high (nothing grows).  prune_too_big: iter > reset_every.
std::tuple<at::Tensor, at::Tensor> adc_classify(const at::Tensor densification_info, const at::Tensor scaling_raw,
                                                const at::Tensor rotation_raw, const at::Tensor opacity_raw,
                                                const float grad_threshold, const float grow_scale3d,
                                                const float prune_scale3d, const float scene_scale,
                                                const float prune_opacity, const bool prune_too_big,
                                                const bool revised_opacity);
// The final (params, exp_avg, exp_avg_sq, zeroed densification_info [2, n_final]) in freshly allocated tensors, rows in
// the reference's order; n_split = counts[1], n_final = counts[3]; z = torch::randn({2, n_split, 3}).
std::tuple<std::vector<at::Tensor>, std::vector<at::Tensor>, std::vector<at::Tensor>, at::Tensor>
adc_apply(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &exp_avg,
          const std::vector<at::Tensor> &exp_avg_sq, const at::Tensor workspace, const at::Tensor counts,
          const int64_t n_split, const int64_t n_final, const c10::optional<at::Tensor> z, const bool revised_opacity);
// reset_opacity (:251-290) in place: opacity_raw = min(opacity_raw, logit(2 prune_opacity)), its moments zeroed
void adc_reset_opacity(at::Tensor opacity_raw, c10::optional<at::Tensor> exp_avg, c10::optional<at::Tensor> exp_avg_sq,
                       const float prune_opacity);

// ADMM opacity sparsification (src/training/components/sparsity_optimizer.cpp).  k = (int)(prune_ratio * N), the
// caller's float product.  Nothing is read back to the host.
//
// initialize (u = 0, z = prune_z(sigmoid(o))) or update_state (z = prune_z(sigmoid(o) + u), u += sigmoid(o) - z) in
// place on z and u ([N] float, opacity_raw's element count)
void sparsity_update(const at::Tensor opacity_raw, at::Tensor z, at::Tensor u, const int64_t k, const bool initialize);
// 0.5 rho ||sigmoid(o) - z + u||^2 as a [1] device tensor; its gradient added into v_opacity.  rho: a [1] device
// tensor (0: zero loss, v_opacity untouched)
at::Tensor sparsity_loss(const at::Tensor opacity_raw, const at::Tensor z, const at::Tensor u, const at::Tensor rho,
                         at::Tensor v_opacity);
// the final prune: (counts [8], workspace) for adc_apply(..., n_split = 0, n_final = N - n_prune), which then removes
// exactly the n_prune rows of lowest sigmoid(opacity_raw) (ties at the boundary: the first in index order)
std::tuple<at::Tensor, at::Tensor> sparsity_prune_classify(const at::Tensor opacity_raw, const int64_t n_prune);

// Evaluation metrics of one view (src/training/metrics/metrics.cpp:40-116 after the clamp at :441): (psnr, ssim) of
// clamp(image, 0, 1) against target [3,H,W] written as float32 into out (a [2] device tensor), no host read-back.
// image: [3,H,W], or [H,W,3] (the from-world blend's layout, read in place) when image_hwc.
void image_metrics(const at::Tensor image, const at::Tensor target, const bool image_hwc, at::Tensor out);

// Model set-up (src/core/splat_data.cpp:63-111, compute_mean_neighbor_distances): for each point of points [N,3]
// (float32, CUDA) the mean distance to its nearest neighbours, [N] float32 on the device.  The same semantics as the
// reference's function, but the search is exact where the reference's (nanoflann, eps = 10) is approximate: the first
// (up to 3) of the min(4, N) smallest squared distances, the point itself included, that exceed 1e-8; 0.01 when none
// does.  Raises c10::Error on a bad shape, dtype or device, or on a NaN or infinite coordinate (one read-back).
at::Tensor mean_neighbor_distances(const at::Tensor points);
// The same into out [N] float32, with status [1] int32 set to 0 or GSB_KNN_NONFINITE on the device and not read back,
// so the call can be captured in a CUDA graph.
void mean_neighbor_distances_out(const at::Tensor points, at::Tensor out, at::Tensor status);

} // namespace gsplat
