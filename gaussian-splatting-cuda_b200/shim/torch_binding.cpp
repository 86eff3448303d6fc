// torch_binding.cpp -- exposes the gsplat:: shim to Python as torch.ops.gsplat_b200.* so that the
// parity tests and bench.py drive exactly the functions the reference's C++ callers link against
// (same argument order and meaning as include/gsplat/Ops.h; enums and the UT struct are flattened
// to ints/floats because the dispatcher only carries primitive types).
#include <torch/library.h>

#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include "FusedOps.h"
#include "Ops.h"
#include "gsb200.h"

namespace {

using at::Tensor;
using OT = std::optional<at::Tensor>;

UnscentedTransformParameters make_ut(double alpha, double beta, double kappa, double margin, bool require_all) {
    UnscentedTransformParameters ut;
    ut.alpha = (float)alpha;
    ut.beta = (float)beta;
    ut.kappa = (float)kappa;
    ut.in_image_margin_factor = (float)margin;
    ut.require_all_sigma_points_valid = require_all;
    return ut;
}

Tensor sh_fwd(int64_t degree, const Tensor &dirs, const Tensor &coeffs, const OT &masks) {
    return gsplat::spherical_harmonics_fwd((uint32_t)degree, dirs, coeffs, masks);
}

std::tuple<Tensor, Tensor> sh_bwd(int64_t K, int64_t degree, const Tensor &dirs, const Tensor &coeffs, const OT &masks,
                                  const Tensor &v_colors, bool compute_v_dirs) {
    auto r = gsplat::spherical_harmonics_bwd((uint32_t)K, (uint32_t)degree, dirs, coeffs, masks, v_colors, compute_v_dirs);
    Tensor v_dirs = std::get<1>(r);
    if (!v_dirs.defined()) v_dirs = at::empty({0}, dirs.options());
    return std::make_tuple(std::get<0>(r), v_dirs);
}

std::tuple<Tensor, Tensor, Tensor> intersect_tile(const Tensor &means2d, const Tensor &radii, const Tensor &depths,
                                                  int64_t C, int64_t tile_size, int64_t tile_width,
                                                  int64_t tile_height, bool sort) {
    return gsplat::intersect_tile(means2d, radii, depths, c10::nullopt, c10::nullopt, (uint32_t)C, (uint32_t)tile_size,
                                  (uint32_t)tile_width, (uint32_t)tile_height, sort);
}

Tensor intersect_offset(const Tensor &isect_ids, int64_t C, int64_t tile_width, int64_t tile_height) {
    return gsplat::intersect_offset(isect_ids, (uint32_t)C, (uint32_t)tile_width, (uint32_t)tile_height);
}

std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor> projection_ut(
    const Tensor &means, const Tensor &quats, const Tensor &scales, const OT &opacities, const Tensor &viewmats0,
    const OT &viewmats1, const Tensor &Ks, int64_t width, int64_t height, double eps2d, double near_plane,
    double far_plane, double radius_clip, bool calc_compensations, int64_t camera_model, double ut_alpha,
    double ut_beta, double ut_kappa, double ut_margin, bool ut_require_all, int64_t rs_type, const OT &radial,
    const OT &tangential, const OT &thin_prism) {
    auto r = gsplat::projection_ut_3dgs_fused(
        means, quats, scales, opacities, viewmats0, viewmats1, Ks, (uint32_t)width, (uint32_t)height, (float)eps2d,
        (float)near_plane, (float)far_plane, (float)radius_clip, calc_compensations,
        static_cast<gsplat::CameraModelType>(camera_model), make_ut(ut_alpha, ut_beta, ut_kappa, ut_margin, ut_require_all),
        static_cast<ShutterType>(rs_type), radial, tangential, thin_prism);
    Tensor comp = std::get<4>(r);
    if (!comp.defined()) comp = at::empty({0}, means.options());
    return std::make_tuple(std::get<0>(r), std::get<1>(r), std::get<2>(r), std::get<3>(r), comp);
}

std::tuple<Tensor, Tensor, Tensor> raster_fwd(const Tensor &means, const Tensor &quats, const Tensor &scales,
                                              const Tensor &colors, const Tensor &opacities, const OT &backgrounds,
                                              const OT &masks, int64_t width, int64_t height, int64_t tile_size,
                                              const Tensor &viewmats0, const OT &viewmats1, const Tensor &Ks,
                                              int64_t camera_model, int64_t rs_type, const OT &radial,
                                              const OT &tangential, const OT &thin_prism, const Tensor &tile_offsets,
                                              const Tensor &flatten_ids) {
    return gsplat::rasterize_to_pixels_from_world_3dgs_fwd(
        means, quats, scales, colors, opacities, backgrounds, masks, (uint32_t)width, (uint32_t)height,
        (uint32_t)tile_size, viewmats0, viewmats1, Ks, static_cast<gsplat::CameraModelType>(camera_model),
        UnscentedTransformParameters{}, static_cast<ShutterType>(rs_type), radial, tangential, thin_prism, tile_offsets,
        flatten_ids);
}

std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor> raster_bwd(
    const Tensor &means, const Tensor &quats, const Tensor &scales, const Tensor &colors, const Tensor &opacities,
    const OT &backgrounds, const OT &masks, int64_t width, int64_t height, int64_t tile_size, const Tensor &viewmats0,
    const OT &viewmats1, const Tensor &Ks, int64_t camera_model, int64_t rs_type, const OT &radial, const OT &tangential,
    const OT &thin_prism, const Tensor &tile_offsets, const Tensor &flatten_ids, const Tensor &render_alphas,
    const Tensor &last_ids, const Tensor &v_render_colors, const Tensor &v_render_alphas) {
    return gsplat::rasterize_to_pixels_from_world_3dgs_bwd(
        means, quats, scales, colors, opacities, backgrounds, masks, (uint32_t)width, (uint32_t)height,
        (uint32_t)tile_size, viewmats0, viewmats1, Ks, static_cast<gsplat::CameraModelType>(camera_model),
        UnscentedTransformParameters{}, static_cast<ShutterType>(rs_type), radial, tangential, thin_prism, tile_offsets,
        flatten_ids, render_alphas, last_ids, v_render_colors, v_render_alphas);
}

// Extension for the multi-GPU exchange step (not part of the reference's Ops.h): include/gsb200.h, gsb_sh_bwd_views.
// Returns v_coeffs [M, K, 3]; v_means [M, 3] is accumulated in place.
Tensor sh_bwd_views(int64_t degree, const Tensor &means, const Tensor &campos, const Tensor &coeffs,
                    const Tensor &v_colors, Tensor v_means) {
    TORCH_CHECK(means.is_cuda() && campos.is_cuda() && coeffs.is_cuda() && v_colors.is_cuda() && v_means.is_cuda(),
                "sh_bwd_views: CUDA tensors expected");
    TORCH_CHECK(means.is_contiguous() && campos.is_contiguous() && coeffs.is_contiguous() && v_colors.is_contiguous() &&
                    v_means.is_contiguous(),
                "sh_bwd_views: contiguous tensors expected");
    TORCH_CHECK(means.scalar_type() == at::kFloat && coeffs.scalar_type() == at::kFloat &&
                    v_colors.scalar_type() == at::kFloat && campos.scalar_type() == at::kFloat &&
                    v_means.scalar_type() == at::kFloat,
                "sh_bwd_views: float32 tensors expected");
    const int64_t M = means.size(0), V = campos.size(0), K = coeffs.size(-2);
    TORCH_CHECK(coeffs.numel() == M * K * 3 && v_colors.numel() == V * M * 3 && v_means.numel() == M * 3,
                "sh_bwd_views: shape mismatch");
    const c10::cuda::CUDAGuard guard(means.device());
    Tensor v_coeffs = at::empty_like(coeffs);
    const int rc = gsb_sh_bwd_views((uint32_t)M, (uint32_t)K, (uint32_t)degree, (uint32_t)V, means.data_ptr<float>(),
                                    campos.data_ptr<float>(), coeffs.data_ptr<float>(), v_colors.data_ptr<float>(),
                                    v_coeffs.data_ptr<float>(), v_means.data_ptr<float>(),
                                    c10::cuda::getCurrentCUDAStream().stream());
    TORCH_CHECK(rc == 0, "gsb_sh_bwd_views failed: ", gsb_error_string(rc));
    return v_coeffs;
}

// The same step reading every view through its own device address (include/gsb200.h, gsb_sh_bwd_views_peer): the
// addresses are those of NVLink-mapped symmetric-memory buffers of the V ranks (torch.distributed._symmetric_memory
// buffer_ptrs), so they arrive as integers; view v's block is [M*3 colour gradients | 3 camera position] floats.
Tensor sh_bwd_views_peer(int64_t degree, const Tensor &means, const Tensor &coeffs, std::vector<int64_t> view_addrs,
                         Tensor v_means) {
    TORCH_CHECK(means.is_cuda() && coeffs.is_cuda() && v_means.is_cuda(), "sh_bwd_views_peer: CUDA tensors expected");
    TORCH_CHECK(means.is_contiguous() && coeffs.is_contiguous() && v_means.is_contiguous(),
                "sh_bwd_views_peer: contiguous tensors expected");
    TORCH_CHECK(means.scalar_type() == at::kFloat && coeffs.scalar_type() == at::kFloat &&
                    v_means.scalar_type() == at::kFloat,
                "sh_bwd_views_peer: float32 tensors expected");
    const int64_t M = means.size(0), K = coeffs.size(-2), V = (int64_t)view_addrs.size();
    TORCH_CHECK(coeffs.numel() == M * K * 3 && v_means.numel() == M * 3, "sh_bwd_views_peer: shape mismatch");
    std::vector<const float *> vc((size_t)V), cp((size_t)V);
    for (int64_t v = 0; v < V; ++v) {
        TORCH_CHECK(view_addrs[(size_t)v] != 0 && (view_addrs[(size_t)v] & 3) == 0, "sh_bwd_views_peer: bad view address");
        vc[(size_t)v] = reinterpret_cast<const float *>(static_cast<uintptr_t>(view_addrs[(size_t)v]));
        cp[(size_t)v] = vc[(size_t)v] + M * 3;
    }
    const c10::cuda::CUDAGuard guard(means.device());
    Tensor v_coeffs = at::empty_like(coeffs);
    const int rc = gsb_sh_bwd_views_peer((uint32_t)M, (uint32_t)K, (uint32_t)degree, (uint32_t)V, means.data_ptr<float>(),
                                         cp.data(), coeffs.data_ptr<float>(), vc.data(), v_coeffs.data_ptr<float>(),
                                         v_means.data_ptr<float>(), c10::cuda::getCurrentCUDAStream().stream());
    TORCH_CHECK(rc == 0, "gsb_sh_bwd_views_peer failed: ", gsb_error_string(rc));
    return v_coeffs;
}

// Extended operators (include/gsplat/FusedOps.h).  Flattened like the rest: the result struct becomes a tuple.
std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor> fused_fwd(
    const Tensor &means, const Tensor &sh0, const Tensor &shN, const Tensor &scaling_raw, const Tensor &rotation_raw,
    const Tensor &opacity_raw, int64_t sh_degree, double scaling_modifier, const Tensor &viewmat, const Tensor &K,
    int64_t width, int64_t height, double eps2d, double near_plane, double far_plane, double radius_clip,
    const OT &backgrounds, int64_t camera_model, const OT &radial, const OT &tangential, const OT &thin_prism,
    int64_t isect_capacity, bool prepare_backward) {
    auto r = gsplat::rasterize_from_world_fused_fwd(
        means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, (uint32_t)sh_degree, (float)scaling_modifier, viewmat, K,
        (uint32_t)width, (uint32_t)height, (float)eps2d, (float)near_plane, (float)far_plane, (float)radius_clip,
        backgrounds, static_cast<gsplat::CameraModelType>(camera_model), UnscentedTransformParameters{}, radial, tangential,
        thin_prism, isect_capacity, prepare_backward);
    return std::make_tuple(r.renders, r.alphas, r.radii, r.means2d, r.depths, r.last_ids, r.tile_offsets, r.flatten_ids,
                           r.workspace, r.n_isects);
}

std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor, Tensor> fused_bwd(
    const Tensor &means, const Tensor &sh0, const Tensor &shN, const Tensor &scaling_raw, const Tensor &rotation_raw,
    const Tensor &opacity_raw, int64_t sh_degree, double scaling_modifier, const Tensor &viewmat, const Tensor &K,
    int64_t width, int64_t height, const OT &backgrounds, int64_t camera_model, const OT &radial, const OT &tangential,
    const OT &thin_prism, const Tensor &radii, const Tensor &tile_offsets, const Tensor &flatten_ids, Tensor workspace,
    const Tensor &render_alphas, const Tensor &last_ids, const Tensor &v_render_colors, const Tensor &v_render_alphas) {
    auto r = gsplat::rasterize_from_world_fused_bwd(
        means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, (uint32_t)sh_degree, (float)scaling_modifier, viewmat, K,
        (uint32_t)width, (uint32_t)height, backgrounds, static_cast<gsplat::CameraModelType>(camera_model),
        UnscentedTransformParameters{}, radial, tangential, thin_prism, radii, tile_offsets, flatten_ids, workspace,
        render_alphas, last_ids, v_render_colors, v_render_alphas);
    Tensor v_shN = std::get<2>(r);
    if (!v_shN.defined()) v_shN = at::empty({0}, means.options());
    return std::make_tuple(std::get<0>(r), std::get<1>(r), v_shN, std::get<3>(r), std::get<4>(r), std::get<5>(r));
}

// The RenderMode overloads (render_mode = gsplat::RenderMode as an int)
std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor> fused_fwd_mode(
    const Tensor &means, const Tensor &sh0, const Tensor &shN, const Tensor &scaling_raw, const Tensor &rotation_raw,
    const Tensor &opacity_raw, int64_t sh_degree, double scaling_modifier, const Tensor &viewmat, const Tensor &K,
    int64_t width, int64_t height, double eps2d, double near_plane, double far_plane, double radius_clip,
    const OT &backgrounds, int64_t camera_model, const OT &radial, const OT &tangential, const OT &thin_prism,
    int64_t isect_capacity, bool prepare_backward, int64_t render_mode) {
    TORCH_CHECK(render_mode >= 0 && render_mode <= 4, "invalid render mode ", render_mode);
    auto r = gsplat::rasterize_from_world_fused_fwd(
        means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, (uint32_t)sh_degree, (float)scaling_modifier, viewmat, K,
        (uint32_t)width, (uint32_t)height, (float)eps2d, (float)near_plane, (float)far_plane, (float)radius_clip,
        backgrounds, static_cast<gsplat::CameraModelType>(camera_model), UnscentedTransformParameters{}, radial, tangential,
        thin_prism, isect_capacity, prepare_backward, static_cast<gsplat::RenderMode>(render_mode));
    return std::make_tuple(r.renders, r.alphas, r.radii, r.means2d, r.depths, r.last_ids, r.tile_offsets, r.flatten_ids,
                           r.workspace, r.n_isects);
}

std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor, Tensor> fused_bwd_mode(
    const Tensor &means, const Tensor &sh0, const Tensor &shN, const Tensor &scaling_raw, const Tensor &rotation_raw,
    const Tensor &opacity_raw, int64_t sh_degree, double scaling_modifier, const Tensor &viewmat, const Tensor &K,
    int64_t width, int64_t height, const OT &backgrounds, int64_t camera_model, const OT &radial, const OT &tangential,
    const OT &thin_prism, const Tensor &radii, const Tensor &tile_offsets, const Tensor &flatten_ids, Tensor workspace,
    const Tensor &render_alphas, const Tensor &last_ids, const Tensor &v_render_colors, const Tensor &v_render_alphas,
    const Tensor &depths, int64_t render_mode) {
    TORCH_CHECK(render_mode >= 0 && render_mode <= 4, "invalid render mode ", render_mode);
    auto r = gsplat::rasterize_from_world_fused_bwd(
        means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, (uint32_t)sh_degree, (float)scaling_modifier, viewmat, K,
        (uint32_t)width, (uint32_t)height, backgrounds, static_cast<gsplat::CameraModelType>(camera_model),
        UnscentedTransformParameters{}, radial, tangential, thin_prism, radii, tile_offsets, flatten_ids, workspace,
        render_alphas, last_ids, v_render_colors, v_render_alphas, depths, static_cast<gsplat::RenderMode>(render_mode));
    Tensor v_shN = std::get<2>(r);
    if (!v_shN.defined()) v_shN = at::empty({0}, means.options());
    return std::make_tuple(std::get<0>(r), std::get<1>(r), v_shN, std::get<3>(r), std::get<4>(r), std::get<5>(r));
}

std::tuple<Tensor, Tensor> loss_fused(const Tensor &renders, const Tensor &target, double lambda_dssim, bool compute_grad) {
    auto r = gsplat::photometric_loss_fused(renders, target, (float)lambda_dssim, compute_grad);
    Tensor v = std::get<1>(r);
    if (!v.defined()) v = at::empty({0}, renders.options());
    return std::make_tuple(std::get<0>(r), v);
}

std::tuple<Tensor, Tensor> loss_fused_unclamped(const Tensor &renders, const Tensor &target, double lambda_dssim,
                                                bool compute_grad) {
    auto r = gsplat::photometric_loss_fused_unclamped(renders, target, (float)lambda_dssim, compute_grad);
    Tensor v = std::get<1>(r);
    if (!v.defined()) v = at::empty({0}, renders.options());
    return std::make_tuple(std::get<0>(r), v);
}

void adam_step(std::vector<Tensor> params, std::vector<Tensor> grads, std::vector<Tensor> exp_avg,
               std::vector<Tensor> exp_avg_sq, std::vector<double> lr, double beta1, double beta2, double eps,
               std::vector<int64_t> step_counts) {
    gsplat::fused_adam_step(params, grads, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, step_counts);
}

void adam_step_dynamic(std::vector<Tensor> params, std::vector<Tensor> grads, std::vector<Tensor> exp_avg,
                       std::vector<Tensor> exp_avg_sq, const Tensor &dynamic_scalars, double beta1, double beta2,
                       double eps) {
    gsplat::fused_adam_step_dynamic(params, grads, exp_avg, exp_avg_sq, dynamic_scalars, beta1, beta2, eps);
}

Tensor quats_to_rotmats(const Tensor &quats) { return gsplat::quats_to_rotmats(quats); }

std::tuple<Tensor, Tensor> relocation(const Tensor &opacities, const Tensor &scales, const Tensor &ratios,
                                      const Tensor &binoms, int64_t n_max) {
    return gsplat::relocation(opacities, scales, ratios, binoms, (int)n_max);
}

void add_noise(const Tensor &raw_opacities, const Tensor &raw_scales, const Tensor &raw_quats, const Tensor &noise,
               Tensor means, double current_lr) {
    gsplat::add_noise(raw_opacities, raw_scales, raw_quats, noise, means, (float)current_lr);
}

void image_metrics(const Tensor &image, const Tensor &target, bool image_hwc, Tensor out) {
    gsplat::image_metrics(image, target, image_hwc, out);
}

Tensor mean_neighbor_distances(const Tensor &points) { return gsplat::mean_neighbor_distances(points); }

void mean_neighbor_distances_out(const Tensor &points, Tensor out, Tensor status) {
    gsplat::mean_neighbor_distances_out(points, out, status);
}

} // namespace

TORCH_LIBRARY(gsplat_b200, m) {
    m.def("spherical_harmonics_fwd", &sh_fwd);
    m.def("spherical_harmonics_bwd", &sh_bwd);
    m.def("intersect_tile", &intersect_tile);
    m.def("intersect_offset", &intersect_offset);
    m.def("projection_ut_3dgs_fused", &projection_ut);
    m.def("rasterize_to_pixels_from_world_3dgs_fwd", &raster_fwd);
    m.def("rasterize_to_pixels_from_world_3dgs_bwd", &raster_bwd);
    m.def("spherical_harmonics_bwd_views(int degree, Tensor means, Tensor campos, Tensor coeffs, Tensor v_colors, "
          "Tensor(a!) v_means) -> Tensor",
          &sh_bwd_views);
    m.def("spherical_harmonics_bwd_views_peer(int degree, Tensor means, Tensor coeffs, int[] view_addrs, "
          "Tensor(a!) v_means) -> Tensor",
          &sh_bwd_views_peer);
    m.def("rasterize_from_world_fused_fwd", &fused_fwd);
    m.def("rasterize_from_world_fused_bwd(Tensor means, Tensor sh0, Tensor shN, Tensor scaling_raw, Tensor rotation_raw, "
          "Tensor opacity_raw, int sh_degree, float scaling_modifier, Tensor viewmat, Tensor K, int width, int height, "
          "Tensor? backgrounds, int camera_model, Tensor? radial, Tensor? tangential, Tensor? thin_prism, Tensor radii, "
          "Tensor tile_offsets, Tensor flatten_ids, Tensor(a!) workspace, Tensor render_alphas, Tensor last_ids, "
          "Tensor v_render_colors, Tensor v_render_alphas) -> (Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)",
          &fused_bwd);
    m.def("rasterize_from_world_fused_fwd_mode", &fused_fwd_mode);
    m.def("rasterize_from_world_fused_bwd_mode(Tensor means, Tensor sh0, Tensor shN, Tensor scaling_raw, "
          "Tensor rotation_raw, Tensor opacity_raw, int sh_degree, float scaling_modifier, Tensor viewmat, Tensor K, "
          "int width, int height, Tensor? backgrounds, int camera_model, Tensor? radial, Tensor? tangential, "
          "Tensor? thin_prism, Tensor radii, Tensor tile_offsets, Tensor flatten_ids, Tensor(a!) workspace, "
          "Tensor render_alphas, Tensor last_ids, Tensor v_render_colors, Tensor v_render_alphas, Tensor depths, "
          "int render_mode) -> (Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)",
          &fused_bwd_mode);
    m.def("photometric_loss_fused", &loss_fused);
    m.def("photometric_loss_fused_unclamped", &loss_fused_unclamped);
    m.def("fused_adam_step(Tensor(a!)[] params, Tensor[] grads, Tensor(b!)[] exp_avg, Tensor(c!)[] exp_avg_sq, float[] lr, "
          "float beta1, float beta2, float eps, int[] step_counts) -> ()",
          &adam_step);
    m.def("fused_adam_step_dynamic(Tensor(a!)[] params, Tensor[] grads, Tensor(b!)[] exp_avg, Tensor(c!)[] exp_avg_sq, "
          "Tensor dynamic_scalars, float beta1, float beta2, float eps) -> ()",
          &adam_step_dynamic);
    m.def("quats_to_rotmats", &quats_to_rotmats);
    m.def("relocation", &relocation);
    m.def("add_noise(Tensor raw_opacities, Tensor raw_scales, Tensor raw_quats, Tensor noise, Tensor(a!) means, float current_lr) -> ()",
          &add_noise);
    m.def("image_metrics(Tensor image, Tensor target, bool image_hwc, Tensor(a!) out) -> ()", &image_metrics);
    m.def("mean_neighbor_distances", &mean_neighbor_distances);
    m.def("mean_neighbor_distances_out(Tensor points, Tensor(a!) out, Tensor(b!) status) -> ()",
          &mean_neighbor_distances_out);
}
