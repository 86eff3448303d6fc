// FusedOps.cpp -- host side of the extended operators (include/gsplat/FusedOps.h) on top of the C ABI
// (include/gsb200.h: gsb_fused_front, gsb_isect_plan, gsb_isect_emit_planned, gsb_raster_fwd_recs /
// gsb_raster_bwd_recs, gsb_fused_back).  Allocation through the torch caching allocator, launches on the current
// stream, errors as c10::Error -- the conventions of Ops.cpp.  Nothing here computes.
#include <ATen/Functions.h>
#include <ATen/core/Tensor.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include <cmath>

#include "FusedOps.h"
#include "gsb200.h"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace {

inline gsb_stream_t cur_stream() { return reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()); }

inline void gsb_check(int rc, const char *op) {
    TORCH_CHECK(rc == GSB_OK, "gsplat::", op, " (CUDA backend) failed: ", gsb_error_string(rc), " [code ", rc, "]");
}

inline const float *opt_f32(const at::optional<at::Tensor> &t) {
    return (t.has_value() && t->defined() && t->numel() > 0) ? t->data_ptr<float>() : nullptr;
}

#define CHECK_F32(x)                                                                                    \
    TORCH_CHECK((x).is_cuda() && (x).is_contiguous() && (x).scalar_type() == at::kFloat, #x " must be a contiguous " \
                                                                                            "float32 CUDA tensor")

struct Splats {
    GsbSplatRaw raw;
};

Splats make_splats(const at::Tensor &means, const at::Tensor &sh0, const at::Tensor &shN, const at::Tensor &scaling_raw,
                   const at::Tensor &rotation_raw, const at::Tensor &opacity_raw, uint32_t sh_degree,
                   float scaling_modifier) {
    CHECK_F32(means);
    CHECK_F32(sh0);
    CHECK_F32(scaling_raw);
    CHECK_F32(rotation_raw);
    CHECK_F32(opacity_raw);
    const int64_t N = means.size(0);
    TORCH_CHECK(means.numel() == N * 3 && scaling_raw.numel() == N * 3 && rotation_raw.numel() == N * 4 &&
                    opacity_raw.numel() == N && sh0.numel() == N * 3,
                "fused rasterizer: inconsistent SplatData shapes");
    int64_t rest = 0;
    if (shN.defined() && shN.numel() > 0) {
        CHECK_F32(shN);
        TORCH_CHECK(N > 0 && shN.numel() % (N * 3) == 0, "shN must be [N, K-1, 3]");
        rest = shN.numel() / (N * 3);
    }
    Splats s;
    s.raw.N = (uint32_t)N;
    s.raw.sh_coeffs = (uint32_t)(1 + rest);
    s.raw.sh_degree = sh_degree;
    s.raw.scaling_modifier = scaling_modifier;
    s.raw.means = means.data_ptr<float>();
    s.raw.sh0 = sh0.data_ptr<float>();
    s.raw.shN = rest ? shN.data_ptr<float>() : nullptr;
    s.raw.scaling_raw = scaling_raw.data_ptr<float>();
    s.raw.rotation_raw = rotation_raw.data_ptr<float>();
    s.raw.opacity_raw = opacity_raw.data_ptr<float>();
    TORCH_CHECK((sh_degree + 1) * (sh_degree + 1) <= s.raw.sh_coeffs, "sh_degree ", sh_degree, " needs ",
                (sh_degree + 1) * (sh_degree + 1), " coefficients, the tensors hold ", s.raw.sh_coeffs);
    return s;
}

struct Cam {
    GsbCamera cam;
    at::Tensor radial, tangential, thin_prism;
};

Cam make_cam(const at::Tensor &viewmat, const at::Tensor &K, gsplat::CameraModelType model,
             const UnscentedTransformParameters &ut, const at::optional<at::Tensor> &radial,
             const at::optional<at::Tensor> &tangential, const at::optional<at::Tensor> &thin_prism) {
    CHECK_F32(viewmat);
    CHECK_F32(K);
    TORCH_CHECK(viewmat.numel() == 16 && K.numel() == 9, "the fused rasterizer renders one camera per call (C == 1)");
    Cam c;
    c.cam.viewmats0 = viewmat.data_ptr<float>();
    c.cam.viewmats1 = nullptr;
    c.cam.Ks = K.data_ptr<float>();
    c.cam.camera_model = static_cast<int32_t>(model);
    c.cam.shutter_type = GSB_SHUTTER_GLOBAL;
    auto fill = [&](const at::optional<at::Tensor> &t, at::Tensor &keep, const float *&ptr, int32_t &count) {
        ptr = nullptr;
        count = 0;
        if (t.has_value() && t->defined() && t->numel() > 0) {
            keep = t->contiguous();
            ptr = keep.data_ptr<float>();
            count = static_cast<int32_t>(keep.numel());
        }
    };
    fill(radial, c.radial, c.cam.radial_coeffs, c.cam.radial_count);
    fill(tangential, c.tangential, c.cam.tangential_coeffs, c.cam.tangential_count);
    fill(thin_prism, c.thin_prism, c.cam.thin_prism_coeffs, c.cam.thin_prism_count);
    c.cam.ut.alpha = ut.alpha;
    c.cam.ut.beta = ut.beta;
    c.cam.ut.kappa = ut.kappa;
    c.cam.ut.in_image_margin_factor = ut.in_image_margin_factor;
    c.cam.ut.require_all_sigma_points_valid = ut.require_all_sigma_points_valid ? 1 : 0;
    return c;
}

} // namespace

namespace gsplat {

namespace {
uint32_t mode_channels(RenderMode m) {
    switch (m) {
        case RenderMode::RGB: return 3;
        case RenderMode::D:
        case RenderMode::ED: return 1;
        case RenderMode::RGB_D:
        case RenderMode::RGB_ED: return 4;
    }
    TORCH_CHECK(false, "fused rasterizer: invalid render mode ", static_cast<int>(m));
}
} // namespace

GSB_EXPORT FusedForwardResult rasterize_from_world_fused_fwd(
    const at::Tensor means, const at::Tensor sh0, const at::Tensor shN, const at::Tensor scaling_raw,
    const at::Tensor rotation_raw, const at::Tensor opacity_raw, const uint32_t sh_degree, const float scaling_modifier,
    const at::Tensor viewmat, const at::Tensor K, const uint32_t image_width, const uint32_t image_height,
    const float eps2d, const float near_plane, const float far_plane, const float radius_clip,
    const at::optional<at::Tensor> backgrounds, const CameraModelType camera_model,
    const UnscentedTransformParameters ut_params, const at::optional<at::Tensor> radial_coeffs,
    const at::optional<at::Tensor> tangential_coeffs, const at::optional<at::Tensor> thin_prism_coeffs,
    const int64_t isect_capacity, const bool prepare_backward) {
    return rasterize_from_world_fused_fwd(means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, sh_degree,
                                          scaling_modifier, viewmat, K, image_width, image_height, eps2d, near_plane,
                                          far_plane, radius_clip, backgrounds, camera_model, ut_params, radial_coeffs,
                                          tangential_coeffs, thin_prism_coeffs, isect_capacity, prepare_backward,
                                          RenderMode::RGB);
}

GSB_EXPORT FusedForwardResult rasterize_from_world_fused_fwd(
    const at::Tensor means, const at::Tensor sh0, const at::Tensor shN, const at::Tensor scaling_raw,
    const at::Tensor rotation_raw, const at::Tensor opacity_raw, const uint32_t sh_degree, const float scaling_modifier,
    const at::Tensor viewmat, const at::Tensor K, const uint32_t image_width, const uint32_t image_height,
    const float eps2d, const float near_plane, const float far_plane, const float radius_clip,
    const at::optional<at::Tensor> backgrounds, const CameraModelType camera_model,
    const UnscentedTransformParameters ut_params, const at::optional<at::Tensor> radial_coeffs,
    const at::optional<at::Tensor> tangential_coeffs, const at::optional<at::Tensor> thin_prism_coeffs,
    const int64_t isect_capacity, const bool prepare_backward, const RenderMode render_mode) {
    const uint32_t channels = mode_channels(render_mode);
    TORCH_CHECK(render_mode == RenderMode::RGB || !backgrounds.has_value() || !backgrounds->defined() ||
                    backgrounds->numel() == 0 || backgrounds->numel() == channels,
                "fused rasterizer: backgrounds must be [1,", channels, "] in this render mode");
    const c10::cuda::CUDAGuard guard(means.device());
    Splats sp = make_splats(means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, sh_degree, scaling_modifier);
    Cam cam = make_cam(viewmat, K, camera_model, ut_params, radial_coeffs, tangential_coeffs, thin_prism_coeffs);
    const uint32_t N = sp.raw.N;
    const uint32_t tw = (image_width + 15) / 16, th = (image_height + 15) / 16;
    const auto f32 = means.options();
    const auto i32 = means.options().dtype(at::kInt);
    FusedForwardResult r;
    r.radii = at::empty({1, N, 2}, i32);
    r.means2d = at::empty({1, N, 2}, f32);
    r.depths = at::empty({1, N}, f32);
    const size_t ws_bytes = gsb_fused_workspace(N);
    r.workspace = at::empty({(int64_t)ws_bytes}, means.options().dtype(at::kByte));
    gsb_check(gsb_fused_front_mode(&sp.raw, &cam.cam, image_width, image_height, eps2d, near_plane, far_plane,
                                   radius_clip, prepare_backward ? 1 : 0, static_cast<int>(render_mode),
                                   r.radii.data_ptr<int32_t>(), r.means2d.data_ptr<float>(), r.depths.data_ptr<float>(),
                                   r.workspace.data_ptr(), ws_bytes, cur_stream()),
              "rasterize_from_world_fused_fwd/front");

    // intersect: plan (everything that needs no host-side count), then the direct placement
    at::Tensor tiles_per_gauss = at::empty({1, N}, i32);
    r.tile_offsets = at::empty({(int64_t)tw * th + 1}, i32);
    r.n_isects = at::empty({1}, means.options().dtype(at::kLong));
    const size_t plan_bytes = gsb_isect_plan_workspace(1, N, tw, th);
    at::Tensor plan_ws = at::empty({(int64_t)plan_bytes}, means.options().dtype(at::kByte));
    gsb_check(gsb_isect_plan(1, N, r.means2d.data_ptr<float>(), r.radii.data_ptr<int32_t>(), r.depths.data_ptr<float>(), 16,
                             tw, th, tiles_per_gauss.data_ptr<int32_t>(), r.n_isects.data_ptr<int64_t>(),
                             r.tile_offsets.data_ptr<int32_t>(), 1, plan_ws.data_ptr(), plan_bytes, cur_stream()),
              "rasterize_from_world_fused_fwd/plan");
    int64_t capacity = isect_capacity;
    if (capacity <= 0) { // exact allocation: the one read-back of the operator API (Intersect.cpp:76)
        capacity = r.n_isects.item<int64_t>();
    }
    TORCH_CHECK(capacity <= 0x7fffffffLL, "isect capacity out of range");
    r.flatten_ids = at::empty({capacity}, i32);
    if (capacity > 0 && N > 0) {
        gsb_check(gsb_isect_emit_planned(1, N, r.depths.data_ptr<float>(), tw, th, (uint64_t)capacity, plan_ws.data_ptr(), plan_bytes, nullptr,
                                         r.flatten_ids.data_ptr<int32_t>(), cur_stream()),
                  "rasterize_from_world_fused_fwd/emit");
    }
    r.renders = at::empty({1, image_height, image_width, channels}, f32);
    r.alphas = at::empty({1, image_height, image_width, 1}, f32);
    r.last_ids = at::empty({1, image_height, image_width}, i32);
    gsb_check(gsb_raster_fwd_recs_nc(N, (uint32_t)capacity, channels, r.workspace.data_ptr(), ws_bytes,
                                     r.depths.data_ptr<float>(), opt_f32(backgrounds), nullptr, image_width,
                                     image_height, &cam.cam, r.tile_offsets.data_ptr<int32_t>(),
                                     capacity ? r.flatten_ids.data_ptr<int32_t>() : nullptr, r.renders.data_ptr<float>(),
                                     r.alphas.data_ptr<float>(), r.last_ids.data_ptr<int32_t>(), cur_stream()),
              "rasterize_from_world_fused_fwd/blend");
    return r;
}

GSB_EXPORT std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor>
rasterize_from_world_fused_bwd(const at::Tensor means, const at::Tensor sh0, const at::Tensor shN,
                               const at::Tensor scaling_raw, const at::Tensor rotation_raw, const at::Tensor opacity_raw,
                               const uint32_t sh_degree, const float scaling_modifier, const at::Tensor viewmat,
                               const at::Tensor K, const uint32_t image_width, const uint32_t image_height,
                               const at::optional<at::Tensor> backgrounds, const CameraModelType camera_model,
                               const UnscentedTransformParameters ut_params,
                               const at::optional<at::Tensor> radial_coeffs,
                               const at::optional<at::Tensor> tangential_coeffs,
                               const at::optional<at::Tensor> thin_prism_coeffs, const at::Tensor radii,
                               const at::Tensor tile_offsets, const at::Tensor flatten_ids, at::Tensor workspace,
                               const at::Tensor render_alphas, const at::Tensor last_ids,
                               const at::Tensor v_render_colors, const at::Tensor v_render_alphas) {
    return rasterize_from_world_fused_bwd(means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, sh_degree,
                                          scaling_modifier, viewmat, K, image_width, image_height, backgrounds,
                                          camera_model, ut_params, radial_coeffs, tangential_coeffs, thin_prism_coeffs,
                                          radii, tile_offsets, flatten_ids, workspace, render_alphas, last_ids,
                                          v_render_colors, v_render_alphas, at::Tensor(), RenderMode::RGB);
}

GSB_EXPORT std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor>
rasterize_from_world_fused_bwd(const at::Tensor means, const at::Tensor sh0, const at::Tensor shN,
                               const at::Tensor scaling_raw, const at::Tensor rotation_raw, const at::Tensor opacity_raw,
                               const uint32_t sh_degree, const float scaling_modifier, const at::Tensor viewmat,
                               const at::Tensor K, const uint32_t image_width, const uint32_t image_height,
                               const at::optional<at::Tensor> backgrounds, const CameraModelType camera_model,
                               const UnscentedTransformParameters ut_params,
                               const at::optional<at::Tensor> radial_coeffs,
                               const at::optional<at::Tensor> tangential_coeffs,
                               const at::optional<at::Tensor> thin_prism_coeffs, const at::Tensor radii,
                               const at::Tensor tile_offsets, const at::Tensor flatten_ids, at::Tensor workspace,
                               const at::Tensor render_alphas, const at::Tensor last_ids,
                               const at::Tensor v_render_colors, const at::Tensor v_render_alphas,
                               const at::Tensor depths, const RenderMode render_mode) {
    const uint32_t channels = mode_channels(render_mode);
    TORCH_CHECK(render_mode == RenderMode::RGB || !backgrounds.has_value() || !backgrounds->defined() ||
                    backgrounds->numel() == 0 || backgrounds->numel() == channels,
                "fused rasterizer: backgrounds must be [1,", channels, "] in this render mode");
    const c10::cuda::CUDAGuard guard(means.device());
    Splats sp = make_splats(means, sh0, shN, scaling_raw, rotation_raw, opacity_raw, sh_degree, scaling_modifier);
    Cam cam = make_cam(viewmat, K, camera_model, ut_params, radial_coeffs, tangential_coeffs, thin_prism_coeffs);
    CHECK_F32(render_alphas);
    CHECK_F32(v_render_colors);
    CHECK_F32(v_render_alphas);
    TORCH_CHECK(radii.is_cuda() && radii.is_contiguous() && tile_offsets.is_contiguous() && flatten_ids.is_contiguous() &&
                    last_ids.is_contiguous() && workspace.is_contiguous(),
                "fused backward: contiguous CUDA context tensors expected");
    const uint32_t N = sp.raw.N;
    const size_t ws_bytes = (size_t)workspace.numel();
    const int64_t capacity = flatten_ids.numel();
    TORCH_CHECK(v_render_colors.numel() == (int64_t)image_width * image_height * channels,
                "fused backward: v_render_colors must be [1,H,W,", channels, "]");
    // RGB_D / RGB_ED: the blend reads the fourth channel from the forward's depths, by the record's Gaussian index
    if (channels == 4) {
        CHECK_F32(depths);
        TORCH_CHECK(depths.numel() == (int64_t)N, "fused backward: depths must be the forward's [1,N] depths");
    }
    gsb_check(gsb_raster_bwd_recs_nc(N, (uint32_t)capacity, channels, workspace.data_ptr(), ws_bytes,
                                     channels == 4 ? depths.data_ptr<float>() : nullptr, opt_f32(backgrounds), nullptr,
                                     image_width, image_height, &cam.cam, tile_offsets.data_ptr<int32_t>(),
                                     capacity ? flatten_ids.data_ptr<int32_t>() : nullptr,
                                     render_alphas.data_ptr<float>(), last_ids.data_ptr<int32_t>(),
                                     v_render_colors.data_ptr<float>(), v_render_alphas.data_ptr<float>(),
                                     cur_stream()),
              "rasterize_from_world_fused_bwd/blend");
    at::Tensor v_means = at::empty_like(means), v_sh0 = at::empty_like(sh0), v_scaling = at::empty_like(scaling_raw);
    at::Tensor v_rotation = at::empty_like(rotation_raw), v_opacity = at::empty_like(opacity_raw);
    at::Tensor v_shN = shN.defined() ? at::empty_like(shN) : at::Tensor();
    gsb_check(gsb_fused_back_mode(&sp.raw, &cam.cam, image_width, image_height, static_cast<int>(render_mode),
                                  radii.data_ptr<int32_t>(), workspace.data_ptr(), ws_bytes, v_means.data_ptr<float>(), v_sh0.data_ptr<float>(),
                             (v_shN.defined() && v_shN.numel()) ? v_shN.data_ptr<float>() : nullptr,
                             v_scaling.data_ptr<float>(), v_rotation.data_ptr<float>(), v_opacity.data_ptr<float>(),
                             cur_stream()),
              "rasterize_from_world_fused_bwd/back");
    return std::make_tuple(v_means, v_sh0, v_shN, v_scaling, v_rotation, v_opacity);
}

namespace {
std::tuple<at::Tensor, at::Tensor> photometric_loss_impl(const at::Tensor &renders, const at::Tensor &target,
                                                         const float lambda_dssim, const bool compute_grad, const int flags) {
    const c10::cuda::CUDAGuard guard(renders.device());
    CHECK_F32(renders);
    CHECK_F32(target);
    // [1,H,W,3] (the from-world blend's output) or [3,H,W] planes (the fastgs path's image)
    const bool r_chw = renders.dim() == 3 && renders.size(0) == 3;
    TORCH_CHECK(r_chw || (renders.dim() == 4 && renders.size(0) == 1 && renders.size(3) == 3),
                "renders must be [1,H,W,3] or [3,H,W]");
    const int64_t H = renders.size(1), W = renders.size(2); // the same two dimensions in both layouts
    TORCH_CHECK(target.numel() == 3 * H * W, "target must hold 3*H*W elements");
    const bool hwc = target.dim() == 4 && target.size(-1) == 3 && target.size(1) == H;
    const bool chw = (target.dim() == 3 && target.size(0) == 3) || (target.dim() == 4 && target.size(1) == 3 && !hwc);
    TORCH_CHECK(hwc || chw, "target must be [3,H,W], [1,3,H,W] or [1,H,W,3]");
    at::Tensor stats = at::empty({3}, renders.options());
    at::Tensor v_renders;
    if (compute_grad) v_renders = at::empty_like(renders);
    at::Tensor ws = at::empty({(int64_t)gsb_ssim_l1_workspace()}, renders.options().dtype(at::kByte));
    gsb_check(gsb_ssim_l1((uint32_t)W, (uint32_t)H, renders.data_ptr<float>(), target.data_ptr<float>(),
                          (chw ? GSB_LOSS_TARGET_CHW : 0) | (r_chw ? GSB_LOSS_RENDERS_CHW : 0) | flags,
                          lambda_dssim, 1.0f, compute_grad ? v_renders.data_ptr<float>() : nullptr, stats.data_ptr<float>(),
                          ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
              "photometric_loss_fused");
    return std::make_tuple(stats, v_renders);
}
} // namespace

GSB_EXPORT std::tuple<at::Tensor, at::Tensor> photometric_loss_fused(const at::Tensor renders, const at::Tensor target,
                                                                     const float lambda_dssim, const bool compute_grad) {
    return photometric_loss_impl(renders, target, lambda_dssim, compute_grad, 0);
}

GSB_EXPORT std::tuple<at::Tensor, at::Tensor> photometric_loss_fused_unclamped(const at::Tensor renders,
                                                                               const at::Tensor target,
                                                                               const float lambda_dssim,
                                                                               const bool compute_grad) {
    return photometric_loss_impl(renders, target, lambda_dssim, compute_grad, GSB_LOSS_NO_CLAMP);
}

namespace {
// Validates one entry per group in every list and packs the groups' tensors and hyperparameters into g; the learning
// rate and the bias corrections are the caller's.  Returns the number of groups.
uint32_t pack_adam_groups(const char *op, GsbAdamGroup (&g)[8], const std::vector<at::Tensor> &params,
                          const std::vector<at::Tensor> &grads, const std::vector<at::Tensor> &exp_avg,
                          const std::vector<at::Tensor> &exp_avg_sq, const double beta1, const double beta2,
                          const double eps) {
    const size_t n = params.size();
    TORCH_CHECK(n > 0 && n <= 8, op, ": 1..8 parameter groups");
    TORCH_CHECK(grads.size() == n && exp_avg.size() == n && exp_avg_sq.size() == n, op,
                ": one entry per group in every list");
    for (size_t i = 0; i < n; ++i) {
        CHECK_F32(params[i]);
        CHECK_F32(grads[i]);
        CHECK_F32(exp_avg[i]);
        CHECK_F32(exp_avg_sq[i]);
        TORCH_CHECK(grads[i].numel() == params[i].numel() && exp_avg[i].numel() == params[i].numel() &&
                        exp_avg_sq[i].numel() == params[i].numel(),
                    op, ": group ", i, " has mismatching sizes");
        g[i].param = params[i].data_ptr<float>();
        g[i].grad = grads[i].data_ptr<float>();
        g[i].exp_avg = exp_avg[i].data_ptr<float>();
        g[i].exp_avg_sq = exp_avg_sq[i].data_ptr<float>();
        g[i].n = (uint64_t)params[i].numel();
        g[i].lr = 0.f;
        g[i].beta1 = (float)beta1;
        g[i].beta2 = (float)beta2;
        g[i].eps = (float)eps;
        g[i].bias_correction1_rcp = g[i].bias_correction2_sqrt_rcp = 1.f;
    }
    return (uint32_t)n;
}
} // namespace

GSB_EXPORT void fused_adam_step(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &grads,
                                const std::vector<at::Tensor> &exp_avg, const std::vector<at::Tensor> &exp_avg_sq,
                                const std::vector<double> &lr, const double beta1, const double beta2, const double eps,
                                const std::vector<int64_t> &step_counts) {
    TORCH_CHECK(lr.size() == params.size() && step_counts.size() == params.size(),
                "fused_adam_step: one entry per group in every list");
    GsbAdamGroup g[8];
    const uint32_t n = pack_adam_groups("fused_adam_step", g, params, grads, exp_avg, exp_avg_sq, beta1, beta2, eps);
    const c10::cuda::CUDAGuard guard(params[0].device());
    for (uint32_t i = 0; i < n; ++i) {
        g[i].lr = (float)lr[i];
        // fused_adam.cpp:80-81
        g[i].bias_correction1_rcp = (float)(1.0 / (1.0 - std::pow(beta1, (double)step_counts[i])));
        g[i].bias_correction2_sqrt_rcp = (float)(1.0 / std::sqrt(1.0 - std::pow(beta2, (double)step_counts[i])));
    }
    gsb_check(gsb_adam_step(g, n, cur_stream()), "fused_adam_step");
}

GSB_EXPORT void fused_adam_step_dynamic(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &grads,
                                        const std::vector<at::Tensor> &exp_avg, const std::vector<at::Tensor> &exp_avg_sq,
                                        const at::Tensor dynamic_scalars, const double beta1, const double beta2,
                                        const double eps) {
    GsbAdamGroup g[8];
    const uint32_t n =
        pack_adam_groups("fused_adam_step_dynamic", g, params, grads, exp_avg, exp_avg_sq, beta1, beta2, eps);
    CHECK_F32(dynamic_scalars);
    TORCH_CHECK(dynamic_scalars.numel() == (int64_t)n * 4, "dynamic_scalars must be [n_groups, 4]");
    const c10::cuda::CUDAGuard guard(params[0].device());
    gsb_check(gsb_adam_step_dynamic(g, n, dynamic_scalars.data_ptr<float>(), cur_stream()), "fused_adam_step_dynamic");
}

} // namespace gsplat
