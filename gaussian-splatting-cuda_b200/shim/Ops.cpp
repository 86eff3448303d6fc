// Ops.cpp -- the reference's gsplat:: operator API on top of the C ABI (include/gsb200.h).
//
// Host-side mirror of the reference's launch layer (gsplat/{Projection,Intersect,Rasterization,
// SphericalHarmonics,QuatToRotmat,Relocation}.cpp): same argument checks, same output shapes /
// dtypes / allocation through the torch caching allocator, same stream (the current CUDA stream),
// same error convention (c10::Error).  All arithmetic lives behind the C ABI; nothing here computes.
#include <ATen/Functions.h>
#include <ATen/TensorUtils.h>
#include <ATen/core/Tensor.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include <tuple>

#include "Ops.h"
#include "gsb200.h"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace {

inline gsb_stream_t cur_stream() { return reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()); }

inline void gsb_check(int rc, const char *op) {
    TORCH_CHECK(rc == GSB_OK, "gsplat::", op, " (CUDA backend) failed: ", gsb_error_string(rc), " [code ", rc, "]");
}

inline at::Tensor byte_workspace(size_t bytes, const at::Tensor &like) {
    // 256-byte aligned by the caching allocator (512-byte granularity)
    return at::empty({(int64_t)bytes}, like.options().dtype(at::kByte));
}

inline const float *opt_f32(const at::optional<at::Tensor> &t) {
    return (t.has_value() && t->defined() && t->numel() > 0) ? t->data_ptr<float>() : nullptr;
}

struct CameraArgs {
    GsbCamera cam;
    at::Tensor radial, tangential, thin_prism; // keep converted tensors alive
};

CameraArgs make_camera(const at::Tensor &viewmats0, const at::optional<at::Tensor> &viewmats1, const at::Tensor &Ks,
                       gsplat::CameraModelType camera_model, const UnscentedTransformParameters &ut,
                       ShutterType rs_type, const at::optional<at::Tensor> &radial,
                       const at::optional<at::Tensor> &tangential, const at::optional<at::Tensor> &thin_prism) {
    CameraArgs a;
    const int64_t C = Ks.size(0);
    a.cam.viewmats0 = viewmats0.data_ptr<float>();
    a.cam.viewmats1 = opt_f32(viewmats1);
    a.cam.Ks = Ks.data_ptr<float>();
    a.cam.camera_model = static_cast<int32_t>(camera_model);
    a.cam.shutter_type = static_cast<int32_t>(rs_type);
    auto fill = [&](const at::optional<at::Tensor> &t, at::Tensor &keep, const float *&ptr, int32_t &count) {
        ptr = nullptr;
        count = 0;
        if (t.has_value() && t->defined() && t->numel() > 0) {
            keep = t->contiguous();
            ptr = keep.data_ptr<float>();
            count = static_cast<int32_t>(keep.numel() / std::max<int64_t>(C, 1));
        }
    };
    fill(radial, a.radial, a.cam.radial_coeffs, a.cam.radial_count);
    fill(tangential, a.tangential, a.cam.tangential_coeffs, a.cam.tangential_count);
    fill(thin_prism, a.thin_prism, a.cam.thin_prism_coeffs, a.cam.thin_prism_count);
    a.cam.ut.alpha = ut.alpha;
    a.cam.ut.beta = ut.beta;
    a.cam.ut.kappa = ut.kappa;
    a.cam.ut.in_image_margin_factor = ut.in_image_margin_factor;
    a.cam.ut.require_all_sigma_points_valid = ut.require_all_sigma_points_valid ? 1 : 0;
    return a;
}

} // namespace

namespace gsplat {

// ---------------------------------------------------------------------------------------------
// SphericalHarmonics.cpp:15-75
// ---------------------------------------------------------------------------------------------
GSB_EXPORT at::Tensor spherical_harmonics_fwd(const uint32_t degrees_to_use, const at::Tensor dirs,
                                              const at::Tensor coeffs, const at::optional<at::Tensor> masks) {
    DEVICE_GUARD(dirs);
    CHECK_INPUT(dirs);
    CHECK_INPUT(coeffs);
    if (masks.has_value()) {
        CHECK_INPUT(masks.value());
    }
    TORCH_CHECK(coeffs.size(-1) == 3, "coeffs must have last dimension 3");
    TORCH_CHECK(dirs.size(-1) == 3, "dirs must have last dimension 3");
    at::Tensor colors = at::empty_like(dirs);
    const uint32_t K = coeffs.size(-2);
    const uint32_t M = dirs.numel() / 3;
    gsb_check(gsb_sh_fwd(M, K, degrees_to_use, dirs.data_ptr<float>(), coeffs.data_ptr<float>(),
                         masks.has_value() ? reinterpret_cast<const uint8_t *>(masks->data_ptr<bool>()) : nullptr,
                         colors.data_ptr<float>(), cur_stream()),
              "spherical_harmonics_fwd");
    return colors;
}

GSB_EXPORT std::tuple<at::Tensor, at::Tensor> spherical_harmonics_bwd(
    const uint32_t K, const uint32_t degrees_to_use, const at::Tensor dirs, const at::Tensor coeffs,
    const at::optional<at::Tensor> masks, const at::Tensor v_colors, bool compute_v_dirs) {
    DEVICE_GUARD(dirs);
    CHECK_INPUT(dirs);
    CHECK_INPUT(coeffs);
    CHECK_INPUT(v_colors);
    if (masks.has_value()) {
        CHECK_INPUT(masks.value());
    }
    TORCH_CHECK(v_colors.size(-1) == 3, "v_colors must have last dimension 3");
    TORCH_CHECK(coeffs.size(-1) == 3, "coeffs must have last dimension 3");
    TORCH_CHECK(dirs.size(-1) == 3, "dirs must have last dimension 3");
    const uint32_t M = dirs.numel() / 3;
    // the kernel writes every element (zeros included): no 192 B/Gaussian memset as in the reference
    at::Tensor v_coeffs = at::empty_like(coeffs);
    at::Tensor v_dirs;
    if (compute_v_dirs) v_dirs = at::empty_like(dirs);
    gsb_check(gsb_sh_bwd(M, (uint32_t)coeffs.size(-2), degrees_to_use, dirs.data_ptr<float>(),
                         coeffs.data_ptr<float>(),
                         masks.has_value() ? reinterpret_cast<const uint8_t *>(masks->data_ptr<bool>()) : nullptr,
                         v_colors.data_ptr<float>(), v_coeffs.data_ptr<float>(),
                         compute_v_dirs ? v_dirs.data_ptr<float>() : nullptr, cur_stream()),
              "spherical_harmonics_bwd");
    (void)K;
    return std::make_tuple(v_coeffs, v_dirs);
}

// ---------------------------------------------------------------------------------------------
// Intersect.cpp:15-137
// ---------------------------------------------------------------------------------------------
GSB_EXPORT std::tuple<at::Tensor, at::Tensor, at::Tensor> intersect_tile(
    const at::Tensor means2d, const at::Tensor radii, const at::Tensor depths,
    const at::optional<at::Tensor> camera_ids, const at::optional<at::Tensor> gaussian_ids, const uint32_t C,
    const uint32_t tile_size, const uint32_t tile_width, const uint32_t tile_height, const bool sort) {
    DEVICE_GUARD(means2d);
    CHECK_INPUT(means2d);
    CHECK_INPUT(radii);
    CHECK_INPUT(depths);
    const bool packed = means2d.dim() == 2;
    TORCH_CHECK(!packed, "gsplat::intersect_tile (CUDA backend): packed mode is not supported "
                         "(the reference's caller rejects it too, rasterizer.cpp:56)");
    (void)camera_ids;
    (void)gaussian_ids;
    TORCH_CHECK(radii.scalar_type() == at::kInt, "radii must be int32");
    const uint32_t n_elements = means2d.numel() / 2;
    const uint32_t N = C ? n_elements / C : 0;

    at::Tensor tiles_per_gauss = at::empty_like(depths, depths.options().dtype(at::kInt));
    int64_t n_isects = 0;
    if (n_elements && sort) {
        // Planned sorted path (gsb_intersect.cu): count, depth order, run table and the per-tile histogram are
        // enqueued before the one host read-back the API forces (Intersect.cpp:76); the number lands in pinned memory.
        const size_t plan_bytes = gsb_isect_plan_workspace(C, N, tile_width, tile_height);
        at::Tensor plan_ws = byte_workspace(plan_bytes, depths);
        at::Tensor n_host = at::empty({1}, at::TensorOptions().dtype(at::kLong).pinned_memory(true));
        gsb_check(gsb_isect_plan(C, N, means2d.data_ptr<float>(), radii.data_ptr<int32_t>(), depths.data_ptr<float>(),
                                 tile_size, tile_width, tile_height, tiles_per_gauss.data_ptr<int32_t>(),
                                 n_host.data_ptr<int64_t>(), nullptr, 0, plan_ws.data_ptr(), plan_bytes, cur_stream()),
                  "intersect_tile/plan");
        c10::cuda::getCurrentCUDAStream().synchronize();
        n_isects = n_host.data_ptr<int64_t>()[0];
        at::Tensor isect_ids_sorted = at::empty({n_isects}, depths.options().dtype(at::kLong));
        at::Tensor flatten_ids_sorted = at::empty({n_isects}, depths.options().dtype(at::kInt));
        if (n_isects) {
            gsb_check(gsb_isect_emit_planned(C, N, depths.data_ptr<float>(), tile_width, tile_height, (uint64_t)n_isects, plan_ws.data_ptr(),
                                             plan_bytes, isect_ids_sorted.data_ptr<int64_t>(),
                                             flatten_ids_sorted.data_ptr<int32_t>(), cur_stream()),
                      "intersect_tile/emit_planned");
        }
        return std::make_tuple(tiles_per_gauss, isect_ids_sorted, flatten_ids_sorted);
    }
    at::Tensor cum_tiles;
    if (n_elements) {
        cum_tiles = at::empty({(int64_t)n_elements}, depths.options().dtype(at::kLong));
        const size_t ws_bytes = gsb_isect_count_workspace(n_elements);
        at::Tensor ws = byte_workspace(ws_bytes, depths);
        gsb_check(gsb_isect_count(C, N, means2d.data_ptr<float>(), radii.data_ptr<int32_t>(), tile_size, tile_width,
                                  tile_height, tiles_per_gauss.data_ptr<int32_t>(), cum_tiles.data_ptr<int64_t>(),
                                  ws.data_ptr(), ws_bytes, cur_stream()),
                  "intersect_tile/count");
        n_isects = cum_tiles[-1].item<int64_t>(); // the one host sync the API forces (Intersect.cpp:76)
    }
    at::Tensor isect_ids = at::empty({n_isects}, depths.options().dtype(at::kLong));
    at::Tensor flatten_ids = at::empty({n_isects}, depths.options().dtype(at::kInt));
    if (n_isects) {
        gsb_check(gsb_isect_emit(C, N, means2d.data_ptr<float>(), radii.data_ptr<int32_t>(), depths.data_ptr<float>(),
                                 cum_tiles.data_ptr<int64_t>(), tile_size, tile_width, tile_height,
                                 isect_ids.data_ptr<int64_t>(), flatten_ids.data_ptr<int32_t>(), cur_stream()),
                  "intersect_tile/emit");
    }
    return std::make_tuple(tiles_per_gauss, isect_ids, flatten_ids);
}

GSB_EXPORT at::Tensor intersect_offset(const at::Tensor isect_ids, const uint32_t C, const uint32_t tile_width,
                                       const uint32_t tile_height) {
    DEVICE_GUARD(isect_ids);
    CHECK_INPUT(isect_ids);
    at::Tensor offsets = at::empty({C, tile_height, tile_width}, isect_ids.options().dtype(at::kInt));
    gsb_check(gsb_isect_offsets((uint64_t)isect_ids.size(0), isect_ids.numel() ? isect_ids.data_ptr<int64_t>() : nullptr,
                                C, tile_width, tile_height, offsets.data_ptr<int32_t>(), cur_stream()),
              "intersect_offset");
    return offsets;
}

// ---------------------------------------------------------------------------------------------
// QuatToRotmat.cpp:13-26, Relocation.cpp:15-50
// ---------------------------------------------------------------------------------------------
GSB_EXPORT at::Tensor quats_to_rotmats(const at::Tensor quats) {
    DEVICE_GUARD(quats);
    CHECK_INPUT(quats);
    const uint32_t N = quats.size(0);
    at::Tensor rotmats = at::empty({N, 3, 3}, quats.options());
    gsb_check(gsb_quat_to_rotmat(N, quats.data_ptr<float>(), rotmats.data_ptr<float>(), cur_stream()),
              "quats_to_rotmats");
    return rotmats;
}

GSB_EXPORT std::tuple<at::Tensor, at::Tensor> relocation(at::Tensor opacities, at::Tensor scales, at::Tensor ratios,
                                                         at::Tensor binoms, const int n_max) {
    DEVICE_GUARD(opacities);
    CHECK_INPUT(opacities);
    CHECK_INPUT(scales);
    CHECK_INPUT(ratios);
    CHECK_INPUT(binoms);
    at::Tensor new_opacities = at::empty_like(opacities);
    at::Tensor new_scales = at::empty_like(scales);
    gsb_check(gsb_relocation((uint32_t)opacities.size(0), opacities.data_ptr<float>(), scales.data_ptr<float>(),
                             ratios.data_ptr<int32_t>(), binoms.data_ptr<float>(), n_max,
                             new_opacities.data_ptr<float>(), new_scales.data_ptr<float>(), cur_stream()),
              "relocation");
    return std::make_tuple(new_opacities, new_scales);
}

GSB_EXPORT void add_noise(at::Tensor raw_opacities, at::Tensor raw_scales, at::Tensor raw_quats, at::Tensor noise,
                          at::Tensor means, const float current_lr) {
    DEVICE_GUARD(raw_opacities);
    CHECK_INPUT(raw_opacities);
    CHECK_INPUT(raw_scales);
    CHECK_INPUT(raw_quats);
    CHECK_INPUT(noise);
    CHECK_INPUT(means);
    gsb_check(gsb_add_noise((uint32_t)raw_opacities.size(0), raw_opacities.data_ptr<float>(),
                            raw_scales.data_ptr<float>(), raw_quats.data_ptr<float>(), noise.data_ptr<float>(),
                            means.data_ptr<float>(), current_lr, cur_stream()),
              "add_noise");
}

// ---------------------------------------------------------------------------------------------
// Projection.cpp:16-110
// ---------------------------------------------------------------------------------------------
GSB_EXPORT std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> projection_ut_3dgs_fused(
    const at::Tensor means, const at::Tensor quats, const at::Tensor scales,
    const at::optional<at::Tensor> opacities, const at::Tensor viewmats0, const at::optional<at::Tensor> viewmats1,
    const at::Tensor Ks, const uint32_t image_width, const uint32_t image_height, const float eps2d,
    const float near_plane, const float far_plane, const float radius_clip, const bool calc_compensations,
    const CameraModelType camera_model, const UnscentedTransformParameters ut_params, ShutterType rs_type,
    const at::optional<at::Tensor> radial_coeffs, const at::optional<at::Tensor> tangential_coeffs,
    const at::optional<at::Tensor> thin_prism_coeffs) {
    DEVICE_GUARD(means);
    CHECK_INPUT(means);
    CHECK_INPUT(quats);
    CHECK_INPUT(scales);
    if (opacities.has_value()) {
        CHECK_INPUT(opacities.value());
    }
    CHECK_INPUT(viewmats0);
    if (viewmats1.has_value()) {
        CHECK_INPUT(viewmats1.value());
    }
    CHECK_INPUT(Ks);
    if (radial_coeffs.has_value()) {
        CHECK_INPUT(radial_coeffs.value());
    }
    if (tangential_coeffs.has_value()) {
        CHECK_INPUT(tangential_coeffs.value());
    }
    if (thin_prism_coeffs.has_value()) {
        CHECK_INPUT(thin_prism_coeffs.value());
    }
    const uint32_t N = means.size(0);
    const uint32_t C = Ks.size(0);
    at::Tensor radii = at::empty({C, N, 2}, means.options().dtype(at::kInt));
    at::Tensor means2d = at::empty({C, N, 2}, means.options());
    at::Tensor depths = at::empty({C, N}, means.options());
    at::Tensor conics = at::empty({C, N, 3}, means.options());
    at::Tensor compensations;
    if (calc_compensations) compensations = at::zeros({C, N}, means.options());
    CameraArgs ca = make_camera(viewmats0, viewmats1, Ks, camera_model, ut_params, rs_type, radial_coeffs,
                                tangential_coeffs, thin_prism_coeffs);
    gsb_check(gsb_projection_ut(C, N, means.data_ptr<float>(), quats.data_ptr<float>(), scales.data_ptr<float>(),
                                (opacities.has_value() && opacities->defined()) ? opacities->data_ptr<float>() : nullptr,
                                &ca.cam, image_width, image_height, eps2d, near_plane, far_plane, radius_clip,
                                radii.data_ptr<int32_t>(), means2d.data_ptr<float>(), depths.data_ptr<float>(),
                                conics.data_ptr<float>(), calc_compensations ? compensations.data_ptr<float>() : nullptr,
                                cur_stream()),
              "projection_ut_3dgs_fused");
    return std::make_tuple(radii, means2d, depths, conics, compensations);
}

// ---------------------------------------------------------------------------------------------
// Rasterization.cpp:20-261
// ---------------------------------------------------------------------------------------------
GSB_EXPORT std::tuple<at::Tensor, at::Tensor, at::Tensor> rasterize_to_pixels_from_world_3dgs_fwd(
    const at::Tensor means, const at::Tensor quats, const at::Tensor scales, const at::Tensor colors,
    const at::Tensor opacities, const at::optional<at::Tensor> backgrounds, const at::optional<at::Tensor> masks,
    const uint32_t image_width, const uint32_t image_height, const uint32_t tile_size, const at::Tensor viewmats0,
    const at::optional<at::Tensor> viewmats1, const at::Tensor Ks, const CameraModelType camera_model,
    const UnscentedTransformParameters ut_params, ShutterType rs_type, const at::optional<at::Tensor> radial_coeffs,
    const at::optional<at::Tensor> tangential_coeffs, const at::optional<at::Tensor> thin_prism_coeffs,
    const at::Tensor tile_offsets, const at::Tensor flatten_ids) {
    DEVICE_GUARD(means);
    CHECK_INPUT(means);
    CHECK_INPUT(quats);
    CHECK_INPUT(scales);
    CHECK_INPUT(colors);
    CHECK_INPUT(opacities);
    CHECK_INPUT(tile_offsets);
    CHECK_INPUT(flatten_ids);
    if (backgrounds.has_value()) {
        CHECK_INPUT(backgrounds.value());
    }
    if (masks.has_value()) {
        CHECK_INPUT(masks.value());
    }
    const uint32_t C = tile_offsets.size(0);
    const uint32_t N = means.size(0);
    const uint32_t channels = colors.size(-1);
    // 3 = RGB; 1 and 4 are the depth render modes (D / ED, RGB_D / RGB_ED: rasterizer.cpp:272-298)
    TORCH_CHECK(channels == 1 || channels == 3 || channels == 4, "Unsupported number of channels: ", channels);
    TORCH_CHECK(channels == 3 || !backgrounds.has_value() || backgrounds->numel() == (int64_t)C * channels,
                "backgrounds must be [C, ", channels, "]");
    at::Tensor renders = at::empty({C, image_height, image_width, channels}, means.options());
    at::Tensor alphas = at::empty({C, image_height, image_width, 1}, means.options());
    at::Tensor last_ids = at::empty({C, image_height, image_width}, means.options().dtype(at::kInt));
    CameraArgs ca = make_camera(viewmats0, viewmats1, Ks, camera_model, ut_params, rs_type, radial_coeffs,
                                tangential_coeffs, thin_prism_coeffs);
    const size_t ws_bytes = gsb_raster_fwd_workspace(N);
    at::Tensor ws = byte_workspace(ws_bytes, means);
    gsb_check(gsb_raster_fwd_nc(C, N, (uint64_t)flatten_ids.size(0), channels, means.data_ptr<float>(), quats.data_ptr<float>(),
                             scales.data_ptr<float>(), colors.data_ptr<float>(), opacities.data_ptr<float>(),
                             opt_f32(backgrounds),
                             masks.has_value() ? reinterpret_cast<const uint8_t *>(masks->data_ptr<bool>()) : nullptr,
                             image_width, image_height, tile_size, &ca.cam, tile_offsets.data_ptr<int32_t>(),
                             flatten_ids.numel() ? flatten_ids.data_ptr<int32_t>() : nullptr, renders.data_ptr<float>(),
                             alphas.data_ptr<float>(), last_ids.data_ptr<int32_t>(), ws.data_ptr(), ws_bytes,
                             cur_stream()),
              "rasterize_to_pixels_from_world_3dgs_fwd");
    return std::make_tuple(renders, alphas, last_ids);
}

GSB_EXPORT std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor>
rasterize_to_pixels_from_world_3dgs_bwd(
    const at::Tensor means, const at::Tensor quats, const at::Tensor scales, const at::Tensor colors,
    const at::Tensor opacities, const at::optional<at::Tensor> backgrounds, const at::optional<at::Tensor> masks,
    const uint32_t image_width, const uint32_t image_height, const uint32_t tile_size, const at::Tensor viewmats0,
    const at::optional<at::Tensor> viewmats1, const at::Tensor Ks, const CameraModelType camera_model,
    const UnscentedTransformParameters ut_params, ShutterType rs_type, const at::optional<at::Tensor> radial_coeffs,
    const at::optional<at::Tensor> tangential_coeffs, const at::optional<at::Tensor> thin_prism_coeffs,
    const at::Tensor tile_offsets, const at::Tensor flatten_ids, const at::Tensor render_alphas,
    const at::Tensor last_ids, const at::Tensor v_render_colors, const at::Tensor v_render_alphas) {
    DEVICE_GUARD(means);
    CHECK_INPUT(means);
    CHECK_INPUT(quats);
    CHECK_INPUT(scales);
    CHECK_INPUT(colors);
    CHECK_INPUT(opacities);
    CHECK_INPUT(tile_offsets);
    CHECK_INPUT(flatten_ids);
    CHECK_INPUT(render_alphas);
    CHECK_INPUT(last_ids);
    CHECK_INPUT(v_render_colors);
    CHECK_INPUT(v_render_alphas);
    if (backgrounds.has_value()) {
        CHECK_INPUT(backgrounds.value());
    }
    if (masks.has_value()) {
        CHECK_INPUT(masks.value());
    }
    const uint32_t C = tile_offsets.size(0);
    const uint32_t N = means.size(0);
    const uint32_t channels = colors.size(-1);
    TORCH_CHECK(channels == 1 || channels == 3 || channels == 4, "Unsupported number of channels: ", channels);
    TORCH_CHECK(channels == 3 || !backgrounds.has_value() || backgrounds->numel() == (int64_t)C * channels,
                "backgrounds must be [C, ", channels, "]");
    // every element is written by the backend: no five zero-fills as in Rasterization.cpp:190-194
    at::Tensor v_means = at::empty_like(means);
    at::Tensor v_quats = at::empty_like(quats);
    at::Tensor v_scales = at::empty_like(scales);
    at::Tensor v_colors = at::empty_like(colors);
    at::Tensor v_opacities = at::empty_like(opacities);
    CameraArgs ca = make_camera(viewmats0, viewmats1, Ks, camera_model, ut_params, rs_type, radial_coeffs,
                                tangential_coeffs, thin_prism_coeffs);
    const size_t ws_bytes = gsb_raster_bwd_workspace(N);
    at::Tensor ws = byte_workspace(ws_bytes, means);
    gsb_check(gsb_raster_bwd_nc(C, N, (uint64_t)flatten_ids.size(0), channels, means.data_ptr<float>(), quats.data_ptr<float>(),
                             scales.data_ptr<float>(), colors.data_ptr<float>(), opacities.data_ptr<float>(),
                             opt_f32(backgrounds),
                             masks.has_value() ? reinterpret_cast<const uint8_t *>(masks->data_ptr<bool>()) : nullptr,
                             image_width, image_height, tile_size, &ca.cam, tile_offsets.data_ptr<int32_t>(),
                             flatten_ids.numel() ? flatten_ids.data_ptr<int32_t>() : nullptr,
                             render_alphas.data_ptr<float>(), last_ids.data_ptr<int32_t>(),
                             v_render_colors.data_ptr<float>(), v_render_alphas.data_ptr<float>(),
                             v_means.data_ptr<float>(), v_quats.data_ptr<float>(), v_scales.data_ptr<float>(),
                             v_colors.data_ptr<float>(), v_opacities.data_ptr<float>(), ws.data_ptr(), ws_bytes,
                             cur_stream()),
              "rasterize_to_pixels_from_world_3dgs_bwd");
    return std::make_tuple(v_means, v_quats, v_scales, v_colors, v_opacities);
}

} // namespace gsplat
