// ref_binding.cpp -- exposes the REFERENCE's own gsplat:: operators (compiled from
// /root/reference/gsplat by oracle/build_ref.py) as torch.ops.gsplat_ref.* .
// TEST INFRASTRUCTURE ONLY: the checker that pins the oracle / the H100 path on the rows the
// reference's tests do not cover (UT projection, from-world blend fwd/bwd), and the same-box GPU
// baseline of bench.py.  Same flattening of enums / UT params as the product's torch_binding.cpp.
#include <torch/library.h>

#include "Ops.h"

namespace {
using at::Tensor;
using OT = std::optional<at::Tensor>;

UnscentedTransformParameters make_ut(double a, double b, double k, double m, bool r) {
    UnscentedTransformParameters ut;
    ut.alpha = (float)a; ut.beta = (float)b; ut.kappa = (float)k;
    ut.in_image_margin_factor = (float)m; ut.require_all_sigma_points_valid = r;
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
Tensor quats_to_rotmats(const Tensor &quats) { return gsplat::quats_to_rotmats(quats); }
std::tuple<Tensor, Tensor> relocation(const Tensor &opacities, const Tensor &scales, const Tensor &ratios,
                                      const Tensor &binoms, int64_t n_max) {
    return gsplat::relocation(opacities, scales, ratios, binoms, (int)n_max);
}
void add_noise(const Tensor &raw_opacities, const Tensor &raw_scales, const Tensor &raw_quats, const Tensor &noise,
               Tensor means, double current_lr) {
    gsplat::add_noise(raw_opacities, raw_scales, raw_quats, noise, means, (float)current_lr);
}
} // namespace

#ifndef REF_NS
#define REF_NS gsplat_ref
#endif
#define REF_TORCH_LIBRARY(ns, m) TORCH_LIBRARY(ns, m) // expands REF_NS before TORCH_LIBRARY pastes it

REF_TORCH_LIBRARY(REF_NS, m) {
    m.def("spherical_harmonics_fwd", &sh_fwd);
    m.def("spherical_harmonics_bwd", &sh_bwd);
    m.def("intersect_tile", &intersect_tile);
    m.def("intersect_offset", &intersect_offset);
    m.def("projection_ut_3dgs_fused", &projection_ut);
    m.def("rasterize_to_pixels_from_world_3dgs_fwd", &raster_fwd);
    m.def("rasterize_to_pixels_from_world_3dgs_bwd", &raster_bwd);
    m.def("quats_to_rotmats", &quats_to_rotmats);
    m.def("relocation", &relocation);
    m.def("add_noise(Tensor raw_opacities, Tensor raw_scales, Tensor raw_quats, Tensor noise, Tensor(a!) means, float current_lr) -> ()",
          &add_noise);
}
