// FastGs.cpp -- fast_gs::rasterization::forward_wrapper / backward_wrapper (include/fastgs/rasterization_api.h, the
// reference's fastgs/rasterization/src/rasterization_api.cu:15-181) on top of the C ABI (gsb_fastgs_*, include/gsb200.h).
// Allocation through the torch caching allocator, launches on the current stream, failures as c10::Error.  No compute.
// (The backward is not handed opacities_raw / sh_coefficients_0 -- rasterization_api.h:46-75; the blend records in
// per_primitive_buffers carry the activated opacity and the colour clamp mask instead.)
#include <ATen/Functions.h>
#include <ATen/core/Tensor.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime_api.h>

#include "fastgs/rasterization_api.h"
#include "fastgs/rasterization_ext.h"
#include "gsb200.h"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace {

inline gsb_stream_t cur_stream() { return reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()); }

inline void fgs_check(int rc, const char *op) {
    TORCH_CHECK(rc == GSB_OK, "fast_gs::rasterization::", op, " (CUDA backend) failed: ", gsb_error_string(rc), " [code ", rc,
                "]");
}

#define FGS_F32(x)                                                                                                   \
    TORCH_CHECK((x).is_cuda() && (x).is_contiguous() && (x).scalar_type() == at::kFloat, #x " must be a contiguous " \
                                                                                            "float32 CUDA tensor")

struct View {
    GsbFastgsView v;
    at::Tensor w2c, campos;
};
View make_view(const at::Tensor &w2c, const at::Tensor &cam_position, int active_sh_bases, int64_t rest, int width, int height,
               float fx, float fy, float cx, float cy, float near_plane, float far_plane) {
    TORCH_CHECK(w2c.numel() == 16, "w2c must hold one 4x4 matrix");
    TORCH_CHECK(cam_position.numel() == 3, "cam_position must hold 3 floats");
    TORCH_CHECK(width > 0 && height > 0, "image size must be positive");
    View r;
    r.w2c = w2c.detach().to(at::kFloat).contiguous();
    r.campos = cam_position.detach().to(r.w2c.device(), at::kFloat).contiguous();
    r.v.w2c = r.w2c.data_ptr<float>();
    r.v.cam_position = r.campos.data_ptr<float>();
    r.v.width = (uint32_t)width; r.v.height = (uint32_t)height;
    r.v.focal_x = fx; r.v.focal_y = fy; r.v.center_x = cx; r.v.center_y = cy;
    r.v.near_plane = near_plane; r.v.far_plane = far_plane;
    r.v.active_sh_bases = (uint32_t)active_sh_bases;
    r.v.total_bases_sh_rest = (uint32_t)rest;
    return r;
}

} // namespace

namespace fast_gs::rasterization {

namespace {
struct ForwardOut {
    at::Tensor image, alpha, per_primitive, per_tile, per_instance, n_instances_dev;
    int64_t n_instances;
};
// capacity < 0: exact -- the instance count is read back (one stream synchronisation) and sizes per_instance_buffers.
// capacity >= 0: the instance buffer holds `capacity` entries, the count stays on the device (n_instances_dev), nothing
// in the call reads a device value on the host: the call can be captured in a CUDA graph.
ForwardOut forward_impl(const torch::Tensor &means, const torch::Tensor &scales_raw, const torch::Tensor &rotations_raw,
                        const torch::Tensor &opacities_raw, const torch::Tensor &sh_coefficients_0,
                        const torch::Tensor &sh_coefficients_rest, const torch::Tensor &w2c, const torch::Tensor &cam_position,
                        const int active_sh_bases, const int width, const int height, const float focal_x, const float focal_y,
                        const float center_x, const float center_y, const float near_plane, const float far_plane,
                        const int64_t capacity) {
    FGS_F32(means); FGS_F32(scales_raw); FGS_F32(rotations_raw); FGS_F32(opacities_raw); FGS_F32(sh_coefficients_0);
    FGS_F32(sh_coefficients_rest);
    const c10::cuda::CUDAGuard guard(means.device());
    const int64_t N = means.size(0);
    TORCH_CHECK(means.numel() == N * 3 && scales_raw.numel() == N * 3 && rotations_raw.numel() == N * 4 &&
                    opacities_raw.numel() == N && sh_coefficients_0.numel() == N * 3,
                "fastgs forward: inconsistent parameter shapes");
    const int64_t rest = sh_coefficients_rest.dim() >= 2 ? sh_coefficients_rest.size(1) : 0;
    TORCH_CHECK(sh_coefficients_rest.numel() == N * rest * 3, "sh_coefficients_rest must be [N, B-1, 3]");
    TORCH_CHECK(active_sh_bases == 1 || active_sh_bases == 4 || active_sh_bases == 9 || active_sh_bases == 16,
                "active_sh_bases must be 1, 4, 9 or 16");
    TORCH_CHECK(active_sh_bases <= rest + 1, "active_sh_bases exceeds the stored SH coefficients");
    TORCH_CHECK(capacity <= 0x7fffffffLL, "fastgs forward: capacity beyond 2^31 instances");
    View view = make_view(w2c, cam_position, active_sh_bases, rest, width, height, focal_x, focal_y, center_x, center_y,
                          near_plane, far_plane);
    const auto f32 = means.options().dtype(at::kFloat);
    const auto u8 = means.options().dtype(at::kByte);
    ForwardOut o;
    o.image = at::empty({3, height, width}, f32);
    o.alpha = at::empty({1, height, width}, f32);
    const size_t prim_core = gsb_fastgs_primitive_bytes((uint32_t)N, (uint32_t)width, (uint32_t)height);
    o.per_primitive = at::empty({(int64_t)(prim_core + 256)}, u8);
    const size_t tile_bytes = gsb_fastgs_tile_bytes((uint32_t)width, (uint32_t)height);
    o.per_tile = at::empty({(int64_t)(tile_bytes + 256)}, u8);
    char *prim = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(o.per_primitive.data_ptr()) + 255) & ~(uintptr_t)255);
    char *tile = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(o.per_tile.data_ptr()) + 255) & ~(uintptr_t)255);
    const bool exact = capacity < 0;
    at::Tensor n_host;
    int64_t *n_out;
    if (exact) {
        n_host = at::empty({1}, at::TensorOptions().dtype(at::kLong).pinned_memory(true));
        n_host.data_ptr<int64_t>()[0] = 0;
        n_out = n_host.data_ptr<int64_t>();
    } else {
        o.n_instances_dev = at::empty({1}, means.options().dtype(at::kLong));
        n_out = o.n_instances_dev.data_ptr<int64_t>();
    }
    fgs_check(gsb_fastgs_forward_plan((uint32_t)N, means.data_ptr<float>(), scales_raw.data_ptr<float>(),
                                      rotations_raw.data_ptr<float>(), opacities_raw.data_ptr<float>(),
                                      sh_coefficients_0.data_ptr<float>(), rest ? sh_coefficients_rest.data_ptr<float>() : nullptr,
                                      &view.v, prim, prim_core, tile, tile_bytes, n_out, cur_stream()),
              "forward (plan)");
    o.n_instances = capacity;
    if (exact) {
        at::cuda::getCurrentCUDAStream().synchronize(); // the one read-back: sizes per_instance_buffers
        o.n_instances = n_host.data_ptr<int64_t>()[0];
        TORCH_CHECK(o.n_instances <= 0x7fffffffLL, "fastgs forward: more than 2^31 instances");
    }
    o.per_instance = at::empty({o.n_instances * 4}, u8);
    fgs_check(gsb_fastgs_forward_blend((uint32_t)N, &view.v, prim, prim_core, tile, tile_bytes,
                                       o.n_instances ? reinterpret_cast<int32_t *>(o.per_instance.data_ptr()) : nullptr,
                                       (uint64_t)o.n_instances, o.image.data_ptr<float>(), o.alpha.data_ptr<float>(),
                                       cur_stream()),
              "forward (blend)");
    return o;
}
} // namespace

GSB_EXPORT std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, int, int, int, int, int>
forward_wrapper(const torch::Tensor &means, const torch::Tensor &scales_raw, const torch::Tensor &rotations_raw,
                const torch::Tensor &opacities_raw, const torch::Tensor &sh_coefficients_0,
                const torch::Tensor &sh_coefficients_rest, const torch::Tensor &w2c, const torch::Tensor &cam_position,
                const int active_sh_bases, const int width, const int height, const float focal_x, const float focal_y,
                const float center_x, const float center_y, const float near_plane, const float far_plane) {
    ForwardOut o = forward_impl(means, scales_raw, rotations_raw, opacities_raw, sh_coefficients_0, sh_coefficients_rest, w2c,
                                cam_position, active_sh_bases, width, height, focal_x, focal_y, center_x, center_y, near_plane,
                                far_plane, -1);
    at::Tensor per_bucket = at::empty({0}, means.options().dtype(at::kByte));
    return {o.image, o.alpha, o.per_primitive, o.per_tile, o.per_instance, per_bucket, -1, (int)o.n_instances, 0, 0, 0};
}

GSB_EXPORT std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
forward_capacity(const torch::Tensor &means, const torch::Tensor &scales_raw, const torch::Tensor &rotations_raw,
                 const torch::Tensor &opacities_raw, const torch::Tensor &sh_coefficients_0,
                 const torch::Tensor &sh_coefficients_rest, const torch::Tensor &w2c, const torch::Tensor &cam_position,
                 const int active_sh_bases, const int width, const int height, const float focal_x, const float focal_y,
                 const float center_x, const float center_y, const float near_plane, const float far_plane,
                 const int64_t instance_capacity) {
    TORCH_CHECK(instance_capacity >= 0, "forward_capacity: instance_capacity must be >= 0");
    ForwardOut o = forward_impl(means, scales_raw, rotations_raw, opacities_raw, sh_coefficients_0, sh_coefficients_rest, w2c,
                                cam_position, active_sh_bases, width, height, focal_x, focal_y, center_x, center_y, near_plane,
                                far_plane, instance_capacity);
    return {o.image, o.alpha, o.per_primitive, o.per_tile, o.per_instance, o.n_instances_dev};
}

GSB_EXPORT std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
backward_wrapper(torch::Tensor &densification_info, const torch::Tensor &grad_image, const torch::Tensor &grad_alpha,
                 const torch::Tensor &image, const torch::Tensor &alpha, const torch::Tensor &means,
                 const torch::Tensor &scales_raw, const torch::Tensor &rotations_raw, const torch::Tensor &sh_coefficients_rest,
                 const torch::Tensor &per_primitive_buffers, const torch::Tensor &per_tile_buffers,
                 const torch::Tensor &per_instance_buffers, const torch::Tensor &per_bucket_buffers, const torch::Tensor &w2c,
                 const torch::Tensor &cam_position, const int active_sh_bases, const int width, const int height,
                 const float focal_x, const float focal_y, const float center_x, const float center_y, const float near_plane,
                 const float far_plane, const int n_visible_primitives, const int n_instances, const int n_buckets,
                 const int primitive_primitive_indices_selector, const int instance_primitive_indices_selector) {
    FGS_F32(means); FGS_F32(scales_raw); FGS_F32(rotations_raw); FGS_F32(sh_coefficients_rest); FGS_F32(alpha);
    const c10::cuda::CUDAGuard guard(means.device());
    const int64_t N = means.size(0);
    const int64_t rest = sh_coefficients_rest.dim() >= 2 ? sh_coefficients_rest.size(1) : 0;
    View view = make_view(w2c, cam_position, active_sh_bases, rest, width, height, focal_x, focal_y, center_x, center_y,
                          near_plane, far_plane);
    const auto f32 = means.options().dtype(at::kFloat);
    at::Tensor grad_means = at::empty({N, 3}, f32), grad_scales_raw = at::empty({N, 3}, f32);
    at::Tensor grad_rotations_raw = at::empty({N, 4}, f32), grad_opacities_raw = at::empty({N, 1}, f32);
    at::Tensor grad_sh0 = at::empty({N, 1, 3}, f32), grad_shN = at::empty({N, rest, 3}, f32);
    at::Tensor grad_w2c;
    if (w2c.requires_grad()) grad_w2c = at::zeros_like(w2c, f32);
    const bool update_dens = densification_info.defined() && densification_info.numel() > 0 && densification_info.size(0) > 0;
    if (update_dens) {
        FGS_F32(densification_info);
        TORCH_CHECK(densification_info.numel() == 2 * N, "densification_info must be [2, N]");
    }
    if (N == 0) return {grad_means, grad_scales_raw, grad_rotations_raw, grad_opacities_raw, grad_sh0, grad_shN, grad_w2c};
    at::Tensor gi = grad_image.contiguous(), ga = grad_alpha.contiguous();
    FGS_F32(gi); FGS_F32(ga);
    TORCH_CHECK(gi.numel() == (int64_t)3 * width * height && ga.numel() == (int64_t)width * height &&
                    alpha.numel() == (int64_t)width * height,
                "fastgs backward: image gradients do not match the image size");
    const size_t prim_core = gsb_fastgs_primitive_bytes((uint32_t)N, (uint32_t)width, (uint32_t)height);
    const size_t tile_bytes = gsb_fastgs_tile_bytes((uint32_t)width, (uint32_t)height);
    TORCH_CHECK(per_primitive_buffers.is_cuda() && (size_t)per_primitive_buffers.numel() >= prim_core + 256 &&
                    per_tile_buffers.is_cuda() && (size_t)per_tile_buffers.numel() >= tile_bytes + 256 &&
                    per_instance_buffers.numel() >= (int64_t)n_instances * 4,
                "fastgs backward: the buffers do not come from this backend's forward_wrapper");
    char *prim = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(per_primitive_buffers.data_ptr()) + 255) & ~(uintptr_t)255);
    char *tile = reinterpret_cast<char *>((reinterpret_cast<uintptr_t>(per_tile_buffers.data_ptr()) + 255) & ~(uintptr_t)255);
    fgs_check(gsb_fastgs_backward(
                  (uint32_t)N, means.data_ptr<float>(), scales_raw.data_ptr<float>(), rotations_raw.data_ptr<float>(),
                  rest ? sh_coefficients_rest.data_ptr<float>() : nullptr, &view.v, prim, prim_core, tile, tile_bytes,
                  n_instances ? reinterpret_cast<const int32_t *>(per_instance_buffers.data_ptr()) : nullptr,
                  (uint64_t)n_instances, alpha.data_ptr<float>(), gi.data_ptr<float>(), ga.data_ptr<float>(),
                  grad_means.data_ptr<float>(), grad_scales_raw.data_ptr<float>(), grad_rotations_raw.data_ptr<float>(),
                  grad_opacities_raw.data_ptr<float>(), grad_sh0.data_ptr<float>(), rest ? grad_shN.data_ptr<float>() : nullptr,
                  grad_w2c.defined() ? grad_w2c.data_ptr<float>() : nullptr,
                  update_dens ? densification_info.data_ptr<float>() : nullptr, cur_stream()),
              "backward");
    return {grad_means, grad_scales_raw, grad_rotations_raw, grad_opacities_raw, grad_sh0, grad_shN, grad_w2c};
}

} // namespace fast_gs::rasterization
