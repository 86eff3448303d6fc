// Init.cpp -- the initial scales of SplatData::init_model_from_pointcloud (src/core/splat_data.cpp:63-111,
// compute_mean_neighbor_distances) on this library's exact nearest-neighbour kernel (csrc/gsb_knn.cu), registered as
// torch.ops.gsplat_b200.mean_neighbor_distances[_out] (torch_binding.cpp) for the Python set-up (model.py).
#include <ATen/Functions.h>
#include <ATen/core/Tensor.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include "FusedOps.h"
#include "SplatRows.h"
#include "gsb200.h"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace gsplat {

GSB_EXPORT void mean_neighbor_distances_out(const at::Tensor points, at::Tensor out, at::Tensor status) {
    using gsb_shim::check_cuda;
    check_cuda(points, at::kFloat, "points");
    check_cuda(out, at::kFloat, "out");
    check_cuda(status, at::kInt, "status");
    TORCH_CHECK(points.dim() == 2 && points.size(1) == 3, "mean_neighbor_distances: points must be [N,3]");
    const int64_t N = points.size(0);
    TORCH_CHECK(N <= (int64_t)GSB_KNN_MAX_POINTS, "mean_neighbor_distances: at most ", GSB_KNN_MAX_POINTS, " points");
    TORCH_CHECK(out.numel() == N, "mean_neighbor_distances: out must hold N floats");
    TORCH_CHECK(status.numel() == 1, "mean_neighbor_distances: status must hold one int32");
    TORCH_CHECK(out.device() == points.device() && status.device() == points.device(),
                "mean_neighbor_distances: points, out and status must be on one device");
    const c10::cuda::CUDAGuard guard(points.device());
    at::Tensor ws = at::empty({(int64_t)gsb_knn_mean_dist_workspace((uint32_t)N)}, points.options().dtype(at::kByte));
    const int rc = gsb_knn_mean_dist((uint32_t)N, N ? points.data_ptr<float>() : nullptr,
                                     N ? out.data_ptr<float>() : nullptr, ws.data_ptr(), (size_t)ws.numel(),
                                     reinterpret_cast<uint32_t *>(status.data_ptr<int32_t>()),
                                     reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()));
    TORCH_CHECK(rc == 0, "gsb_knn_mean_dist failed: ", gsb_error_string(rc));
}

GSB_EXPORT at::Tensor mean_neighbor_distances(const at::Tensor points) {
    TORCH_CHECK(points.defined() && points.is_cuda(), "mean_neighbor_distances: points must be a CUDA tensor");
    TORCH_CHECK(points.scalar_type() == at::kFloat, "mean_neighbor_distances: points must be float32");
    TORCH_CHECK(points.dim() == 2 && points.size(1) == 3, "mean_neighbor_distances: points must be [N,3]");
    const at::Tensor p = points.contiguous();
    at::Tensor out = at::empty({p.size(0)}, p.options());
    at::Tensor status = at::empty({1}, p.options().dtype(at::kInt));
    mean_neighbor_distances_out(p, out, status);
    // the one read-back of the call (the set-up reads scene_scale back anyway)
    TORCH_CHECK(status.item<int32_t>() == 0, "mean_neighbor_distances: points must be finite (NaN or infinity found)");
    return out;
}

} // namespace gsplat
