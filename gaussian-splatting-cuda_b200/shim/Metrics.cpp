// Metrics.cpp -- PSNR and SSIM of one view (src/training/metrics/metrics.cpp:40-116, PSNR::compute and SSIM::compute
// after the clamp at :441) on this library's kernel (csrc/gsb_metrics.cu), registered as
// torch.ops.gsplat_b200.image_metrics (torch_binding.cpp) for the Python evaluator (metrics.py).  The result goes into a
// caller-given [2] device tensor; nothing is read back to the host.
#include <ATen/Functions.h>
#include <ATen/core/Tensor.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include "FusedOps.h"
#include "SplatRows.h"
#include "gsb200.h"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace gsplat {

GSB_EXPORT void image_metrics(const at::Tensor image, const at::Tensor target, const bool image_hwc, at::Tensor out) {
    using gsb_shim::check_cuda;
    check_cuda(image, at::kFloat, "image");
    check_cuda(target, at::kFloat, "target");
    check_cuda(out, at::kFloat, "out");
    TORCH_CHECK(target.dim() == 3 && target.size(0) == 3, "image_metrics: target must be [3,H,W]");
    const int64_t H = target.size(1), W = target.size(2);
    TORCH_CHECK(H >= 1 && W >= 1, "image_metrics: the image must have at least one pixel");
    if (image_hwc) {
        TORCH_CHECK(image.dim() == 3 && image.size(0) == H && image.size(1) == W && image.size(2) == 3,
                    "image_metrics: image must be [H,W,3] with the target's H and W");
    } else {
        TORCH_CHECK(image.sizes() == target.sizes(), "image_metrics: image must be [3,H,W] like the target");
    }
    TORCH_CHECK(3 * H * W <= INT32_MAX, "image_metrics: at most INT32_MAX values per image");
    TORCH_CHECK(out.numel() == 2, "image_metrics: out must hold two floats (psnr, ssim)");
    TORCH_CHECK(image.device() == target.device() && out.device() == target.device(),
                "image_metrics: image, target and out must be on one device");
    const c10::cuda::CUDAGuard guard(target.device());
    at::Tensor ws = at::empty({(int64_t)gsb_image_metrics_workspace()}, target.options().dtype(at::kByte));
    const int rc = gsb_image_metrics((uint32_t)W, (uint32_t)H, image.data_ptr<float>(), target.data_ptr<float>(),
                                     image_hwc ? GSB_METRICS_IMAGE_HWC : 0, out.data_ptr<float>(), ws.data_ptr(),
                                     (size_t)ws.numel(),
                                     reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()));
    TORCH_CHECK(rc == 0, "gsb_image_metrics failed: ", gsb_error_string(rc));
}

} // namespace gsplat
