// BilateralGrid.cpp -- SURVEY.md 8 f5: the bilateral grid on this library's kernels (csrc/gsb_bilagrid.cu).
//
//  * gs::bilateral_grid::* -- the drop-in kernel API of the reference's include/kernels/bilateral_grid.cuh
//    (include/kernels/bilateral_grid.cuh here), which its BilateralGrid component (components/bilateral_grid.cpp) calls;
//  * torch.ops.gsplat_b200.bilagrid_* -- the ops behind the Python mirror (bilateral.py) and the training step: the
//    image index is a device tensor and the slice backward adds into a caller-owned grid-gradient buffer, so that the
//    TV gradient of all grids and the slice gradient of one image meet in one buffer without a zero-fill.
#include <ATen/Functions.h>
#include <ATen/core/Tensor.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include "gsb200.h"
#include "kernels/bilateral_grid.cuh"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace {

using at::Tensor;

inline gsb_stream_t cur_stream() { return reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()); }

inline void check(int rc, const char *op) { TORCH_CHECK(rc == 0, op, " failed: ", gsb_error_string(rc)); }

inline void check_f32(const Tensor &t, const char *name) {
    TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == at::kFloat, name, " must be float32");
    TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}

struct GridDims {
    uint32_t n, l, h, w;
};

// [N, 12, L, H, W] or one image's [12, L, H, W]
GridDims grid_dims(const Tensor &grids) {
    check_f32(grids, "grids");
    const bool one = grids.dim() == 4;
    TORCH_CHECK((one || grids.dim() == 5) && grids.size(one ? 0 : 1) == 12, "grids must be [N,12,L,H,W] or [12,L,H,W]");
    const int64_t o = one ? 0 : 1;
    return {one ? 1u : (uint32_t)grids.size(0), (uint32_t)grids.size(o + 1), (uint32_t)grids.size(o + 2),
            (uint32_t)grids.size(o + 3)};
}

// (height, width) of an image [..., 3, H, W] (chw) or [..., H, W, 3]
std::pair<uint32_t, uint32_t> image_dims(const Tensor &image, bool chw) {
    check_f32(image, "image");
    TORCH_CHECK(image.dim() >= 3, "image must have at least three dimensions");
    if (chw) {
        TORCH_CHECK(image.size(-3) == 3 && image.numel() == 3 * image.size(-2) * image.size(-1), "image must be [3,H,W]");
        return {(uint32_t)image.size(-2), (uint32_t)image.size(-1)};
    }
    TORCH_CHECK(image.size(-1) == 3 && image.numel() == 3 * image.size(-3) * image.size(-2), "image must be [H,W,3]");
    return {(uint32_t)image.size(-3), (uint32_t)image.size(-2)};
}

const int32_t *index_ptr(const c10::optional<Tensor> &image_idx) {
    if (!image_idx.has_value() || !image_idx->defined()) return nullptr;
    TORCH_CHECK(image_idx->is_cuda() && image_idx->scalar_type() == at::kInt && image_idx->numel() == 1,
                "image_idx must be a one-element int32 CUDA tensor");
    return image_idx->data_ptr<int32_t>();
}

void slice_into(const Tensor &grids, const Tensor &image, const c10::optional<Tensor> &image_idx, bool chw, Tensor &out) {
    const c10::cuda::CUDAGuard guard(image.device());
    const GridDims g = grid_dims(grids);
    const auto [h, w] = image_dims(image, chw);
    check_f32(out, "output");
    TORCH_CHECK(out.numel() == image.numel(), "output must be shaped like the image");
    check(gsb_bilagrid_slice_fwd(g.w, g.h, g.l, g.n, grids.data_ptr<float>(), index_ptr(image_idx), w, h,
                                 chw ? GSB_BILAGRID_CHW : 0, image.data_ptr<float>(), out.data_ptr<float>(), cur_stream()),
          "gsb_bilagrid_slice_fwd");
}

Tensor slice(const Tensor &grids, const Tensor &image, const c10::optional<Tensor> &image_idx, bool chw) {
    Tensor out = at::empty_like(image);
    slice_into(grids, image, image_idx, chw, out);
    return out;
}

Tensor slice_backward(const Tensor &grids, const Tensor &image, const c10::optional<Tensor> &image_idx,
                      const Tensor &v_output, Tensor v_grids, bool chw) {
    const c10::cuda::CUDAGuard guard(image.device());
    const GridDims g = grid_dims(grids);
    const auto [h, w] = image_dims(image, chw);
    check_f32(v_output, "v_output");
    check_f32(v_grids, "v_grids");
    TORCH_CHECK(v_output.numel() == image.numel(), "v_output must be shaped like the image");
    TORCH_CHECK(v_grids.numel() == grids.numel(), "v_grids must be shaped like the grids");
    Tensor v_image = at::empty_like(image);
    check(gsb_bilagrid_slice_bwd(g.w, g.h, g.l, g.n, grids.data_ptr<float>(), index_ptr(image_idx), w, h,
                                 chw ? GSB_BILAGRID_CHW : 0, image.data_ptr<float>(), v_output.data_ptr<float>(),
                                 v_grids.data_ptr<float>(), v_image.data_ptr<float>(), cur_stream()),
          "gsb_bilagrid_slice_bwd");
    return v_image;
}

// (loss: 0-dim tensor, gradient scaled by *weight or an empty tensor)
std::tuple<Tensor, Tensor> tv(const Tensor &grids, const c10::optional<Tensor> &weight, bool compute_grad) {
    const c10::cuda::CUDAGuard guard(grids.device());
    const GridDims g = grid_dims(grids);
    const float *wp = nullptr;
    if (weight.has_value() && weight->defined()) {
        check_f32(*weight, "weight");
        TORCH_CHECK(weight->numel() == 1, "weight must hold one element");
        wp = weight->data_ptr<float>();
    }
    Tensor loss = at::empty({}, grids.options());
    Tensor v = compute_grad ? at::empty_like(grids) : at::empty({0}, grids.options());
    Tensor ws = at::empty({(int64_t)gsb_bilagrid_tv_workspace()}, grids.options().dtype(at::kByte));
    check(gsb_bilagrid_tv(g.w, g.h, g.l, g.n, grids.data_ptr<float>(), wp, loss.data_ptr<float>(),
                          compute_grad ? v.data_ptr<float>() : nullptr, ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
          "gsb_bilagrid_tv");
    return std::make_tuple(loss, v);
}

} // namespace

namespace gs {
    namespace bilateral_grid {

        GSB_EXPORT void slice_forward_cuda(const torch::Tensor &grid, const torch::Tensor &rgb, torch::Tensor &output,
                                           bool /*use_uniform_coords: the reference's kernels only have this mode*/) {
            TORCH_CHECK(grid.dim() == 4, "grid must be [12,L,H,W]");
            TORCH_CHECK(output.sizes() == rgb.sizes(), "output must be shaped like rgb");
            slice_into(grid.contiguous(), rgb.contiguous(), c10::nullopt, false, output);
        }

        // d rgb is taken with respect to the unclamped rgb: zero where rgb < 0 or rgb > 1 (DESIGN.md section 1)
        GSB_EXPORT std::tuple<torch::Tensor, torch::Tensor> slice_backward_cuda(const torch::Tensor &grid,
                                                                                const torch::Tensor &rgb,
                                                                                const torch::Tensor &grad_output) {
            TORCH_CHECK(grid.dim() == 4, "grid must be [12,L,H,W]");
            const Tensor g = grid.contiguous();
            Tensor v_grid = at::zeros_like(g);
            Tensor v_rgb = slice_backward(g, rgb.contiguous(), c10::nullopt, grad_output.contiguous(), v_grid, false);
            return std::make_tuple(v_grid, v_rgb);
        }

        GSB_EXPORT torch::Tensor tv_loss_forward_cuda(const torch::Tensor &grids) {
            TORCH_CHECK(grids.dim() == 5 && grids.size(1) == 12, "grids must be [N,12,L,H,W]");
            return std::get<0>(tv(grids.contiguous(), c10::nullopt, false));
        }

        GSB_EXPORT torch::Tensor tv_loss_backward_cuda(const torch::Tensor &grids, const torch::Tensor &grad_output) {
            TORCH_CHECK(grids.dim() == 5 && grids.size(1) == 12, "grids must be [N,12,L,H,W]");
            // read on the device (the reference reads it with .item(), a host synchronisation)
            const Tensor w = grad_output.to(grids.device(), at::kFloat).contiguous().reshape({1});
            return std::get<1>(tv(grids.contiguous(), w, true));
        }

    } // namespace bilateral_grid
} // namespace gs

TORCH_LIBRARY_FRAGMENT(gsplat_b200, m) {
    m.def("bilagrid_slice(Tensor grids, Tensor image, Tensor? image_idx, bool chw) -> Tensor", &slice);
    m.def("bilagrid_slice_backward(Tensor grids, Tensor image, Tensor? image_idx, Tensor v_output, Tensor(a!) v_grids, "
          "bool chw) -> Tensor",
          &slice_backward);
    m.def("bilagrid_tv(Tensor grids, Tensor? weight, bool compute_grad) -> (Tensor, Tensor)", &tv);
}
