// kernels/bilateral_grid.cuh -- the bilateral-grid kernel API (SURVEY.md 8 f5) that the reference's BilateralGrid
// component (src/training/components/bilateral_grid.cpp) calls, served by libgsplat_b200.so (shim/BilateralGrid.cpp)
// on top of the C ABI of include/gsb200.h.  Same namespace, names, parameter lists and return types as the reference's
// include/kernels/bilateral_grid.cuh, so that component compiles unchanged against this header and links against this
// library.  Deviations (DESIGN.md section 1): everything launches on the current torch stream, tv_loss_backward_cuda reads
// its upstream gradient on the device (no host synchronisation), the slice clamps its input to [0, 1] itself, and the
// slice backward returns the gradient with respect to the unclamped input (zero where rgb < 0 or rgb > 1).
#pragma once
#include <torch/torch.h>

#include <tuple>

namespace gs {
    namespace bilateral_grid {

        // output [h, w, 3] = rgb [h, w, 3] sliced through one image's grid [12, L, H, W]
        void slice_forward_cuda(const torch::Tensor& grid, const torch::Tensor& rgb, torch::Tensor& output,
                                bool use_uniform_coords = true);

        // (d grid [12, L, H, W], d rgb [h, w, 3]) for an upstream gradient [h, w, 3]
        std::tuple<torch::Tensor, torch::Tensor> slice_backward_cuda(const torch::Tensor& grid, const torch::Tensor& rgb,
                                                                     const torch::Tensor& grad_output);

        // total-variation loss (0-dim tensor) of all grids [N, 12, L, H, W]
        torch::Tensor tv_loss_forward_cuda(const torch::Tensor& grids);

        // its gradient [N, 12, L, H, W], scaled by grad_output (a one-element device tensor)
        torch::Tensor tv_loss_backward_cuda(const torch::Tensor& grids, const torch::Tensor& grad_output);

    } // namespace bilateral_grid
} // namespace gs
