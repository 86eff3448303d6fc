// ref_bilagrid_harness.cpp -- runs the REFERENCE's BilateralGrid component (src/training/components/bilateral_grid.cpp,
// compiled unmodified by oracle/build_ref_bilagrid.py) on THIS repository's drop-in kernels (libgsplat_b200.so,
// include/kernels/bilateral_grid.cuh): torch.ops.bilagrid_component.run.
// TEST INFRASTRUCTURE ONLY (tests/test_gpu_bilagrid_reference.py compares it with the Python mirror, bilateral.py).
#include <torch/library.h>
#include <torch/torch.h>

#include "bilateral_grid.hpp"

namespace {
using at::Tensor;

// A BilateralGrid of grids_init's shape, loaded with grids_init; out = apply(rgb, idx), tv = tv_loss(); then
// backward of sum(out * v_out) + tv_weight * tv.  Returns (out, tv, d grids, d rgb).
std::tuple<Tensor, Tensor, Tensor, Tensor> run(const Tensor &grids_init, const Tensor &rgb, int64_t idx,
                                               const Tensor &v_out, double tv_weight) {
    gs::training::BilateralGrid bg((int)grids_init.size(0), (int)grids_init.size(4), (int)grids_init.size(3),
                                   (int)grids_init.size(2));
    {
        torch::NoGradGuard ng;
        bg.parameters().copy_(grids_init);
    }
    Tensor x = rgb.detach().clone().set_requires_grad(true);
    Tensor out = bg.apply(x, (int)idx);
    Tensor tv = bg.tv_loss();
    ((out * v_out).sum() + tv * tv_weight).backward();
    return std::make_tuple(out.detach(), tv.detach(), bg.parameters().grad(), x.grad());
}
} // namespace

TORCH_LIBRARY(bilagrid_component, m) { m.def("run", &run); }
