// ref_bilagrid_binding.cpp -- exposes the REFERENCE's own bilateral-grid kernels (src/training/kernels/
// bilateral_grid_{forward,backward,tv}.cu, compiled unmodified by oracle/build_ref_bilagrid.py) as
// torch.ops.bilagrid_ref.*, with the reference's own signatures (include/kernels/bilateral_grid.cuh).
// TEST INFRASTRUCTURE ONLY: the live checker of SURVEY.md 8 f5, the source of tests/golden/ref_bilagrid_small.npz and the
// same-box baseline of bench_bilateral_grid.py.
#include <torch/library.h>
#include <torch/torch.h>

#include "kernels/bilateral_grid.cuh"

namespace {
using at::Tensor;

Tensor slice_forward(const Tensor &grid, const Tensor &rgb) {
    Tensor out = torch::empty_like(rgb);
    gs::bilateral_grid::slice_forward_cuda(grid.contiguous(), rgb.contiguous(), out, true);
    return out;
}
std::tuple<Tensor, Tensor> slice_backward(const Tensor &grid, const Tensor &rgb, const Tensor &grad_output) {
    return gs::bilateral_grid::slice_backward_cuda(grid.contiguous(), rgb.contiguous(), grad_output.contiguous());
}
Tensor tv_forward(const Tensor &grids) { return gs::bilateral_grid::tv_loss_forward_cuda(grids.contiguous()); }
Tensor tv_backward(const Tensor &grids, const Tensor &grad_output) {
    return gs::bilateral_grid::tv_loss_backward_cuda(grids.contiguous(), grad_output);
}
} // namespace

TORCH_LIBRARY(bilagrid_ref, m) {
    m.def("slice_forward", &slice_forward);
    m.def("slice_backward", &slice_backward);
    m.def("tv_forward", &tv_forward);
    m.def("tv_backward", &tv_backward);
}
