// Sparsity.cpp -- the ADMM opacity-sparsity phase (src/training/components/sparsity_optimizer.cpp) on this library's
// kernels (csrc/gsb_sparsity.cu, gsb_adc.cu): extended operators (FusedOps.h) registered as
// torch.ops.gsplat_b200.sparsity_* for the Python sparsifier (sparsity.py).
//
//   sparsity_update          initialize / update_state: z and u written in place
//   sparsity_loss            the loss on the device, its gradient added into v_opacity (rho read from the device)
//   sparsity_prune_classify  (counts, workspace) for adc_apply: the n_prune lowest-opacity rows removed
// None of them reads anything back to the host.
#include <ATen/Functions.h>
#include <ATen/core/Tensor.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include "FusedOps.h"
#include "SplatRows.h"
#include "gsb200.h"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace {

using at::Tensor;
using namespace gsb_shim;

inline gsb_stream_t cur_stream() { return reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()); }

inline void check(int rc, const char *op) { TORCH_CHECK(rc == 0, op, " failed: ", gsb_error_string(rc)); }

int64_t checked_rows(const Tensor &opacity_raw) {
    check_cuda(opacity_raw, at::kFloat, "opacity_raw");
    const int64_t N = opacity_raw.numel();
    TORCH_CHECK(N <= INT32_MAX / 2, "at most INT32_MAX / 2 rows");
    return N;
}

void check_state(const Tensor &t, int64_t N, const char *name) {
    check_cuda(t, at::kFloat, name);
    TORCH_CHECK(t.numel() == N, name, " must have opacity_raw's number of elements");
}

Tensor workspace(int64_t bytes, const Tensor &like) { return at::empty({bytes}, like.options().dtype(at::kByte)); }

} // namespace

namespace gsplat {

GSB_EXPORT void sparsity_update(const at::Tensor opacity_raw, at::Tensor z, at::Tensor u, const int64_t k,
                                const bool initialize) {
    const int64_t N = checked_rows(opacity_raw);
    check_state(z, N, "z");
    check_state(u, N, "u");
    TORCH_CHECK(k >= 0 && k <= N, "sparsity_update: k must be in [0, N]");
    if (N == 0) return;
    const c10::cuda::CUDAGuard guard(opacity_raw.device());
    Tensor ws = workspace((int64_t)gsb_sparsity_workspace((uint32_t)N), opacity_raw);
    check(gsb_sparsity_update((uint32_t)N, opacity_raw.data_ptr<float>(), z.data_ptr<float>(), u.data_ptr<float>(),
                              (uint32_t)k, initialize ? 1 : 0, ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
          "gsb_sparsity_update");
}

GSB_EXPORT at::Tensor sparsity_loss(const at::Tensor opacity_raw, const at::Tensor z, const at::Tensor u,
                                    const at::Tensor rho, at::Tensor v_opacity) {
    const int64_t N = checked_rows(opacity_raw);
    check_state(z, N, "z");
    check_state(u, N, "u");
    check_state(v_opacity, N, "v_opacity");
    check_cuda(rho, at::kFloat, "rho");
    TORCH_CHECK(rho.numel() == 1, "rho must be a one-element device tensor");
    const c10::cuda::CUDAGuard guard(opacity_raw.device());
    Tensor loss = at::empty({1}, opacity_raw.options());
    Tensor ws = workspace((int64_t)gsb_sparsity_workspace((uint32_t)N), opacity_raw);
    check(gsb_sparsity_loss((uint32_t)N, N ? opacity_raw.data_ptr<float>() : nullptr, N ? z.data_ptr<float>() : nullptr,
                            N ? u.data_ptr<float>() : nullptr, rho.data_ptr<float>(),
                            N ? v_opacity.data_ptr<float>() : nullptr, loss.data_ptr<float>(), ws.data_ptr(),
                            (size_t)ws.numel(), cur_stream()),
          "gsb_sparsity_loss");
    return loss;
}

GSB_EXPORT std::tuple<at::Tensor, at::Tensor> sparsity_prune_classify(const at::Tensor opacity_raw,
                                                                      const int64_t n_prune) {
    const int64_t N = checked_rows(opacity_raw);
    TORCH_CHECK(n_prune >= 0 && n_prune <= N, "sparsity_prune_classify: n_prune must be in [0, N]");
    const c10::cuda::CUDAGuard guard(opacity_raw.device());
    Tensor counts = at::empty({8}, opacity_raw.options().dtype(at::kInt));
    Tensor ws = workspace((int64_t)gsb_adc_workspace((uint32_t)N), opacity_raw);
    check(gsb_adc_prune_classify((uint32_t)N, N ? opacity_raw.data_ptr<float>() : nullptr, (uint32_t)n_prune,
                                 counts.data_ptr<int32_t>(), ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
          "gsb_adc_prune_classify");
    return std::make_tuple(counts, ws);
}

} // namespace gsplat

namespace {

void update_op(const Tensor &opacity_raw, Tensor z, Tensor u, int64_t k, bool initialize) {
    gsplat::sparsity_update(opacity_raw, z, u, k, initialize);
}
Tensor loss_op(const Tensor &opacity_raw, const Tensor &z, const Tensor &u, const Tensor &rho, Tensor v_opacity) {
    return gsplat::sparsity_loss(opacity_raw, z, u, rho, v_opacity);
}
std::tuple<Tensor, Tensor> prune_op(const Tensor &opacity_raw, int64_t n_prune) {
    return gsplat::sparsity_prune_classify(opacity_raw, n_prune);
}

} // namespace

TORCH_LIBRARY_FRAGMENT(gsplat_b200, m) {
    m.def("sparsity_update(Tensor opacity_raw, Tensor(a!) z, Tensor(b!) u, int k, bool initialize) -> ()", &update_op);
    m.def("sparsity_loss(Tensor opacity_raw, Tensor z, Tensor u, Tensor rho, Tensor(a!) v_opacity) -> Tensor",
          &loss_op);
    m.def("sparsity_prune_classify(Tensor opacity_raw, int n_prune) -> (Tensor, Tensor)", &prune_op);
}
