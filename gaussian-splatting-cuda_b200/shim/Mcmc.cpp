// Mcmc.cpp -- SURVEY.md 8 f6: the MCMC strategy's refine, noise and regularisers on this library's kernels
// (csrc/gsb_mcmc.cu), as extended operators over the raw SplatData tensors and their Adam moments (FusedOps.h) and as
// torch.ops.gsplat_b200.mcmc_* for the Python strategy (mcmc.py).  Every operator works in place on the caller's
// tensors, allocates only its outputs and a workspace from the caching allocator, and never reads a device value on
// the host, so a refine can sit between two captured parts of a training iteration without a synchronisation.
#include <ATen/Functions.h>
#include <ATen/core/Tensor.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <mutex>

#include "FusedOps.h"
#include "SplatRows.h"
#include "gsb200.h"

#define GSB_EXPORT __attribute__((visibility("default")))

namespace {

using at::Tensor;
using namespace gsb_shim;

inline gsb_stream_t cur_stream() { return reinterpret_cast<gsb_stream_t>(at::cuda::getCurrentCUDAStream().stream()); }

inline void check(int rc, const char *op) { TORCH_CHECK(rc == 0, op, " failed: ", gsb_error_string(rc)); }

Tensor workspace(uint32_t N, const Tensor &like) {
    return at::empty({(int64_t)gsb_mcmc_workspace(N)}, like.options().dtype(at::kByte));
}

const uint32_t *count_ptr(const c10::optional<Tensor> &n) {
    if (!n.has_value() || !n->defined()) return nullptr;
    check_cuda(*n, at::kInt, "sample count");
    TORCH_CHECK(n->numel() == 1, "the sample count must hold one element");
    return reinterpret_cast<const uint32_t *>(n->data_ptr<int32_t>());
}

void apply(const std::vector<Tensor> &params, const std::vector<Tensor> &exp_avg, const std::vector<Tensor> &exp_avg_sq,
           int64_t N, const Tensor &samples, const c10::optional<Tensor> &n_samples, const int32_t *targets,
           const Tensor &binoms, double min_opacity) {
    check_cuda(samples, at::kInt, "samples");
    check_cuda(binoms, at::kFloat, "binoms");
    TORCH_CHECK(binoms.dim() == 2 && binoms.size(0) == binoms.size(1), "binoms must be [n_max, n_max]");
    const int64_t n = samples.numel();
    const GsbMcmcRows r = make_rows(params, exp_avg, exp_avg_sq, targets ? N : N + n);
    if (N == 0 || n == 0) return;
    const c10::cuda::CUDAGuard guard(samples.device());
    Tensor ws = workspace((uint32_t)N, samples);
    check(gsb_mcmc_apply((uint32_t)N, &r, samples.data_ptr<int32_t>(), (uint32_t)n, count_ptr(n_samples), targets,
                         binoms.data_ptr<float>(), (int32_t)binoms.size(0), (float)min_opacity, ws.data_ptr(),
                         (size_t)ws.numel(), cur_stream()),
          "gsb_mcmc_apply");
}

} // namespace

namespace gsplat {

GSB_EXPORT std::tuple<at::Tensor, at::Tensor, at::Tensor> mcmc_dead(const at::Tensor opacity_raw,
                                                                    const at::Tensor rotation_raw,
                                                                    const float min_opacity) {
    check_cuda(opacity_raw, at::kFloat, "opacity_raw");
    check_cuda(rotation_raw, at::kFloat, "rotation_raw");
    const int64_t N = rotation_raw.size(0);
    TORCH_CHECK(rotation_raw.numel() == 4 * N && opacity_raw.numel() == N, "opacity_raw [N] / [N,1], rotation_raw [N,4]");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(rotation_raw.data_ptr()) & 15) == 0, "rotation_raw must be 16-byte aligned");
    const c10::cuda::CUDAGuard guard(opacity_raw.device());
    Tensor dead = at::empty({N}, opacity_raw.options().dtype(at::kInt));
    Tensor n_dead = at::zeros({1}, opacity_raw.options().dtype(at::kInt));
    Tensor weights = at::empty({N}, opacity_raw.options());
    if (N == 0) return std::make_tuple(dead, n_dead, weights);
    Tensor ws = workspace((uint32_t)N, opacity_raw);
    check(gsb_mcmc_dead((uint32_t)N, opacity_raw.data_ptr<float>(), rotation_raw.data_ptr<float>(), min_opacity,
                        dead.data_ptr<int32_t>(), reinterpret_cast<uint32_t *>(n_dead.data_ptr<int32_t>()),
                        weights.data_ptr<float>(), ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
          "gsb_mcmc_dead");
    return std::make_tuple(dead, n_dead, weights);
}

GSB_EXPORT at::Tensor mcmc_sample(const at::Tensor weights, const int64_t n_samples,
                                  const c10::optional<at::Tensor> n_samples_dev, const c10::optional<at::Tensor> uniforms,
                                  const bool weights_are_logits) {
    check_cuda(weights, at::kFloat, "weights");
    TORCH_CHECK(n_samples >= 0 && n_samples <= INT32_MAX, "n_samples out of range");
    const int64_t N = weights.numel();
    const c10::cuda::CUDAGuard guard(weights.device());
    Tensor samples = at::empty({n_samples}, weights.options().dtype(at::kInt));
    if (N == 0 || n_samples == 0) return samples;
    const double *u = nullptr;
    GsbPhilox ph{};
    if (uniforms.has_value() && uniforms->defined()) {
        check_cuda(*uniforms, at::kDouble, "uniforms");
        TORCH_CHECK(uniforms->numel() >= n_samples, "uniforms must hold n_samples values");
        u = uniforms->data_ptr<double>();
    } else {
        // torch's default CUDA generator: torch.manual_seed governs the draws, and under graph capture the seed and
        // offset are device pointers that each replay advances (Note [CUDA Graph-safe RNG states])
        auto *gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(
            c10::nullopt, at::cuda::detail::getDefaultCUDAGenerator(weights.device().index()));
        at::PhiloxCudaState st;
        {
            std::lock_guard<std::mutex> lock(gen->mutex_);
            st = gen->philox_cuda_state(4);
        }
        if (st.captured_) {
            ph.seed_ptr = reinterpret_cast<const uint64_t *>(st.seed_.ptr);
            ph.offset_ptr = st.offset_.ptr;
            ph.offset_intragraph = st.offset_intragraph_;
        } else {
            ph.seed = st.seed_.val;
            ph.offset = st.offset_.val;
        }
    }
    Tensor ws = workspace((uint32_t)N, weights);
    check(gsb_mcmc_sample((uint32_t)N, weights.data_ptr<float>(), weights_are_logits ? 1 : 0, (uint32_t)n_samples,
                          count_ptr(n_samples_dev), u, u ? nullptr : &ph, samples.data_ptr<int32_t>(), ws.data_ptr(),
                          (size_t)ws.numel(), cur_stream()),
          "gsb_mcmc_sample");
    return samples;
}

GSB_EXPORT void mcmc_relocate(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &exp_avg,
                              const std::vector<at::Tensor> &exp_avg_sq, const at::Tensor samples,
                              const at::Tensor dead_indices, const at::Tensor n_dead, const at::Tensor binoms,
                              const float min_opacity) {
    check_cuda(dead_indices, at::kInt, "dead_indices");
    TORCH_CHECK(params.size() == 6, "params must hold six tensors");
    const int64_t N = params[0].size(0);
    TORCH_CHECK(samples.numel() <= dead_indices.numel(), "dead_indices must hold one target per sample");
    apply(params, exp_avg, exp_avg_sq, N, samples, n_dead, dead_indices.data_ptr<int32_t>(), binoms, min_opacity);
}

GSB_EXPORT void mcmc_grow(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &exp_avg,
                          const std::vector<at::Tensor> &exp_avg_sq, const int64_t n_rows, const at::Tensor samples,
                          const at::Tensor binoms, const float min_opacity) {
    TORCH_CHECK(n_rows >= 0 && n_rows + samples.numel() <= UINT32_MAX, "n_rows out of range");
    apply(params, exp_avg, exp_avg_sq, n_rows, samples, c10::nullopt, nullptr, binoms, min_opacity);
}

GSB_EXPORT void mcmc_add_noise(const at::Tensor raw_opacities, const at::Tensor raw_scales, const at::Tensor raw_quats,
                               const at::Tensor noise, at::Tensor means, const at::Tensor lr, const float lr_scale) {
    for (const Tensor *t : std::initializer_list<const Tensor *>{&raw_opacities, &raw_scales, &raw_quats, &noise, &means, &lr})
        check_cuda(*t, at::kFloat, "add_noise argument");
    const int64_t N = means.size(0);
    TORCH_CHECK(means.numel() == 3 * N && noise.numel() == 3 * N && raw_scales.numel() == 3 * N &&
                    raw_quats.numel() == 4 * N && raw_opacities.numel() == N && lr.numel() >= 1,
                "add_noise: means/noise/scales [N,3], quats [N,4], opacities [N], lr a device scalar");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(raw_quats.data_ptr()) & 15) == 0, "raw_quats must be 16-byte aligned");
    const c10::cuda::CUDAGuard guard(means.device());
    check(gsb_mcmc_add_noise((uint32_t)N, raw_opacities.data_ptr<float>(), raw_scales.data_ptr<float>(),
                             raw_quats.data_ptr<float>(), noise.data_ptr<float>(), means.data_ptr<float>(),
                             lr.data_ptr<float>(), lr_scale, cur_stream()),
          "gsb_mcmc_add_noise");
}

GSB_EXPORT at::Tensor mcmc_regularize(const at::Tensor scaling_raw, const at::Tensor opacity_raw, const float scale_reg,
                                      const float opacity_reg, c10::optional<at::Tensor> v_scaling,
                                      c10::optional<at::Tensor> v_opacity) {
    check_cuda(scaling_raw, at::kFloat, "scaling_raw");
    check_cuda(opacity_raw, at::kFloat, "opacity_raw");
    const int64_t N = opacity_raw.numel();
    TORCH_CHECK(scaling_raw.numel() == 3 * N, "scaling_raw must be [N,3]");
    const c10::cuda::CUDAGuard guard(opacity_raw.device());
    Tensor loss = at::zeros({2}, opacity_raw.options());
    float *vs = nullptr, *vo = nullptr;
    if (v_scaling.has_value() && v_scaling->defined()) {
        check_cuda(*v_scaling, at::kFloat, "v_scaling");
        TORCH_CHECK(v_scaling->numel() == 3 * N, "v_scaling must be shaped like scaling_raw");
        vs = v_scaling->data_ptr<float>();
    }
    if (v_opacity.has_value() && v_opacity->defined()) {
        check_cuda(*v_opacity, at::kFloat, "v_opacity");
        TORCH_CHECK(v_opacity->numel() == N, "v_opacity must be shaped like opacity_raw");
        vo = v_opacity->data_ptr<float>();
    }
    if (N == 0) return loss;
    Tensor ws = workspace((uint32_t)N, opacity_raw);
    check(gsb_mcmc_regularize((uint32_t)N, scaling_raw.data_ptr<float>(), opacity_raw.data_ptr<float>(), scale_reg,
                              opacity_reg, vs, vo, loss.data_ptr<float>(), ws.data_ptr(), (size_t)ws.numel(),
                              cur_stream()),
          "gsb_mcmc_regularize");
    return loss;
}

} // namespace gsplat

namespace {

std::tuple<Tensor, Tensor, Tensor> dead_op(const Tensor &opacity_raw, const Tensor &rotation_raw, double min_opacity) {
    return gsplat::mcmc_dead(opacity_raw, rotation_raw, (float)min_opacity);
}
Tensor sample_op(const Tensor &weights, int64_t n_samples, const c10::optional<Tensor> &n_samples_dev,
                 const c10::optional<Tensor> &uniforms, bool weights_are_logits) {
    return gsplat::mcmc_sample(weights, n_samples, n_samples_dev, uniforms, weights_are_logits);
}
void relocate_op(std::vector<Tensor> params, std::vector<Tensor> exp_avg, std::vector<Tensor> exp_avg_sq,
                 const Tensor &samples, const Tensor &dead_indices, const Tensor &n_dead, const Tensor &binoms,
                 double min_opacity) {
    gsplat::mcmc_relocate(params, exp_avg, exp_avg_sq, samples, dead_indices, n_dead, binoms, (float)min_opacity);
}
void grow_op(std::vector<Tensor> params, std::vector<Tensor> exp_avg, std::vector<Tensor> exp_avg_sq, int64_t n_rows,
             const Tensor &samples, const Tensor &binoms, double min_opacity) {
    gsplat::mcmc_grow(params, exp_avg, exp_avg_sq, n_rows, samples, binoms, (float)min_opacity);
}
void noise_op(const Tensor &raw_opacities, const Tensor &raw_scales, const Tensor &raw_quats, const Tensor &noise,
              Tensor means, const Tensor &lr, double lr_scale) {
    gsplat::mcmc_add_noise(raw_opacities, raw_scales, raw_quats, noise, means, lr, (float)lr_scale);
}
Tensor regularize_op(const Tensor &scaling_raw, const Tensor &opacity_raw, double scale_reg, double opacity_reg,
                     c10::optional<Tensor> v_scaling, c10::optional<Tensor> v_opacity) {
    return gsplat::mcmc_regularize(scaling_raw, opacity_raw, (float)scale_reg, (float)opacity_reg, v_scaling, v_opacity);
}

} // namespace

TORCH_LIBRARY_FRAGMENT(gsplat_b200, m) {
    m.def("mcmc_dead(Tensor opacity_raw, Tensor rotation_raw, float min_opacity) -> (Tensor, Tensor, Tensor)", &dead_op);
    m.def("mcmc_sample(Tensor weights, int n_samples, Tensor? n_samples_dev, Tensor? uniforms, bool weights_are_logits) "
          "-> Tensor",
          &sample_op);
    m.def("mcmc_relocate(Tensor(a!)[] params, Tensor(b!)[] exp_avg, Tensor(c!)[] exp_avg_sq, Tensor samples, "
          "Tensor dead_indices, Tensor n_dead, Tensor binoms, float min_opacity) -> ()",
          &relocate_op);
    m.def("mcmc_grow(Tensor(a!)[] params, Tensor(b!)[] exp_avg, Tensor(c!)[] exp_avg_sq, int n_rows, Tensor samples, "
          "Tensor binoms, float min_opacity) -> ()",
          &grow_op);
    m.def("mcmc_add_noise(Tensor raw_opacities, Tensor raw_scales, Tensor raw_quats, Tensor noise, Tensor(a!) means, "
          "Tensor lr, float lr_scale) -> ()",
          &noise_op);
    m.def("mcmc_regularize(Tensor scaling_raw, Tensor opacity_raw, float scale_reg, float opacity_reg, "
          "Tensor(a!)? v_scaling, Tensor(b!)? v_opacity) -> Tensor",
          &regularize_op);
}
