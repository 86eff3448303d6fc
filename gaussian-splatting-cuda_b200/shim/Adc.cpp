// Adc.cpp -- adaptive density control, the reference's default strategy (default_strategy.cpp:164-290), on this
// library's kernels (csrc/gsb_adc.cu): extended operators over the raw SplatData tensors and their Adam moments
// (FusedOps.h), registered as torch.ops.gsplat_b200.adc_* for the Python strategy (adc.py).
//
//   adc_classify -> (counts, workspace): counts stay on the device; the caller reads them back once to size the output
//   adc_apply    -> the final parameters, moments and zeroed statistics in freshly allocated exact-size tensors
//   adc_reset_opacity: in place
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

GsbAdcParams adc_params(float grad_threshold, float grow_scale3d, float prune_scale3d, float scene_scale,
                        float prune_opacity, bool prune_too_big, bool revised_opacity) {
    GsbAdcParams p;
    p.grad_threshold = grad_threshold;
    p.grow_scale3d = grow_scale3d;
    p.prune_scale3d = prune_scale3d;
    p.scene_scale = scene_scale;
    p.prune_opacity = prune_opacity;
    p.prune_too_big = prune_too_big ? 1 : 0;
    p.revised_opacity = revised_opacity ? 1 : 0;
    return p;
}

std::vector<Tensor> like_rows(const std::vector<Tensor> &ts, int64_t rows) {
    std::vector<Tensor> out;
    out.reserve(ts.size());
    for (const Tensor &t : ts) {
        std::vector<int64_t> shape = t.sizes().vec();
        shape[0] = rows;
        out.push_back(at::empty(shape, t.options()));
    }
    return out;
}

} // namespace

namespace gsplat {

GSB_EXPORT std::tuple<at::Tensor, at::Tensor>
adc_classify(const at::Tensor densification_info, const at::Tensor scaling_raw, const at::Tensor rotation_raw,
             const at::Tensor opacity_raw, const float grad_threshold, const float grow_scale3d,
             const float prune_scale3d, const float scene_scale, const float prune_opacity, const bool prune_too_big,
             const bool revised_opacity) {
    check_cuda(scaling_raw, at::kFloat, "scaling_raw");
    check_cuda(rotation_raw, at::kFloat, "rotation_raw");
    check_cuda(opacity_raw, at::kFloat, "opacity_raw");
    const int64_t N = rotation_raw.size(0);
    TORCH_CHECK(rotation_raw.numel() == 4 * N && scaling_raw.numel() == 3 * N && opacity_raw.numel() == N,
                "scaling_raw [N,3], rotation_raw [N,4], opacity_raw [N] / [N,1]");
    TORCH_CHECK(N <= INT32_MAX / 2, "adc_classify: at most INT32_MAX / 2 rows");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(rotation_raw.data_ptr()) & 15) == 0, "rotation_raw must be 16-byte aligned");
    const float *info = nullptr;
    if (densification_info.defined() && densification_info.numel() > 0) {
        check_cuda(densification_info, at::kFloat, "densification_info");
        TORCH_CHECK(densification_info.numel() == 2 * N, "densification_info must be [2, N]");
        info = densification_info.data_ptr<float>();
    }
    const c10::cuda::CUDAGuard guard(opacity_raw.device());
    Tensor counts = at::empty({8}, opacity_raw.options().dtype(at::kInt));
    Tensor ws = at::empty({(int64_t)gsb_adc_workspace((uint32_t)N)}, opacity_raw.options().dtype(at::kByte));
    const GsbAdcParams p = adc_params(grad_threshold, grow_scale3d, prune_scale3d, scene_scale, prune_opacity,
                                      prune_too_big, revised_opacity);
    check(gsb_adc_classify((uint32_t)N, info, N ? scaling_raw.data_ptr<float>() : nullptr,
                           N ? rotation_raw.data_ptr<float>() : nullptr, N ? opacity_raw.data_ptr<float>() : nullptr,
                           &p, counts.data_ptr<int32_t>(), ws.data_ptr(), (size_t)ws.numel(), cur_stream()),
          "gsb_adc_classify");
    return std::make_tuple(counts, ws);
}

GSB_EXPORT std::tuple<std::vector<at::Tensor>, std::vector<at::Tensor>, std::vector<at::Tensor>, at::Tensor>
adc_apply(const std::vector<at::Tensor> &params, const std::vector<at::Tensor> &exp_avg,
          const std::vector<at::Tensor> &exp_avg_sq, const at::Tensor workspace, const at::Tensor counts,
          const int64_t n_split, const int64_t n_final, const c10::optional<at::Tensor> z, const bool revised_opacity) {
    TORCH_CHECK(params.size() == 6, "params must hold six tensors");
    const int64_t N = params[0].size(0);
    check_cuda(counts, at::kInt, "counts");
    TORCH_CHECK(counts.numel() == 8, "counts must be adc_classify's [8]");
    check_cuda(workspace, at::kByte, "workspace");
    TORCH_CHECK(n_split >= 0 && n_split <= N && n_final >= 0 && n_final <= 2 * N, "n_split / n_final out of range");
    const float *zp = nullptr;
    if (n_split > 0) {
        TORCH_CHECK(z.has_value() && z->defined(), "z [2, n_split, 3] is needed when rows are split");
        check_cuda(*z, at::kFloat, "z");
        TORCH_CHECK(z->numel() == 6 * n_split, "z must be [2, n_split, 3]");
        zp = z->data_ptr<float>();
    }
    const c10::cuda::CUDAGuard guard(counts.device());
    std::vector<Tensor> np = like_rows(params, n_final), m1 = like_rows(exp_avg, n_final),
                        m2 = like_rows(exp_avg_sq, n_final);
    Tensor info = at::empty({2, n_final}, params[0].options());
    if (n_final == 0) return std::make_tuple(np, m1, m2, info); // everything pruned
    const GsbMcmcRows src = make_rows(params, exp_avg, exp_avg_sq, N);
    const GsbMcmcRows dst = make_rows(np, m1, m2, n_final);
    GsbAdcParams p = adc_params(0.f, 0.f, 0.f, 0.f, 0.f, false, revised_opacity);
    check(gsb_adc_apply((uint32_t)N, &src, &dst, (uint32_t)n_split, (uint32_t)n_final, zp, &p,
                        counts.data_ptr<int32_t>(), info.data_ptr<float>(), workspace.data_ptr(),
                        (size_t)workspace.numel(), cur_stream()),
          "gsb_adc_apply");
    return std::make_tuple(np, m1, m2, info);
}

GSB_EXPORT void adc_reset_opacity(at::Tensor opacity_raw, c10::optional<at::Tensor> exp_avg,
                                  c10::optional<at::Tensor> exp_avg_sq, const float prune_opacity) {
    check_cuda(opacity_raw, at::kFloat, "opacity_raw");
    const int64_t N = opacity_raw.numel();
    float *m[2] = {nullptr, nullptr};
    int k = 0;
    for (c10::optional<at::Tensor> *t : {&exp_avg, &exp_avg_sq}) {
        if (t->has_value() && (*t)->defined()) {
            check_cuda(**t, at::kFloat, "opacity moment");
            TORCH_CHECK((*t)->numel() == N, "the opacity moments must have opacity_raw's number of elements");
            m[k] = N ? (*t)->data_ptr<float>() : nullptr;
        }
        ++k;
    }
    if (N == 0) return;
    const c10::cuda::CUDAGuard guard(opacity_raw.device());
    check(gsb_adc_reset_opacity((uint32_t)N, opacity_raw.data_ptr<float>(), prune_opacity, m[0], m[1], cur_stream()),
          "gsb_adc_reset_opacity");
}

} // namespace gsplat

namespace {

std::tuple<Tensor, Tensor> classify_op(const c10::optional<Tensor> &info, const Tensor &scaling_raw,
                                       const Tensor &rotation_raw, const Tensor &opacity_raw, double grad_threshold,
                                       double grow_scale3d, double prune_scale3d, double scene_scale,
                                       double prune_opacity, bool prune_too_big, bool revised_opacity) {
    return gsplat::adc_classify(info.has_value() ? *info : Tensor(), scaling_raw, rotation_raw, opacity_raw,
                                (float)grad_threshold, (float)grow_scale3d, (float)prune_scale3d, (float)scene_scale,
                                (float)prune_opacity, prune_too_big, revised_opacity);
}
std::tuple<std::vector<Tensor>, std::vector<Tensor>, std::vector<Tensor>, Tensor>
apply_op(std::vector<Tensor> params, std::vector<Tensor> exp_avg, std::vector<Tensor> exp_avg_sq, const Tensor &workspace,
         const Tensor &counts, int64_t n_split, int64_t n_final, const c10::optional<Tensor> &z, bool revised_opacity) {
    return gsplat::adc_apply(params, exp_avg, exp_avg_sq, workspace, counts, n_split, n_final, z, revised_opacity);
}
void reset_op(Tensor opacity_raw, c10::optional<Tensor> exp_avg, c10::optional<Tensor> exp_avg_sq,
              double prune_opacity) {
    gsplat::adc_reset_opacity(opacity_raw, exp_avg, exp_avg_sq, (float)prune_opacity);
}

} // namespace

TORCH_LIBRARY_FRAGMENT(gsplat_b200, m) {
    m.def("adc_classify(Tensor? densification_info, Tensor scaling_raw, Tensor rotation_raw, Tensor opacity_raw, "
          "float grad_threshold, float grow_scale3d, float prune_scale3d, float scene_scale, float prune_opacity, "
          "bool prune_too_big, bool revised_opacity) -> (Tensor, Tensor)",
          &classify_op);
    m.def("adc_apply(Tensor[] params, Tensor[] exp_avg, Tensor[] exp_avg_sq, Tensor workspace, Tensor counts, "
          "int n_split, int n_final, Tensor? z, bool revised_opacity) -> (Tensor[], Tensor[], Tensor[], Tensor)",
          &apply_op);
    m.def("adc_reset_opacity(Tensor(a!) opacity_raw, Tensor(b!)? exp_avg, Tensor(c!)? exp_avg_sq, "
          "float prune_opacity) -> ()",
          &reset_op);
}
