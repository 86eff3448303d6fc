// SplatRows.h -- the six raw SplatData tensors and their Adam moments as a GsbMcmcRows (gsb200.h), shared by the
// densification strategies' operators (Mcmc.cpp, Adc.cpp).
#pragma once

#include <ATen/core/Tensor.h>

#include <vector>

#include "gsb200.h"

namespace gsb_shim {

using at::Tensor;

inline void check_cuda(const Tensor &t, at::ScalarType type, const char *name) {
    TORCH_CHECK(t.defined() && t.is_cuda(), name, " must be a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == type, name, " has the wrong dtype");
    TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}

const char *const kGroups[6] = {"means", "sh0", "shN", "scaling_raw", "rotation_raw", "opacity_raw"};
const int64_t kWidth[6] = {3, 3, -1, 3, 4, 1}; // floats per row; shN: any multiple of 3

// rows: the tensors must hold at least `rows` rows
inline GsbMcmcRows make_rows(const std::vector<Tensor> &params, const std::vector<Tensor> &exp_avg,
                      const std::vector<Tensor> &exp_avg_sq, int64_t rows) {
    TORCH_CHECK(params.size() == 6, "params must be the six SplatData tensors (means, sh0, shN, scaling_raw, "
                                    "rotation_raw, opacity_raw)");
    TORCH_CHECK(exp_avg.empty() || exp_avg.size() == 6, "exp_avg must be empty or hold six tensors");
    TORCH_CHECK(exp_avg_sq.size() == exp_avg.size(), "exp_avg_sq must match exp_avg");
    GsbMcmcRows r{};
    float *p[6];
    for (int g = 0; g < 6; ++g) {
        const Tensor &t = params[g];
        check_cuda(t, at::kFloat, kGroups[g]);
        TORCH_CHECK(t.dim() >= 1 && t.size(0) >= rows, kGroups[g], " must hold ", rows, " rows");
        const int64_t w = t.size(0) ? t.numel() / t.size(0) : 0;
        TORCH_CHECK(kWidth[g] < 0 ? w % 3 == 0 : w == kWidth[g], kGroups[g], " has the wrong row width");
        p[g] = t.numel() ? t.data_ptr<float>() : nullptr;
        if (!exp_avg.empty()) {
            for (const Tensor *m : {&exp_avg[g], &exp_avg_sq[g]}) {
                check_cuda(*m, at::kFloat, "Adam moment");
                TORCH_CHECK(m->numel() == 0 || m->numel() == t.numel(), "the moments of ", kGroups[g],
                            " must have its number of elements");
            }
            r.exp_avg[g] = exp_avg[g].numel() ? exp_avg[g].data_ptr<float>() : nullptr;
            r.exp_avg_sq[g] = exp_avg_sq[g].numel() ? exp_avg_sq[g].data_ptr<float>() : nullptr;
        }
    }
    TORCH_CHECK((reinterpret_cast<uintptr_t>(p[4]) & 15) == 0, "rotation_raw must be 16-byte aligned");
    r.means = p[0]; r.sh0 = p[1]; r.shN = p[2]; r.scaling_raw = p[3]; r.rotation_raw = p[4]; r.opacity_raw = p[5];
    r.shN_rows = params[2].size(0) ? (uint32_t)(params[2].numel() / params[2].size(0) / 3) : 0;
    if (!r.shN_rows) r.shN = nullptr;
    return r;
}

} // namespace gsb_shim
