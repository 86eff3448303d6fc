// gsb_optim.cu -- SURVEY.md 8(f3): the optimizer step of the training iteration, all parameter groups in ONE launch.
//
// The reference steps Adam with one kernel launch per parameter tensor (six per iteration, scalar 4-byte accesses:
// fastgs/optimizer/include/adam_kernels.cuh:13-36 driven by src/training/optimizers/fused_adam.cpp:22-95).  The
// update is a pure stream -- read param / grad / exp_avg / exp_avg_sq, write param / exp_avg / exp_avg_sq:
// 28 B per element, 1.65 GB per step at 1 M Gaussians -- so this version walks all groups in a single grid with
// 128-bit accesses.  The arithmetic is the reference kernel's, operation for operation (float32).
#include "gsb_common.cuh"

namespace gsb {

constexpr int kAdamThreads = 256;
constexpr int kAdamMaxGroups = 8;

struct AdamGroupDev {
    float *param, *exp_avg, *exp_avg_sq;
    const float *grad;
    unsigned long long n;          // elements
    unsigned long long chunk_end;  // cumulative number of 4-element chunks up to and including this group
    float lr, beta1, beta2, eps, bc1_rcp, bc2_sqrt_rcp;
    int vec;                       // all four pointers 16-byte aligned
};
struct AdamArgs {
    AdamGroupDev g[kAdamMaxGroups];
    int n_groups;
    const float *dyn; // optional DEVICE array [n_groups][4] = (lr, bias_correction1_rcp, bias_correction2_sqrt_rcp, enabled)
};

__device__ __forceinline__ void adam_one(float &p, float &m, float &v, float grad, const AdamGroupDev &g) {
    const float moment1 = g.beta1 * m + (1.0f - g.beta1) * grad;
    const float moment2 = g.beta2 * v + (1.0f - g.beta2) * grad * grad;
    const float denom = sqrtf(moment2) * g.bc2_sqrt_rcp + g.eps;
    const float step_size = g.lr * g.bc1_rcp;
    p -= step_size * moment1 / denom;
    m = moment1;
    v = moment2;
}

__global__ void __launch_bounds__(kAdamThreads) adam_multi_kernel(const AdamArgs a) {
    const unsigned long long c = (unsigned long long)blockIdx.x * kAdamThreads + threadIdx.x;
    int gi = 0;
    unsigned long long base = 0;
    while (gi < a.n_groups && c >= a.g[gi].chunk_end) { base = a.g[gi].chunk_end; ++gi; }
    if (gi >= a.n_groups) return;
    AdamGroupDev g = a.g[gi];
    if (a.dyn) { // step-dependent scalars come from device memory: the launch can be replayed from a CUDA graph
        const float4 d = reinterpret_cast<const float4 *>(a.dyn)[gi];
        if (d.w == 0.0f) return;
        g.lr = d.x; g.bc1_rcp = d.y; g.bc2_sqrt_rcp = d.z;
    }
    const unsigned long long e0 = (c - base) * 4ull;
    if (e0 + 4 <= g.n && g.vec) {
        float4 p = reinterpret_cast<float4 *>(g.param)[c - base];
        float4 m = reinterpret_cast<float4 *>(g.exp_avg)[c - base];
        float4 v = reinterpret_cast<float4 *>(g.exp_avg_sq)[c - base];
        const float4 gr = reinterpret_cast<const float4 *>(g.grad)[c - base];
        adam_one(p.x, m.x, v.x, gr.x, g); adam_one(p.y, m.y, v.y, gr.y, g);
        adam_one(p.z, m.z, v.z, gr.z, g); adam_one(p.w, m.w, v.w, gr.w, g);
        reinterpret_cast<float4 *>(g.param)[c - base] = p;
        reinterpret_cast<float4 *>(g.exp_avg)[c - base] = m;
        reinterpret_cast<float4 *>(g.exp_avg_sq)[c - base] = v;
    } else {
        for (unsigned long long e = e0; e < e0 + 4 && e < g.n; ++e) {
            float p = g.param[e], m = g.exp_avg[e], v = g.exp_avg_sq[e];
            adam_one(p, m, v, g.grad[e], g);
            g.param[e] = p; g.exp_avg[e] = m; g.exp_avg_sq[e] = v;
        }
    }
}

} // namespace gsb

extern "C" int gsb_adam_step_dynamic(const GsbAdamGroup *groups, uint32_t n_groups, const float *dynamic_scalars,
                                     gsb_stream_t stream);

extern "C" int gsb_adam_step(const GsbAdamGroup *groups, uint32_t n_groups, gsb_stream_t stream) {
    return gsb_adam_step_dynamic(groups, n_groups, nullptr, stream);
}

extern "C" int gsb_adam_step_dynamic(const GsbAdamGroup *groups, uint32_t n_groups, const float *dynamic_scalars,
                                     gsb_stream_t stream) {
    using namespace gsb;
    if (n_groups == 0) return GSB_OK;
    if (!groups || n_groups > (uint32_t)kAdamMaxGroups) return GSB_E_INVALID;
    if (reinterpret_cast<uintptr_t>(dynamic_scalars) & 15) return GSB_E_INVALID;
    AdamArgs a;
    a.dyn = dynamic_scalars;
    a.n_groups = 0;
    unsigned long long chunks = 0;
    for (uint32_t i = 0; i < n_groups; ++i) {
        const GsbAdamGroup &g = groups[i];
        if (g.n == 0 && !dynamic_scalars) continue; // (with dynamic scalars the group index must stay aligned)
        // an empty tensor has no storage: a zero-size group kept for its row of the scalar table may hold null pointers
        if (g.n && (!g.param || !g.grad || !g.exp_avg || !g.exp_avg_sq)) return GSB_E_INVALID;
        AdamGroupDev &d = a.g[a.n_groups++];
        d.param = g.param; d.grad = g.grad; d.exp_avg = g.exp_avg; d.exp_avg_sq = g.exp_avg_sq;
        d.n = g.n;
        chunks += (g.n + 3) / 4;
        d.chunk_end = chunks;
        d.lr = g.lr; d.beta1 = g.beta1; d.beta2 = g.beta2; d.eps = g.eps;
        d.bc1_rcp = g.bias_correction1_rcp; d.bc2_sqrt_rcp = g.bias_correction2_sqrt_rcp;
        const uintptr_t bits = reinterpret_cast<uintptr_t>(g.param) | reinterpret_cast<uintptr_t>(g.grad) |
                               reinterpret_cast<uintptr_t>(g.exp_avg) | reinterpret_cast<uintptr_t>(g.exp_avg_sq);
        d.vec = (bits & 15) == 0 ? 1 : 0;
    }
    if (chunks == 0) return GSB_OK;
    if ((chunks + kAdamThreads - 1) / kAdamThreads > 0x7fffffffull) return GSB_E_INVALID;
    cudaStream_t s = as_stream(stream);
    {
        ProfScope ps("adam_step", s);
        adam_multi_kernel<<<(unsigned)((chunks + kAdamThreads - 1) / kAdamThreads), kAdamThreads, 0, s>>>(a);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
