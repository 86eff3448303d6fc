// gsb_mcmc.cu -- SURVEY.md 8 f6: the MCMC densification strategy's refine on the device
// (src/training/strategies/mcmc.cpp:112-347 relocate_gs / add_new_gs, trainer.cpp:132-158 regularisers).
//
//   gsb_mcmc_dead        dead mask (sigmoid(opacity_raw) <= min_opacity or |rotation_raw|^2 < 1e-8, IEEE expf as torch
//                        computes it), the ascending dead indices by a scan of the flags, their count on the device and
//                        the sampling weights (opacity where alive, 0 where dead).  20 B read per Gaussian.
//   gsb_mcmc_sample      weighted draw with replacement: float64 inclusive prefix C of the weights, sample j takes the
//                        first i with C[i] > u_j * C[N-1] (moved to the nearest positive weight should rounding of the
//                        prefix leave a gap at a zero weight).  A zero weight is never drawn, and drawing over all N
//                        Gaussians with zero weights on the dead ones selects the same Gaussian as drawing over the
//                        compacted alive list that mcmc.cpp builds, so no alive compaction is needed.  u_j comes from
//                        torch's Philox state (seed / offset, possibly device pointers under graph capture) or from
//                        the caller.  Works for any N (the reference falls back to a host loop above 2^24).
//   gsb_mcmc_apply       relocation (targets = dead indices) or growth (targets = N + j): per-index copy counts with
//                        integer atomics, ratio = min(count + 1, n_max), relocation_one, clamp, logit / log, written to
//                        the target row together with copies of means, sh0, shN and rotation; Adam moments zeroed at
//                        the sampled rows (relocation) or the new rows (growth).  The sampled rows receive their new
//                        opacity and scale in a second launch: a sample drawn twice would otherwise let one thread
//                        read a row another thread has already rewritten.
//   gsb_mcmc_regularize  scale_reg * mean(exp(scaling_raw)) and opacity_reg * mean(sigmoid(opacity_raw)): gradients
//                        added into the caller's tensors, losses reduced deterministically (per-CTA partials, the last
//                        CTA sums them in a fixed order).
// Nothing here reads a device value on the host: the dead count and the sample count stay in device memory.
#include <curand_kernel.h>

#include "gsb_common.cuh"
#include "gsb_devsort.cuh"
#include "gsb_relocation.cuh"

namespace gsb {

constexpr int kMcmcThreads = 256;
constexpr uint32_t kMcmcScanBlocks = 264; // two CTAs of 1024 threads per SM of an H100 SXM
constexpr uint32_t kRegBlocks = 128;

struct McmcWs {
    unsigned int *done; // regulariser ticket
    void *bsum;         // [kMcmcScanBlocks] 8-byte block sums / [2 kRegBlocks] regulariser partials
    void *rows;         // 8 N bytes: flags + ranks, the float64 prefix, or the copy counts
};

static size_t mcmc_ws_bytes(uint32_t N) { return 256 + (size_t)kMcmcScanBlocks * 8 + (size_t)N * 8; }

static int mcmc_ws(uint32_t N, void *workspace, size_t bytes, McmcWs &w) {
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || bytes < mcmc_ws_bytes(N)) return GSB_E_WORKSPACE;
    char *b = static_cast<char *>(workspace);
    w.done = reinterpret_cast<unsigned int *>(b);
    w.bsum = b + 256;
    w.rows = b + 256 + (size_t)kMcmcScanBlocks * 8;
    return GSB_OK;
}

struct ScanPlan {
    uint32_t nblocks, seg;
};
static ScanPlan scan_plan(uint64_t n) {
    uint64_t nb = (n + 4095) / 4096;
    if (nb < 1) nb = 1;
    if (nb > kMcmcScanBlocks) nb = kMcmcScanBlocks;
    return {(uint32_t)nb, (uint32_t)((n + nb - 1) / nb)};
}

// torch's sigmoid for float (1 / (1 + exp(-x)) with the IEEE expf, not __expf)
__device__ __forceinline__ float sigmoid_ieee(float x) { return 1.0f / (1.0f + expf(-x)); }

// ---- dead mask and compaction -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMcmcThreads) mcmc_mask_kernel(uint32_t N, const float *__restrict__ opacity_raw,
                                                                 const float *__restrict__ rotation_raw,
                                                                 float min_opacity, int32_t *__restrict__ flags,
                                                                 float *__restrict__ weights) {
    const uint32_t i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= N) return;
    const float op = sigmoid_ieee(opacity_raw[i]);
    const float4 q = reinterpret_cast<const float4 *>(rotation_raw)[i];
    const float q2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    const bool dead = op <= min_opacity || q2 < 1e-8f;
    flags[i] = dead ? 1 : 0;
    weights[i] = dead ? 0.f : op;
}

__global__ void __launch_bounds__(kMcmcThreads) mcmc_compact_kernel(uint32_t N, const int32_t *__restrict__ flags,
                                                                    const int32_t *__restrict__ ranks,
                                                                    int32_t *__restrict__ dead_idx,
                                                                    uint32_t *__restrict__ n_dead) {
    const uint32_t i = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (i >= N) return;
    if (flags[i]) dead_idx[ranks[i] - 1] = (int32_t)i;
    if (i == N - 1) *n_dead = (uint32_t)ranks[i];
}

// ---- weighted sampling with replacement ---------------------------------------------------------------------------
struct LoadWeight {
    const float *w;
    bool logits;
    __device__ __forceinline__ double operator()(uint64_t i) const {
        const float x = w[i];
        return (double)(logits ? sigmoid_ieee(x) : x);
    }
};

// 53 random bits -> [0, 1).  Thread j uses Philox subsequence j at the caller's offset (4 32-bit values per thread,
// torch's convention for philox_cuda_state(4)).
__device__ __forceinline__ double philox_uniform(const GsbPhilox &p, uint64_t j) {
    const uint64_t seed = p.seed_ptr ? *p.seed_ptr : p.seed;
    const uint64_t offset = p.offset_ptr ? (uint64_t)*p.offset_ptr + p.offset_intragraph : p.offset;
    curandStatePhilox4_32_10_t st;
    curand_init(seed, j, offset, &st);
    const uint4 r = curand4(&st);
    return ((double)(r.x >> 5) * 67108864.0 + (double)(r.y >> 6)) * (1.0 / 9007199254740992.0);
}

__global__ void __launch_bounds__(kMcmcThreads) mcmc_draw_kernel(uint32_t N, const double *__restrict__ prefix,
                                                                 const LoadWeight load, uint32_t n_samples,
                                                                 const uint32_t *__restrict__ n_dev,
                                                                 const double *__restrict__ uniforms, GsbPhilox philox,
                                                                 int32_t *__restrict__ samples) {
    const uint32_t j = blockIdx.x * kMcmcThreads + threadIdx.x;
    if (j >= n_samples || (n_dev && j >= *n_dev)) return;
    const double total = prefix[N - 1];
    if (!(total > 0.0)) { // nothing to draw from (no alive Gaussian): the apply skips the sample
        samples[j] = -1;
        return;
    }
    const double u = uniforms ? uniforms[j] : philox_uniform(philox, j);
    double t = u * total;
    if (!(t < total)) t = nextafter(total, 0.0); // u * total rounded up to total: keep the last positive weight
    uint32_t lo = 0, hi = N - 1; // first i with prefix[i] > t; prefix[N-1] > t holds
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (prefix[mid] > t) hi = mid;
        else lo = mid + 1;
    }
    // The prefix of a block starts from a carry summed in another order than the previous block's own prefix, so at a
    // block boundary it may step up by an ulp at a zero weight; a draw landing in that gap (~2^-53) moves to the
    // nearest positive weight, so that a dead row is never drawn (it would be both a sample and a target).
    while (lo + 1 < N && !(load(lo) > 0.0)) ++lo;
    while (lo > 0 && !(load(lo) > 0.0)) --lo;
    samples[j] = (int32_t)lo;
}

// ---- relocation / growth ------------------------------------------------------------------------------------------
struct ApplyArgs {
    GsbMcmcRows r;
    uint32_t N, n_samples;
    const uint32_t *n_dev;    // nullable
    const int32_t *samples;
    const int32_t *targets;   // null: growth, target N + j
    const float *binoms;
    int32_t n_max;
    float min_opacity;
    int32_t *counts;          // [N], zeroed before the count launch
};

__device__ __forceinline__ bool apply_sample(const ApplyArgs &a, uint32_t j, int32_t &s, uint32_t &t) {
    if (j >= a.n_samples || (a.n_dev && j >= *a.n_dev)) return false;
    s = a.samples[j];
    if (s < 0) return false;
    t = a.targets ? (uint32_t)a.targets[j] : a.N + j;
    return true;
}

__global__ void __launch_bounds__(kMcmcThreads) mcmc_count_kernel(const ApplyArgs a) {
    const uint32_t j = blockIdx.x * kMcmcThreads + threadIdx.x;
    int32_t s;
    uint32_t t;
    if (apply_sample(a, j, s, t)) atomicAdd(&a.counts[s], 1);
}

__device__ __forceinline__ void zero_row(float *m, size_t row, int width) {
    if (!m) return;
    for (int k = 0; k < width; ++k) m[row * width + k] = 0.f;
}

__global__ void __launch_bounds__(kMcmcThreads) mcmc_apply_kernel(const ApplyArgs a) {
    const uint32_t j = blockIdx.x * kMcmcThreads + threadIdx.x;
    int32_t si;
    uint32_t t;
    if (!apply_sample(a, j, si, t)) return;
    const size_t s = (size_t)si;
    const GsbMcmcRows &r = a.r;
    int copies = a.counts[s] + 1;
    if (copies > a.n_max) copies = a.n_max;
    // mcmc.cpp:147-167 (relocate_gs) / :225-245 (add_new_gs)
    float o_new;
    const float grow = relocation_one(sigmoid_ieee(r.opacity_raw[s]), copies, a.binoms, a.n_max, &o_new);
    const float hi = 1.0f - 1e-7f;
    o_new = o_new < a.min_opacity ? a.min_opacity : (o_new > hi ? hi : o_new); // torch::clamp, NaN kept
    r.opacity_raw[t] = logf(o_new / (1.0f - o_new));
#pragma unroll
    for (int k = 0; k < 3; ++k) r.scaling_raw[(size_t)t * 3 + k] = logf(grow * expf(r.scaling_raw[s * 3 + k]));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        r.means[(size_t)t * 3 + k] = r.means[s * 3 + k];
        r.sh0[(size_t)t * 3 + k] = r.sh0[s * 3 + k];
    }
    reinterpret_cast<float4 *>(r.rotation_raw)[t] = reinterpret_cast<const float4 *>(r.rotation_raw)[s];
    const size_t kn = (size_t)r.shN_rows * 3;
    for (size_t k = 0; k < kn; ++k) r.shN[(size_t)t * kn + k] = r.shN[s * kn + k];
    // moments: the sampled rows when relocating (update_optimizer_for_relocate, mcmc.cpp:84-109, leaves the dead rows'
    // moments as they were), the new rows when growing (zeros concatenated, :281-284)
    const size_t row = a.targets ? s : (size_t)t;
    const int width[6] = {3, 3, (int)kn, 3, 4, 1};
#pragma unroll
    for (int g = 0; g < 6; ++g) {
        zero_row(r.exp_avg[g], row, width[g]);
        zero_row(r.exp_avg_sq[g], row, width[g]);
    }
}

// the sampled row takes the opacity and scale its copies received (all copies of one sample hold the same values)
__global__ void __launch_bounds__(kMcmcThreads) mcmc_writeback_kernel(const ApplyArgs a) {
    const uint32_t j = blockIdx.x * kMcmcThreads + threadIdx.x;
    int32_t s;
    uint32_t t;
    if (!apply_sample(a, j, s, t)) return;
    const GsbMcmcRows &r = a.r;
    r.opacity_raw[s] = r.opacity_raw[t];
#pragma unroll
    for (int k = 0; k < 3; ++k) r.scaling_raw[(size_t)s * 3 + k] = r.scaling_raw[(size_t)t * 3 + k];
}

// ---- regularisers -------------------------------------------------------------------------------------------------
__device__ __forceinline__ double mcmc_block_sum(double v, double *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int k = 0; k < kMcmcThreads / 32; ++k) t += red[k]; // fixed order: deterministic
    return t;
}

struct RegArgs {
    uint32_t N;
    const float *scaling_raw, *opacity_raw;
    float *v_scaling, *v_opacity; // added into; null: that term is skipped
    float scale_reg, opacity_reg;
    float scale_g, opacity_g;     // scale_reg / (3N), opacity_reg / N: mean's backward as torch computes it
    float *loss_out;              // [2]
    double *partials;             // [gridDim.x][2]
    unsigned int *done;
};

__global__ void __launch_bounds__(kMcmcThreads) mcmc_regularize_kernel(const RegArgs a) {
    __shared__ double red[kMcmcThreads / 32];
    __shared__ bool last;
    float se = 0.f, so = 0.f;
    for (uint32_t i = blockIdx.x * kMcmcThreads + threadIdx.x; i < a.N; i += gridDim.x * kMcmcThreads) {
        if (a.v_scaling) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float e = expf(a.scaling_raw[(size_t)i * 3 + k]);
                a.v_scaling[(size_t)i * 3 + k] += a.scale_g * e; // exp backward: grad * result
                se += e;
            }
        }
        if (a.v_opacity) {
            const float sg = sigmoid_ieee(a.opacity_raw[i]);
            a.v_opacity[i] += a.opacity_g * (1.0f - sg) * sg; // sigmoid backward: grad * (1 - y) * y
            so += sg;
        }
    }
    const double be = mcmc_block_sum((double)se, red), bo = mcmc_block_sum((double)so, red);
    if (threadIdx.x == 0) {
        a.partials[2 * blockIdx.x] = be;
        a.partials[2 * blockIdx.x + 1] = bo;
        __threadfence();
        last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double te = 0.0, to = 0.0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += kMcmcThreads) {
        const volatile double *q = a.partials + 2 * b;
        te += q[0];
        to += q[1];
    }
    te = mcmc_block_sum(te, red);
    to = mcmc_block_sum(to, red);
    if (threadIdx.x == 0) {
        a.loss_out[0] = a.v_scaling ? (float)((double)a.scale_reg * te / (3.0 * (double)a.N)) : 0.f;
        a.loss_out[1] = a.v_opacity ? (float)((double)a.opacity_reg * to / (double)a.N) : 0.f;
    }
}

static unsigned blocks_for(uint64_t n) { return (unsigned)((n + kMcmcThreads - 1) / kMcmcThreads); }

} // namespace gsb

extern "C" size_t gsb_mcmc_workspace(uint32_t N) { return gsb::mcmc_ws_bytes(N); }

extern "C" int gsb_mcmc_dead(uint32_t N, const float *opacity_raw, const float *rotation_raw, float min_opacity,
                             int32_t *dead_idx, uint32_t *n_dead, float *weights, void *workspace,
                             size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (N == 0) return GSB_OK;
    if (!opacity_raw || !rotation_raw || !dead_idx || !n_dead || !weights) return GSB_E_INVALID;
    if (reinterpret_cast<uintptr_t>(rotation_raw) & 15) return GSB_E_INVALID;
    McmcWs w;
    if (int rc = mcmc_ws(N, workspace, workspace_bytes, w)) return rc;
    cudaStream_t s = as_stream(stream);
    int32_t *flags = static_cast<int32_t *>(w.rows);
    int32_t *ranks = flags + N;
    long long *bsum = static_cast<long long *>(w.bsum);
    ProfScope ps("mcmc_dead", s);
    mcmc_mask_kernel<<<blocks_for(N), kMcmcThreads, 0, s>>>(N, opacity_raw, rotation_raw, min_opacity, flags, weights);
    GSB_LAUNCH_CHECK();
    const ScanPlan sp = scan_plan(N);
    scan_blocksum_kernel<<<sp.nblocks, kSortThreads, 0, s>>>(LoadI32{flags}, N, sp.seg, bsum);
    GSB_LAUNCH_CHECK();
    scan_apply_kernel<<<sp.nblocks, kSortThreads, 0, s>>>(LoadI32{flags}, N, sp.seg, bsum, ranks);
    GSB_LAUNCH_CHECK();
    mcmc_compact_kernel<<<blocks_for(N), kMcmcThreads, 0, s>>>(N, flags, ranks, dead_idx, n_dead);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_mcmc_sample(uint32_t N, const float *weights, int weights_are_logits, uint32_t n_samples,
                               const uint32_t *n_samples_dev, const double *uniforms, const GsbPhilox *philox,
                               int32_t *samples, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (N == 0 || n_samples == 0) return GSB_OK;
    if (!weights || !samples || (!uniforms && !philox)) return GSB_E_INVALID;
    McmcWs w;
    if (int rc = mcmc_ws(N, workspace, workspace_bytes, w)) return rc;
    cudaStream_t s = as_stream(stream);
    double *prefix = static_cast<double *>(w.rows);
    double *bsum = static_cast<double *>(w.bsum);
    const LoadWeight load{weights, weights_are_logits != 0};
    const GsbPhilox ph = philox ? *philox : GsbPhilox{};
    ProfScope ps("mcmc_sample", s);
    const ScanPlan sp = scan_plan(N);
    scan_blocksum_kernel<<<sp.nblocks, kSortThreads, 0, s>>>(load, N, sp.seg, bsum);
    GSB_LAUNCH_CHECK();
    scan_apply_kernel<<<sp.nblocks, kSortThreads, 0, s>>>(load, N, sp.seg, bsum, prefix);
    GSB_LAUNCH_CHECK();
    mcmc_draw_kernel<<<blocks_for(n_samples), kMcmcThreads, 0, s>>>(N, prefix, load, n_samples, n_samples_dev, uniforms, ph,
                                                                    samples);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_mcmc_apply(uint32_t N, const GsbMcmcRows *rows, const int32_t *samples, uint32_t n_samples,
                              const uint32_t *n_samples_dev, const int32_t *targets, const float *binoms, int32_t n_max,
                              float min_opacity, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (N == 0 || n_samples == 0) return GSB_OK;
    if (!rows || !samples || !binoms || n_max < 1) return GSB_E_INVALID;
    const GsbMcmcRows &r = *rows;
    if (!r.means || !r.sh0 || !r.scaling_raw || !r.rotation_raw || !r.opacity_raw || (r.shN_rows && !r.shN))
        return GSB_E_INVALID;
    if (reinterpret_cast<uintptr_t>(r.rotation_raw) & 15) return GSB_E_INVALID;
    if (!targets && (uint64_t)N + n_samples > 0xffffffffull) return GSB_E_INVALID;
    McmcWs w;
    if (int rc = mcmc_ws(N, workspace, workspace_bytes, w)) return rc;
    cudaStream_t s = as_stream(stream);
    ApplyArgs a;
    a.r = r; a.N = N; a.n_samples = n_samples; a.n_dev = n_samples_dev; a.samples = samples; a.targets = targets;
    a.binoms = binoms; a.n_max = n_max; a.min_opacity = min_opacity;
    a.counts = static_cast<int32_t *>(w.rows);
    ProfScope ps(targets ? "mcmc_relocate" : "mcmc_grow", s);
    GSB_CUDA_TRY(cudaMemsetAsync(a.counts, 0, (size_t)N * sizeof(int32_t), s));
    const unsigned nb = blocks_for(n_samples);
    mcmc_count_kernel<<<nb, kMcmcThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    mcmc_apply_kernel<<<nb, kMcmcThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    mcmc_writeback_kernel<<<nb, kMcmcThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_mcmc_regularize(uint32_t N, const float *scaling_raw, const float *opacity_raw, float scale_reg,
                                   float opacity_reg, float *v_scaling, float *v_opacity, float *loss_out,
                                   void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (N == 0) return GSB_OK;
    if (!loss_out || (v_scaling && !scaling_raw) || (v_opacity && !opacity_raw)) return GSB_E_INVALID;
    McmcWs w;
    if (int rc = mcmc_ws(N, workspace, workspace_bytes, w)) return rc;
    cudaStream_t s = as_stream(stream);
    RegArgs a;
    a.N = N; a.scaling_raw = scaling_raw; a.opacity_raw = opacity_raw; a.v_scaling = v_scaling; a.v_opacity = v_opacity;
    a.scale_reg = scale_reg; a.opacity_reg = opacity_reg;
    a.scale_g = scale_reg * (1.0f / (float)(3.0 * N)); // torch divides by a scalar through its reciprocal
    a.opacity_g = opacity_reg * (1.0f / (float)N);
    a.loss_out = loss_out; a.partials = static_cast<double *>(w.bsum); a.done = w.done;
    GSB_CUDA_TRY(cudaMemsetAsync(w.done, 0, sizeof(unsigned int), s));
    unsigned nb = blocks_for(N);
    if (nb > kRegBlocks) nb = kRegBlocks;
    ProfScope ps("mcmc_regularize", s);
    mcmc_regularize_kernel<<<nb, kMcmcThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
