// gsb_adc.cu -- adaptive density control, the reference's default densification strategy, on the device
// (src/training/strategies/default_strategy.cpp:164-290: grow_gs, prune_gs, reset_opacity).
//
// A refine (grow_gs then prune_gs) is one compaction.  Everything an original row i contributes to the final set is
// known from row i alone -- a duplicate copy equals its source, and the two copies of a split row agree in everything
// prune_gs reads -- so:
//   gsb_adc_classify  per row: dup = high & small, split = high & !small, whether the row (and its duplicate copy)
//                     survives the prune, whether its split copies do (read from the copies' stored scaling_raw and,
//                     with revised_opacity, their stored opacity, computed as torch computes them); then one scan of
//                     four counters over those flags (gsb_devsort.cuh's scan kernels with a Cnt4 accumulator):
//                     rank among split rows (indexes z), among kept rest rows, kept duplicate copies and kept split
//                     rows.  The totals go to a small DEVICE array: the one value a refine reads back.
//   gsb_adc_apply     the final row of every output is a segment base plus a rank, in the reference's order
//                     (rest rows, duplicate copies, copy 0 of the split rows, copy 1 of the split rows).  A map kernel
//                     writes each output row's source and kind; a row kernel writes the narrow groups (means with the
//                     split offset R(q) (s * z), scaling_raw, opacity_raw, rotation_raw, sh0 and their moments); an
//                     element kernel copies shN and its moments float by float, so that the widest group (180 of the
//                     236 parameter bytes per row at degree 3) is read and written by consecutive threads.  New rows
//                     get zero moments.
//   gsb_adc_reset_opacity   opacity_raw = min(opacity_raw, logit(2 prune_opacity)) in place, the group's moments zeroed.
//   gsb_adc_prune_classify  the ADMM sparsifier's final prune as flags and ranks for gsb_adc_apply: the n_prune-th
//                     smallest sigmoid(opacity_raw) v by gsb_select.cuh's device select, every row below v removed,
//                     rows equal to v removed in index order until n_prune rows are gone (one scan ranks the ties).
// No fast-math: the flags compare exp / log / sigmoid values with thresholds, bit for bit as torch computes them.
#include <cmath>

#include "gsb_common.cuh"
#include "gsb_devsort.cuh"
#include "gsb_select.cuh"

namespace gsb {
namespace adc {

constexpr int kThreads = 256;
constexpr uint32_t kScanBlocks = 264; // two CTAs of 1024 threads per SM of an H100 SXM
constexpr uint32_t kShnRowsPerBlock = 32;
constexpr float kInvSplitScale = 1.0f / 1.6f; // log(s / 1.6): torch divides by a CPU scalar through its reciprocal

enum : uint8_t { kSplit = 1, kKeepRest = 2, kKeepDup = 4, kKeepSplit = 8 };
enum : uint32_t { kKindRest = 0, kKindDup = 1, kKindSplit0 = 2, kKindSplit1 = 3 };
constexpr uint32_t kSrcMask = 0x3fffffffu; // map entry: source row | kind << 30 (N < 2^30)

// four int32 counters scanned at once: (split, kept rest, kept duplicate, kept split)
struct Cnt4 {
    int32_t split, rest, dup, spl;
    Cnt4() = default;
    __device__ __forceinline__ Cnt4(int v) : split(v), rest(v), dup(v), spl(v) {}
    __device__ __forceinline__ Cnt4 &operator+=(const Cnt4 &o) {
        split += o.split; rest += o.rest; dup += o.dup; spl += o.spl;
        return *this;
    }
    __device__ __forceinline__ Cnt4 operator+(const Cnt4 &o) const { Cnt4 r = *this; return r += o; }
};
// found by argument-dependent lookup from block_scan_inclusive
__device__ __forceinline__ Cnt4 __shfl_up_sync(unsigned mask, const Cnt4 &v, int delta) {
    Cnt4 r;
    r.split = ::__shfl_up_sync(mask, v.split, delta);
    r.rest = ::__shfl_up_sync(mask, v.rest, delta);
    r.dup = ::__shfl_up_sync(mask, v.dup, delta);
    r.spl = ::__shfl_up_sync(mask, v.spl, delta);
    return r;
}

struct LoadFlags {
    const uint8_t *f;
    __device__ __forceinline__ Cnt4 operator()(uint64_t i) const {
        const uint32_t x = f[i];
        Cnt4 c;
        c.split = x & kSplit ? 1 : 0;
        c.rest = x & kKeepRest ? 1 : 0;
        c.dup = x & kKeepDup ? 1 : 0;
        c.spl = x & kKeepSplit ? 1 : 0;
        return c;
    }
};

struct Ws {
    Cnt4 *bsum;     // [kScanBlocks]
    uint8_t *flags; // [N]
    Cnt4 *ranks;    // [N] inclusive
    uint32_t *map;  // [2N] output row -> source | kind
};

static size_t ws_bytes(uint32_t N) {
    return 256 + (size_t)kScanBlocks * sizeof(Cnt4) + (((size_t)N + 15) & ~(size_t)15) + (size_t)N * sizeof(Cnt4) +
           (size_t)N * 2 * sizeof(uint32_t);
}

static int ws_carve(uint32_t N, void *workspace, size_t bytes, Ws &w) {
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || bytes < ws_bytes(N)) return GSB_E_WORKSPACE;
    char *b = static_cast<char *>(workspace) + 256;
    w.bsum = reinterpret_cast<Cnt4 *>(b);
    b += (size_t)kScanBlocks * sizeof(Cnt4);
    w.flags = reinterpret_cast<uint8_t *>(b);
    b += ((size_t)N + 15) & ~(size_t)15;
    w.ranks = reinterpret_cast<Cnt4 *>(b);
    b += (size_t)N * sizeof(Cnt4);
    w.map = reinterpret_cast<uint32_t *>(b);
    return GSB_OK;
}

struct Thresholds {
    float grad_threshold, grow_limit, prune_opacity, prune_limit;
    bool prune_big, revised;
};

static Thresholds thresholds(const GsbAdcParams &p) {
    // float products, as default_strategy.cpp:173,241 form them
    return {p.grad_threshold, p.grow_scale3d * p.scene_scale, p.prune_opacity, p.prune_scale3d * p.scene_scale,
            p.prune_too_big != 0, p.revised_opacity != 0};
}

// torch's float logit on CUDA (IEEE logf); sigmoid_f is gsb_common.cuh's
__device__ __forceinline__ float logit_f(float x) { return logf(x / (1.0f - x)); }
// torch::max over the last dim propagates NaN
__device__ __forceinline__ float max_nan(float a, float b) { return (a > b || a != a) ? a : b; }
// default_strategy.cpp:121-122: logit(1 - sqrt(1 - sigmoid(o)))
__device__ __forceinline__ float revised_opacity(float o) { return logit_f(1.0f - sqrtf(1.0f - sigmoid_f(o))); }
__device__ __forceinline__ float split_scaling(float sr) { return logf(expf(sr) * kInvSplitScale); }

// ---- classify -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) classify_kernel(uint32_t N, const float *__restrict__ info,
                                                            const float *__restrict__ scaling_raw,
                                                            const float4 *__restrict__ rotation_raw,
                                                            const float *__restrict__ opacity_raw, const Thresholds t,
                                                            uint8_t *__restrict__ flags, int32_t *__restrict__ n_dup) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    bool dup = false;
    if (i < N) {
        const float sr0 = scaling_raw[(size_t)i * 3], sr1 = scaling_raw[(size_t)i * 3 + 1],
                    sr2 = scaling_raw[(size_t)i * 3 + 2];
        const float smax = max_nan(max_nan(expf(sr0), expf(sr1)), expf(sr2));
        bool high = false;
        if (info) { // grow_gs (:167-171): info[1] / clamp_min(info[0], 1) > grad_threshold
            const float c = info[i];
            high = info[(size_t)N + i] / (c < 1.0f ? 1.0f : c) > t.grad_threshold;
        }
        const bool small = smax <= t.grow_limit;
        dup = high && small;
        const bool split = high && !small;
        const float o = opacity_raw[i];
        const float4 q = rotation_raw[i];
        const bool bad_rot = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w < 1e-8f;
        // prune_gs (:229-249) on the row, which also decides its duplicate copy
        const bool prune_row = sigmoid_f(o) < t.prune_opacity || bad_rot || (t.prune_big && smax > t.prune_limit);
        uint8_t f = 0;
        if (split) {
            f |= kSplit;
            const float cmax = max_nan(max_nan(expf(split_scaling(sr0)), expf(split_scaling(sr1))),
                                       expf(split_scaling(sr2)));
            const float oc = t.revised ? revised_opacity(o) : o;
            const bool prune_copy = sigmoid_f(oc) < t.prune_opacity || bad_rot || (t.prune_big && cmax > t.prune_limit);
            if (!prune_copy) f |= kKeepSplit;
        } else if (!prune_row) {
            f |= kKeepRest;
        }
        if (dup && !prune_row) f |= kKeepDup;
        flags[i] = f;
    }
    const int c = __syncthreads_count(dup);
    if (threadIdx.x == 0 && c) atomicAdd(n_dup, c);
}

// counts: [0] duplicated, [1] split, [2] pruned (of the grown set), [3] final rows, [4..6] kept rest / duplicate /
// split rows
__global__ void totals_kernel(uint32_t N, const Cnt4 *__restrict__ ranks, int32_t *__restrict__ counts) {
    const Cnt4 t = ranks[N - 1];
    const int32_t n_final = t.rest + t.dup + 2 * t.spl;
    counts[1] = t.split;
    counts[2] = (int32_t)N + counts[0] + t.split - n_final;
    counts[3] = n_final;
    counts[4] = t.rest;
    counts[5] = t.dup;
    counts[6] = t.spl;
}

// ---- apply --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) map_kernel(uint32_t N, const uint8_t *__restrict__ flags,
                                                       const Cnt4 *__restrict__ ranks,
                                                       const int32_t *__restrict__ counts,
                                                       uint32_t *__restrict__ map) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= N) return;
    const uint8_t f = flags[i];
    if (!(f & (kKeepRest | kKeepDup | kKeepSplit))) return;
    const Cnt4 r = ranks[i];
    const uint32_t k_rest = (uint32_t)counts[4], k_dup = (uint32_t)counts[5], k_spl = (uint32_t)counts[6];
    if (f & kKeepRest) map[r.rest - 1] = i | (kKindRest << 30);
    if (f & kKeepDup) map[k_rest + r.dup - 1] = i | (kKindDup << 30);
    if (f & kKeepSplit) {
        const uint32_t d = k_rest + k_dup + r.spl - 1;
        map[d] = i | (kKindSplit0 << 30);
        map[d + k_spl] = i | (kKindSplit1 << 30);
    }
}

template <int W>
__device__ __forceinline__ void copy_row(const float *__restrict__ s, float *__restrict__ d, size_t src, size_t dst) {
#pragma unroll
    for (int k = 0; k < W; ++k) d[dst * W + k] = s[src * W + k];
}

template <int W>
__device__ __forceinline__ void moments_row(const float *s, float *d, size_t src, size_t dst, bool keep) {
    if (!d) return;
#pragma unroll
    for (int k = 0; k < W; ++k) d[dst * W + k] = keep ? s[src * W + k] : 0.f;
}

struct RowsArgs {
    GsbMcmcRows src, dst;
    uint32_t n_final;
    const uint32_t *map;
    const Cnt4 *ranks;
    const float *z;       // [2, n_split, 3]
    uint32_t n_split;
    bool revised;
};

__global__ void __launch_bounds__(kThreads) rows_kernel(const RowsArgs a) {
    const uint32_t d = blockIdx.x * kThreads + threadIdx.x;
    if (d >= a.n_final) return;
    const uint32_t e = a.map[d];
    const size_t s = e & kSrcMask;
    const uint32_t kind = e >> 30;
    const GsbMcmcRows &S = a.src, &D = a.dst;
    const float4 q = reinterpret_cast<const float4 *>(S.rotation_raw)[s];
    reinterpret_cast<float4 *>(D.rotation_raw)[d] = q;
    copy_row<3>(S.sh0, D.sh0, s, d);
    if (kind < kKindSplit0) {
        copy_row<3>(S.means, D.means, s, d);
        copy_row<3>(S.scaling_raw, D.scaling_raw, s, d);
        D.opacity_raw[d] = S.opacity_raw[s];
    } else {
        // split (:94-118): means + R(normalize(q)) (s * z[b, rank]), z drawn by torch::randn({2, n_split, 3})
        const float s0 = expf(S.scaling_raw[s * 3]), s1 = expf(S.scaling_raw[s * 3 + 1]),
                    s2 = expf(S.scaling_raw[s * 3 + 2]);
        const float nq = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f); // F::normalize
        const M3<float> R = quat_to_rotmat_norm(q.x / nq, q.y / nq, q.z / nq, q.w / nq, __int_as_float(0x7f800000));
        const uint32_t b = kind - kKindSplit0;
        const float *zz = a.z + ((size_t)b * a.n_split + (uint32_t)(a.ranks[s].split - 1)) * 3;
        const float z0 = zz[0], z1 = zz[1], z2 = zz[2];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float off = R.m[r][0] * s0 * z0 + R.m[r][1] * s1 * z1 + R.m[r][2] * s2 * z2;
            D.means[(size_t)d * 3 + r] = S.means[s * 3 + r] + off;
        }
        D.scaling_raw[(size_t)d * 3] = logf(s0 * kInvSplitScale);
        D.scaling_raw[(size_t)d * 3 + 1] = logf(s1 * kInvSplitScale);
        D.scaling_raw[(size_t)d * 3 + 2] = logf(s2 * kInvSplitScale);
        const float o = S.opacity_raw[s];
        D.opacity_raw[d] = a.revised ? revised_opacity(o) : o;
    }
    const bool keep = kind == kKindRest;
    moments_row<3>(S.exp_avg[0], D.exp_avg[0], s, d, keep);
    moments_row<3>(S.exp_avg_sq[0], D.exp_avg_sq[0], s, d, keep);
    moments_row<3>(S.exp_avg[1], D.exp_avg[1], s, d, keep);
    moments_row<3>(S.exp_avg_sq[1], D.exp_avg_sq[1], s, d, keep);
    moments_row<3>(S.exp_avg[3], D.exp_avg[3], s, d, keep);
    moments_row<3>(S.exp_avg_sq[3], D.exp_avg_sq[3], s, d, keep);
    moments_row<4>(S.exp_avg[4], D.exp_avg[4], s, d, keep);
    moments_row<4>(S.exp_avg_sq[4], D.exp_avg_sq[4], s, d, keep);
    moments_row<1>(S.exp_avg[5], D.exp_avg[5], s, d, keep);
    moments_row<1>(S.exp_avg_sq[5], D.exp_avg_sq[5], s, d, keep);
}

// shN and its moments: a block owns kShnRowsPerBlock output rows and walks their floats with consecutive threads
__global__ void __launch_bounds__(kThreads) shn_kernel(const RowsArgs a) {
    const uint32_t kn = a.src.shN_rows * 3;
    const uint32_t r0 = blockIdx.x * kShnRowsPerBlock;
    const uint32_t rows = min(kShnRowsPerBlock, a.n_final - r0);
    const uint32_t n = rows * kn;
    const float *sp = a.src.shN, *s1 = a.src.exp_avg[2], *s2 = a.src.exp_avg_sq[2];
    float *dp = a.dst.shN, *d1 = a.dst.exp_avg[2], *d2 = a.dst.exp_avg_sq[2];
    for (uint32_t l = threadIdx.x; l < n; l += kThreads) {
        const uint32_t rr = l / kn, c = l - rr * kn;
        const uint32_t e = a.map[r0 + rr];
        const size_t src = (size_t)(e & kSrcMask) * kn + c;
        const size_t dst = (size_t)(r0 + rr) * kn + c;
        const bool keep = (e >> 30) == kKindRest;
        dp[dst] = sp[src];
        if (d1) d1[dst] = keep ? s1[src] : 0.f;
        if (d2) d2[dst] = keep ? s2[src] : 0.f;
    }
}

__global__ void __launch_bounds__(kThreads) reset_opacity_kernel(uint32_t N, float *__restrict__ o, float thr) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= N) return;
    const float v = o[i];
    o[i] = v > thr ? thr : v; // torch::clamp_max: NaN stays
}

// ---- the sparsifier's final prune (gsb_adc_prune_classify) --------------------------------------------------------
// Workspace reuse: the keys live in `map` (written by gsb_adc_apply only), the select's histograms in `bsum` (before
// the scan uses it), its state in the 256-byte head.
static_assert(sel::kHistBytes <= kScanBlocks * sizeof(Cnt4), "the select histograms must fit the scan's block sums");
static_assert(sizeof(sel::SelectState) <= 256, "the select state must fit the workspace head");

__global__ void __launch_bounds__(kThreads) prune_keys_kernel(uint32_t N, const float *__restrict__ opacity_raw,
                                                              uint32_t *__restrict__ keys) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i < N) keys[i] = sel::float_key(sigmoid_f(opacity_raw[i]));
}

// below the n_prune-th smallest key: pruned; equal to it: a tie (kSplit marks it for the scan); above: kept
__global__ void __launch_bounds__(kThreads) prune_flags_kernel(uint32_t N, const uint32_t *__restrict__ keys,
                                                               const sel::SelectState *__restrict__ st, bool none,
                                                               uint8_t *__restrict__ flags) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= N) return;
    if (none) {
        flags[i] = kKeepRest;
        return;
    }
    const uint32_t k = keys[i], v = st->prefix;
    flags[i] = k > v ? kKeepRest : (k == v ? kSplit : 0);
}

// After the scan (split = rank among ties, rest = rank among rows above the boundary): the first n_prune - n_less
// ties in index order are pruned, the others kept, and every kept row's rank becomes its rank among all kept rows.
__global__ void __launch_bounds__(kThreads) prune_ranks_kernel(uint32_t N, uint32_t n_prune,
                                                               const sel::SelectState *__restrict__ st, bool none,
                                                               uint8_t *__restrict__ flags, Cnt4 *__restrict__ ranks,
                                                               int32_t *__restrict__ counts) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i == 0) {
        const int32_t kept = (int32_t)(N - n_prune);
        counts[0] = 0; counts[1] = 0; counts[2] = (int32_t)n_prune; counts[3] = kept;
        counts[4] = kept; counts[5] = 0; counts[6] = 0; counts[7] = 0;
    }
    if (i >= N || none) return;
    const int32_t tie_pruned = (int32_t)(n_prune - st->n_less);
    const uint8_t f = flags[i];
    Cnt4 r = ranks[i];
    const int32_t kept_ties = r.split > tie_pruned ? r.split - tie_pruned : 0;
    if (f & kSplit) flags[i] = r.split > tie_pruned ? kKeepRest : 0;
    r.rest += kept_ties;
    ranks[i] = r;
}

static unsigned blocks_for(uint64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

static bool rows_valid(const GsbMcmcRows &r) {
    if (!r.means || !r.sh0 || !r.scaling_raw || !r.rotation_raw || !r.opacity_raw || (r.shN_rows && !r.shN)) return false;
    return (reinterpret_cast<uintptr_t>(r.rotation_raw) & 15) == 0;
}

} // namespace adc
} // namespace gsb

extern "C" size_t gsb_adc_workspace(uint32_t N) { return gsb::adc::ws_bytes(N); }

extern "C" int gsb_adc_classify(uint32_t N, const float *densification_info, const float *scaling_raw,
                                const float *rotation_raw, const float *opacity_raw, const GsbAdcParams *params,
                                int32_t *counts, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::adc;
    if (!params || !counts) return GSB_E_INVALID;
    if ((uint64_t)N * 2 > (uint64_t)INT32_MAX) return GSB_E_INVALID; // N + n_dup + n_split <= 2N must fit int32
    cudaStream_t s = as_stream(stream);
    if (N == 0) {
        GSB_CUDA_TRY(cudaMemsetAsync(counts, 0, 8 * sizeof(int32_t), s));
        return GSB_OK;
    }
    if (!scaling_raw || !rotation_raw || !opacity_raw) return GSB_E_INVALID;
    if (reinterpret_cast<uintptr_t>(rotation_raw) & 15) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_carve(N, workspace, workspace_bytes, w)) return rc;
    const Thresholds t = thresholds(*params);
    ProfScope ps("adc_classify", s);
    GSB_CUDA_TRY(cudaMemsetAsync(counts, 0, 8 * sizeof(int32_t), s));
    classify_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, densification_info, scaling_raw,
                                                       reinterpret_cast<const float4 *>(rotation_raw), opacity_raw, t,
                                                       w.flags, counts);
    GSB_LAUNCH_CHECK();
    uint64_t nb = (N + 4095) / 4096;
    if (nb > kScanBlocks) nb = kScanBlocks;
    const uint32_t seg = (uint32_t)((N + nb - 1) / nb);
    const LoadFlags load{w.flags};
    scan_blocksum_kernel<<<(unsigned)nb, kSortThreads, 0, s>>>(load, N, seg, w.bsum);
    GSB_LAUNCH_CHECK();
    scan_apply_kernel<<<(unsigned)nb, kSortThreads, 0, s>>>(load, N, seg, w.bsum, w.ranks);
    GSB_LAUNCH_CHECK();
    totals_kernel<<<1, 1, 0, s>>>(N, w.ranks, counts);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_adc_apply(uint32_t N, const GsbMcmcRows *src, const GsbMcmcRows *dst, uint32_t n_split,
                             uint32_t n_final, const float *z, const GsbAdcParams *params, const int32_t *counts,
                             float *densification_info, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::adc;
    if (!params || !counts || !src || !dst) return GSB_E_INVALID;
    if ((uint64_t)N * 2 > (uint64_t)INT32_MAX || n_final > 2 * (uint64_t)N || n_split > N) return GSB_E_INVALID;
    if (n_split && !z) return GSB_E_INVALID;
    cudaStream_t s = as_stream(stream);
    if (densification_info && n_final)
        GSB_CUDA_TRY(cudaMemsetAsync(densification_info, 0, (size_t)n_final * 2 * sizeof(float), s));
    if (n_final == 0) return GSB_OK;
    if (!rows_valid(*src) || !rows_valid(*dst) || src->shN_rows != dst->shN_rows) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_carve(N, workspace, workspace_bytes, w)) return rc;
    RowsArgs a;
    a.src = *src; a.dst = *dst; a.n_final = n_final; a.map = w.map; a.ranks = w.ranks; a.z = z; a.n_split = n_split;
    a.revised = params->revised_opacity != 0;
    ProfScope ps("adc_apply", s);
    map_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, w.flags, w.ranks, counts, w.map);
    GSB_LAUNCH_CHECK();
    rows_kernel<<<blocks_for(n_final), kThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    if (a.src.shN_rows) {
        shn_kernel<<<(n_final + kShnRowsPerBlock - 1) / kShnRowsPerBlock, kThreads, 0, s>>>(a);
        GSB_LAUNCH_CHECK();
    }
    return GSB_OK;
}

extern "C" int gsb_adc_prune_classify(uint32_t N, const float *opacity_raw, uint32_t n_prune, int32_t *counts,
                                      void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::adc;
    if (!counts || n_prune > N) return GSB_E_INVALID;
    if ((uint64_t)N * 2 > (uint64_t)INT32_MAX) return GSB_E_INVALID; // gsb_adc_apply's bound
    cudaStream_t s = as_stream(stream);
    if (N == 0) {
        GSB_CUDA_TRY(cudaMemsetAsync(counts, 0, 8 * sizeof(int32_t), s));
        return GSB_OK;
    }
    if (!opacity_raw) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_carve(N, workspace, workspace_bytes, w)) return rc;
    uint32_t *keys = w.map;
    uint32_t *hist = reinterpret_cast<uint32_t *>(w.bsum);
    sel::SelectState *st = static_cast<sel::SelectState *>(workspace);
    const bool none = n_prune == 0;
    ProfScope ps("adc_prune_classify", s);
    GSB_CUDA_TRY(cudaMemsetAsync(st, 0, sizeof(sel::SelectState), s));
    if (!none) {
        prune_keys_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, opacity_raw, keys);
        GSB_LAUNCH_CHECK();
        if (int rc = sel::select_kth(keys, N, n_prune, hist, st, s)) return rc;
    }
    prune_flags_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, keys, st, none, w.flags);
    GSB_LAUNCH_CHECK();
    uint64_t nb = (N + 4095) / 4096;
    if (nb > kScanBlocks) nb = kScanBlocks;
    const uint32_t seg = (uint32_t)((N + nb - 1) / nb);
    const LoadFlags load{w.flags};
    scan_blocksum_kernel<<<(unsigned)nb, kSortThreads, 0, s>>>(load, N, seg, w.bsum);
    GSB_LAUNCH_CHECK();
    scan_apply_kernel<<<(unsigned)nb, kSortThreads, 0, s>>>(load, N, seg, w.bsum, w.ranks);
    GSB_LAUNCH_CHECK();
    prune_ranks_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, n_prune, st, none, w.flags, w.ranks, counts);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_adc_reset_opacity(uint32_t N, float *opacity_raw, float prune_opacity, float *exp_avg,
                                     float *exp_avg_sq, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::adc;
    if (N == 0) return GSB_OK;
    if (!opacity_raw) return GSB_E_INVALID;
    cudaStream_t s = as_stream(stream);
    // torch::logit(torch::tensor(2.0f * prune_opacity)).item() (:254-260): a float logit on the host
    const float x = 2.0f * prune_opacity;
    const float thr = std::log(x / (1.0f - x));
    ProfScope ps("adc_reset_opacity", s);
    reset_opacity_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, opacity_raw, thr);
    GSB_LAUNCH_CHECK();
    if (exp_avg) GSB_CUDA_TRY(cudaMemsetAsync(exp_avg, 0, (size_t)N * sizeof(float), s));
    if (exp_avg_sq) GSB_CUDA_TRY(cudaMemsetAsync(exp_avg_sq, 0, (size_t)N * sizeof(float), s));
    return GSB_OK;
}
