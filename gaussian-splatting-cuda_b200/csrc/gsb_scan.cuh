// gsb_scan.cuh -- device-wide inclusive scan, hand-written for sm_90a.
//
// Replaces at::cumsum (gsplat/Intersect.cpp:71) and serves every stage that ranks or prefixes per-Gaussian values: the
// intersect stage's cum_tiles and run table, the MCMC dead ranks and sampling prefix, the ADC and final-prune ranks.
//   * scan_blocksum_kernel / scan_apply_kernel -- two-launch inclusive scan (per-CTA sums, then every CTA adds the
//     sums of its predecessors and scans its own segment), launched together by scan_launch.
//   * scan_plan -- the CTA count and segment length of a scan over n items.  A float64 scan's result depends on the
//     partition, so every caller keeps its own cap on the CTA count: changing it changes, e.g., which Gaussian a
//     seeded MCMC draw picks.
// The kernels are stream-ordered and keep no state outside the caller's workspace.
#pragma once

#include "gsb_common.cuh"

namespace gsb {

constexpr int kScanThreads = 1024;
constexpr int kScanWarps = kScanThreads / 32;

struct SegRange {
    uint64_t lo, hi;
};
__device__ __forceinline__ SegRange cta_segment(uint64_t n, uint32_t seg) {
    SegRange r;
    r.lo = (uint64_t)blockIdx.x * seg;
    r.hi = r.lo + seg < n ? r.lo + seg : n;
    if (r.lo > n) r.lo = n;
    return r;
}

// CTAs of about 4096 items each (four per thread), at most max_blocks of them
struct ScanPlan {
    uint32_t nblocks, seg;
};
static inline ScanPlan scan_plan(uint64_t n, uint32_t max_blocks) {
    uint64_t nb = ceil_div(n, 4096);
    if (nb < 1) nb = 1;
    if (nb > max_blocks) nb = max_blocks;
    return {(uint32_t)nb, (uint32_t)ceil_div(n, nb)};
}

// ---- block-wide inclusive scan of one value per thread (kScanThreads threads) ---------------------------------------
// T is an integer, a floating-point type or a struct of them with +=, +, construction from the int 0 and a
// __shfl_up_sync overload found by argument-dependent lookup (a hidden friend: adc::Cnt4, RunAcc).  kUnroll unrolls
// the loop over the warps' sums: the run table's 16-byte sums are read faster all at once (kScanWarps).
template <typename T, int kUnroll = 8>
__device__ __forceinline__ T block_scan_inclusive(T v, T *s_warp /* [kScanWarps] */, T &total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= (uint32_t)o) v += t;
    }
    __syncthreads(); // s_warp may still be read by the previous call
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    T add = 0, tot = 0;
#pragma unroll kUnroll
    for (int w = 0; w < kScanWarps; ++w) {
        const T x = s_warp[w];
        if ((uint32_t)w < warp) add += x;
        tot += x;
    }
    total = tot;
    return v + add;
}

// ---- inclusive scan of loader values: Load is `Acc operator()(uint64_t i) const` ---------------------------
// Instantiated for int32 counts -> int64 (the unsorted intersect path's cum_tiles; Intersect.cpp:71), 0/1 flags ->
// int32 ranks and float weights -> a float64 prefix (gsb_mcmc.cu), and four-counter flags (gsb_adc.cu).
struct LoadI32 {
    const int32_t *p;
    __device__ __forceinline__ long long operator()(uint64_t i) const { return p[i]; }
};

template <typename Load, typename Acc>
__global__ void __launch_bounds__(kScanThreads) scan_blocksum_kernel(const Load load, uint64_t n, uint32_t seg,
                                                                     Acc *__restrict__ bsum) {
    __shared__ Acc s_warp[kScanWarps];
    const SegRange r = cta_segment(n, seg);
    Acc acc = 0;
    for (uint64_t i = r.lo + threadIdx.x; i < r.hi; i += kScanThreads) acc += load(i);
    Acc tot;
    block_scan_inclusive<Acc>(acc, s_warp, tot);
    if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}

template <typename Load, typename Acc, typename Out>
__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(const Load load, uint64_t n, uint32_t seg,
                                                                  const Acc *__restrict__ bsum, Out *__restrict__ cum) {
    __shared__ Acc s_warp[kScanWarps];
    Acc carry;
    {
        Acc part = 0;
        for (uint32_t bb = threadIdx.x; bb < blockIdx.x; bb += kScanThreads) part += bsum[bb];
        block_scan_inclusive<Acc>(part, s_warp, carry);
    }
    const SegRange r = cta_segment(n, seg);
    for (uint64_t i0 = r.lo; i0 < r.hi; i0 += kScanThreads) {
        const uint64_t i = i0 + threadIdx.x;
        const Acc v = i < r.hi ? load(i) : (Acc)0;
        Acc tot;
        const Acc inc = block_scan_inclusive<Acc>(v, s_warp, tot);
        if (i < r.hi) cum[i] = (Out)(carry + inc);
        carry += tot;
    }
}

// cum[i] = load(0) + ... + load(i) for i < n; bsum holds sp.nblocks block sums
template <typename Load, typename Acc, typename Out>
static inline int scan_launch(const Load &load, uint64_t n, const ScanPlan &sp, Acc *bsum, Out *cum, cudaStream_t s) {
    scan_blocksum_kernel<<<sp.nblocks, kScanThreads, 0, s>>>(load, n, sp.seg, bsum);
    GSB_LAUNCH_CHECK();
    scan_apply_kernel<<<sp.nblocks, kScanThreads, 0, s>>>(load, n, sp.seg, bsum, cum);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

} // namespace gsb
