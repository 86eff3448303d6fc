// gsb_devsort.cuh -- device-wide radix sort of the intersect stage, hand-written for sm_90a.
//
// Replaces the library sort of the reference's intersect_tile (cub::DeviceRadixSort::SortPairs,
// gsplat/IntersectTile.cu:300-314) with this repository's own kernels:
//   * radix_count_kernel / radix_scatter_kernel -- stable LSD radix sort of (key, value) pairs, 8 bits per
//     pass, two launches per pass.  Each CTA owns one contiguous segment; its 32 warps own contiguous
//     sub-segments and rank their keys with match.any, so equal digits keep their input order.  The
//     exclusive prefix over (digit, CTA) is recomputed by every CTA from the small CTA x 256 histogram
//     matrix (148 KB in L2) instead of a third launch.  A pass whose digit is the same for every ACTIVE key
//     (SortCtl::key_or / key_and, e.g. the exponent byte of depths within one octave) is skipped by both
//     kernels; which buffer currently holds the data is derived from the same control block, so no host
//     round trip is needed.  Any subset of the passes may be skipped, all four included (one Gaussian with
//     tiles, or all of them at one depth): the caller therefore writes the values (the identity permutation)
//     into v0 together with the keys, so that whichever pass runs first -- or, when none does, the run
//     table itself -- reads a valid permutation from v0.
// The CTA segments are gsb_scan.cuh's.  The kernels are stream-ordered and keep no state outside the caller's
// workspace.
#pragma once

#include "gsb_scan.cuh"

namespace gsb {

constexpr int kSortThreads = 1024;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kRadixBins = 256;

// Control block of the planned intersect path (device memory, inside the plan workspace).
struct SortCtl {
    uint32_t key_or;          // OR of the depth keys of all Gaussians that touch a tile
    uint32_t key_nor;         // OR of their complements (AND of the keys = ~key_nor): both start at zero
    uint32_t n_runs;          // Gaussians with at least one tile (length of the run table)
    uint32_t pad0;
    unsigned long long n_isects;
    unsigned long long pad1;
};

// Pass `pass` (digit bits [8 pass, 8 pass + 8)) is skipped when all active keys agree on that digit.
__device__ __forceinline__ bool radix_pass_skipped(const SortCtl *ctl, int pass) {
    if (!ctl) return false;
    return (((ctl->key_or ^ ~ctl->key_nor) >> (8 * pass)) & 0xffu) == 0u;
}
// Number of passes before `pass` that actually moved data: its parity says which buffer is current.
__device__ __forceinline__ int radix_passes_done(const SortCtl *ctl, int pass) {
    int done = 0;
    for (int p = 0; p < pass; ++p) done += radix_pass_skipped(ctl, p) ? 0 : 1;
    return done;
}

template <typename KeyT>
__device__ __forceinline__ uint32_t radix_digit(KeyT k, uint32_t shift, uint32_t mask) {
    return (uint32_t)(k >> shift) & mask;
}

// ---- pass kernel 1: per-CTA digit histogram -------------------------------------------------------------
// With ctl != nullptr the source is buffer (passes done so far) & 1 of {k0, k1}; otherwise k0.
template <typename KeyT>
__global__ void __launch_bounds__(kSortThreads) radix_count_kernel(const KeyT *__restrict__ k0,
                                                                   const KeyT *__restrict__ k1, uint64_t n,
                                                                   uint32_t seg, int pass, uint32_t shift,
                                                                   uint32_t mask, const SortCtl *__restrict__ ctl,
                                                                   uint32_t *__restrict__ H) {
    if (radix_pass_skipped(ctl, pass)) return;
    const KeyT *src = (ctl && (radix_passes_done(ctl, pass) & 1)) ? k1 : k0;
    __shared__ uint32_t h[kRadixBins];
    if (threadIdx.x < kRadixBins) h[threadIdx.x] = 0;
    __syncthreads();
    const SegRange r = cta_segment(n, seg);
    for (uint64_t i = r.lo + threadIdx.x; i < r.hi; i += kSortThreads) atomicAdd(&h[radix_digit(src[i], shift, mask)], 1u);
    __syncthreads();
    if (threadIdx.x < kRadixBins) H[(size_t)blockIdx.x * kRadixBins + threadIdx.x] = h[threadIdx.x];
}

// ---- pass kernel 2: stable scatter ----------------------------------------------------------------------
// Source / destination: without a control block k0/v0 -> k1/v1 (the host alternates the buffers); with one,
// buffer (passes executed so far) & 1 is the source.
template <typename KeyT>
__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(
    KeyT *k0, KeyT *k1, uint32_t *v0, uint32_t *v1, uint64_t n, uint32_t seg, uint32_t nblocks, int pass,
    uint32_t shift, uint32_t mask, const SortCtl *__restrict__ ctl, const uint32_t *__restrict__ H) {
    if (radix_pass_skipped(ctl, pass)) return;
    const int done = ctl ? radix_passes_done(ctl, pass) : 0;
    const KeyT *__restrict__ ksrc = (done & 1) ? k1 : k0;
    KeyT *__restrict__ kdst = (done & 1) ? k0 : k1;
    const uint32_t *__restrict__ vsrc = (done & 1) ? v1 : v0;
    uint32_t *__restrict__ vdst = (done & 1) ? v0 : v1;

    __shared__ uint32_t s_w[kSortWarps][kRadixBins]; // warp histograms, then warp write cursors
    __shared__ uint32_t s_tot[4][kRadixBins], s_pre[4][kRadixBins];
    __shared__ uint32_t s_scan[kRadixBins / 32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t b = blockIdx.x;

    // (a) column sums of the CTA x digit matrix: total per digit and the part owned by CTAs before this one
    {
        const uint32_t d = tid & (kRadixBins - 1), q = tid >> 8;
        uint32_t tot = 0, pre = 0;
        for (uint32_t bb = q; bb < nblocks; bb += 4) {
            const uint32_t v = H[(size_t)bb * kRadixBins + d];
            tot += v;
            if (bb < b) pre += v;
        }
        s_tot[q][d] = tot;
        s_pre[q][d] = pre;
    }
    for (uint32_t i = tid; i < kSortWarps * kRadixBins; i += kSortThreads) (&s_w[0][0])[i] = 0;
    __syncthreads();
    uint32_t gbase = 0; // threads < 256: first output slot of digit `tid` for this CTA
    if (tid < kRadixBins) {
        const uint32_t tot = s_tot[0][tid] + s_tot[1][tid] + s_tot[2][tid] + s_tot[3][tid];
        const uint32_t pre = s_pre[0][tid] + s_pre[1][tid] + s_pre[2][tid] + s_pre[3][tid];
        // exclusive scan of tot over the 256 digits (8 warps)
        uint32_t inc = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= (uint32_t)o) inc += t;
        }
        if (lane == 31) s_scan[warp] = inc;
        gbase = inc - tot + pre;
    }
    __syncthreads();
    if (tid < kRadixBins) {
        uint32_t add = 0;
        for (uint32_t w = 0; w < warp; ++w) add += s_scan[w];
        gbase += add;
    }

    // (b) warp histograms over the warp's contiguous sub-segment
    const SegRange r = cta_segment(n, seg);
    const uint64_t len = r.hi - r.lo;
    const uint64_t wseg = (len + kSortWarps - 1) / kSortWarps;
    uint64_t wlo = r.lo + (uint64_t)warp * wseg, whi = wlo + wseg;
    if (wlo > r.hi) wlo = r.hi;
    if (whi > r.hi) whi = r.hi;
    for (uint64_t i = wlo + lane; i < whi; i += 32) atomicAdd(&s_w[warp][radix_digit(ksrc[i], shift, mask)], 1u);
    __syncthreads();
    // (c) histograms -> write cursors: digit d of warp w starts at gbase[d] + sum of earlier warps' counts
    if (tid < kRadixBins) {
        uint32_t run = gbase;
#pragma unroll 4
        for (int w = 0; w < kSortWarps; ++w) {
            const uint32_t c = s_w[w][tid];
            s_w[w][tid] = run;
            run += c;
        }
    }
    __syncthreads();
    // (d) ranked scatter: 32 keys per step, equal digits keep lane (= input) order.  The set of lanes with the same
    //     digit comes from eight ballots (one per digit bit), not from match.any, whose cost grows with the number of
    //     DISTINCT values in the warp; the next step's key is loaded before this step's rank is computed.
    uint32_t *cur = s_w[warp];
    KeyT key_next = 0;
    if (wlo + lane < whi) key_next = ksrc[wlo + lane];
    for (uint64_t i0 = wlo; i0 < whi; i0 += 32) {
        const uint64_t i = i0 + lane;
        const bool valid = i < whi;
        const KeyT key = key_next;
        if (i + 32 < whi) key_next = ksrc[i + 32];
        const uint32_t dgt = radix_digit(key, shift, mask);
        uint32_t peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
        for (int bit = 0; bit < 8; ++bit) {
            const bool one = (dgt >> bit) & 1u;
            const uint32_t m = __ballot_sync(0xffffffffu, one);
            peers &= one ? m : ~m;
        }
        uint32_t base = 0;
        if (valid) base = cur[dgt];
        __syncwarp();
        if (valid) {
            const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
            const uint32_t pos = base + rank;
            kdst[pos] = key;
            vdst[pos] = vsrc[i];
            if ((peers >> lane) == 1u) cur[dgt] = base + __popc(peers); // highest lane of the group
        }
        __syncwarp();
    }
}

} // namespace gsb
