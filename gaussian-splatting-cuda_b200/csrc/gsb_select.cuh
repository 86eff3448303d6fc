// gsb_select.cuh -- the k-th smallest of N floats on the device, for the ADMM sparsifier (gsb_sparsity.cu: the
// threshold of prune_z, a torch::sort(x)[k - 1] in sparsity_optimizer.cpp:157-165) and its final prune (gsb_adc.cu:
// the boundary value of torch::topk(sigmoid(o), n_prune, largest=false)).
//
// Each float becomes an order-preserving uint32 key (float_key: -0 as +0, every NaN last, as torch.sort puts it),
// written by the caller into a key array.  Four radix passes of 8 bits then narrow a prefix down to the exact k-th
// key: a histogram kernel counts the digit of every key that matches the prefix so far, and a one-CTA kernel finds
// the bin holding the k-th key, extends the prefix and keeps the remaining rank and the number of keys below the
// prefix.  Everything stays in device memory (SelectState): no host read-back, so the select can be captured in a
// CUDA graph.  The bins are counted in shared memory and flushed with one global atomic per non-empty bin per CTA.
#pragma once

#include "gsb_common.cuh"

namespace gsb {
namespace sel {

constexpr int kThreads = 256;
constexpr int kBins = 256;
constexpr int kPasses = 4;
constexpr uint32_t kMaxBlocks = 1056; // eight CTAs per SM of an H100 SXM

struct SelectState {
    uint32_t prefix; // the key bits found so far; after the last pass, the k-th smallest key
    uint32_t k;      // rank (1-based) still to find among the keys matching the prefix
    uint32_t n_less; // keys below the prefix; after the last pass, keys strictly below the k-th key
    uint32_t pad;
};
constexpr size_t kHistBytes = (size_t)kPasses * kBins * sizeof(uint32_t);

// float -> uint32 with a < b  <=>  key(a) < key(b) for non-NaN floats; -0 and +0 share a key, NaN is the largest
__device__ __forceinline__ uint32_t float_key(float f) {
    if (f != f) return 0xffffffffu;
    uint32_t b = __float_as_uint(f);
    if (b == 0x80000000u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
// the inverse (the NaN key gives a NaN)
__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <int Pass>
__global__ void __launch_bounds__(kThreads) hist_kernel(const uint32_t *__restrict__ keys, uint32_t N,
                                                        const SelectState *__restrict__ st,
                                                        uint32_t *__restrict__ hist) {
    constexpr uint32_t shift = 24 - 8 * Pass;
    constexpr uint32_t hi_mask = Pass == 0 ? 0u : (0xffffffffu << (32 - 8 * Pass));
    __shared__ uint32_t h[kBins];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t prefix = Pass == 0 ? 0u : st->prefix;
    const uint32_t stride = gridDim.x * kThreads;
    for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < N; i += stride) {
        const uint32_t k = keys[i];
        if ((k & hi_mask) == prefix) atomicAdd(&h[(k >> shift) & 0xffu], 1u);
    }
    __syncthreads();
    const uint32_t c = h[threadIdx.x];
    if (c) atomicAdd(&hist[threadIdx.x], c);
}

// one CTA of kBins threads: the bin holding the k-th key of this pass
template <int Pass>
__global__ void __launch_bounds__(kBins) find_kernel(const uint32_t *__restrict__ hist, uint32_t k0,
                                                     SelectState *st) {
    constexpr uint32_t shift = 24 - 8 * Pass;
    __shared__ uint32_t s_warp[kBins / 32];
    __shared__ uint32_t s_bin, s_before;
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t k = Pass == 0 ? k0 : st->k;
    const uint32_t c = hist[t];
    uint32_t inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (uint32_t)o) inc += v;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    for (uint32_t w = 0; w < warp; ++w) inc += s_warp[w];
    const uint32_t exc = inc - c;
    if (exc < k && k <= inc) { // exactly one bin while 1 <= k <= the matching keys
        s_bin = t;
        s_before = exc;
    }
    __syncthreads();
    if (t == 0) {
        st->prefix = (Pass == 0 ? 0u : st->prefix) | (s_bin << shift);
        st->k = k - s_before;
        st->n_less = (Pass == 0 ? 0u : st->n_less) + s_before;
    }
}

// The k-th smallest (1 <= k <= N) of keys[0, N) into st->prefix, the count of smaller keys into st->n_less.
// hist: kHistBytes of device memory, st: one SelectState; both are overwritten.
static inline int select_kth(const uint32_t *keys, uint32_t N, uint32_t k, uint32_t *hist, SelectState *st,
                             cudaStream_t s) {
    GSB_CUDA_TRY(cudaMemsetAsync(hist, 0, kHistBytes, s));
    uint64_t nb = ((uint64_t)N + kThreads - 1) / kThreads;
    if (nb > kMaxBlocks) nb = kMaxBlocks;
    const unsigned g = (unsigned)nb;
    hist_kernel<0><<<g, kThreads, 0, s>>>(keys, N, st, hist);
    GSB_LAUNCH_CHECK();
    find_kernel<0><<<1, kBins, 0, s>>>(hist, k, st);
    GSB_LAUNCH_CHECK();
    hist_kernel<1><<<g, kThreads, 0, s>>>(keys, N, st, hist + kBins);
    GSB_LAUNCH_CHECK();
    find_kernel<1><<<1, kBins, 0, s>>>(hist + kBins, k, st);
    GSB_LAUNCH_CHECK();
    hist_kernel<2><<<g, kThreads, 0, s>>>(keys, N, st, hist + 2 * kBins);
    GSB_LAUNCH_CHECK();
    find_kernel<2><<<1, kBins, 0, s>>>(hist + 2 * kBins, k, st);
    GSB_LAUNCH_CHECK();
    hist_kernel<3><<<g, kThreads, 0, s>>>(keys, N, st, hist + 3 * kBins);
    GSB_LAUNCH_CHECK();
    find_kernel<3><<<1, kBins, 0, s>>>(hist + 3 * kBins, k, st);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

} // namespace sel
} // namespace gsb
