// gsb_reduce.cuh -- deterministic float64 reductions, hand-written for sm_90a: the losses that end in a device scalar
// (gsb_mcmc.cu's regularisers, gsb_sparsity.cu's ADMM loss, gsb_bilagrid.cu's TV loss).  The order of every addition
// is fixed by the launch shape alone, so a loss repeats bit for bit from run to run:
//   * block_sum -- a butterfly per warp, then the warps' sums added in index order;
//   * grid_sum_last -- per-CTA block sums into a partials array; the last CTA to take a ticket reads them back, each
//     thread summing the CTAs strided by the block size, and finishes with another block sum.
#pragma once

#include "gsb_common.cuh"

namespace gsb {

template <int kThreads>
__device__ __forceinline__ double block_sum(double v, double *red /* [kThreads / 32] */) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int k = 0; k < kThreads / 32; ++k) t += red[k]; // fixed order: deterministic
    return t;
}

// Grid-wide sums of K values per thread.  Every thread of every CTA calls it.  It returns true in the CTA that finishes
// last, whose threads all receive the K grid totals in `tot`, and false in every other CTA.
// partials: gridDim.x * K doubles; ticket: zeroed before the launch.
template <int kThreads, int K>
__device__ __forceinline__ bool grid_sum_last(const double (&v)[K], double *partials, unsigned int *ticket,
                                              double (&tot)[K]) {
    __shared__ double red[kThreads / 32];
    __shared__ bool last;
    double b[K];
#pragma unroll
    for (int k = 0; k < K; ++k) b[k] = block_sum<kThreads>(v[k], red);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) partials[(size_t)K * blockIdx.x + k] = b[k];
        __threadfence(); // the partials are visible before the ticket is taken
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return false;
    __threadfence(); // every other CTA's partials are read after its ticket
#pragma unroll
    for (int k = 0; k < K; ++k) tot[k] = 0.0;
    for (uint32_t c = threadIdx.x; c < gridDim.x; c += kThreads) {
        const volatile double *q = partials + (size_t)K * c;
#pragma unroll
        for (int k = 0; k < K; ++k) tot[k] += q[k];
    }
#pragma unroll
    for (int k = 0; k < K; ++k) tot[k] = block_sum<kThreads>(tot[k], red);
    return true;
}

} // namespace gsb
