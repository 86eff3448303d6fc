// gsb_relocation.cuh -- the per-Gaussian body of gsplat::relocation (RelocationCUDA.cu:12-43), shared by the
// link-surface kernel (gsb_misc.cu) and the MCMC refine (gsb_mcmc.cu) so that both compute the same bits.
#pragma once

#include "gsb_common.cuh"

namespace gsb {

// Eq. (9) of "3D Gaussian Splatting as Markov Chain Monte Carlo".
// A Gaussian split into n copies keeps its appearance with opacity o' = 1 - (1 - o)^(1/n) and scales multiplied by
//     o / sum_{i=1..n} sum_{k=0..i-1} C(i-1, k) (-1)^k o'^(k+1) / sqrt(k+1).
// The double sum is evaluated k-major here: the power of o' and 1/sqrt(k+1) are built once per k (no powf in the
// loop) and multiplied by the column sum of the caller's binomial table, sum_{i=k+1..n} binoms[i-1][k].
// Returns the factor the scales are multiplied by; *o_new receives o'.
__device__ __forceinline__ float relocation_one(float o, int copies, const float *__restrict__ binoms, int32_t n_max,
                                                float *o_new) {
    const float on = 1.0f - powf(1.0f - o, 1.0f / (float)copies);
    *o_new = on;
    float series = 0.0f;
    float pw = on; // (-1)^k o'^(k+1), k = 0
    for (int k = 0; k < copies; ++k) {
        float column = 0.0f;
        for (int i = k + 1; i <= copies; ++i) column += binoms[(i - 1) * n_max + k];
        series += column * pw * rsqrtf((float)(k + 1));
        pw *= -on;
    }
    return o / series;
}

} // namespace gsb
