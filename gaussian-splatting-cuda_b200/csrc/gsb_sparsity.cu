// gsb_sparsity.cu -- the ADMM opacity-sparsity phase of the reference's trainer on the device
// (src/training/components/sparsity_optimizer.cpp).  With s = sigmoid(opacity_raw) and k = (int)(prune_ratio * N)
// (the caller's float product):
//   gsb_sparsity_update  initialize (u = 0, z = prune_z(s + u)) or update_state (zt = s + u, z = prune_z(zt),
//                        u += s - z), where prune_z(x) = (x > x_(k)) * x with x_(k) the k-th smallest of x
//                        (sort(x)[k - 1]) and 0 when k == 0.  The select is gsb_select.cuh's: the threshold never
//                        leaves the device.  Elementwise float, bit for bit as torch computes it.
//   gsb_sparsity_loss    0.5 rho ||s - z + u||^2 into a device scalar (per-CTA double partials summed in a fixed
//                        order by the last CTA: deterministic) and its gradient rho (s - z + u) s (1 - s) added into
//                        v_opacity.  rho is read from the device, so one captured graph serves the whole phase; a
//                        zero rho writes a zero loss and leaves the gradient alone.
// No fast-math; the elementwise arithmetic uses the explicit _rn intrinsics so that nothing is contracted.
#include <cmath>

#include "gsb_common.cuh"
#include "gsb_select.cuh"

namespace gsb {
namespace sparsity {

constexpr int kThreads = 256;
constexpr uint32_t kLossBlocks = 264;

struct Ws {
    sel::SelectState *st;
    unsigned int *done;
    uint32_t *hist;   // [kPasses * kBins]
    double *partials; // [kLossBlocks]
    uint32_t *keys;   // [N]
};

static size_t ws_bytes(uint32_t N) { return 256 + sel::kHistBytes + (size_t)kLossBlocks * sizeof(double) + (size_t)N * 4; }

static int ws_carve(uint32_t N, void *workspace, size_t bytes, Ws &w) {
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || bytes < ws_bytes(N)) return GSB_E_WORKSPACE;
    char *b = static_cast<char *>(workspace);
    w.st = reinterpret_cast<sel::SelectState *>(b);
    w.done = reinterpret_cast<unsigned int *>(b + 128);
    b += 256;
    w.hist = reinterpret_cast<uint32_t *>(b);
    b += sel::kHistBytes;
    w.partials = reinterpret_cast<double *>(b);
    b += (size_t)kLossBlocks * sizeof(double);
    w.keys = reinterpret_cast<uint32_t *>(b);
    return GSB_OK;
}

// zt = s + u (u = 0 when initialising), as an order key
__global__ void __launch_bounds__(kThreads) keys_kernel(uint32_t N, const float *__restrict__ opacity_raw,
                                                        const float *__restrict__ u, bool init,
                                                        uint32_t *__restrict__ keys) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= N) return;
    const float zt = __fadd_rn(sigmoid_f(opacity_raw[i]), init ? 0.0f : u[i]);
    keys[i] = sel::float_key(zt);
}

// z = (zt > thr) * zt; update: u = u + (s - z).  k == 0: z = 0 (torch::zeros_like).
__global__ void __launch_bounds__(kThreads) update_kernel(uint32_t N, const float *__restrict__ opacity_raw,
                                                          float *__restrict__ z, float *__restrict__ u, bool init,
                                                          bool zero, const sel::SelectState *__restrict__ st) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= N) return;
    const float s = sigmoid_f(opacity_raw[i]);
    const float u0 = init ? 0.0f : u[i];
    float zi = 0.0f;
    if (!zero) {
        const float thr = sel::key_float(st->prefix);
        const float zt = __fadd_rn(s, u0);
        zi = __fmul_rn(zt > thr ? 1.0f : 0.0f, zt);
    }
    z[i] = zi;
    u[i] = init ? 0.0f : __fadd_rn(u0, __fsub_rn(s, zi));
}

__device__ __forceinline__ double block_sum(double v, double *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int k = 0; k < kThreads / 32; ++k) t += red[k]; // fixed order: deterministic
    return t;
}

struct LossArgs {
    uint32_t N;
    const float *opacity_raw, *z, *u, *rho;
    float *v_opacity, *loss_out;
    double *partials;
    unsigned int *done;
};

__global__ void __launch_bounds__(kThreads) loss_kernel(const LossArgs a) {
    __shared__ double red[kThreads / 32];
    __shared__ bool last;
    const float rho = *a.rho;
    if (rho == 0.0f) { // no loss this iteration (the prune iteration of a captured phase)
        if (blockIdx.x == 0 && threadIdx.x == 0) a.loss_out[0] = 0.0f;
        return;
    }
    double acc = 0.0;
    for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < a.N; i += gridDim.x * kThreads) {
        const float s = sigmoid_f(a.opacity_raw[i]);
        const float diff = __fadd_rn(__fsub_rn(s, a.z[i]), a.u[i]);
        acc += (double)diff * (double)diff;
        // norm / pow backward: rho * diff; sigmoid backward: grad * (1 - y) * y
        const float g = __fmul_rn(__fmul_rn(__fmul_rn(rho, diff), __fsub_rn(1.0f, s)), s);
        a.v_opacity[i] = __fadd_rn(a.v_opacity[i], g);
    }
    const double b = block_sum(acc, red);
    if (threadIdx.x == 0) {
        a.partials[blockIdx.x] = b;
        __threadfence();
        last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double t = 0.0;
    for (uint32_t bb = threadIdx.x; bb < gridDim.x; bb += kThreads) t += ((const volatile double *)a.partials)[bb];
    t = block_sum(t, red);
    if (threadIdx.x == 0) a.loss_out[0] = (float)((double)__fmul_rn(0.5f, rho) * t);
}

static unsigned blocks_for(uint64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

} // namespace sparsity
} // namespace gsb

extern "C" size_t gsb_sparsity_workspace(uint32_t N) { return gsb::sparsity::ws_bytes(N); }

extern "C" int gsb_sparsity_update(uint32_t N, const float *opacity_raw, float *z, float *u, uint32_t k,
                                   int initialize, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::sparsity;
    if (k > N) return GSB_E_INVALID;
    if (N == 0) return GSB_OK;
    if (!opacity_raw || !z || !u) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_carve(N, workspace, workspace_bytes, w)) return rc;
    cudaStream_t s = as_stream(stream);
    const bool init = initialize != 0, zero = k == 0;
    ProfScope ps(init ? "sparsity_initialize" : "sparsity_update", s);
    if (!zero) {
        keys_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, opacity_raw, u, init, w.keys);
        GSB_LAUNCH_CHECK();
        if (int rc = sel::select_kth(w.keys, N, k, w.hist, w.st, s)) return rc;
    }
    update_kernel<<<blocks_for(N), kThreads, 0, s>>>(N, opacity_raw, z, u, init, zero, w.st);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_sparsity_loss(uint32_t N, const float *opacity_raw, const float *z, const float *u,
                                 const float *rho, float *v_opacity, float *loss_out, void *workspace,
                                 size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::sparsity;
    if (!loss_out || !rho) return GSB_E_INVALID;
    cudaStream_t s = as_stream(stream);
    if (N == 0) {
        GSB_CUDA_TRY(cudaMemsetAsync(loss_out, 0, sizeof(float), s));
        return GSB_OK;
    }
    if (!opacity_raw || !z || !u || !v_opacity) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_carve(N, workspace, workspace_bytes, w)) return rc;
    LossArgs a;
    a.N = N; a.opacity_raw = opacity_raw; a.z = z; a.u = u; a.rho = rho; a.v_opacity = v_opacity;
    a.loss_out = loss_out; a.partials = w.partials; a.done = w.done;
    unsigned nb = blocks_for(N);
    if (nb > kLossBlocks) nb = kLossBlocks;
    ProfScope ps("sparsity_loss", s);
    GSB_CUDA_TRY(cudaMemsetAsync(w.done, 0, sizeof(unsigned int), s));
    loss_kernel<<<nb, kThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
