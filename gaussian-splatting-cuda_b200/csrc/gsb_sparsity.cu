// gsb_sparsity.cu -- the ADMM opacity-sparsity phase of the reference's trainer on the device
// (src/training/components/sparsity_optimizer.cpp).  With s = sigmoid(opacity_raw) and k = (int)(prune_ratio * N)
// (the caller's float product):
//   gsb_sparsity_update  initialize (u = 0, z = prune_z(s + u)) or update_state (zt = s + u, z = prune_z(zt),
//                        u += s - z), where prune_z(x) = (x > x_(k)) * x with x_(k) the k-th smallest of x
//                        (sort(x)[k - 1]) and 0 when k == 0.  The select is gsb_select.cuh's: the threshold never
//                        leaves the device.  Elementwise float, bit for bit as torch computes it.
//   gsb_sparsity_loss    0.5 rho ||s - z + u||^2 into a device scalar (reduced deterministically, gsb_reduce.cuh) and
//                        its gradient rho (s - z + u) s (1 - s) added into v_opacity.  rho is read from the device,
//                        so one captured graph serves the whole phase; a zero rho writes a zero loss and leaves the
//                        gradient alone.
// No fast-math; the elementwise arithmetic uses the explicit _rn intrinsics so that nothing is contracted.
#include <cmath>

#include "gsb_common.cuh"
#include "gsb_reduce.cuh"
#include "gsb_select.cuh"

namespace gsb {
namespace sparsity {

constexpr int kThreads = 256;
constexpr uint32_t kLossBlocks = 264;

struct Ws {
    sel::SelectState *st;
    unsigned int *done; // loss ticket
    uint32_t *hist;     // [kPasses * kBins]
    double *partials;   // [kLossBlocks]
    uint32_t *keys;     // [N]
};

// the buffers of a workspace at `base` (null: sizing only); returns its size
static size_t ws_layout(uint32_t N, void *base, Ws &w) {
    WsLayout l{static_cast<char *>(base)};
    w.st = l.carve<sel::SelectState>(1);
    w.done = l.carve<unsigned int>(1);
    w.hist = l.carve<uint32_t>(sel::kHistBytes / sizeof(uint32_t));
    w.partials = l.carve<double>(kLossBlocks);
    w.keys = l.carve<uint32_t>(N);
    return l.bytes;
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

struct LossArgs {
    uint32_t N;
    const float *opacity_raw, *z, *u, *rho;
    float *v_opacity, *loss_out;
    double *partials;
    unsigned int *done;
};

__global__ void __launch_bounds__(kThreads) loss_kernel(const LossArgs a) {
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
    double t[1];
    if (!grid_sum_last<kThreads, 1>({acc}, a.partials, a.done, t)) return;
    if (threadIdx.x == 0) a.loss_out[0] = (float)((double)__fmul_rn(0.5f, rho) * t[0]);
}

} // namespace sparsity
} // namespace gsb

extern "C" size_t gsb_sparsity_workspace(uint32_t N) {
    gsb::sparsity::Ws w;
    return gsb::sparsity::ws_layout(N, nullptr, w);
}

extern "C" int gsb_sparsity_update(uint32_t N, const float *opacity_raw, float *z, float *u, uint32_t k,
                                   int initialize, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::sparsity;
    if (k > N) return GSB_E_INVALID;
    if (N == 0) return GSB_OK;
    if (!opacity_raw || !z || !u) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_check(workspace, workspace_bytes, ws_layout(N, workspace, w))) return rc;
    cudaStream_t s = as_stream(stream);
    const bool init = initialize != 0, zero = k == 0;
    ProfScope ps(init ? "sparsity_initialize" : "sparsity_update", s);
    if (!zero) {
        keys_kernel<<<ceil_div(N, kThreads), kThreads, 0, s>>>(N, opacity_raw, u, init, w.keys);
        GSB_LAUNCH_CHECK();
        if (int rc = sel::select_kth(w.keys, N, k, w.hist, w.st, s)) return rc;
    }
    update_kernel<<<ceil_div(N, kThreads), kThreads, 0, s>>>(N, opacity_raw, z, u, init, zero, w.st);
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
    if (int rc = ws_check(workspace, workspace_bytes, ws_layout(N, workspace, w))) return rc;
    LossArgs a;
    a.N = N; a.opacity_raw = opacity_raw; a.z = z; a.u = u; a.rho = rho; a.v_opacity = v_opacity;
    a.loss_out = loss_out; a.partials = w.partials; a.done = w.done;
    unsigned nb = (unsigned)ceil_div(N, kThreads);
    if (nb > kLossBlocks) nb = kLossBlocks;
    ProfScope ps("sparsity_loss", s);
    GSB_CUDA_TRY(cudaMemsetAsync(w.done, 0, sizeof(unsigned int), s));
    loss_kernel<<<nb, kThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
