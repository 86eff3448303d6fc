// gsb_misc.cu -- link-surface operators used by the densification strategies, plus library
// housekeeping.  References: gsplat/QuatToRotmatCUDA.cu:14-39 (gsplat::quats_to_rotmats, caller
// default_strategy.cpp:96), gsplat/RelocationCUDA.cu:12-43 (gsplat::relocation, mcmc.cpp:153,231),
// gsplat/RelocationCUDA.cu:86-144 (gsplat::add_noise, mcmc.cpp:360).
#include <atomic>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "gsb_common.cuh"
#include "gsb_relocation.cuh"

namespace gsb {

// ---- diagnostics: launch counter and opt-in event timing --------------------------------------
// Off by default; the compute path holds no mutable state.  bench.py enables it to time the
// dominant kernel with CUDA events on the launching stream (roofline.achieved).
static std::atomic<uint64_t> g_launches{0};
static std::atomic<int> g_prof_on{0};
struct ProfRec { std::string name; cudaEvent_t e0, e1; };
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof;

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

ProfScope::ProfScope(const char *n, cudaStream_t s) : name(n), stream(s), slot(nullptr) {
    if (!g_prof_on.load(std::memory_order_relaxed)) return;
    ProfRec *r = new ProfRec();
    r->name = n;
    cudaEventCreate(&r->e0);
    cudaEventCreate(&r->e1);
    cudaEventRecord(r->e0, s);
    slot = r;
}
ProfScope::~ProfScope() {
    if (!slot) return;
    ProfRec *r = static_cast<ProfRec *>(slot);
    cudaEventRecord(r->e1, stream);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof.push_back(*r);
    delete r;
}

constexpr int kMiscThreads = 256;

// quat_to_rotmat_norm (gsb_common.cuh) is shared with the ADC split (gsb_adc.cu)
__global__ void __launch_bounds__(kMiscThreads) quat_to_rotmat_kernel(uint32_t N, const float *__restrict__ quats,
                                                                       float *__restrict__ rotmats) {
    const uint32_t i = blockIdx.x * kMiscThreads + threadIdx.x;
    if (i >= N) return;
    const float4 q = reinterpret_cast<const float4 *>(quats)[i];
    const M3<float> R = quat_to_rotmat_norm(q.x, q.y, q.z, q.w, __int_as_float(0x7f800000));
    float *o = rotmats + (size_t)i * 9;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) o[r * 3 + c] = R.m[r][c];
}

// gsplat::relocation (RelocationCUDA.cu:12-43); the body is relocation_one (gsb_relocation.cuh).
__global__ void __launch_bounds__(kMiscThreads) relocation_kernel(uint32_t N, const float *__restrict__ opacities,
                                                                   const float *__restrict__ scales,
                                                                   const int32_t *__restrict__ ratios,
                                                                   const float *__restrict__ binoms, int32_t n_max,
                                                                   float *__restrict__ new_opacities,
                                                                   float *__restrict__ new_scales) {
    const uint32_t g = blockIdx.x * kMiscThreads + threadIdx.x;
    if (g >= N) return;
    const float grow = relocation_one(opacities[g], ratios[g], binoms, n_max, &new_opacities[g]);
    new_scales[(size_t)g * 3] = grow * scales[(size_t)g * 3];
    new_scales[(size_t)g * 3 + 1] = grow * scales[(size_t)g * 3 + 1];
    new_scales[(size_t)g * 3 + 2] = grow * scales[(size_t)g * 3 + 2];
}

// kLrOnDevice: the rate is *lr_dev * lr_scale, read at run time (gsb_mcmc_add_noise), so a captured CUDA graph
// follows the learning-rate schedule; otherwise it is the launch argument current_lr (gsb_add_noise).
template <bool kLrOnDevice>
__global__ void __launch_bounds__(kMiscThreads) add_noise_kernel(uint32_t N, const float *__restrict__ raw_opacities,
                                                                  const float *__restrict__ raw_scales,
                                                                  const float *__restrict__ raw_quats,
                                                                  const float *__restrict__ noise,
                                                                  float *__restrict__ means, float current_lr,
                                                                  const float *__restrict__ lr_dev, float lr_scale) {
    const uint32_t idx = blockIdx.x * kMiscThreads + threadIdx.x;
    if (idx >= N) return;
    if (kLrOnDevice) current_lr = __ldg(lr_dev) * lr_scale; // mcmc.cpp:353: (float)lr * _noise_lr
    const size_t i3 = (size_t)idx * 3;
    const float e0 = expf(2.f * raw_scales[i3]), e1 = expf(2.f * raw_scales[i3 + 1]), e2 = expf(2.f * raw_scales[i3 + 2]);
    const float4 q = reinterpret_cast<const float4 *>(raw_quats)[idx];
    const M3<float> R = quat_to_rotmat_norm(q.x, q.y, q.z, q.w, 1e12f); // "match torch normalize" (:88)
    const V3<float> nz = {noise[i3], noise[i3 + 1], noise[i3 + 2]};
    // covariance * noise = R diag(e) R^T noise
    V3<float> tmp = mulTv(R, nz);
    tmp.x *= e0; tmp.y *= e1; tmp.z *= e2;
    const V3<float> tn = mulv(R, tmp);
    const float opacity = 1.0f / (1.0f + expf(-raw_opacities[idx]));
    const float op_sigmoid = 1.0f / (1.0f + expf(100.f * opacity - 0.5f));
    const float nf = current_lr * op_sigmoid;
    means[i3] += nf * tn.x;
    means[i3 + 1] += nf * tn.y;
    means[i3 + 2] += nf * tn.z;
}

} // namespace gsb

extern "C" int gsb_quat_to_rotmat(uint32_t N, const float *quats, float *rotmats, gsb_stream_t stream) {
    if (N == 0) return GSB_OK;
    if (!quats || !rotmats) return GSB_E_INVALID;
    gsb::quat_to_rotmat_kernel<<<(N + gsb::kMiscThreads - 1) / gsb::kMiscThreads, gsb::kMiscThreads, 0,
                                 gsb::as_stream(stream)>>>(N, quats, rotmats);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_relocation(uint32_t N, const float *opacities, const float *scales, const int32_t *ratios,
                              const float *binoms, int32_t n_max, float *new_opacities, float *new_scales,
                              gsb_stream_t stream) {
    if (N == 0) return GSB_OK;
    if (!opacities || !scales || !ratios || !binoms || !new_opacities || !new_scales) return GSB_E_INVALID;
    gsb::relocation_kernel<<<(N + gsb::kMiscThreads - 1) / gsb::kMiscThreads, gsb::kMiscThreads, 0,
                             gsb::as_stream(stream)>>>(N, opacities, scales, ratios, binoms, n_max, new_opacities,
                                                       new_scales);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_add_noise(uint32_t N, const float *raw_opacities, const float *raw_scales, const float *raw_quats,
                             const float *noise, float *means, float current_lr, gsb_stream_t stream) {
    if (N == 0) return GSB_OK;
    if (!raw_opacities || !raw_scales || !raw_quats || !noise || !means) return GSB_E_INVALID;
    gsb::add_noise_kernel<false><<<(N + gsb::kMiscThreads - 1) / gsb::kMiscThreads, gsb::kMiscThreads, 0,
                                   gsb::as_stream(stream)>>>(N, raw_opacities, raw_scales, raw_quats, noise, means,
                                                             current_lr, nullptr, 0.f);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_mcmc_add_noise(uint32_t N, const float *raw_opacities, const float *raw_scales,
                                  const float *raw_quats, const float *noise, float *means, const float *lr,
                                  float lr_scale, gsb_stream_t stream) {
    if (N == 0) return GSB_OK;
    if (!raw_opacities || !raw_scales || !raw_quats || !noise || !means || !lr) return GSB_E_INVALID;
    if (reinterpret_cast<uintptr_t>(raw_quats) & 15) return GSB_E_INVALID;
    gsb::add_noise_kernel<true><<<(N + gsb::kMiscThreads - 1) / gsb::kMiscThreads, gsb::kMiscThreads, 0,
                                  gsb::as_stream(stream)>>>(N, raw_opacities, raw_scales, raw_quats, noise, means,
                                                            0.f, lr, lr_scale);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" const char *gsb_error_string(int code) {
    switch (code) {
    case GSB_OK: return "ok";
    case GSB_E_INVALID: return "invalid argument";
    case GSB_E_UNSUPPORTED: return "configuration not supported by the CUDA backend (see DESIGN.md, out of scope)";
    case GSB_E_WORKSPACE: return "workspace too small or misaligned";
    default: break;
    }
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "unknown error";
}

extern "C" int gsb_version(void) { return 100; }

extern "C" uint64_t gsb_launch_count(void) { return gsb::g_launches.load(); }

extern "C" void gsb_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(gsb::g_prof_mu);
    for (auto &r : gsb::g_prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    gsb::g_prof.clear();
    gsb::g_prof_on.store(on ? 1 : 0);
}

// Sum of the recorded durations of kernel `name` since gsb_profile_enable(1); synchronises on the
// recorded events.  Returns the number of launches found.
extern "C" int gsb_profile_read(const char *name, double *total_ms) {
    std::lock_guard<std::mutex> lk(gsb::g_prof_mu);
    int n = 0;
    double tot = 0.0;
    for (auto &r : gsb::g_prof) {
        if (r.name != name) continue;
        if (cudaEventSynchronize(r.e1) != cudaSuccess) continue;
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) { tot += ms; ++n; }
    }
    if (total_ms) *total_ms = tot;
    return n;
}
