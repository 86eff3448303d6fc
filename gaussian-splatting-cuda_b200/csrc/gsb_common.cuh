// gsb_common.cuh -- shared device helpers for the sm_90a 3DGUT hot path.
// No torch, no GLM: plain CUDA C++ with a few inline-PTX wrappers
// (mbarrier, cp.async.bulk, vector red) for the Hopper async-copy (TMA) path.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gsb200.h"

#define GSB_LAUNCH_CHECK()                         \
    do {                                           \
        cudaError_t e__ = cudaPeekAtLastError();   \
        if (e__ != cudaSuccess) return (int)e__;   \
        gsb::count_launch();                       \
    } while (0)

#define GSB_CUDA_TRY(expr)                         \
    do {                                           \
        cudaError_t e__ = (expr);                  \
        if (e__ != cudaSuccess) return (int)e__;   \
    } while (0)

namespace gsb {

// launch counter + opt-in per-kernel event timing (gsb_misc.cu); both are diagnostics only
void count_launch();
struct ProfScope {
    const char *name;
    cudaStream_t stream;
    void *slot;
    ProfScope(const char *name, cudaStream_t stream);
    ~ProfScope();
};

constexpr float kAlphaThreshold = 1.0f / 255.0f; // gsplat/Common.h:53
constexpr float kMaxAlpha = 0.999f;              // RasterizeToPixelsFromWorld3DGSFwd.cu:239
constexpr float kMinTransmittance = 1e-4f;       // RasterizeToPixelsFromWorld3DGSFwd.cu:245

static inline cudaStream_t as_stream(gsb_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

static inline uint32_t bit_width_u32(uint32_t n) { // floor(log2 n) + 1, Intersect.cpp:46-47
    uint32_t b = 0;
    while (n) { ++b; n >>= 1; }
    return b;
}

// ------------------------------------------------------------------------------------------
// tiny fixed-size linear algebra, templated on the scalar so the per-Gaussian set-up can run
// in double (it is cancellation-sensitive, see DESIGN.md) while the per-pixel work is float.
// Matrices are ROW-major math matrices: m[r][c].
// ------------------------------------------------------------------------------------------
template <typename T> struct V3 { T x, y, z; };
template <typename T> struct M3 { T m[3][3]; };

template <typename T> __host__ __device__ inline V3<T> mk3(T x, T y, T z) { return V3<T>{x, y, z}; }
template <typename T> __host__ __device__ inline V3<T> operator+(V3<T> a, V3<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename T> __host__ __device__ inline V3<T> operator-(V3<T> a, V3<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename T> __host__ __device__ inline V3<T> operator*(V3<T> a, T s) { return {a.x * s, a.y * s, a.z * s}; }
template <typename T> __host__ __device__ inline T dot(V3<T> a, V3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> __host__ __device__ inline V3<T> cross(V3<T> a, V3<T> b) {
    return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
template <typename T> __host__ __device__ inline V3<T> mulv(const M3<T> &a, V3<T> v) {
    return {a.m[0][0] * v.x + a.m[0][1] * v.y + a.m[0][2] * v.z,
            a.m[1][0] * v.x + a.m[1][1] * v.y + a.m[1][2] * v.z,
            a.m[2][0] * v.x + a.m[2][1] * v.y + a.m[2][2] * v.z};
}
template <typename T> __host__ __device__ inline V3<T> mulTv(const M3<T> &a, V3<T> v) { // a^T v
    return {a.m[0][0] * v.x + a.m[1][0] * v.y + a.m[2][0] * v.z,
            a.m[0][1] * v.x + a.m[1][1] * v.y + a.m[2][1] * v.z,
            a.m[0][2] * v.x + a.m[1][2] * v.y + a.m[2][2] * v.z};
}
template <typename T> __host__ __device__ inline M3<T> matmul(const M3<T> &a, const M3<T> &b) {
    M3<T> r;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
    return r;
}
template <typename T> __host__ __device__ inline V3<T> col(const M3<T> &a, int j) { return {a.m[0][j], a.m[1][j], a.m[2][j]}; }
template <typename T> __host__ __device__ inline M3<T> inverse3(const M3<T> &a) {
    M3<T> r;
    T c00 = a.m[1][1] * a.m[2][2] - a.m[1][2] * a.m[2][1];
    T c01 = a.m[1][2] * a.m[2][0] - a.m[1][0] * a.m[2][2];
    T c02 = a.m[1][0] * a.m[2][1] - a.m[1][1] * a.m[2][0];
    T det = a.m[0][0] * c00 + a.m[0][1] * c01 + a.m[0][2] * c02;
    T id = T(1) / det;
    r.m[0][0] = c00 * id;
    r.m[0][1] = (a.m[0][2] * a.m[2][1] - a.m[0][1] * a.m[2][2]) * id;
    r.m[0][2] = (a.m[0][1] * a.m[1][2] - a.m[0][2] * a.m[1][1]) * id;
    r.m[1][0] = c01 * id;
    r.m[1][1] = (a.m[0][0] * a.m[2][2] - a.m[0][2] * a.m[2][0]) * id;
    r.m[1][2] = (a.m[0][2] * a.m[1][0] - a.m[0][0] * a.m[1][2]) * id;
    r.m[2][0] = c02 * id;
    r.m[2][1] = (a.m[0][1] * a.m[2][0] - a.m[0][0] * a.m[2][1]) * id;
    r.m[2][2] = (a.m[0][0] * a.m[1][1] - a.m[0][1] * a.m[1][0]) * id;
    return r;
}

// Rotation matrix of a (w,x,y,z) quaternion WITHOUT normalising it (what GLM's mat3_cast does,
// used on the camera pose by gsplat/Cameras.cuh:261-265) ...
template <typename T> __host__ __device__ inline M3<T> rotmat_raw(T w, T x, T y, T z) {
    M3<T> r;
    r.m[0][0] = T(1) - T(2) * (y * y + z * z);
    r.m[0][1] = T(2) * (x * y - w * z);
    r.m[0][2] = T(2) * (x * z + w * y);
    r.m[1][0] = T(2) * (x * y + w * z);
    r.m[1][1] = T(1) - T(2) * (x * x + z * z);
    r.m[1][2] = T(2) * (y * z - w * x);
    r.m[2][0] = T(2) * (x * z - w * y);
    r.m[2][1] = T(2) * (y * z + w * x);
    r.m[2][2] = T(1) - T(2) * (x * x + y * y);
    return r;
}

#ifdef __CUDACC__
// normalised quaternion -> row-major rotation (Utils.cuh:80-102): gsb_quat_to_rotmat, add_noise and the ADC split
__device__ __forceinline__ M3<float> quat_to_rotmat_norm(float w, float x, float y, float z, float max_inv_norm) {
    float inv_norm = rsqrtf(x * x + y * y + z * z + w * w);
    inv_norm = fminf(inv_norm, max_inv_norm);
    return rotmat_raw(w * inv_norm, x * inv_norm, y * inv_norm, z * inv_norm);
}

// torch's float sigmoid on CUDA (IEEE expf, no fast-math): the ADC flags and the sparsifier compare its values
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
#endif

// Camera pose the way the reference derives it (gsplat/Cameras.cuh:33-71): the rotation block
// of the row-major view matrix goes through a float quaternion (GLM quat_cast); t is column 3.
struct CamPose {
    float qw, qx, qy, qz; // quat_cast(R), float32 like the reference
    float tx, ty, tz;
};

__host__ __device__ inline CamPose cam_pose_from_viewmat(const float *v) {
    // R[r][c] = v[r*4+c]
    const float r00 = v[0], r01 = v[1], r02 = v[2];
    const float r10 = v[4], r11 = v[5], r12 = v[6];
    const float r20 = v[8], r21 = v[9], r22 = v[10];
    const float fx = r00 - r11 - r22, fy = r11 - r00 - r22, fz = r22 - r00 - r11, fw = r00 + r11 + r22;
    int bi = 0;
    float fb = fw;
    if (fx > fb) { fb = fx; bi = 1; }
    if (fy > fb) { fb = fy; bi = 2; }
    if (fz > fb) { fb = fz; bi = 3; }
    const float bv = sqrtf(fb + 1.0f) * 0.5f;
    const float mult = 0.25f / bv;
    CamPose p;
    // glm m[c][r] == R[r][c]
    if (bi == 0) { p.qw = bv; p.qx = (r21 - r12) * mult; p.qy = (r02 - r20) * mult; p.qz = (r10 - r01) * mult; }
    else if (bi == 1) { p.qw = (r21 - r12) * mult; p.qx = bv; p.qy = (r10 + r01) * mult; p.qz = (r02 + r20) * mult; }
    else if (bi == 2) { p.qw = (r02 - r20) * mult; p.qx = (r10 + r01) * mult; p.qy = bv; p.qz = (r21 + r12) * mult; }
    else { p.qw = (r10 - r01) * mult; p.qx = (r02 + r20) * mult; p.qy = (r21 + r12) * mult; p.qz = bv; }
    p.tx = v[3]; p.ty = v[7]; p.tz = v[11];
    return p;
}

// ------------------------------------------------------------------------------------------
// PTX wrappers (sm_90a): mbarrier + bulk async copy (TMA unit, non-tensor form).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    // make the init visible to the async (TMA) proxy
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-byte aligned.
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared -> global bulk store (bulk async-group completion)
__device__ __forceinline__ void bulk_s2g(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// fire-and-forget float reductions to global memory
__device__ __forceinline__ void red_add_f32(float *addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_ex2(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// ---- fp32 pairs: two values carried side by side (the SSIM window sums of gsb_loss.cu) ----
// Each pair operation is two scalar IEEE-rn FFMA / FMUL / FADD (the explicit __f*_rn intrinsics keep
// ptxas from contracting or reassociating them).
struct f2 {
    float lo, hi;
};
__device__ __forceinline__ f2 f2_make(float lo, float hi) { return f2{lo, hi}; }
__device__ __forceinline__ f2 f2_bc(float a) { return f2{a, a}; }
__device__ __forceinline__ float f2_lo(f2 a) { return a.lo; }
__device__ __forceinline__ float f2_hi(f2 a) { return a.hi; }
__device__ __forceinline__ f2 f2_fma(f2 a, f2 b, f2 c) { return f2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ f2 f2_mul(f2 a, f2 b) { return f2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 f2_add(f2 a, f2 b) { return f2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }

} // namespace gsb
