// gsb_sh.cu -- a3/a4: spherical-harmonics colour evaluation and its gradient.
//
// Implements gsplat::spherical_harmonics_fwd / _bwd (reference:
// gsplat/SphericalHarmonicsCUDA.cu:21-110 fwd, :113-371 vjp, :374-481 kernels).
// Real SH basis in Sloan's ordering, degrees 0..4, constants as in the reference.
//
// Design differences from the reference (same results):
//  * one thread per element evaluates the basis ONCE and produces all three channels (the
//    reference runs one thread per channel and re-evaluates the basis three times, reading the
//    coefficient rows at a 12-byte stride);
//  * the backward writes every v_coeffs / v_dirs element itself (zeros where the reference
//    relies on a 192 B/Gaussian memset) and needs no atomics for v_dirs because the three
//    channels live in one thread.
#include "gsb_sh.cuh"

namespace gsb {

constexpr int kShThreads = 128;

template <int DEG>
__global__ void __launch_bounds__(kShThreads) sh_fwd_kernel(uint32_t M, uint32_t K, const float *__restrict__ dirs,
                                                            const float *__restrict__ coeffs,
                                                            const uint8_t *__restrict__ masks,
                                                            float *__restrict__ colors) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    const uint32_t e = blockIdx.x * kShThreads + threadIdx.x;
    if (e >= M) return;
    if (masks != nullptr && !masks[e]) return; // masked rows stay untouched (:391-393)
    float b[NB];
    float x = dirs[(size_t)e * 3], y = dirs[(size_t)e * 3 + 1], z = dirs[(size_t)e * 3 + 2];
    if constexpr (DEG >= 1) {
        const float inorm = rsqrtf(x * x + y * y + z * z);
        x *= inorm; y *= inorm; z *= inorm;
    }
    sh_basis<DEG>(x, y, z, b);
    const float *c = coeffs + (size_t)e * K * 3;
    float r0 = 0.f, r1 = 0.f, r2 = 0.f;
    // a contiguous view may start at any 4-byte offset (e.g. coeffs[1:]): the 128-bit loads need the base aligned too
    if ((K * 3) % 4 == 0 && NB * 3 % 4 == 0 && (reinterpret_cast<uintptr_t>(coeffs) & 15) == 0) {
        // 16-byte aligned rows: 128-bit loads (K = 16, deg 3: twelve LDG.128 per element)
        const float4 *c4 = reinterpret_cast<const float4 *>(c);
        float f[NB * 3];
#pragma unroll
        for (int i = 0; i < NB * 3 / 4; ++i) {
            const float4 v = __ldg(c4 + i);
            f[i * 4] = v.x; f[i * 4 + 1] = v.y; f[i * 4 + 2] = v.z; f[i * 4 + 3] = v.w;
        }
#pragma unroll
        for (int k = 0; k < NB; ++k) {
            r0 += b[k] * f[k * 3]; r1 += b[k] * f[k * 3 + 1]; r2 += b[k] * f[k * 3 + 2];
        }
    } else {
#pragma unroll
        for (int k = 0; k < NB; ++k) {
            r0 += b[k] * __ldg(c + k * 3);
            r1 += b[k] * __ldg(c + k * 3 + 1);
            r2 += b[k] * __ldg(c + k * 3 + 2);
        }
    }
    colors[(size_t)e * 3] = r0;
    colors[(size_t)e * 3 + 1] = r1;
    colors[(size_t)e * 3 + 2] = r2;
}

template <int DEG>
__global__ void __launch_bounds__(kShThreads) sh_bwd_kernel(uint32_t M, uint32_t K, const float *__restrict__ dirs,
                                                            const float *__restrict__ coeffs,
                                                            const uint8_t *__restrict__ masks,
                                                            const float *__restrict__ v_colors,
                                                            float *__restrict__ v_coeffs,
                                                            float *__restrict__ v_dirs) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    const uint32_t e = blockIdx.x * kShThreads + threadIdx.x;
    if (e >= M) return;
    float *vc = v_coeffs + (size_t)e * K * 3;
    const bool active = (masks == nullptr) || masks[e];
    if (!active) {
        for (uint32_t i = 0; i < K * 3; ++i) vc[i] = 0.f;
        if (v_dirs) { v_dirs[(size_t)e * 3] = 0.f; v_dirs[(size_t)e * 3 + 1] = 0.f; v_dirs[(size_t)e * 3 + 2] = 0.f; }
        return;
    }
    float b[NB];
    const float dx = dirs[(size_t)e * 3], dy = dirs[(size_t)e * 3 + 1], dz = dirs[(size_t)e * 3 + 2];
    float x = dx, y = dy, z = dz, inorm = 1.f;
    if constexpr (DEG >= 1) {
        inorm = rsqrtf(dx * dx + dy * dy + dz * dz);
        x *= inorm; y *= inorm; z *= inorm;
    }
    sh_basis<DEG>(x, y, z, b);
    const float g0 = v_colors[(size_t)e * 3], g1 = v_colors[(size_t)e * 3 + 1], g2 = v_colors[(size_t)e * 3 + 2];
    const float *c = coeffs + (size_t)e * K * 3;
    float w[NB];
    if ((K * 3) % 4 == 0 && NB * 3 % 4 == 0 &&
        ((reinterpret_cast<uintptr_t>(coeffs) | reinterpret_cast<uintptr_t>(v_coeffs)) & 15) == 0) {
        float4 *vc4 = reinterpret_cast<float4 *>(vc);
        const float4 *c4 = reinterpret_cast<const float4 *>(c);
        float f[NB * 3], o[NB * 3];
        if (v_dirs) {
#pragma unroll
            for (int i = 0; i < NB * 3 / 4; ++i) {
                const float4 v = __ldg(c4 + i);
                f[i * 4] = v.x; f[i * 4 + 1] = v.y; f[i * 4 + 2] = v.z; f[i * 4 + 3] = v.w;
            }
        }
#pragma unroll
        for (int k = 0; k < NB; ++k) {
            o[k * 3] = b[k] * g0; o[k * 3 + 1] = b[k] * g1; o[k * 3 + 2] = b[k] * g2;
            if (v_dirs) w[k] = g0 * f[k * 3] + g1 * f[k * 3 + 1] + g2 * f[k * 3 + 2];
        }
#pragma unroll
        for (int i = 0; i < NB * 3 / 4; ++i) vc4[i] = make_float4(o[i * 4], o[i * 4 + 1], o[i * 4 + 2], o[i * 4 + 3]);
    } else {
#pragma unroll
        for (int k = 0; k < NB; ++k) {
            vc[k * 3] = b[k] * g0; vc[k * 3 + 1] = b[k] * g1; vc[k * 3 + 2] = b[k] * g2;
            if (v_dirs) w[k] = g0 * __ldg(c + k * 3) + g1 * __ldg(c + k * 3 + 1) + g2 * __ldg(c + k * 3 + 2);
        }
    }
    for (uint32_t i = NB * 3; i < K * 3; ++i) vc[i] = 0.f; // inactive degrees: zero (reference: memset)
    if (v_dirs) {
        float vx = 0.f, vy = 0.f, vz = 0.f;
        if constexpr (DEG >= 1) {
            sh_basis_vjp<DEG>(x, y, z, w, vx, vy, vz);
            const float d = vx * x + vy * y + vz * z;
            vx = (vx - d * x) * inorm; vy = (vy - d * y) * inorm; vz = (vz - d * z) * inorm;
        }
        v_dirs[(size_t)e * 3] = vx; v_dirs[(size_t)e * 3 + 1] = vy; v_dirs[(size_t)e * 3 + 2] = vz;
    }
}

// ------------------------------------------------------------------------------------------
// K == 16 fast path (SH degree <= 3 with the reference's [N,16,3] layout, 192-byte rows).
// Every thread moves ITS OWN 192-byte coefficient row with one TMA bulk copy (global -> shared
// through an mbarrier, shared -> global through a bulk group), so all global traffic is full,
// aligned 32-byte sectors regardless of the 192-byte element stride, and the per-thread shared rows
// are padded to 208 bytes: float4 slot (13 t + i) mod 8 is conflict-free for 8 consecutive lanes.
// ------------------------------------------------------------------------------------------
constexpr int kRow16 = 48;        // floats per row
constexpr int kRowStride16 = 52;  // padded row stride in floats (208 B)

template <int DEG>
__global__ void __launch_bounds__(kShThreads) sh_fwd_k16_kernel(uint32_t M, const float *__restrict__ dirs,
                                                                const float *__restrict__ coeffs,
                                                                const uint8_t *__restrict__ masks,
                                                                float *__restrict__ colors) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    extern __shared__ __align__(128) float s_rows[]; // [kShThreads][kRowStride16]
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t tid = threadIdx.x;
    const uint32_t e = blockIdx.x * kShThreads + tid;
    const bool active = (e < M) && (masks == nullptr || masks[e]);
    if (tid == 0) { mbar_init(&s_bar, kShThreads); mbar_fence_init(); }
    __syncthreads();
    float *row = s_rows + tid * kRowStride16;
    constexpr uint32_t kInBytes = (NB * 12 + 15) / 16 * 16; // only the active degrees' bytes
    if (active) {
        mbar_arrive_expect_tx(&s_bar, kInBytes);
        bulk_g2s(row, coeffs + (size_t)e * kRow16, kInBytes, &s_bar);
    } else {
        mbar_arrive(&s_bar);
    }
    float b[NB];
    float x = 0.f, y = 0.f, z = 1.f;
    if (active) { x = dirs[(size_t)e * 3]; y = dirs[(size_t)e * 3 + 1]; z = dirs[(size_t)e * 3 + 2]; }
    if constexpr (DEG >= 1) {
        const float inorm = rsqrtf(x * x + y * y + z * z);
        x *= inorm; y *= inorm; z *= inorm;
    }
    sh_basis<DEG>(x, y, z, b);
    mbar_wait(&s_bar, 0);
    if (!active) return; // masked rows stay untouched
    float r0 = 0.f, r1 = 0.f, r2 = 0.f;
    const float4 *r4 = reinterpret_cast<const float4 *>(row);
    float f[(NB * 3 + 3) / 4 * 4];
#pragma unroll
    for (int i = 0; i < (NB * 3 + 3) / 4; ++i) {
        const float4 v = r4[i];
        f[i * 4] = v.x; f[i * 4 + 1] = v.y; f[i * 4 + 2] = v.z; f[i * 4 + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < NB; ++k) { r0 += b[k] * f[k * 3]; r1 += b[k] * f[k * 3 + 1]; r2 += b[k] * f[k * 3 + 2]; }
    colors[(size_t)e * 3] = r0; colors[(size_t)e * 3 + 1] = r1; colors[(size_t)e * 3 + 2] = r2;
}

template <int DEG>
__global__ void __launch_bounds__(kShThreads) sh_bwd_k16_kernel(uint32_t M, const float *__restrict__ dirs,
                                                                const float *__restrict__ coeffs,
                                                                const uint8_t *__restrict__ masks,
                                                                const float *__restrict__ v_colors,
                                                                float *__restrict__ v_coeffs,
                                                                float *__restrict__ v_dirs) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    extern __shared__ __align__(128) float s_rows[]; // in rows [T][52] then out rows [T][52]
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t tid = threadIdx.x;
    const uint32_t e = blockIdx.x * kShThreads + tid;
    const bool inside = e < M;
    const bool active = inside && (masks == nullptr || masks[e]);
    const bool need_in = active && (v_dirs != nullptr) && (DEG >= 1);
    if (tid == 0) { mbar_init(&s_bar, kShThreads); mbar_fence_init(); }
    __syncthreads();
    float *row_in = s_rows + tid * kRowStride16;
    float *row_out = s_rows + (kShThreads + tid) * kRowStride16;
    constexpr uint32_t kInBytes = (NB * 12 + 15) / 16 * 16;
    if (need_in) {
        mbar_arrive_expect_tx(&s_bar, kInBytes);
        bulk_g2s(row_in, coeffs + (size_t)e * kRow16, kInBytes, &s_bar);
    } else {
        mbar_arrive(&s_bar);
    }
    float b[NB];
    float x = 0.f, y = 0.f, z = 1.f, inorm = 1.f, g0 = 0.f, g1 = 0.f, g2 = 0.f;
    if (active) {
        x = dirs[(size_t)e * 3]; y = dirs[(size_t)e * 3 + 1]; z = dirs[(size_t)e * 3 + 2];
        g0 = v_colors[(size_t)e * 3]; g1 = v_colors[(size_t)e * 3 + 1]; g2 = v_colors[(size_t)e * 3 + 2];
    }
    if constexpr (DEG >= 1) {
        inorm = rsqrtf(x * x + y * y + z * z);
        x *= inorm; y *= inorm; z *= inorm;
    }
    sh_basis<DEG>(x, y, z, b);
    // v_coeffs row: b_k * g_c for the active degrees, zeros elsewhere (and for masked elements)
    float4 *o4 = reinterpret_cast<float4 *>(row_out);
    {
        float o[kRow16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const float bk = (k < NB) ? b[k < NB ? k : 0] : 0.f;
            o[k * 3] = bk * g0; o[k * 3 + 1] = bk * g1; o[k * 3 + 2] = bk * g2;
        }
#pragma unroll
        for (int i = 0; i < kRow16 / 4; ++i) o4[i] = make_float4(o[i * 4], o[i * 4 + 1], o[i * 4 + 2], o[i * 4 + 3]);
    }
    if (inside) {
        fence_proxy_async(); // this thread's generic-proxy writes -> visible to its bulk store
        bulk_s2g(v_coeffs + (size_t)e * kRow16, row_out, kRow16 * 4);
        bulk_commit();
    }
    mbar_wait(&s_bar, 0);
    if (inside && v_dirs != nullptr) {
        float vx = 0.f, vy = 0.f, vz = 0.f;
        if constexpr (DEG >= 1) {
            if (active) {
                float w[NB];
                const float4 *r4 = reinterpret_cast<const float4 *>(row_in);
                float f[(NB * 3 + 3) / 4 * 4];
#pragma unroll
                for (int i = 0; i < (NB * 3 + 3) / 4; ++i) {
                    const float4 v = r4[i];
                    f[i * 4] = v.x; f[i * 4 + 1] = v.y; f[i * 4 + 2] = v.z; f[i * 4 + 3] = v.w;
                }
#pragma unroll
                for (int k = 0; k < NB; ++k) w[k] = g0 * f[k * 3] + g1 * f[k * 3 + 1] + g2 * f[k * 3 + 2];
                sh_basis_vjp<DEG>(x, y, z, w, vx, vy, vz);
                const float d = vx * x + vy * y + vz * z;
                vx = (vx - d * x) * inorm; vy = (vy - d * y) * inorm; vz = (vz - d * z) * inorm;
            }
        }
        v_dirs[(size_t)e * 3] = vx; v_dirs[(size_t)e * 3 + 1] = vy; v_dirs[(size_t)e * 3 + 2] = vz;
    }
    if (inside) bulk_wait_read_all(); // the row must stay in shared memory until the bulk store has read it
}

// ------------------------------------------------------------------------------------------
// Multi-view SH backward (the multi-GPU exchange step, SURVEY.md 8e).  The SH gradient of one view is the
// rank-1 row  v_coeffs[n] = Y(dir_v(n)) (x) v_color_v[n]  -- 192 B per Gaussian made from 12 B.  Ranks
// therefore exchange the 12-byte colour gradients (all-gather) instead of all-reducing the 192-byte rows,
// and every rank expands and sums all V views here: one thread per Gaussian, the coefficient row comes in
// and the summed gradient row goes out with one TMA bulk copy each (K = 16), views whose colour gradient is
// exactly zero (Gaussian not blended in that view) cost one 12-byte load.  The gradient w.r.t. the view
// directions is chained to the Gaussian's position (dir = mean - campos) and ACCUMULATED into v_means.
// ------------------------------------------------------------------------------------------
// kTable: view v's colour gradients and camera position are read through a table of per-view pointers instead of
// from one stacked tensor -- the pointers may be PEER memory (NVLink-mapped buffers of the other ranks,
// gsb_sh_bwd_views_peer): the all-gather of the exchange step then happens inside this kernel, overlapped with the
// expansion, and the gathered tensor never exists.
constexpr int kMaxViewPtrs = 16;
struct ViewTable {
    const float *vc[kMaxViewPtrs]; // [M,3] each
    const float *cp[kMaxViewPtrs]; // [3] each
};

template <int DEG, bool kRow16Path, bool kTable>
__global__ void __launch_bounds__(kShThreads) sh_bwd_views_kernel(uint32_t M, uint32_t K, uint32_t V,
                                                                  const float *__restrict__ means,
                                                                  const float *__restrict__ campos,
                                                                  const float *__restrict__ coeffs,
                                                                  const float *__restrict__ v_colors,
                                                                  float *__restrict__ v_coeffs,
                                                                  float *__restrict__ v_means, const ViewTable tbl) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    extern __shared__ __align__(128) float s_rows[]; // row path: in rows [T][52] then out rows [T][52]
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ float s_cp[kMaxViewPtrs * 3];
    const uint32_t tid = threadIdx.x;
    if constexpr (kTable) { // camera positions once per CTA (remote loads), not once per thread and view
        if (tid < V * 3) s_cp[tid] = tbl.cp[tid / 3][tid % 3];
        __syncthreads();
    }
    const uint32_t e = blockIdx.x * kShThreads + tid;
    const bool inside = e < M;
    float *row_in = nullptr, *row_out = nullptr;
    if constexpr (kRow16Path) {
        if (tid == 0) { mbar_init(&s_bar, kShThreads); mbar_fence_init(); }
        __syncthreads();
        row_in = s_rows + tid * kRowStride16;
        row_out = s_rows + (kShThreads + tid) * kRowStride16;
        constexpr uint32_t kInBytes = (NB * 12 + 15) / 16 * 16;
        if (inside && DEG >= 1) {
            mbar_arrive_expect_tx(&s_bar, kInBytes);
            bulk_g2s(row_in, coeffs + (size_t)e * kRow16, kInBytes, &s_bar);
        } else {
            mbar_arrive(&s_bar);
        }
    }
    float acc[NB * 3];
#pragma unroll
    for (int i = 0; i < NB * 3; ++i) acc[i] = 0.f;
    float mx = 0.f, my = 0.f, mz = 0.f, vmx = 0.f, vmy = 0.f, vmz = 0.f;
    if (inside) { mx = means[(size_t)e * 3]; my = means[(size_t)e * 3 + 1]; mz = means[(size_t)e * 3 + 2]; }
    if constexpr (kRow16Path) mbar_wait(&s_bar, 0);
    if (inside) {
        float n0 = 0.f, n1 = 0.f, n2 = 0.f; // table path: the next view's colours are in flight during this view's math
        if constexpr (kTable) {
            if (V > 0) { const float *gc = tbl.vc[0] + (size_t)e * 3; n0 = gc[0]; n1 = gc[1]; n2 = gc[2]; }
        }
        for (uint32_t v = 0; v < V; ++v) {
            float g0, g1, g2;
            const float *cpv;
            if constexpr (kTable) {
                g0 = n0; g1 = n1; g2 = n2;
                if (v + 1 < V) { const float *gc = tbl.vc[v + 1] + (size_t)e * 3; n0 = gc[0]; n1 = gc[1]; n2 = gc[2]; }
                cpv = s_cp + v * 3;
            } else {
                const float *gc = v_colors + ((size_t)v * M + e) * 3;
                g0 = gc[0]; g1 = gc[1]; g2 = gc[2];
                cpv = campos + v * 3;
            }
            if (g0 == 0.f && g1 == 0.f && g2 == 0.f) continue;
            float x = mx - cpv[0], y = my - cpv[1], z = mz - cpv[2], inorm = 1.f;
            if constexpr (DEG >= 1) {
                inorm = rsqrtf(x * x + y * y + z * z);
                x *= inorm; y *= inorm; z *= inorm;
            }
            float b[NB];
            sh_basis<DEG>(x, y, z, b);
#pragma unroll
            for (int k = 0; k < NB; ++k) {
                acc[k * 3] = fmaf(b[k], g0, acc[k * 3]);
                acc[k * 3 + 1] = fmaf(b[k], g1, acc[k * 3 + 1]);
                acc[k * 3 + 2] = fmaf(b[k], g2, acc[k * 3 + 2]);
            }
            if constexpr (DEG >= 1) {
                float w[NB];
#pragma unroll
                for (int k = 0; k < NB; ++k) {
                    float f0, f1, f2;
                    if constexpr (kRow16Path) { f0 = row_in[k * 3]; f1 = row_in[k * 3 + 1]; f2 = row_in[k * 3 + 2]; }
                    else {
                        const float *f = coeffs + ((size_t)e * K + k) * 3;
                        f0 = f[0]; f1 = f[1]; f2 = f[2];
                    }
                    w[k] = g0 * f0 + g1 * f1 + g2 * f2;
                }
                float vx = 0.f, vy = 0.f, vz = 0.f;
                sh_basis_vjp<DEG>(x, y, z, w, vx, vy, vz);
                const float d = vx * x + vy * y + vz * z;
                vmx += (vx - d * x) * inorm; vmy += (vy - d * y) * inorm; vmz += (vz - d * z) * inorm;
            }
        }
    }
    if constexpr (kRow16Path) {
        float4 *o4 = reinterpret_cast<float4 *>(row_out);
#pragma unroll
        for (int i = 0; i < kRow16 / 4; ++i) {
            float t[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) t[j] = (i * 4 + j < NB * 3) ? acc[(i * 4 + j < NB * 3) ? i * 4 + j : 0] : 0.f;
            o4[i] = make_float4(t[0], t[1], t[2], t[3]);
        }
        if (inside) {
            fence_proxy_async();
            bulk_s2g(v_coeffs + (size_t)e * kRow16, row_out, kRow16 * 4);
            bulk_commit();
        }
    } else if (inside) {
        float *o = v_coeffs + (size_t)e * K * 3;
        for (uint32_t k = 0; k < K; ++k)
            for (int c = 0; c < 3; ++c) o[k * 3 + c] = (k < (uint32_t)NB) ? acc[(k < (uint32_t)NB ? k : 0) * 3 + c] : 0.f;
    }
    if (inside && DEG >= 1) {
        v_means[(size_t)e * 3] += vmx; v_means[(size_t)e * 3 + 1] += vmy; v_means[(size_t)e * 3 + 2] += vmz;
    }
    if constexpr (kRow16Path) {
        if (inside) bulk_wait_read_all();
    }
}

static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

} // namespace gsb

extern "C" int gsb_sh_fwd(uint32_t M, uint32_t K, uint32_t degree, const float *dirs, const float *coeffs,
                          const uint8_t *masks, float *colors, gsb_stream_t stream) {
    if (M == 0) return GSB_OK;
    if (!dirs || !coeffs || !colors) return GSB_E_INVALID;
    if (degree > 4 || (degree + 1) * (degree + 1) > K) return GSB_E_INVALID;
    const dim3 grid((M + gsb::kShThreads - 1) / gsb::kShThreads);
    cudaStream_t s = gsb::as_stream(stream);
    gsb::ProfScope ps("sh_fwd", s);
    if (K == 16 && degree >= 1 && degree <= 3 && gsb::aligned16(coeffs)) {
        const size_t smem = (size_t)gsb::kShThreads * gsb::kRowStride16 * 4;
        switch (degree) {
        case 1: gsb::sh_fwd_k16_kernel<1><<<grid, gsb::kShThreads, smem, s>>>(M, dirs, coeffs, masks, colors); break;
        case 2: gsb::sh_fwd_k16_kernel<2><<<grid, gsb::kShThreads, smem, s>>>(M, dirs, coeffs, masks, colors); break;
        default: gsb::sh_fwd_k16_kernel<3><<<grid, gsb::kShThreads, smem, s>>>(M, dirs, coeffs, masks, colors); break;
        }
        GSB_LAUNCH_CHECK();
        return GSB_OK;
    }
    switch (degree) {
    case 0: gsb::sh_fwd_kernel<0><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, colors); break;
    case 1: gsb::sh_fwd_kernel<1><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, colors); break;
    case 2: gsb::sh_fwd_kernel<2><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, colors); break;
    case 3: gsb::sh_fwd_kernel<3><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, colors); break;
    default: gsb::sh_fwd_kernel<4><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, colors); break;
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_sh_bwd(uint32_t M, uint32_t K, uint32_t degree, const float *dirs, const float *coeffs,
                          const uint8_t *masks, const float *v_colors, float *v_coeffs, float *v_dirs,
                          gsb_stream_t stream) {
    if (M == 0) return GSB_OK;
    if (!dirs || !coeffs || !v_colors || !v_coeffs) return GSB_E_INVALID;
    if (degree > 4 || (degree + 1) * (degree + 1) > K) return GSB_E_INVALID;
    const dim3 grid((M + gsb::kShThreads - 1) / gsb::kShThreads);
    cudaStream_t s = gsb::as_stream(stream);
    gsb::ProfScope ps("sh_bwd", s);
    if (K == 16 && degree <= 3 && gsb::aligned16(coeffs) && gsb::aligned16(v_coeffs)) {
        const size_t smem = (size_t)2 * gsb::kShThreads * gsb::kRowStride16 * 4; // 53 248 B
        #define GSB_SH_BWD16(D)                                                                                        \
            cudaFuncSetAttribute(gsb::sh_bwd_k16_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   \
            gsb::sh_bwd_k16_kernel<D><<<grid, gsb::kShThreads, smem, s>>>(M, dirs, coeffs, masks, v_colors, v_coeffs, v_dirs)
        switch (degree) {
        case 0: GSB_SH_BWD16(0); break;
        case 1: GSB_SH_BWD16(1); break;
        case 2: GSB_SH_BWD16(2); break;
        default: GSB_SH_BWD16(3); break;
        }
        #undef GSB_SH_BWD16
        GSB_LAUNCH_CHECK();
        return GSB_OK;
    }
    switch (degree) {
    case 0: gsb::sh_bwd_kernel<0><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, v_colors, v_coeffs, v_dirs); break;
    case 1: gsb::sh_bwd_kernel<1><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, v_colors, v_coeffs, v_dirs); break;
    case 2: gsb::sh_bwd_kernel<2><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, v_colors, v_coeffs, v_dirs); break;
    case 3: gsb::sh_bwd_kernel<3><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, v_colors, v_coeffs, v_dirs); break;
    default: gsb::sh_bwd_kernel<4><<<grid, gsb::kShThreads, 0, s>>>(M, K, dirs, coeffs, masks, v_colors, v_coeffs, v_dirs); break;
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

namespace gsb {
template <bool kTable>
static int sh_bwd_views_launch(uint32_t M, uint32_t K, uint32_t degree, uint32_t V, const float *means,
                               const float *campos, const float *coeffs, const float *v_colors, float *v_coeffs,
                               float *v_means, const ViewTable &tbl, cudaStream_t s) {
    const dim3 grid((M + kShThreads - 1) / kShThreads);
    ProfScope ps("sh_bwd_views", s);
    if (K == 16 && degree <= 3 && aligned16(coeffs) && aligned16(v_coeffs)) {
        const size_t smem = (size_t)2 * kShThreads * kRowStride16 * 4;
        #define GSB_SH_VIEWS16(D)                                                                                      \
            cudaFuncSetAttribute(sh_bwd_views_kernel<D, true, kTable>, cudaFuncAttributeMaxDynamicSharedMemorySize,    \
                                 (int)smem);                                                                           \
            sh_bwd_views_kernel<D, true, kTable><<<grid, kShThreads, smem, s>>>(M, K, V, means, campos, coeffs,        \
                                                                                v_colors, v_coeffs, v_means, tbl)
        switch (degree) {
        case 0: GSB_SH_VIEWS16(0); break;
        case 1: GSB_SH_VIEWS16(1); break;
        case 2: GSB_SH_VIEWS16(2); break;
        default: GSB_SH_VIEWS16(3); break;
        }
        #undef GSB_SH_VIEWS16
        GSB_LAUNCH_CHECK();
        return GSB_OK;
    }
    #define GSB_SH_VIEWS(D)                                                                                            \
        sh_bwd_views_kernel<D, false, kTable><<<grid, kShThreads, 0, s>>>(M, K, V, means, campos, coeffs, v_colors,    \
                                                                          v_coeffs, v_means, tbl)
    switch (degree) {
    case 0: GSB_SH_VIEWS(0); break;
    case 1: GSB_SH_VIEWS(1); break;
    case 2: GSB_SH_VIEWS(2); break;
    case 3: GSB_SH_VIEWS(3); break;
    default: GSB_SH_VIEWS(4); break;
    }
    #undef GSB_SH_VIEWS
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
} // namespace gsb

extern "C" int gsb_sh_bwd_views(uint32_t M, uint32_t K, uint32_t degree, uint32_t V, const float *means,
                                const float *campos, const float *coeffs, const float *v_colors, float *v_coeffs,
                                float *v_means, gsb_stream_t stream) {
    if (M == 0) return GSB_OK;
    if (!means || !coeffs || !v_coeffs || !v_means || (V > 0 && (!campos || !v_colors))) return GSB_E_INVALID;
    if (degree > 4 || (degree + 1) * (degree + 1) > K) return GSB_E_INVALID;
    gsb::ViewTable tbl = {};
    return gsb::sh_bwd_views_launch<false>(M, K, degree, V, means, campos, coeffs, v_colors, v_coeffs, v_means, tbl,
                                           gsb::as_stream(stream));
}

extern "C" int gsb_sh_bwd_views_peer(uint32_t M, uint32_t K, uint32_t degree, uint32_t V, const float *means,
                                     const float *const *campos_views, const float *coeffs,
                                     const float *const *v_colors_views, float *v_coeffs, float *v_means,
                                     gsb_stream_t stream) {
    if (M == 0) return GSB_OK;
    if (!means || !coeffs || !v_coeffs || !v_means || (V > 0 && (!campos_views || !v_colors_views))) return GSB_E_INVALID;
    if (degree > 4 || (degree + 1) * (degree + 1) > K) return GSB_E_INVALID;
    if (V > (uint32_t)gsb::kMaxViewPtrs) return GSB_E_UNSUPPORTED;
    gsb::ViewTable tbl = {};
    for (uint32_t v = 0; v < V; ++v) {
        if (!campos_views[v] || !v_colors_views[v]) return GSB_E_INVALID;
        tbl.vc[v] = v_colors_views[v];
        tbl.cp[v] = campos_views[v];
    }
    return gsb::sh_bwd_views_launch<true>(M, K, degree, V, means, nullptr, coeffs, nullptr, v_coeffs, v_means, tbl,
                                          gsb::as_stream(stream));
}
