// gsb_fastgs.cu -- SURVEY.md 8 f4: the reference's default rasterizer ("fastgs": EWA splatting of 2-D conics) on the
// blend engine of this library.
//
// Replaces fast_gs::rasterization::forward / backward (reference: fastgs/rasterization/src/forward.cu:15-199,
// src/backward.cu:14-116, include/kernels_forward.cuh, include/kernels_backward.cuh, include/kernel_utils.cuh) behind the
// same API (rasterization_api.h:25-75 -> include/fastgs/rasterization_api.h, shim/FastGs.cpp).
//
// The reference runs: preprocess -> CUB depth sort of the visible primitives -> instance creation with the exact tile
// test -> CUB sort of all instances by tile -> blend (one thread per pixel; the blend state of every pixel is written out
// every 32 primitives: 16 B x 256 pixels per "bucket") -> bucket-parallel backward (one lane per primitive, 9 atomics per
// lane and bucket) -> preprocess backward.  Three host read-backs size its buffers.
//
// Here an EWA primitive is just a blend record whose denominator form is the constant 1 (gsb_raster.cuh), so the path
// reuses the from-world machinery end to end:
//   fgs_front_kernel   one thread per primitive: cull, covariance, EWA projection, conic, opacity-aware tile bounds and
//                      the EXACT tile count (gsb_ewa.cuh), SH colour straight from sh0 / shN, the 64-byte record; zeroes
//                      the primitive's gradient-moment row.
//   isect_plan_ewa     depth radix sort of the N primitives, run table, per-chunk tile histogram with the tile test,
//                      column scan: closed tile offsets and the instance count (one host read-back, which the API's
//                      exactly-sized instance buffer forces).
//   isect_emit_ewa     instances land directly in their final (tile, depth) slots; no instance is ever sorted.
//   raster_*_kernel<false, true>   blend forward / backward on packed fp32 pairs; backward keeps 9 moments per primitive
//                      (sum of g {1, x, y, x^2, xy, y^2} and the colour gradient) -- no per-bucket state is stored.
//   fgs_back_kernel    one thread per primitive: moments -> (mean2d, conic, opacity, colour) gradients -> the chain rule of
//                      kernels_backward.cuh:18-257 to the raw parameters, SH backward written directly into the sh0 / shN
//                      gradient layouts, optional w2c gradient and densification statistics.
#include "gsb_ewa.cuh"
#include "gsb_raster.cuh"
#include "gsb_sh.cuh"

namespace gsb {

// gsb_intersect.cu
size_t isect_plan_ewa_workspace(uint32_t N, uint32_t tile_width, uint32_t tile_height);
int isect_plan_ewa(uint32_t N, int32_t *counts, const uint2 *boxes, const uint32_t *masks, const float *depths,
                   const float4 *filt0, const float2 *filt1, uint32_t tile_width, uint32_t tile_height,
                   int64_t *n_isects_out, int32_t *tile_offsets_out, void *plan_workspace, size_t plan_workspace_bytes,
                   cudaStream_t s);
int isect_emit_ewa(uint32_t N, const float4 *filt0, const float2 *filt1, const float *depths, uint32_t tile_width,
                   uint32_t tile_height, uint64_t capacity, const void *plan_workspace, size_t plan_workspace_bytes,
                   int32_t *flatten_ids, cudaStream_t s);
// gsb_raster.cu
int raster_ewa_fwd(uint32_t cap, const GaussRec *recs, uint32_t W, uint32_t H, const int32_t *tile_offsets,
                   const int32_t *flatten_ids, float *image, float *alpha, int32_t *last_ids, cudaStream_t s);
int raster_ewa_bwd(uint32_t cap, const GaussRec *recs, uint32_t W, uint32_t H, const int32_t *tile_offsets,
                   const int32_t *flatten_ids, const float *alpha, const int32_t *last_ids, const float *grad_image,
                   const float *grad_alpha, float *moments, cudaStream_t s);

constexpr int kFgsThreads = 128;
constexpr float kDilation = 0.3f;        // rasterization_config.h:16
constexpr uint32_t kSeqTiles = 32;       // boxes up to this many tiles are tested by their own lane: one mask bit per tile

struct FgsParams {
    uint32_t N, rest, active; // rest = SH bases in shN per primitive, active = active bases including sh0
    const float *means, *scales_raw, *rotations_raw, *opacities_raw, *sh0, *shN, *w2c, *campos;
    float W, H, fx, fy, cx, cy, near_, far_;
    uint32_t gw, gh;
    // per-primitive state (front writes, blend / back read)
    GaussRec *recs;
    float *moments;
    int32_t *counts;
    uint2 *boxes;
    uint32_t *masks; // tile-test results of boxes of up to 32 tiles (bit j = tile j of the box, row-major)
    float *depths;
    float4 *filt0;
    float2 *filt1;
    // back outputs
    float *g_means, *g_scales, *g_rot, *g_opac, *g_sh0, *g_shN, *g_w2c, *dens;
};

struct FgsCam {
    float r1[4], r2[4], r3[4]; // rows of w2c
    float campos[3];
};

// Covariance of one primitive: Sigma = R diag(exp(2 s)) R^T, R from the un-normalised quaternion (w, x, y, z)
// (kernels_forward.cuh:78-104).
struct FgsCov {
    float R[3][3], var[3], S[6]; // S: 11 12 13 22 23 33
    float qn2;
};
__device__ __forceinline__ void fgs_cov(const float *s, const float4 q, FgsCov &c) {
    c.var[0] = expf(2.0f * s[0]); c.var[1] = expf(2.0f * s[1]); c.var[2] = expf(2.0f * s[2]);
    const float w = q.x, x = q.y, y = q.z, z = q.w;
    c.qn2 = w * w + x * x + y * y + z * z;
    const float k = 2.0f / c.qn2;
    const float xx = k * x * x, yy = k * y * y, zz = k * z * z, xy = k * x * y, xz = k * x * z, yz = k * y * z;
    const float wx = k * w * x, wy = k * w * y, wz = k * w * z;
    c.R[0][0] = 1.0f - (yy + zz); c.R[0][1] = xy - wz; c.R[0][2] = wy + xz;
    c.R[1][0] = wz + xy; c.R[1][1] = 1.0f - (xx + zz); c.R[1][2] = yz - wx;
    c.R[2][0] = xz - wy; c.R[2][1] = wx + yz; c.R[2][2] = 1.0f - (xx + yy);
    int n = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = i; j < 3; ++j)
            c.S[n++] = c.R[i][0] * c.var[0] * c.R[j][0] + c.R[i][1] * c.var[1] * c.R[j][1] + c.R[i][2] * c.var[2] * c.R[j][2];
}

// EWA projection (kernels_forward.cuh:106-151): J W rows, J W Sigma rows, the dilated 2-D covariance.
struct FgsEwa {
    float depth, x, y, tx, ty, j11, j13, j22, j23;
    float r1[3], r2[3], c1[3], c2[3];
    float a, b, c;
};
__device__ __forceinline__ void fgs_ewa(const FgsParams &p, const FgsCam &cam, const float *m, const FgsCov &cv, FgsEwa &e) {
    e.depth = cam.r3[0] * m[0] + cam.r3[1] * m[1] + cam.r3[2] * m[2] + cam.r3[3];
    const float id = 1.0f / e.depth;
    e.x = (cam.r1[0] * m[0] + cam.r1[1] * m[1] + cam.r1[2] * m[2] + cam.r1[3]) * id;
    e.y = (cam.r2[0] * m[0] + cam.r2[1] * m[1] + cam.r2[2] * m[2] + cam.r2[3]) * id;
    e.tx = fminf(fmaxf(e.x, (-0.15f * p.W - p.cx) / p.fx), (1.15f * p.W - p.cx) / p.fx);
    e.ty = fminf(fmaxf(e.y, (-0.15f * p.H - p.cy) / p.fy), (1.15f * p.H - p.cy) / p.fy);
    e.j11 = p.fx * id; e.j13 = -e.j11 * e.tx;
    e.j22 = p.fy * id; e.j23 = -e.j22 * e.ty;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        e.r1[k] = e.j11 * cam.r1[k] + e.j13 * cam.r3[k];
        e.r2[k] = e.j22 * cam.r2[k] + e.j23 * cam.r3[k];
    }
    const float *S = cv.S;
    e.c1[0] = e.r1[0] * S[0] + e.r1[1] * S[1] + e.r1[2] * S[2];
    e.c1[1] = e.r1[0] * S[1] + e.r1[1] * S[3] + e.r1[2] * S[4];
    e.c1[2] = e.r1[0] * S[2] + e.r1[1] * S[4] + e.r1[2] * S[5];
    e.c2[0] = e.r2[0] * S[0] + e.r2[1] * S[1] + e.r2[2] * S[2];
    e.c2[1] = e.r2[0] * S[1] + e.r2[1] * S[3] + e.r2[2] * S[4];
    e.c2[2] = e.r2[0] * S[2] + e.r2[1] * S[4] + e.r2[2] * S[5];
    e.a = e.c1[0] * e.r1[0] + e.c1[1] * e.r1[1] + e.c1[2] * e.r1[2] + kDilation;
    e.b = e.c1[0] * e.r2[0] + e.c1[1] * e.r2[1] + e.c1[2] * e.r2[2];
    e.c = e.c2[0] * e.r2[0] + e.c2[1] * e.r2[1] + e.c2[2] * e.r2[2] + kDilation;
}

__device__ __forceinline__ void fgs_cam_load(const FgsParams &p, FgsCam &c) {
    if (threadIdx.x < 12) {
        const float v = p.w2c[threadIdx.x];
        if (threadIdx.x < 4) c.r1[threadIdx.x] = v;
        else if (threadIdx.x < 8) c.r2[threadIdx.x - 4] = v;
        else c.r3[threadIdx.x - 8] = v;
    }
    if (threadIdx.x >= 32 && threadIdx.x < 35) c.campos[threadIdx.x - 32] = p.campos[threadIdx.x - 32];
}

// one bulk copy per 128-primitive slab of shN rows when the slab is 16-byte aligned as a whole (as gsb_fused.cu)
__device__ __forceinline__ void fgs_rows_in(float *s_rows, const float *g_rows, uint32_t n_floats, uint64_t *bar, bool bulk) {
    if (n_floats == 0) return;
    if (bulk) {
        if (threadIdx.x == 0) {
            mbar_init(bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(bar, n_floats * 4);
            bulk_g2s(s_rows, g_rows, n_floats * 4, bar);
        }
    } else {
        for (uint32_t i = threadIdx.x; i < n_floats; i += kFgsThreads) s_rows[i] = g_rows[i];
    }
}

__device__ __forceinline__ uint32_t tile_floor(float v, uint32_t lim) { // min(lim, max(0, floor(v / 16)))
    const int t = __float2int_rd(v * 0.0625f);
    return min(lim, (uint32_t)max(t, 0));
}
__device__ __forceinline__ uint32_t tile_ceil(float v, uint32_t lim) {
    const int t = __float2int_ru(v * 0.0625f);
    return min(lim, (uint32_t)max(t, 0));
}

template <int DEG>
__global__ void __launch_bounds__(kFgsThreads) fgs_front_kernel(const FgsParams p) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    extern __shared__ __align__(128) float s_rows[]; // [kFgsThreads][rest * 3]
    __shared__ FgsCam s_cam;
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint32_t g0 = blockIdx.x * kFgsThreads;
    const uint32_t cnt = min((uint32_t)kFgsThreads, p.N - g0);
    const uint32_t g = g0 + tid;
    const uint32_t rowf = p.rest * 3;
    const float *g_rows = p.shN ? p.shN + (size_t)g0 * rowf : nullptr;
    const bool want_rows = (DEG >= 1) && rowf > 0 && g_rows != nullptr;
    const uint32_t n_floats = want_rows ? cnt * rowf : 0u;
    const bool bulk = want_rows && ((reinterpret_cast<uintptr_t>(g_rows) & 15) == 0) && ((n_floats & 3u) == 0);

    fgs_cam_load(p, s_cam);
    fgs_rows_in(s_rows, g_rows, n_floats, &s_bar, bulk);
    __syncthreads();

    bool active = tid < cnt;
    float m[3] = {0.f, 0.f, 1.f};
    float opacity = 0.f;
    EwaFilter flt = {0.f, 0.f, 1.f, 0.f, 1.f, 0.f};
    uint32_t x0 = 0, y0 = 0, bw = 0, bh = 0;
    float depth = 0.f, mx = 0.f, my = 0.f;
    if (active) {
        m[0] = p.means[(size_t)g * 3]; m[1] = p.means[(size_t)g * 3 + 1]; m[2] = p.means[(size_t)g * 3 + 2];
        float4 *m4 = reinterpret_cast<float4 *>(p.moments + (size_t)g * kMomFloats);
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        m4[0] = z; m4[1] = z; m4[2] = z; m4[3] = z;
        const float sr[3] = {p.scales_raw[(size_t)g * 3], p.scales_raw[(size_t)g * 3 + 1], p.scales_raw[(size_t)g * 3 + 2]};
        FgsCov cv;
        fgs_cov(sr, reinterpret_cast<const float4 *>(p.rotations_raw)[g], cv);
        FgsEwa e;
        fgs_ewa(p, s_cam, m, cv, e);
        depth = e.depth;
        opacity = 1.0f / (1.0f + expf(-p.opacities_raw[g]));
        const float det = e.a * e.c - e.b * e.b;
        // kernels_forward.cuh:60-64,72-74,88-89,153-155 (the comparisons are written so that a NaN culls)
        active = (depth >= p.near_) && (depth <= p.far_) && (opacity >= kAlphaThreshold) && (cv.qn2 >= 1e-8f) && (det >= 1e-8f);
        if (active) {
            const float idet = 1.0f / det;
            flt.ca = e.c * idet; flt.cb = -e.b * idet; flt.cc = e.a * idet;
            mx = e.x * p.fx + p.cx; my = e.y * p.fy + p.cy;
            flt.mx = mx - 0.5f; flt.my = my - 0.5f;
            flt.thr = logf(opacity * 255.0f);
            const float fac = sqrtf(2.0f * flt.thr);
            const float ex = fmaxf(fac * sqrtf(e.a) - 0.5f, 0.0f), ey = fmaxf(fac * sqrtf(e.c) - 0.5f, 0.0f);
            x0 = tile_floor(mx - ex, p.gw); y0 = tile_floor(my - ey, p.gh);
            bw = tile_ceil(mx + ex, p.gw) - x0; bh = tile_ceil(my + ey, p.gh) - y0;
            active = bw * bh > 0;
        }
    }
    // exact number of tiles (kernels_forward.cuh:180-187, kernel_utils.cuh:141-209): small boxes by their own lane,
    // large ones by the whole warp
    const uint32_t area = active ? bw * bh : 0u;
    uint32_t n_tiles = 0, tmask = 0;
    if (area > 0 && area <= kSeqTiles) {
        uint32_t x = x0, y = y0;
        for (uint32_t j = 0; j < area; ++j) {
            tmask |= (ewa_tile_contributes(flt, x, y) ? 1u : 0u) << j;
            if (++x == x0 + bw) { x = x0; ++y; }
        }
        n_tiles = __popc(tmask);
    }
    uint32_t big = __ballot_sync(0xffffffffu, area > kSeqTiles);
    while (big) {
        const int src = __ffs(big) - 1;
        big &= big - 1;
        EwaFilter bf;
        bf.mx = __shfl_sync(0xffffffffu, flt.mx, src); bf.my = __shfl_sync(0xffffffffu, flt.my, src);
        bf.ca = __shfl_sync(0xffffffffu, flt.ca, src); bf.cb = __shfl_sync(0xffffffffu, flt.cb, src);
        bf.cc = __shfl_sync(0xffffffffu, flt.cc, src); bf.thr = __shfl_sync(0xffffffffu, flt.thr, src);
        const uint32_t bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
        const uint32_t bbw = __shfl_sync(0xffffffffu, bw, src), barea = __shfl_sync(0xffffffffu, area, src);
        uint32_t c = 0;
        for (uint32_t j = lane; j < barea; j += 32) {
            const uint32_t dy = j / bbw, dx = j - dy * bbw;
            c += ewa_tile_contributes(bf, bx0 + dx, by0 + dy) ? 1u : 0u;
        }
        c = __reduce_add_sync(0xffffffffu, c);
        if ((int)lane == src) n_tiles = c;
    }
    const bool visible = active && n_tiles > 0;
    if (tid < cnt) {
        p.counts[g] = visible ? (int32_t)n_tiles : 0;
        p.boxes[g] = make_uint2(x0 | (y0 << 16), bw | (bh << 16));
        p.masks[g] = tmask;
        p.depths[g] = depth;
        p.filt0[g] = make_float4(flt.mx, flt.my, flt.ca, flt.cb);
        p.filt1[g] = make_float2(flt.cc, flt.thr);
    }
    if (bulk) mbar_wait(&s_bar, 0);
    else if (want_rows) __syncthreads();
    if (!visible) {
        if (tid < cnt) { // a record that never passes the rejection test (it is in no tile's list anyway)
            float4 *dst = reinterpret_cast<float4 *>(p.recs + g);
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            dst[0] = z; dst[1] = z; dst[2] = make_float4(0.f, 0.f, 0.f, __int_as_float(0x7f800000));
            dst[3] = make_float4(0.f, 0.f, 0.f, __int_as_float((int32_t)g));
        }
        return;
    }
    // view-dependent colour (kernel_utils.cuh:16-40); the blend clamps it at zero (kernels_forward.cuh:418)
    float b[NB];
    float dx = m[0] - s_cam.campos[0], dy = m[1] - s_cam.campos[1], dz = m[2] - s_cam.campos[2];
    if constexpr (DEG >= 1) {
        const float inorm = rsqrtf(dx * dx + dy * dy + dz * dz);
        dx *= inorm; dy *= inorm; dz *= inorm;
    }
    sh_basis<DEG>(dx, dy, dz, b);
    float col[3];
    col[0] = 0.5f + b[0] * p.sh0[(size_t)g * 3]; col[1] = 0.5f + b[0] * p.sh0[(size_t)g * 3 + 1];
    col[2] = 0.5f + b[0] * p.sh0[(size_t)g * 3 + 2];
    if constexpr (DEG >= 1) {
        const float *row = s_rows + (size_t)tid * rowf;
#pragma unroll
        for (int k = 1; k < NB; ++k) {
            col[0] += b[k] * row[(k - 1) * 3];
            col[1] += b[k] * row[(k - 1) * 3 + 1];
            col[2] += b[k] * row[(k - 1) * 3 + 2];
        }
    }
    // the blend record: Ns = -log2(e) (1/2 ca x^2 + cb x y + 1/2 cc y^2), alpha_raw = 2^(Ns + log2 opacity)
    const float lop = log2f(opacity);
    float4 *dst = reinterpret_cast<float4 *>(p.recs + g);
    dst[0] = make_float4(mx, my, -0.5f * kLog2e * flt.ca, -kLog2e * flt.cb);
    // .y / .z are free in an EWA record (no denominator form): the opacity and the colour clamp mask for the backward
    const int32_t cmask = (col[0] >= 0.f ? 1 : 0) | (col[1] >= 0.f ? 2 : 0) | (col[2] >= 0.f ? 4 : 0);
    dst[1] = make_float4(-0.5f * kLog2e * flt.cc, opacity, __int_as_float(cmask), 0.f);
    dst[2] = make_float4(0.f, 0.f, lop, kLog2AlphaThr - kTauMargin - lop);
    dst[3] = make_float4(fmaxf(col[0], 0.f), fmaxf(col[1], 0.f), fmaxf(col[2], 0.f), __int_as_float((int32_t)g));
}

template <int DEG>
__global__ void __launch_bounds__(kFgsThreads) fgs_back_kernel(const FgsParams p) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    extern __shared__ __align__(128) float s_rows[]; // shN rows in, gradient rows out (each thread owns its row)
    __shared__ FgsCam s_cam;
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ float s_w2c[kFgsThreads / 32][12];
    const uint32_t tid = threadIdx.x;
    const uint32_t g0 = blockIdx.x * kFgsThreads;
    const uint32_t cnt = min((uint32_t)kFgsThreads, p.N - g0);
    const uint32_t g = g0 + tid;
    const uint32_t rowf = p.rest * 3;
    const float *g_rows = p.shN ? p.shN + (size_t)g0 * rowf : nullptr;
    float *g_out = p.g_shN ? p.g_shN + (size_t)g0 * rowf : nullptr;
    const bool have_rows = rowf > 0 && g_rows != nullptr && g_out != nullptr;
    const bool read_rows = have_rows && DEG >= 1;
    const uint32_t n_floats = have_rows ? cnt * rowf : 0u;
    const bool al = have_rows && ((n_floats & 3u) == 0);
    const bool bulk_in = read_rows && al && ((reinterpret_cast<uintptr_t>(g_rows) & 15) == 0);
    const bool bulk_out = al && ((reinterpret_cast<uintptr_t>(g_out) & 15) == 0);

    fgs_cam_load(p, s_cam);
    fgs_rows_in(s_rows, g_rows, read_rows ? n_floats : 0u, &s_bar, bulk_in);
    __syncthreads();
    if (bulk_in) mbar_wait(&s_bar, 0);

    float dcam[3] = {0.f, 0.f, 0.f}, mean[3] = {0.f, 0.f, 0.f};
    float *row = s_rows + (size_t)tid * rowf;
    const bool visible = tid < cnt && p.counts[g] > 0;
    if (tid < cnt) {
        float gm[3] = {0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f}, go = 0.f;
        float g0c[3] = {0.f, 0.f, 0.f};
        if (visible) {
            float mo[16];
            const float4 *m4 = reinterpret_cast<const float4 *>(p.moments + (size_t)g * kMomFloats);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 v = m4[i];
                mo[i * 4] = v.x; mo[i * 4 + 1] = v.y; mo[i * 4 + 2] = v.z; mo[i * 4 + 3] = v.w;
            }
            mean[0] = p.means[(size_t)g * 3]; mean[1] = p.means[(size_t)g * 3 + 1]; mean[2] = p.means[(size_t)g * 3 + 2];
            const float sr[3] = {p.scales_raw[(size_t)g * 3], p.scales_raw[(size_t)g * 3 + 1], p.scales_raw[(size_t)g * 3 + 2]};
            const float4 q = reinterpret_cast<const float4 *>(p.rotations_raw)[g];
            FgsCov cv;
            fgs_cov(sr, q, cv);
            FgsEwa e;
            fgs_ewa(p, s_cam, mean, cv, e);
            const float4 rec1 = reinterpret_cast<const float4 *>(p.recs + g)[1];
            const float opacity = rec1.y;
            const int32_t cmask = __float_as_int(rec1.z);
            go = mo[kS_G] * (1.0f - opacity); // kernels_backward.cuh:440
            // ---- SH backward (kernel_utils.cuh:42-102)
            {
                const float rx = mean[0] - s_cam.campos[0], ry = mean[1] - s_cam.campos[1], rz = mean[2] - s_cam.campos[2];
                float x = rx, y = ry, z = rz, inorm = 1.f;
                if constexpr (DEG >= 1) {
                    inorm = rsqrtf(rx * rx + ry * ry + rz * rz);
                    x *= inorm; y *= inorm; z *= inorm;
                }
                float b[NB];
                sh_basis<DEG>(x, y, z, b);
                // the gradient passes where the unclamped colour was >= 0 (kernels_backward.cuh:310-316)
                const float c0 = (cmask & 1) ? mo[kS_CR] : 0.f, c1 = (cmask & 2) ? mo[kS_CG] : 0.f;
                const float c2 = (cmask & 4) ? mo[kS_CB] : 0.f;
                g0c[0] = b[0] * c0; g0c[1] = b[0] * c1; g0c[2] = b[0] * c2;
                if constexpr (DEG >= 1) {
                    float w[NB];
                    w[0] = 0.f;
#pragma unroll
                    for (int k = 1; k < NB; ++k) {
                        const float s0 = row[(k - 1) * 3], s1 = row[(k - 1) * 3 + 1], s2 = row[(k - 1) * 3 + 2];
                        w[k] = c0 * s0 + c1 * s1 + c2 * s2;
                        row[(k - 1) * 3] = b[k] * c0; row[(k - 1) * 3 + 1] = b[k] * c1; row[(k - 1) * 3 + 2] = b[k] * c2;
                    }
                    float vx = 0.f, vy = 0.f, vz = 0.f;
                    sh_basis_vjp<DEG>(x, y, z, w, vx, vy, vz);
                    const float d = vx * x + vy * y + vz * z; // through the normalisation of the direction
                    gm[0] = (vx - d * x) * inorm; gm[1] = (vy - d * y) * inorm; gm[2] = (vz - d * z) * inorm;
                }
                if (have_rows)
                    for (uint32_t i = (NB - 1) * 3; i < rowf; ++i) row[i] = 0.f; // inactive bases
            }
            // ---- conic / centre gradients from the moments: x = pixel - centre, g = alpha dL/dalpha
            const float a = e.a, bb_ = e.b, c = e.c;
            const float det = a * c - bb_ * bb_, idet = 1.0f / det, idet2 = idet * idet;
            const float ca = c * idet, cb = -bb_ * idet, cc = a * idet;
            const float gmx = ca * mo[kS_W1X] + cb * mo[kS_W1Y], gmy = cb * mo[kS_W1X] + cc * mo[kS_W1Y];
            const float gA = -0.5f * mo[kS_W1XX], gBh = -0.5f * mo[kS_W1XY], gC = -0.5f * mo[kS_W1YY];
            // kernels_backward.cuh:120-130 (the middle entry carries half of dL/db)
            const float dca = idet2 * (2.0f * bb_ * c * gBh - c * c * gA - bb_ * bb_ * gC);
            const float dcb = idet2 * (bb_ * c * gA - (a * c + bb_ * bb_) * gBh + a * bb_ * gC);
            const float dcc = idet2 * (2.0f * a * bb_ * gBh - bb_ * bb_ * gA - a * a * gC);
            float dS[3][3]; // dL/dSigma, symmetric
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int s = r; s < 3; ++s) {
                    dS[r][s] = e.r1[r] * e.r1[s] * dca + (e.r1[r] * e.r2[s] + e.r1[s] * e.r2[r]) * dcb + e.r2[r] * e.r2[s] * dcc;
                    dS[s][r] = dS[r][s];
                }
            float dj11 = 0.f, dj22 = 0.f, dj13 = 0.f, dj23 = 0.f;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float dr1 = 2.0f * (e.c1[k] * dca + e.c2[k] * dcb), dr2 = 2.0f * (e.c1[k] * dcb + e.c2[k] * dcc);
                dj11 += s_cam.r1[k] * dr1; dj22 += s_cam.r2[k] * dr2;
                dj13 += s_cam.r3[k] * dr1; dj23 += s_cam.r3[k] * dr2;
            }
            const float id = 1.0f / e.depth;
            const float h1 = dj11 - 2.0f * e.tx * dj13, h2 = dj22 - 2.0f * e.ty * dj23;
            dcam[0] = e.j11 * (gmx - dj13 * id);
            dcam[1] = e.j22 * (gmy - dj23 * id);
            dcam[2] = -e.j11 * (e.x * gmx + h1 * id) - e.j22 * (e.y * gmy + h2 * id);
#pragma unroll
            for (int k = 0; k < 3; ++k) gm[k] += s_cam.r1[k] * dcam[0] + s_cam.r2[k] * dcam[1] + s_cam.r3[k] * dcam[2];
            // Sigma = R V R^T: dL/dV_m = R[:,m]^T dS R[:,m]; dL/dR[:,m] = 2 V_m dS R[:,m]
            float dR[3][3];
#pragma unroll
            for (int mcol = 0; mcol < 3; ++mcol) {
                float t[3];
#pragma unroll
                for (int r = 0; r < 3; ++r) t[r] = dS[r][0] * cv.R[0][mcol] + dS[r][1] * cv.R[1][mcol] + dS[r][2] * cv.R[2][mcol];
                const float qf = cv.R[0][mcol] * t[0] + cv.R[1][mcol] * t[1] + cv.R[2][mcol] * t[2];
                gs[mcol] = 2.0f * cv.var[mcol] * qf;
#pragma unroll
                for (int r = 0; r < 3; ++r) dR[r][mcol] = 2.0f * cv.var[mcol] * t[r];
            }
            // rotation of q / |q| written with the nine products 2 q_i q_j / |q|^2 (kernels_backward.cuh:228-243)
            const float qw = q.x, qx = q.y, qy = q.z, qz = q.w, k2 = 2.0f / cv.qn2;
            const float dxx = -dR[1][1] - dR[2][2], dyy = -dR[0][0] - dR[2][2], dzz = -dR[0][0] - dR[1][1];
            const float dxy = dR[0][1] + dR[1][0], dxz = dR[0][2] + dR[2][0], dyz = dR[1][2] + dR[2][1];
            const float dwx = dR[2][1] - dR[1][2], dwy = dR[0][2] - dR[2][0], dwz = dR[1][0] - dR[0][1];
            const float hn = k2 * (qx * qx * dxx + qy * qy * dyy + qz * qz * dzz + qx * qy * dxy + qx * qz * dxz + qy * qz * dyz +
                                   qw * qx * dwx + qw * qy * dwy + qw * qz * dwz);
            gq[0] = k2 * (qx * dwx + qy * dwy + qz * dwz - qw * hn);
            gq[1] = k2 * (2.0f * qx * dxx + qy * dxy + qz * dxz + qw * dwx - qx * hn);
            gq[2] = k2 * (2.0f * qy * dyy + qx * dxy + qz * dyz + qw * dwy - qy * hn);
            gq[3] = k2 * (2.0f * qz * dzz + qx * dxz + qy * dyz + qw * dwz - qz * hn);
            if (p.dens) { // kernels_backward.cuh:252-255
                p.dens[g] += 1.0f;
                const float sx = gmx * 0.5f * p.W, sy = gmy * 0.5f * p.H;
                p.dens[(size_t)p.N + g] += sqrtf(sx * sx + sy * sy);
            }
        } else if (have_rows) {
            for (uint32_t i = 0; i < rowf; ++i) row[i] = 0.f;
        }
        p.g_means[(size_t)g * 3] = gm[0]; p.g_means[(size_t)g * 3 + 1] = gm[1]; p.g_means[(size_t)g * 3 + 2] = gm[2];
        p.g_scales[(size_t)g * 3] = gs[0]; p.g_scales[(size_t)g * 3 + 1] = gs[1]; p.g_scales[(size_t)g * 3 + 2] = gs[2];
        reinterpret_cast<float4 *>(p.g_rot)[g] = make_float4(gq[0], gq[1], gq[2], gq[3]);
        p.g_opac[g] = go;
        p.g_sh0[(size_t)g * 3] = g0c[0]; p.g_sh0[(size_t)g * 3 + 1] = g0c[1]; p.g_sh0[(size_t)g * 3 + 2] = g0c[2];
    }
    if (p.g_w2c) { // kernels_backward.cuh:173-186: rows of dL/d(w2c) = dcam (x) (mean, 1); one atomic set per CTA
        float v[12];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            v[r * 4] = dcam[r] * mean[0]; v[r * 4 + 1] = dcam[r] * mean[1]; v[r * 4 + 2] = dcam[r] * mean[2];
            v[r * 4 + 3] = dcam[r];
        }
#pragma unroll
        for (int i = 0; i < 12; ++i) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
        }
        if ((tid & 31) == 0)
            for (int i = 0; i < 12; ++i) s_w2c[tid >> 5][i] = v[i];
        __syncthreads();
        if (tid < 12) {
            float acc = 0.f;
            for (int w = 0; w < kFgsThreads / 32; ++w) acc += s_w2c[w][tid];
            if (acc != 0.f) atomicAdd(p.g_w2c + tid, acc);
        }
    }
    if (!have_rows) return;
    if (bulk_out) {
        fence_proxy_async();
        __syncthreads();
        if (tid == 0) {
            bulk_s2g(g_out, s_rows, n_floats * 4);
            bulk_commit();
            bulk_wait_read_all();
        }
    } else {
        __syncthreads();
        for (uint32_t i = tid; i < n_floats; i += kFgsThreads) g_out[i] = s_rows[i];
    }
}

// layout of the per-primitive buffer (opaque to the caller, carried from forward to backward)
struct PrimLayout {
    size_t recs, moments, counts, boxes, masks, depths, filt0, filt1, plan, plan_bytes, total;
};
static PrimLayout prim_layout(uint32_t N, uint32_t gw, uint32_t gh) {
    PrimLayout l;
    WsLayout w;
    l.recs = w.take((size_t)N * sizeof(GaussRec));
    l.moments = w.take((size_t)N * kMomFloats * 4);
    l.counts = w.take((size_t)N * 4);
    l.boxes = w.take((size_t)N * 8);
    l.masks = w.take((size_t)N * 4);
    l.depths = w.take((size_t)N * 4);
    l.filt0 = w.take((size_t)N * 16);
    l.filt1 = w.take((size_t)N * 8);
    l.plan_bytes = isect_plan_ewa_workspace(N, gw, gh);
    l.plan = w.take(l.plan_bytes);
    l.total = align256(w.bytes) + 256;
    return l;
}
struct TileLayout {
    size_t offsets, last_ids, total;
};
static TileLayout tile_layout(uint32_t W, uint32_t H) {
    const uint32_t gw = (W + 15) / 16, gh = (H + 15) / 16;
    TileLayout l;
    l.offsets = 0;
    l.last_ids = align256(((size_t)gw * gh + 1) * 4);
    l.total = l.last_ids + align256((size_t)W * H * 4) + 256;
    return l;
}

static int check_view(const GsbFastgsView *v) {
    if (!v || !v->w2c || !v->cam_position) return GSB_E_INVALID;
    if (v->width == 0 || v->height == 0) return GSB_E_INVALID;
    if (v->active_sh_bases != 1 && v->active_sh_bases != 4 && v->active_sh_bases != 9 && v->active_sh_bases != 16)
        return GSB_E_INVALID;
    if (v->active_sh_bases > v->total_bases_sh_rest + 1) return GSB_E_INVALID;
    const uint32_t gw = (v->width + 15) / 16, gh = (v->height + 15) / 16;
    if ((uint64_t)gw * gh > 65535ull * 16) return GSB_E_INVALID;
    return GSB_OK;
}

static void fill_params(FgsParams &p, uint32_t N, const GsbFastgsView *v, const float *means, const float *scales_raw,
                        const float *rotations_raw, const float *opacities_raw, const float *sh0, const float *shN,
                        char *prim, const PrimLayout &l) {
    p.N = N; p.rest = v->total_bases_sh_rest; p.active = v->active_sh_bases;
    p.means = means; p.scales_raw = scales_raw; p.rotations_raw = rotations_raw; p.opacities_raw = opacities_raw;
    p.sh0 = sh0; p.shN = shN; p.w2c = v->w2c; p.campos = v->cam_position;
    p.W = (float)v->width; p.H = (float)v->height; p.fx = v->focal_x; p.fy = v->focal_y; p.cx = v->center_x; p.cy = v->center_y;
    p.near_ = v->near_plane; p.far_ = v->far_plane;
    p.gw = (v->width + 15) / 16; p.gh = (v->height + 15) / 16;
    p.recs = reinterpret_cast<GaussRec *>(prim + l.recs);
    p.moments = reinterpret_cast<float *>(prim + l.moments);
    p.counts = reinterpret_cast<int32_t *>(prim + l.counts);
    p.boxes = reinterpret_cast<uint2 *>(prim + l.boxes);
    p.masks = reinterpret_cast<uint32_t *>(prim + l.masks);
    p.depths = reinterpret_cast<float *>(prim + l.depths);
    p.filt0 = reinterpret_cast<float4 *>(prim + l.filt0);
    p.filt1 = reinterpret_cast<float2 *>(prim + l.filt1);
    p.g_means = p.g_scales = p.g_rot = p.g_opac = p.g_sh0 = p.g_shN = p.g_w2c = p.dens = nullptr;
}

#define GSB_FGS_LAUNCH(KERNEL)                                                                                         \
    switch (v->active_sh_bases) {                                                                                      \
        case 1: GSB_FGS_ONE(KERNEL, 0); break;                                                                         \
        case 4: GSB_FGS_ONE(KERNEL, 1); break;                                                                         \
        case 9: GSB_FGS_ONE(KERNEL, 2); break;                                                                         \
        default: GSB_FGS_ONE(KERNEL, 3); break;                                                                        \
    }
#define GSB_FGS_ONE(KERNEL, D)                                                                                         \
    do {                                                                                                               \
        if (smem > 48 * 1024)                                                                                          \
            GSB_CUDA_TRY(cudaFuncSetAttribute(KERNEL<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));     \
        KERNEL<D><<<grid, kFgsThreads, smem, s>>>(p);                                                                  \
    } while (0)

} // namespace gsb

extern "C" size_t gsb_fastgs_primitive_bytes(uint32_t N, uint32_t width, uint32_t height) {
    return gsb::prim_layout(N, (width + 15) / 16, (height + 15) / 16).total;
}
extern "C" size_t gsb_fastgs_tile_bytes(uint32_t width, uint32_t height) { return gsb::tile_layout(width, height).total; }

extern "C" int gsb_fastgs_forward_plan(uint32_t N, const float *means, const float *scales_raw, const float *rotations_raw,
                                       const float *opacities_raw, const float *sh0, const float *shN,
                                       const GsbFastgsView *view, void *per_primitive, size_t per_primitive_bytes,
                                       void *per_tile, size_t per_tile_bytes, int64_t *n_instances_out,
                                       gsb_stream_t stream) {
    using namespace gsb;
    const GsbFastgsView *v = view;
    if (int rc = check_view(v)) return rc;
    if (!n_instances_out) return GSB_E_INVALID;
    const uint32_t gw = (v->width + 15) / 16, gh = (v->height + 15) / 16;
    const PrimLayout l = prim_layout(N, gw, gh);
    const TileLayout tl = tile_layout(v->width, v->height);
    if (!per_primitive || (reinterpret_cast<uintptr_t>(per_primitive) & 255) || per_primitive_bytes < l.total)
        return GSB_E_WORKSPACE;
    if (!per_tile || (reinterpret_cast<uintptr_t>(per_tile) & 255) || per_tile_bytes < tl.total) return GSB_E_WORKSPACE;
    cudaStream_t s = as_stream(stream);
    char *prim = reinterpret_cast<char *>(per_primitive);
    int32_t *tile_offsets = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(per_tile) + tl.offsets);
    if (N > 0) {
        if (!means || !scales_raw || !rotations_raw || !opacities_raw || !sh0) return GSB_E_INVALID;
        if (v->active_sh_bases > 1 && !shN) return GSB_E_INVALID;
        if (reinterpret_cast<uintptr_t>(rotations_raw) & 15) return GSB_E_INVALID;
        FgsParams p;
        fill_params(p, N, v, means, scales_raw, rotations_raw, opacities_raw, sh0, shN, prim, l);
        const uint32_t grid = (N + kFgsThreads - 1) / kFgsThreads;
        const size_t smem = v->active_sh_bases > 1 ? (size_t)kFgsThreads * v->total_bases_sh_rest * 12 : 0;
        {
            ProfScope ps("fgs_front", s);
            GSB_FGS_LAUNCH(fgs_front_kernel);
        }
        GSB_LAUNCH_CHECK();
    }
    FgsParams q;
    fill_params(q, N, v, means, scales_raw, rotations_raw, opacities_raw, sh0, shN, prim, l);
    return isect_plan_ewa(N, q.counts, q.boxes, q.masks, q.depths, q.filt0, q.filt1, gw, gh, n_instances_out, tile_offsets,
                          prim + l.plan, l.plan_bytes, s);
}

extern "C" int gsb_fastgs_forward_blend(uint32_t N, const GsbFastgsView *view, void *per_primitive,
                                        size_t per_primitive_bytes, void *per_tile, size_t per_tile_bytes,
                                        int32_t *instances, uint64_t capacity, float *image, float *alpha,
                                        gsb_stream_t stream) {
    using namespace gsb;
    const GsbFastgsView *v = view;
    if (int rc = check_view(v)) return rc;
    if (!image || !alpha) return GSB_E_INVALID;
    if (capacity > 0x7fffffffull || (capacity > 0 && !instances)) return GSB_E_INVALID;
    const uint32_t gw = (v->width + 15) / 16, gh = (v->height + 15) / 16;
    const PrimLayout l = prim_layout(N, gw, gh);
    const TileLayout tl = tile_layout(v->width, v->height);
    if (!per_primitive || (reinterpret_cast<uintptr_t>(per_primitive) & 255) || per_primitive_bytes < l.total)
        return GSB_E_WORKSPACE;
    if (!per_tile || (reinterpret_cast<uintptr_t>(per_tile) & 255) || per_tile_bytes < tl.total) return GSB_E_WORKSPACE;
    cudaStream_t s = as_stream(stream);
    char *prim = reinterpret_cast<char *>(per_primitive);
    char *tile = reinterpret_cast<char *>(per_tile);
    if (int rc = isect_emit_ewa(N, reinterpret_cast<const float4 *>(prim + l.filt0),
                                reinterpret_cast<const float2 *>(prim + l.filt1),
                                reinterpret_cast<const float *>(prim + l.depths), gw, gh, capacity, prim + l.plan,
                                l.plan_bytes, instances, s))
        return rc;
    return raster_ewa_fwd((uint32_t)capacity, reinterpret_cast<const GaussRec *>(prim + l.recs), v->width, v->height,
                          reinterpret_cast<const int32_t *>(tile + tl.offsets), instances, image, alpha,
                          reinterpret_cast<int32_t *>(tile + tl.last_ids), s);
}

extern "C" int gsb_fastgs_backward(uint32_t N, const float *means, const float *scales_raw, const float *rotations_raw,
                                   const float *shN, const GsbFastgsView *view, void *per_primitive, size_t per_primitive_bytes,
                                   const void *per_tile, size_t per_tile_bytes, const int32_t *instances, uint64_t capacity,
                                   const float *alpha, const float *grad_image, const float *grad_alpha, float *grad_means,
                                   float *grad_scales_raw, float *grad_rotations_raw, float *grad_opacities_raw,
                                   float *grad_sh0, float *grad_shN, float *grad_w2c, float *densification_info,
                                   gsb_stream_t stream) {
    using namespace gsb;
    const GsbFastgsView *v = view;
    if (int rc = check_view(v)) return rc;
    if (N == 0) return GSB_OK;
    if (!means || !scales_raw || !rotations_raw || !alpha || !grad_image || !grad_alpha) return GSB_E_INVALID;
    if (!grad_means || !grad_scales_raw || !grad_rotations_raw || !grad_opacities_raw || !grad_sh0) return GSB_E_INVALID;
    if (v->total_bases_sh_rest > 0 && (!shN || !grad_shN)) return GSB_E_INVALID;
    if ((reinterpret_cast<uintptr_t>(rotations_raw) & 15) || (reinterpret_cast<uintptr_t>(grad_rotations_raw) & 15))
        return GSB_E_INVALID;
    if (capacity > 0x7fffffffull || (capacity > 0 && !instances)) return GSB_E_INVALID;
    const uint32_t gw = (v->width + 15) / 16, gh = (v->height + 15) / 16;
    const PrimLayout l = prim_layout(N, gw, gh);
    const TileLayout tl = tile_layout(v->width, v->height);
    if (!per_primitive || (reinterpret_cast<uintptr_t>(per_primitive) & 255) || per_primitive_bytes < l.total)
        return GSB_E_WORKSPACE;
    if (!per_tile || (reinterpret_cast<uintptr_t>(per_tile) & 255) || per_tile_bytes < tl.total) return GSB_E_WORKSPACE;
    cudaStream_t s = as_stream(stream);
    char *prim = reinterpret_cast<char *>(per_primitive);
    const char *tile = reinterpret_cast<const char *>(per_tile);
    FgsParams p;
    fill_params(p, N, v, means, scales_raw, rotations_raw, nullptr, nullptr, shN, prim, l);
    if (capacity > 0) {
        if (int rc = raster_ewa_bwd((uint32_t)capacity, p.recs, v->width, v->height,
                                    reinterpret_cast<const int32_t *>(tile + tl.offsets), instances, alpha,
                                    reinterpret_cast<const int32_t *>(tile + tl.last_ids), grad_image, grad_alpha,
                                    p.moments, s))
            return rc;
    }
    p.g_means = grad_means; p.g_scales = grad_scales_raw; p.g_rot = grad_rotations_raw; p.g_opac = grad_opacities_raw;
    p.g_sh0 = grad_sh0; p.g_shN = grad_shN; p.g_w2c = grad_w2c; p.dens = densification_info;
    if (grad_w2c) GSB_CUDA_TRY(cudaMemsetAsync(grad_w2c, 0, 16 * sizeof(float), s));
    const uint32_t grid = (N + kFgsThreads - 1) / kFgsThreads;
    const size_t smem = v->total_bases_sh_rest > 0 ? (size_t)kFgsThreads * v->total_bases_sh_rest * 12 : 0;
    {
        ProfScope ps("fgs_back", s);
        GSB_FGS_LAUNCH(fgs_back_kernel);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
