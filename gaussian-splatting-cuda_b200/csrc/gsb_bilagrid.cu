// gsb_bilagrid.cu -- SURVEY.md 8(f5): the bilateral grid of the training iteration (appearance correction per image).
//
// The reference slices the rendered image through a per-image affine bilateral grid before the loss and adds a total
// variation (TV) term over the grids of all images (src/training/components/bilateral_grid.cpp:94-127,
// src/training/trainer.cpp:160-171,662-665,698-705).  Its kernels (src/training/kernels/bilateral_grid_forward.cu,
// _backward.cu, _tv.cu) compute, for pixel (i, j) of an h x w image and a grid A of 12 coefficient volumes [12, L, H, W]:
//
//     x  = clamp(rgb, 0, 1)                                         (bilateral_grid.cpp:110, before the kernel)
//     gx = (j / (w - 1)) * (W - 1),  gy = (i / (h - 1)) * (H - 1),  gz = (0.299 r + 0.587 g + 0.114 b) * (L - 1)
//     corners x0 = floor(gx), x1 = min(x0 + 1, W - 1) (same for y);  z0 = max(floor(gz), 0), z1 = min(max(floor(gz) + 1, 0), L - 1)
//     out_d = sum_s a_{4d+s} x_s + a_{4d+3},  a_c = trilinear interpolation of volume c   (forward.cu:33-88)
//
// and, backward (backward.cu:36-151), the grid gradient sum over pixels of w_corner * x_s * g_d (96 atomicAdds per
// pixel into one image's grid), the input gradient sum_d g_d a_{4d+s} plus the path through the luminance, which is
// zeroed where gz equals z0 or z1 (backward.cu:145-146).  TV (tv.cu:12-142) is (1 / (12 N)) sum over (n, c) of the
// three means of squared neighbour differences, with the gradient read from a host scalar (tv.cu:183: .item()).
//
// Here:
//  * the coordinates are computed in float32 with the reference's operations, written out explicitly (the luminance
//    as the multiply and two FMAs nvcc makes of it), so cell choice and the luminance mask follow the reference's;
//  * the clamp is folded into the slice (forward clamps, backward returns the gradient with respect to the UNCLAMPED
//    input with torch's inclusive clamp mask), and the input may be [H,W,3] (the from-world blend's output) or [3,H,W]
//    (the fastgs image);
//  * the image index is read from device memory, so one captured CUDA graph slices a different image on every replay;
//  * the backward reduces the grid gradient inside the CTA: a warp (one pixel row of 32 columns) stages its pixels in
//    shared memory and its lanes each own a few (x corner, z level, channel) outputs, summing the warp's 32 pixels
//    for them; the warp's sums go into a shared-memory box covering the cells the CTA's 8 x 32 pixel block touches,
//    and the box is added to global memory once per CTA.  Where the box does not fit (grid cells much smaller than
//    the pixel block), the warp sums go to global memory directly -- still one update per (cell, channel) per warp;
//  * the TV loss and its gradient are one launch: the upstream weight comes from device memory, every gradient
//    element is written (no zero-fill), and the loss is reduced deterministically (per-CTA partials, the last CTA
//    sums them in a fixed order) into a device scalar.
#include "gsb_common.cuh"

namespace gsb {

constexpr int kBgThreads = 256;
constexpr int kBwdRows = 8, kBwdCols = 32; // backward CTA: one warp per pixel row of 32 columns
constexpr int kBoxFloats = 6144;           // shared-memory grid-gradient box (24 KB)
constexpr int kTvThreads = 256;
constexpr int kTvMaxBlocks = 1024;

struct BgShape {
    int L, H, W;       // grid guidance depth, height, width
    int n_images;
    int h, w;          // image
    const int32_t *image_idx; // device scalar or null (image 0)
};

struct BgCoords {
    int x0, x1, y0, y1, z0, z1;
    float fx, fy, fz;
    bool zpass; // the gradient through the luminance is kept (gz is neither z0 nor z1)
};

// (i / (n - 1)) * (N - 1) in float32, the reference's operations (forward.cu:34-39).  The division is IEEE here; the
// reference's -use_fast_math build divides approximately, so the two can pick different cells only where a coordinate
// lies within an ulp of an integer -- where the interpolation is continuous and both give the same value to rounding.
__device__ __forceinline__ float bg_axis(int i, int n_img, int n_grid) {
    return __fmul_rn(__fdiv_rn((float)i, (float)(n_img - 1)), (float)(n_grid - 1));
}

__device__ __forceinline__ BgCoords bg_coords(const BgShape &s, int i, int j, float r, float g, float b) {
    BgCoords c;
    const float x = bg_axis(j, s.w, s.W), y = bg_axis(i, s.h, s.H);
    // 0.299 r + 0.587 g + 0.114 b as nvcc contracts it in the reference's build: one multiply, then two FMAs
    const float lum = __fmaf_rn(0.114f, b, __fmaf_rn(0.587f, g, __fmul_rn(0.299f, r)));
    const float z = __fmul_rn(lum, (float)(s.L - 1));
    c.x0 = (int)floorf(x);
    c.y0 = (int)floorf(y);
    const int zf = (int)floorf(z);
    c.x1 = min(c.x0 + 1, s.W - 1);
    c.y1 = min(c.y0 + 1, s.H - 1);
    c.z1 = min(max(zf + 1, 0), s.L - 1);
    c.z0 = max(zf, 0);
    c.fx = x - (float)c.x0;
    c.fy = y - (float)c.y0;
    c.fz = z - (float)c.z0;
    c.zpass = ((float)c.z0 != z) && ((float)c.z1 != z);
    return c;
}

__device__ __forceinline__ float bg_clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// bilinear interpolation of the 12 volumes in the xy plane at depth z
__device__ __forceinline__ void bg_plane(const float *__restrict__ grid, int LHW, int H, int W, int z, const BgCoords &c,
                                         float out[12]) {
    const int r0 = (z * H + c.y0) * W, r1 = (z * H + c.y1) * W;
    const float wx0 = 1.f - c.fx, wy0 = 1.f - c.fy;
#pragma unroll
    for (int ch = 0; ch < 12; ++ch) {
        const float *v = grid + (size_t)ch * LHW;
        const float a = wx0 * __ldg(v + r0 + c.x0) + c.fx * __ldg(v + r0 + c.x1);
        const float b = wx0 * __ldg(v + r1 + c.x0) + c.fx * __ldg(v + r1 + c.x1);
        out[ch] = wy0 * a + c.fy * b;
    }
}

__device__ __forceinline__ int bg_image(const BgShape &s) { return s.image_idx ? __ldg(s.image_idx) : 0; }

template <bool CHW>
__global__ void __launch_bounds__(kBgThreads) bilagrid_slice_fwd_kernel(const BgShape s, const float *__restrict__ grids,
                                                                        const float *__restrict__ in,
                                                                        float *__restrict__ out) {
    const int hw = s.h * s.w;
    const int p = blockIdx.x * kBgThreads + threadIdx.x;
    if (p >= hw) return;
    const size_t o0 = CHW ? (size_t)p : (size_t)p * 3, st = CHW ? (size_t)hw : 1;
    const int img = bg_image(s);
    if (img < 0 || img >= s.n_images) { // an out-of-range index is a caller error: make it visible
        out[o0] = out[o0 + st] = out[o0 + 2 * st] = __int_as_float(0x7fffffff);
        return;
    }
    const int LHW = s.L * s.H * s.W;
    const float *grid = grids + (size_t)img * 12 * LHW;
    const int i = p / s.w, j = p - i * s.w;
    const float r = bg_clamp01(in[o0]), g = bg_clamp01(in[o0 + st]), b = bg_clamp01(in[o0 + 2 * st]);
    const BgCoords c = bg_coords(s, i, j, r, g, b);
    float a0[12], a1[12];
    bg_plane(grid, LHW, s.H, s.W, c.z0, c, a0);
    bg_plane(grid, LHW, s.H, s.W, c.z1, c, a1);
    const float wz0 = 1.f - c.fz;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float a[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) a[k] = wz0 * a0[4 * d + k] + c.fz * a1[4 * d + k];
        out[o0 + d * st] = a[0] * r + a[1] * g + a[2] * b + a[3];
    }
}

struct BwdStage {
    int x0[kBwdRows][kBwdCols], x1[kBwdRows][kBwdCols], z0[kBwdRows][kBwdCols], z1[kBwdRows][kBwdCols];
    float fx[kBwdRows][kBwdCols], fz[kBwdRows][kBwdCols];
    float v[kBwdRows][kBwdCols][12]; // x_s * g_d of channel 4d+s (x_3 = 1)
};

template <bool CHW>
__global__ void __launch_bounds__(kBgThreads) bilagrid_slice_bwd_kernel(const BgShape s, const float *__restrict__ grids,
                                                                        const float *__restrict__ in,
                                                                        const float *__restrict__ v_out,
                                                                        float *__restrict__ v_grids,
                                                                        float *__restrict__ v_in) {
    __shared__ BwdStage S;
    __shared__ float box[kBoxFloats];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tx0 = blockIdx.x * kBwdCols, ty0 = blockIdx.y * kBwdRows;
    const int i = ty0 + warp, j = tx0 + lane;
    const int hw = s.h * s.w;
    const int img = bg_image(s);
    const bool pix = i < s.h && j < s.w;
    const size_t o0 = CHW ? (size_t)i * s.w + j : ((size_t)i * s.w + j) * 3, st = CHW ? (size_t)hw : 1;
    if (img < 0 || img >= s.n_images) {
        if (pix) v_in[o0] = v_in[o0 + st] = v_in[o0 + 2 * st] = __int_as_float(0x7fffffff);
        return;
    }
    const int LHW = s.L * s.H * s.W;
    const float *grid = grids + (size_t)img * 12 * LHW;
    float *vgrid = v_grids + (size_t)img * 12 * LHW;

    // the cells the CTA's pixel block touches: x0 and x1 grow with the column, y0 and y1 with the row
    const int jl = min(tx0 + kBwdCols, s.w) - 1, il = min(ty0 + kBwdRows, s.h) - 1;
    const int bx0 = (int)floorf(bg_axis(tx0, s.w, s.W)), bx1 = min((int)floorf(bg_axis(jl, s.w, s.W)) + 1, s.W - 1);
    const int by0 = (int)floorf(bg_axis(ty0, s.h, s.H)), by1 = min((int)floorf(bg_axis(il, s.h, s.H)) + 1, s.H - 1);
    const int nbx = bx1 - bx0 + 1, nby = by1 - by0 + 1;
    const int nbox = 12 * s.L * nby * nbx;
    const bool use_box = nbox <= kBoxFloats;
    if (use_box)
        for (int e = tid; e < nbox; e += kBgThreads) box[e] = 0.f;

    // (1) per pixel: input gradient, and the staged factors of the grid gradient
    BgCoords c{};
    if (pix) {
        const float raw[3] = {in[o0], in[o0 + st], in[o0 + 2 * st]};
        const float x[4] = {bg_clamp01(raw[0]), bg_clamp01(raw[1]), bg_clamp01(raw[2]), 1.f};
        const float gd[3] = {v_out[o0], v_out[o0 + st], v_out[o0 + 2 * st]};
        c = bg_coords(s, i, j, x[0], x[1], x[2]);
        float a0[12], a1[12];
        bg_plane(grid, LHW, s.H, s.W, c.z0, c, a0);
        bg_plane(grid, LHW, s.H, s.W, c.z1, c, a1);
        const float wz0 = 1.f - c.fz;
        float vx[3] = {0.f, 0.f, 0.f}, dz = 0.f;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int ch = 4 * d + k;
                if (k < 3) vx[k] += gd[d] * (wz0 * a0[ch] + c.fz * a1[ch]);
                dz += (a1[ch] - a0[ch]) * x[k] * gd[d]; // d(out)/d(z) per unit of z
                S.v[warp][lane][ch] = x[k] * gd[d];
            }
        }
        const float gz = c.zpass ? dz * (float)(s.L - 1) : 0.f; // backward.cu:145-146
        const float lum[3] = {0.299f, 0.587f, 0.114f};
#pragma unroll
        for (int k = 0; k < 3; ++k) // torch's clamp backward: the gradient passes where 0 <= raw <= 1
            v_in[o0 + k * st] = (raw[k] >= 0.f && raw[k] <= 1.f) ? vx[k] + lum[k] * gz : 0.f;
        S.x0[warp][lane] = c.x0; S.x1[warp][lane] = c.x1;
        S.z0[warp][lane] = c.z0; S.z1[warp][lane] = c.z1;
        S.fx[warp][lane] = c.fx; S.fz[warp][lane] = c.fz;
    }
    __syncthreads(); // the box is zeroed, the stage is written

    // (2) per warp (one pixel row): lanes own (x corner, z level, channel) outputs and sum the row's pixels for them
    if (i < s.h) {
        const int nvalid = min(kBwdCols, s.w - tx0);
        const int xlo = __reduce_min_sync(0xffffffffu, pix ? c.x0 : 0x7fffffff);
        const int xhi = __reduce_max_sync(0xffffffffu, pix ? c.x1 : -1);
        const int zlo = __reduce_min_sync(0xffffffffu, pix ? c.z0 : 0x7fffffff);
        const int zhi = __reduce_max_sync(0xffffffffu, pix ? c.z1 : -1);
        const float fy = __shfl_sync(0xffffffffu, c.fy, 0);
        const int y0 = __shfl_sync(0xffffffffu, c.y0, 0), y1 = __shfl_sync(0xffffffffu, c.y1, 0);
        const int nz = zhi - zlo + 1, n_out = (xhi - xlo + 1) * nz * 12;
        for (int o = lane; o < n_out; o += 32) {
            const int ch = o % 12, r = o / 12;
            const int zl = zlo + r % nz, xi = xlo + r / nz;
            float sum = 0.f;
            for (int q = 0; q < nvalid; ++q) {
                const float fx = S.fx[warp][q], fz = S.fz[warp][q];
                const float wx = (S.x0[warp][q] == xi ? 1.f - fx : 0.f) + (S.x1[warp][q] == xi ? fx : 0.f);
                const float wz = (S.z0[warp][q] == zl ? 1.f - fz : 0.f) + (S.z1[warp][q] == zl ? fz : 0.f);
                sum = fmaf(wx * wz, S.v[warp][q][ch], sum);
            }
            if (sum != 0.f) {
                if (use_box) {
                    float *b = box + ((ch * s.L + zl) * nby) * nbx + (xi - bx0);
                    atomicAdd(b + (y0 - by0) * nbx, (1.f - fy) * sum);
                    atomicAdd(b + (y1 - by0) * nbx, fy * sum);
                } else {
                    float *g = vgrid + (size_t)ch * LHW + (size_t)zl * s.H * s.W + xi;
                    atomicAdd(g + y0 * s.W, (1.f - fy) * sum);
                    atomicAdd(g + y1 * s.W, fy * sum);
                }
            }
        }
    }
    if (!use_box) return;
    __syncthreads();
    // (3) one global update per touched (cell, channel) of the CTA
    for (int e = tid; e < nbox; e += kBgThreads) {
        const float val = box[e];
        if (val == 0.f) continue;
        const int xr = e % nbx, t = e / nbx;
        const int yr = t % nby, t2 = t / nby;
        const int zl = t2 % s.L, ch = t2 / s.L;
        atomicAdd(vgrid + (size_t)ch * LHW + ((size_t)zl * s.H + by0 + yr) * s.W + bx0 + xr, val);
    }
}

struct TvArgs {
    const float *grids;
    float *v_grids;        // null: loss only
    const float *weight;   // device scalar (upstream gradient of the loss) or null (1)
    float *loss_out;       // device scalar
    double *partials;      // [gridDim.x][3]
    unsigned int *done;    // zeroed before the launch
    long long total;
    int L, H, W, N;
};

__device__ __forceinline__ double bg_block_sum(double v, double *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int k = 0; k < kTvThreads / 32; ++k) t += red[k]; // fixed order: deterministic
    return t;
}

__global__ void __launch_bounds__(kTvThreads) bilagrid_tv_kernel(const TvArgs a) {
    __shared__ double red[kTvThreads / 32];
    __shared__ bool last;
    const int W = a.W, H = a.H, L = a.L, HW = H * W;
    // per-direction 1 / (number of neighbour pairs); a direction of size 1 has none
    const float ix = W > 1 ? 1.f / (float)(L * H * (W - 1)) : 0.f;
    const float iy = H > 1 ? 1.f / (float)(L * (H - 1) * W) : 0.f;
    const float iz = L > 1 ? 1.f / (float)((L - 1) * H * W) : 0.f;
    const float s = (a.weight ? __ldg(a.weight) : 1.f) / (6.f * (float)a.N);
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (long long e = (long long)blockIdx.x * kTvThreads + threadIdx.x; e < a.total; e += (long long)gridDim.x * kTvThreads) {
        const int x = (int)(e % W);
        const long long t = e / W;
        const int y = (int)(t % H), z = (int)((t / H) % L);
        const float *p = a.grids + e;
        const float v = __ldg(p);
        float g = 0.f;
        if (x > 0) { const float d = v - __ldg(p - 1); sx = fmaf(d, d, sx); g += d * ix; }
        if (x < W - 1) g += (v - __ldg(p + 1)) * ix;
        if (y > 0) { const float d = v - __ldg(p - W); sy = fmaf(d, d, sy); g += d * iy; }
        if (y < H - 1) g += (v - __ldg(p + W)) * iy;
        if (z > 0) { const float d = v - __ldg(p - HW); sz = fmaf(d, d, sz); g += d * iz; }
        if (z < L - 1) g += (v - __ldg(p + HW)) * iz;
        if (a.v_grids) a.v_grids[e] = s * g;
    }
    const double bx = bg_block_sum((double)sx, red), by = bg_block_sum((double)sy, red), bz = bg_block_sum((double)sz, red);
    if (threadIdx.x == 0) {
        a.partials[3 * blockIdx.x + 0] = bx;
        a.partials[3 * blockIdx.x + 1] = by;
        a.partials[3 * blockIdx.x + 2] = bz;
        __threadfence();
        last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double tx = 0.0, ty = 0.0, tz = 0.0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += kTvThreads) {
        const volatile double *q = a.partials + 3 * b;
        tx += q[0]; ty += q[1]; tz += q[2];
    }
    tx = bg_block_sum(tx, red); ty = bg_block_sum(ty, red); tz = bg_block_sum(tz, red);
    if (threadIdx.x == 0)
        *a.loss_out = (float)((tx * (double)ix + ty * (double)iy + tz * (double)iz) / (12.0 * (double)a.N));
}

static int bg_check_shape(uint32_t grid_w, uint32_t grid_h, uint32_t grid_l, uint32_t n_images) {
    if (grid_w == 0 || grid_h == 0 || grid_l == 0 || n_images == 0) return GSB_E_INVALID;
    if ((uint64_t)n_images * 12 * grid_l * grid_h * grid_w > 0x7fffffffull) return GSB_E_INVALID;
    return GSB_OK;
}

} // namespace gsb

extern "C" int gsb_bilagrid_slice_fwd(uint32_t grid_w, uint32_t grid_h, uint32_t grid_l, uint32_t n_images,
                                      const float *grids, const int32_t *image_idx, uint32_t image_width,
                                      uint32_t image_height, int layout, const float *input, float *output,
                                      gsb_stream_t stream) {
    using namespace gsb;
    if (bg_check_shape(grid_w, grid_h, grid_l, n_images) != GSB_OK) return GSB_E_INVALID;
    if (!grids || !input || !output) return GSB_E_INVALID;
    if (image_width < 2 || image_height < 2 || (uint64_t)image_width * image_height > 0x7fffffffull) return GSB_E_INVALID;
    const BgShape s{(int)grid_l, (int)grid_h, (int)grid_w, (int)n_images, (int)image_height, (int)image_width, image_idx};
    cudaStream_t st = as_stream(stream);
    const unsigned blocks = (unsigned)((image_width * image_height + kBgThreads - 1) / kBgThreads);
    {
        ProfScope ps("bilagrid_slice_fwd", st);
        if (layout & GSB_BILAGRID_CHW) bilagrid_slice_fwd_kernel<true><<<blocks, kBgThreads, 0, st>>>(s, grids, input, output);
        else bilagrid_slice_fwd_kernel<false><<<blocks, kBgThreads, 0, st>>>(s, grids, input, output);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

extern "C" int gsb_bilagrid_slice_bwd(uint32_t grid_w, uint32_t grid_h, uint32_t grid_l, uint32_t n_images,
                                      const float *grids, const int32_t *image_idx, uint32_t image_width,
                                      uint32_t image_height, int layout, const float *input, const float *v_output,
                                      float *v_grids, float *v_input, gsb_stream_t stream) {
    using namespace gsb;
    if (bg_check_shape(grid_w, grid_h, grid_l, n_images) != GSB_OK) return GSB_E_INVALID;
    if (!grids || !input || !v_output || !v_grids || !v_input) return GSB_E_INVALID;
    if (image_width < 2 || image_height < 2 || (uint64_t)image_width * image_height > 0x7fffffffull) return GSB_E_INVALID;
    const BgShape s{(int)grid_l, (int)grid_h, (int)grid_w, (int)n_images, (int)image_height, (int)image_width, image_idx};
    cudaStream_t st = as_stream(stream);
    const dim3 blocks((image_width + kBwdCols - 1) / kBwdCols, (image_height + kBwdRows - 1) / kBwdRows);
    {
        ProfScope ps("bilagrid_slice_bwd", st);
        if (layout & GSB_BILAGRID_CHW)
            bilagrid_slice_bwd_kernel<true><<<blocks, kBgThreads, 0, st>>>(s, grids, input, v_output, v_grids, v_input);
        else
            bilagrid_slice_bwd_kernel<false><<<blocks, kBgThreads, 0, st>>>(s, grids, input, v_output, v_grids, v_input);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

static unsigned gsb_bilagrid_tv_blocks(uint64_t total) {
    const uint64_t b = (total + gsb::kTvThreads - 1) / gsb::kTvThreads;
    return (unsigned)(b < (uint64_t)gsb::kTvMaxBlocks ? b : (uint64_t)gsb::kTvMaxBlocks);
}

extern "C" size_t gsb_bilagrid_tv_workspace(void) { return 256 + (size_t)gsb::kTvMaxBlocks * 3 * sizeof(double); }

extern "C" int gsb_bilagrid_tv(uint32_t grid_w, uint32_t grid_h, uint32_t grid_l, uint32_t n_images, const float *grids,
                               const float *grad_weight, float *loss_out, float *v_grids, void *workspace,
                               size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (bg_check_shape(grid_w, grid_h, grid_l, n_images) != GSB_OK) return GSB_E_INVALID;
    if (!grids || !loss_out) return GSB_E_INVALID;
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_bilagrid_tv_workspace())
        return GSB_E_WORKSPACE;
    cudaStream_t st = as_stream(stream);
    GSB_CUDA_TRY(cudaMemsetAsync(workspace, 0, sizeof(unsigned int), st));
    TvArgs a;
    a.grids = grids; a.v_grids = v_grids; a.weight = grad_weight; a.loss_out = loss_out;
    a.done = reinterpret_cast<unsigned int *>(workspace);
    a.partials = reinterpret_cast<double *>(reinterpret_cast<char *>(workspace) + 256);
    a.L = (int)grid_l; a.H = (int)grid_h; a.W = (int)grid_w; a.N = (int)n_images;
    a.total = (long long)n_images * 12 * grid_l * grid_h * grid_w;
    {
        ProfScope ps("bilagrid_tv", st);
        bilagrid_tv_kernel<<<gsb_bilagrid_tv_blocks((uint64_t)a.total), kTvThreads, 0, st>>>(a);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
