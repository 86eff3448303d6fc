// gsb_loss.cu -- SURVEY.md 8(f2): the photometric loss of the training step and its gradient in ONE kernel.
//
// The reference computes (src/training/trainer.cpp:103-126)
//     image = clamp(render, 0, 1) permuted to CHW                      (rasterizer.cpp:401)
//     loss  = (1 - lambda) * l1_loss(image, gt) + lambda * (1 - fused_ssim(image, gt, "valid"))
// with fused_ssim = mean over the map cropped by 5 pixels per side of the 11x11 Gaussian-window SSIM evaluated with
// zero padding (src/training/kernels/ssim.cu:64-283, include/kernels/fused_ssim.cuh:27-117), and gets the gradient
// from a second stencil kernel over three stored derivative maps plus the autograd of clamp / permute / l1 / mean
// (ssim.cu:284-420).  Here one kernel reads the blend's [H,W,3] output and the target once and writes the loss and
// dLoss/d(render) -- exactly what gsb_raster_bwd consumes: per 32x16 tile it stages a 52x36 neighbourhood (tile + two
// halos), runs the separable 11-tap window twice (statistics on 42x26, then the three derivative maps back onto the
// tile), and folds in the L1 term, the crop, the means and the clamp mask.  No derivative maps, no permuted copies and
// no 2-million-element reductions go through HBM.  Every stage is cut into about 256 strips (one per thread) and is
// input-stationary -- an input is read from shared memory once and added to every output whose window covers it -- so
// a thread keeps a handful of accumulators instead of a row of inputs (64 registers, three CTAs per SM).
#include "gsb_common.cuh"

namespace gsb {

constexpr int kLossThreads = 256;
constexpr int kTW = 32, kTH = 16; // tile of output pixels per CTA (independent of the blend's tiling)
constexpr int kHalo = 5;          // window radius
constexpr int kSW = kTW + 2 * kHalo, kSH = kTH + 2 * kHalo; // 42 x 26: pixels whose SSIM statistics the tile needs
constexpr int kIW = kTW + 4 * kHalo, kIH = kTH + 4 * kHalo; // 52 x 36: input neighbourhood
// strips: every stage hands one strip of outputs of one row / column to a thread, sized so that a stage has about
// kLossThreads work items: 36 rows x 7 strips of 6 | 42 columns x 6 strips of 5,5,4,4,4,4 | 26 rows x 8 strips of 4 |
// 32 columns x 8 strips of 2
constexpr int kS1 = 6, kN1 = kSW / kS1;  // 7
constexpr int kS2 = 5, kN2 = 6;          // ragged: two strips of 5, four of 4
constexpr int kS3 = 4, kN3 = kTW / kS3;  // 8
constexpr int kS4 = 2, kN4 = kTH / kS4;  // 8
static_assert(kS1 * kN1 == kSW && kS3 * kN3 == kTW && kS4 * kN4 == kTH && 2 * 5 + 4 * 4 == kSH, "strip plan");
// shared-memory rows are padded to an odd number of 8-byte words: a warp whose lanes are rows is conflict-free
constexpr int kIP = kIW + 1, kSP = kSW + 1, kTP = kTW + 1; // 53, 43, 33

__constant__ float c_win[11] = {0.001028380084f, 0.007598758135f, 0.03600077213f, 0.1093606895f, 0.2130055377f,
                                0.2660117249f,   0.2130055377f,   0.1093606895f,  0.03600077213f, 0.007598758135f,
                                0.001028380084f}; // exp(-x^2 / (2 * 1.5^2)) normalised, x = -5..5

struct LossParams {
    uint32_t H, W;
    const float *renders;   // [H,W,3] or [3,H,W] (renders_chw), unclamped
    const float *target;    // [3,H,W] (target_chw) or [H,W,3]
    int target_chw, renders_chw;
    float lambda;           // weight of the SSIM term (lambda_dssim)
    float grad_scale;       // upstream gradient of the scalar loss
    float *v_renders;       // laid out like renders, or null (evaluation)
    double *acc;            // [2] running sums (|x - y|, ssim), zeroed before the launch
    unsigned int *done;     // [1] CTA counter, zeroed before the launch
    float *loss_out;        // [3] loss, l1 mean, ssim mean
    uint32_t y_lo, y_hi, x_lo, x_hi; // valid (cropped) region of the SSIM map
};

struct LossSmem {
    float2 xy[kIH][kIP];        // (clamped render, target), zero outside the image
    float2 h02[kIH + 1][kSP];   // horizontal pass of (X, Y); one spare row for the ragged vertical strips
    float2 h13[kIH + 1][kSP];   //                    (X^2, Y^2)
    float h4[kIH + 1][kSP];     //                    X Y
    float2 m01[kSH][kSP];       // chain * (dm/dmu1, dm/dsigma1^2)
    float m2[kSH][kSP];         // chain * dm/dsigma12
};
// the horizontal pass of the derivative maps reuses the h02 / h4 storage (dead after the vertical statistics pass)
static_assert(sizeof(float2) * kSH * kTP <= sizeof(float2) * (kIH + 1) * kSP, "g01 alias");
static_assert(sizeof(float) * kSH * kTP <= sizeof(float) * (kIH + 1) * kSP, "g2 alias");

// NoClamp (GSB_LOSS_NO_CLAMP): the renders enter as they are and every pixel passes the gradient
template <bool NoClamp>
__global__ void __launch_bounds__(kLossThreads, 3) ssim_l1_kernel(const LossParams p) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    LossSmem &S = *reinterpret_cast<LossSmem *>(s_raw);
    float2 (*g01)[kTP] = reinterpret_cast<float2 (*)[kTP]>(&S.h02[0][0]);
    float (*g2)[kTP] = reinterpret_cast<float (*)[kTP]>(&S.h4[0][0]);
    __shared__ float s_red[2][kLossThreads / 32];
    __shared__ uint8_t s_pass[kTH][kTW];
    const int tid = threadIdx.x;
    const int tx0 = blockIdx.x * kTW, ty0 = blockIdx.y * kTH;
    const int H = (int)p.H, W = (int)p.W;
    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
    const float n_valid = (float)(p.y_hi - p.y_lo) * (float)(p.x_hi - p.x_lo) * 3.0f;
    const float chain = -p.lambda * p.grad_scale / n_valid;
    const float l1_w = (1.0f - p.lambda) * p.grad_scale / ((float)H * (float)W * 3.0f);
    float l1_sum = 0.f, ssim_sum = 0.f;
    f2 w2[6]; // the window is symmetric: tap j and tap 10 - j share a weight
#pragma unroll
    for (int j = 0; j < 6; ++j) w2[j] = f2_bc(c_win[j]);

    for (int c = 0; c < 3; ++c) {
        // (0) neighbourhood of the tile: a warp per row (no index divisions, the row's loads are in flight together)
        for (int r = tid >> 5; r < kIH; r += kLossThreads / 32) {
            const int gy = ty0 + r - 2 * kHalo;
            const bool row_ok = gy >= 0 && gy < H;
            const size_t gyc = row_ok ? (size_t)gy : 0;
            const float *rrow = p.renders_chw ? p.renders + ((size_t)c * H + gyc) * W : p.renders + gyc * W * 3 + c;
            const int rstep = p.renders_chw ? 1 : 3;
            const float *trow = p.target_chw ? p.target + ((size_t)c * H + gyc) * W : p.target + gyc * W * 3 + c;
            const int tstep = p.target_chw ? 1 : 3;
#pragma unroll
            for (int k = 0; k < (kIW + 31) / 32; ++k) {
                const int q = (tid & 31) + 32 * k;
                if (q < kIW) {
                    const int gx = tx0 + q - 2 * kHalo;
                    float X = 0.f, Y = 0.f;
                    if (row_ok && gx >= 0 && gx < W) {
                        const float raw = rrow[gx * rstep];
                        X = NoClamp ? raw : fminf(fmaxf(raw, 0.f), 1.f);
                        Y = trow[gx * tstep];
                        // the tile's own pixels remember whether the clamp was active (dLoss/d(render) = 0 there)
                        const int tr = r - 2 * kHalo, tq = q - 2 * kHalo;
                        if (tr >= 0 && tr < kTH && tq >= 0 && tq < kTW) s_pass[tr][tq] = (NoClamp || (raw >= 0.f && raw <= 1.f)) ? 1 : 0;
                    }
                    S.xy[r][q] = make_float2(X, Y);
                }
            }
        }
        __syncthreads();
        // (1) horizontal window, 36 rows x 42 columns.  Input-stationary: every input is read once and added to the
        //     outputs whose window covers it, so a thread holds kS1 x 5 accumulators and one input, not a row of
        //     inputs.  The five windowed quantities ride on packed fp32 pairs: (X, Y), (X^2, Y^2) and a scalar XY.
        for (int it = tid; it < kIH * kN1; it += kLossThreads) {
            const int r = it % kIH, q0 = (it / kIH) * kS1;
            f2 a02[kS1], a13[kS1];
            float a4[kS1];
#pragma unroll
            for (int o = 0; o < kS1; ++o) { a02[o] = f2_bc(0.f); a13[o] = f2_bc(0.f); a4[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < kS1 + 10; ++k) {
                const float2 v = S.xy[r][q0 + k];
                const f2 xy = f2_make(v.x, v.y);
                const f2 sq = f2_mul(xy, xy);
                const float pr = v.x * v.y;
#pragma unroll
                for (int o = 0; o < kS1; ++o) {
                    const int j = k - o; // tap index of this input in output o's window
                    if (j >= 0 && j <= 10) {
                        const int jj = j <= 5 ? j : 10 - j;
                        a02[o] = f2_fma(w2[jj], xy, a02[o]);
                        a13[o] = f2_fma(w2[jj], sq, a13[o]);
                        a4[o] = fmaf(c_win[jj], pr, a4[o]);
                    }
                }
            }
#pragma unroll
            for (int o = 0; o < kS1; ++o) {
                S.h02[r][q0 + o] = make_float2(f2_lo(a02[o]), f2_hi(a02[o]));
                S.h13[r][q0 + o] = make_float2(f2_lo(a13[o]), f2_hi(a13[o]));
                S.h4[r][q0 + o] = a4[o];
            }
        }
        __syncthreads();
        // (2) vertical window -> statistics of the 26 x 42 pixels -> SSIM value and the three derivative maps
        for (int it = tid; it < kSW * kN2; it += kLossThreads) {
            const int q = it % kSW, st = it / kSW;
            const int r0 = st * 4 + (st < 2 ? st : 2), len = st < 2 ? 5 : 4;
            f2 a02[kS2], a13[kS2];
            float a4[kS2];
#pragma unroll
            for (int o = 0; o < kS2; ++o) { a02[o] = f2_bc(0.f); a13[o] = f2_bc(0.f); a4[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < kS2 + 10; ++k) {
                const float2 u = S.h02[r0 + k][q], v = S.h13[r0 + k][q]; // row r0 + 14 of a short strip: spare row
                const f2 v02 = f2_make(u.x, u.y), v13 = f2_make(v.x, v.y);
                const float v4 = S.h4[r0 + k][q];
#pragma unroll
                for (int o = 0; o < kS2; ++o) {
                    const int j = k - o;
                    if (j >= 0 && j <= 10) {
                        const int jj = j <= 5 ? j : 10 - j;
                        a02[o] = f2_fma(w2[jj], v02, a02[o]);
                        a13[o] = f2_fma(w2[jj], v13, a13[o]);
                        a4[o] = fmaf(c_win[jj], v4, a4[o]);
                    }
                }
            }
#pragma unroll
            for (int o = 0; o < kS2; ++o) {
                if (o < len) {
                    const int r = r0 + o;
                    const int gy = ty0 + r - kHalo, gx = tx0 + q - kHalo;
                    float m0 = 0.f, m1 = 0.f, m2 = 0.f;
                    const bool in_img = gy >= 0 && gy < H && gx >= 0 && gx < W;
                    const bool in_valid = gy >= (int)p.y_lo && gy < (int)p.y_hi && gx >= (int)p.x_lo && gx < (int)p.x_hi;
                    if (in_img && in_valid) {
                        const float mu1 = f2_lo(a02[o]), mu2 = f2_hi(a02[o]);
                        const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2;
                        const float sigma1_sq = f2_lo(a13[o]) - mu1_sq, sigma2_sq = f2_hi(a13[o]) - mu2_sq;
                        const float sigma12 = a4[o] - mu1 * mu2;
                        const float A = mu1_sq + mu2_sq + C1, B = sigma1_sq + sigma2_sq + C2;
                        const float Cc = 2.f * mu1 * mu2 + C1, D = 2.f * sigma12 + C2;
                        const float iAB = 1.0f / (A * B);
                        // ssim.cu:253-263
                        m0 = chain * ((mu2 * 2.f * D) * iAB - (mu2 * 2.f * Cc) * iAB - (mu1 * 2.f * Cc * D) * iAB / A +
                                      (mu1 * 2.f * Cc * D) * iAB / B);
                        m1 = chain * ((-Cc * D) * iAB / B);
                        m2 = chain * ((2.f * Cc) * iAB);
                        // the tile's own pixels add their SSIM value to the mean
                        if (r >= kHalo && r < kHalo + kTH && q >= kHalo && q < kHalo + kTW) ssim_sum += (Cc * D) * iAB;
                    }
                    S.m01[r][q] = make_float2(m0, m1);
                    S.m2[r][q] = m2;
                }
            }
        }
        __syncthreads();
        // (3) horizontal window of the derivative maps: 26 rows x 32 columns; maps 0 and 1 packed
        for (int it = tid; it < kSH * kN3; it += kLossThreads) {
            const int r = it % kSH, q0 = (it / kSH) * kS3;
            f2 a01[kS3];
            float a2[kS3];
#pragma unroll
            for (int o = 0; o < kS3; ++o) { a01[o] = f2_bc(0.f); a2[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < kS3 + 10; ++k) {
                const float2 u = S.m01[r][q0 + k];
                const f2 v01 = f2_make(u.x, u.y);
                const float v2 = S.m2[r][q0 + k];
#pragma unroll
                for (int o = 0; o < kS3; ++o) {
                    const int j = k - o;
                    if (j >= 0 && j <= 10) {
                        const int jj = j <= 5 ? j : 10 - j;
                        a01[o] = f2_fma(w2[jj], v01, a01[o]);
                        a2[o] = fmaf(c_win[jj], v2, a2[o]);
                    }
                }
            }
#pragma unroll
            for (int o = 0; o < kS3; ++o) {
                g01[r][q0 + o] = make_float2(f2_lo(a01[o]), f2_hi(a01[o]));
                g2[r][q0 + o] = a2[o];
            }
        }
        __syncthreads();
        // (4) vertical window + L1 term + clamp mask -> dLoss / d(render): 32 columns x 8 strips of 2 rows
        for (int it = tid; it < kTW * kN4; it += kLossThreads) {
            const int q = it % kTW, r0 = (it / kTW) * kS4;
            f2 a01[kS4];
            float a2[kS4];
#pragma unroll
            for (int o = 0; o < kS4; ++o) { a01[o] = f2_bc(0.f); a2[o] = 0.f; }
#pragma unroll
            for (int k = 0; k < kS4 + 10; ++k) {
                const float2 u = g01[r0 + k][q];
                const f2 v01 = f2_make(u.x, u.y);
                const float v2 = g2[r0 + k][q];
#pragma unroll
                for (int o = 0; o < kS4; ++o) {
                    const int j = k - o;
                    if (j >= 0 && j <= 10) {
                        const int jj = j <= 5 ? j : 10 - j;
                        a01[o] = f2_fma(w2[jj], v01, a01[o]);
                        a2[o] = fmaf(c_win[jj], v2, a2[o]);
                    }
                }
            }
#pragma unroll
            for (int o = 0; o < kS4; ++o) {
                const int gy = ty0 + r0 + o, gx = tx0 + q;
                if (gy < H && gx < W) {
                    const float2 px = S.xy[r0 + o + 2 * kHalo][q + 2 * kHalo];
                    const float d = px.x - px.y;
                    l1_sum += fabsf(d);
                    if (p.v_renders) {
                        float g = f2_lo(a01[o]) + (2.f * px.x) * f2_hi(a01[o]) + px.y * a2[o]; // ssim.cu:411
                        g += l1_w * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
                        const size_t oi = p.renders_chw ? ((size_t)c * H + gy) * W + gx : ((size_t)gy * W + gx) * 3 + c;
                        p.v_renders[oi] = s_pass[r0 + o][q] ? g : 0.f;
                    }
                }
            }
        }
        __syncthreads();
    }

    // loss: CTA sums -> two double atomics; the last CTA turns the sums into the scalar
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        l1_sum += __shfl_xor_sync(0xffffffffu, l1_sum, o);
        ssim_sum += __shfl_xor_sync(0xffffffffu, ssim_sum, o);
    }
    if ((tid & 31) == 0) { s_red[0][tid >> 5] = l1_sum; s_red[1][tid >> 5] = ssim_sum; }
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, b = 0.0;
        for (int w = 0; w < kLossThreads / 32; ++w) { a += (double)s_red[0][w]; b += (double)s_red[1][w]; }
        atomicAdd(&p.acc[0], a);
        atomicAdd(&p.acc[1], b);
        __threadfence();
        const unsigned int ticket = atomicAdd(p.done, 1u);
        if (ticket == gridDim.x * gridDim.y - 1) {
            __threadfence();
            const double l1 = *((volatile double *)&p.acc[0]) / ((double)H * (double)W * 3.0);
            const double ss = *((volatile double *)&p.acc[1]) / (double)n_valid;
            p.loss_out[0] = (float)((1.0 - (double)p.lambda) * l1 + (double)p.lambda * (1.0 - ss));
            p.loss_out[1] = (float)l1;
            p.loss_out[2] = (float)ss;
        }
    }
}

// The workspace: the running sums and the CTA ticket, zeroed together before every launch.
struct LossCtl {
    double acc[2];
    unsigned int done;
};

} // namespace gsb

extern "C" size_t gsb_ssim_l1_workspace(void) { return gsb::align256(sizeof(gsb::LossCtl)); }

extern "C" int gsb_ssim_l1(uint32_t image_width, uint32_t image_height, const float *renders, const float *target,
                           int target_chw, float lambda_dssim, float grad_scale, float *v_renders, float *loss_out,
                           void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (image_width == 0 || image_height == 0) return GSB_E_INVALID;
    if (!renders || !target || !loss_out) return GSB_E_INVALID;
    if (int rc = ws_check(workspace, workspace_bytes, gsb_ssim_l1_workspace())) return rc;
    LossCtl *ctl = static_cast<LossCtl *>(workspace);
    cudaStream_t s = as_stream(stream);
    GSB_CUDA_TRY(cudaMemsetAsync(ctl, 0, sizeof(LossCtl), s));
    LossParams p;
    p.H = image_height; p.W = image_width;
    p.renders = renders; p.target = target;
    p.target_chw = (target_chw & 1) != 0; p.renders_chw = (target_chw & 2) != 0; // GSB_LOSS_TARGET_CHW | GSB_LOSS_RENDERS_CHW
    p.lambda = lambda_dssim; p.grad_scale = grad_scale; p.v_renders = v_renders;
    p.acc = ctl->acc;
    p.done = &ctl->done;
    p.loss_out = loss_out;
    // fused_ssim(..., "valid"): the map is cropped by 5 per side only when both sides exceed 10 (fused_ssim.cuh:63-67)
    const bool crop = image_height > 10 && image_width > 10;
    p.y_lo = crop ? 5 : 0; p.y_hi = crop ? image_height - 5 : image_height;
    p.x_lo = crop ? 5 : 0; p.x_hi = crop ? image_width - 5 : image_width;
    const dim3 grid((image_width + kTW - 1) / kTW, (image_height + kTH - 1) / kTH);
    auto kernel = (target_chw & GSB_LOSS_NO_CLAMP) ? ssim_l1_kernel<true> : ssim_l1_kernel<false>;
    GSB_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(LossSmem)));
    {
        ProfScope ps(v_renders ? "ssim_l1_bwd" : "ssim_l1_fwd", s);
        kernel<<<grid, kLossThreads, sizeof(LossSmem), s>>>(p);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
