// gsb_metrics.cu -- PSNR and SSIM of one rendered view against its ground truth, the evaluation metrics of the
// reference's MetricsEvaluator (src/training/metrics/metrics.cpp:17-116), in one launch per view:
//   x = clamp(image, 0, 1) (metrics.cpp:441), y = target, both 3 x H x W;
//   PSNR = 20 log10(1 / sqrt(max(mean((x - y)^2), 1e-10)))                                    (:40-59)
//   SSIM = mean over all 3 H W of the "same"-size SSIM map: 11 x 11 window, zero padding 5, per channel,
//          C1 = 0.01^2, C2 = 0.03^2, sigma^2 = E[x^2] - mu^2                                   (:62-116)
// The window is the reference's, quirk included: gaussian() computes inv_denom = 1.0f / 2.0f * sigma * sigma = 1.125
// (not 1 / (2 sigma^2)), so the taps are exp(-d^2 * 1.125) normalised in float32, an effective sigma of ~0.67.  It is
// NOT the sigma = 1.5 window of the training loss (gsb_loss.cu), whose crop and gradient differ as well.
//
// One CTA takes a 32 x 16 tile of output pixels at a time, one channel after the other: it stages the tile and its
// 5-pixel halo of (x, y) in shared memory (zero outside the image), runs the 11 taps along rows for the five moments
// (x, y, x^2, y^2, xy), then along columns, and adds up the SSIM map and (x - y)^2 of its pixels in float64.  The grid
// is a fixed kBlocks CTAs (fewer for small images) striding over the tiles, and gsb_reduce.cuh's grid_sum_last adds
// the CTAs' partials in a fixed order: the result depends on the image size only and repeats bit for bit.  The last
// CTA writes (psnr, ssim) as float32; nothing is read back to the host.
#include <cmath>

#include "gsb_common.cuh"
#include "gsb_reduce.cuh"

namespace gsb {
namespace metrics {

constexpr int kThreads = 256;
constexpr int kWin = 11, kHalo = kWin / 2;
constexpr int kTW = 32, kTH = 16;                           // output tile
constexpr int kSW = kTW + 2 * kHalo, kSH = kTH + 2 * kHalo; // 42 x 26 staged neighbourhood
constexpr uint32_t kBlocks = 792;                           // 6 resident CTAs on each of the H100's 132 SMs
constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;   // metrics.hpp:50-51

struct Window {
    float w[kWin];
};

// gaussian(11, 1.5) (metrics.cpp:17-31) in float32, the way the reference builds it
static Window make_window() {
    Window g;
    const float sigma = 1.5f;
    const float inv_denom = 1.0f / 2.0f * sigma * sigma; // 1.125: the reference's operator precedence
    float sum = 0.0f;
    for (int x = 0; x < kWin; ++x) {
        const int d = x - kWin / 2;
        g.w[x] = std::exp(-static_cast<float>(d * d) * inv_denom);
        sum += g.w[x];
    }
    for (int x = 0; x < kWin; ++x) g.w[x] /= sum;
    return g;
}

struct Ws {
    unsigned int *ticket;
    double *partials; // [kBlocks * 2]
};

static size_t ws_layout(void *base, Ws &w) {
    WsLayout l{static_cast<char *>(base)};
    w.ticket = l.carve<unsigned int>(1);
    w.partials = l.carve<double>(2 * kBlocks);
    return l.bytes;
}

struct Args {
    uint32_t W, H, tiles_x, n_tiles;
    bool hwc; // image [H,W,3] instead of [3,H,W]
    const float *image, *target;
    float *out; // [2]: psnr, ssim
    double *partials;
    unsigned int *ticket;
    Window win;
};

// clamp(v, 0, 1) as torch::clamp computes it: NaN stays NaN
__device__ __forceinline__ float clamp01(float v) { return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }

__global__ void __launch_bounds__(kThreads) metrics_kernel(const Args a) {
    __shared__ float s_x[kSH][kSW], s_y[kSH][kSW];
    __shared__ float s_m[5][kSH][kTW]; // row-filtered moments: x, y, x^2, y^2, xy
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t plane = (size_t)a.W * a.H;
    double acc_se = 0.0, acc_ssim = 0.0;

    for (uint32_t t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        const int x0 = (int)(t % a.tiles_x) * kTW, y0 = (int)(t / a.tiles_x) * kTH;
        for (int c = 0; c < 3; ++c) {
            // stage (x, y) over the tile and its halo; zero outside the image (conv2d's zero padding)
            for (int i = threadIdx.x; i < kSH * kSW; i += kThreads) {
                const int r = i / kSW, q = i - r * kSW;
                const int gy = y0 - kHalo + r, gx = x0 - kHalo + q;
                float xv = 0.0f, yv = 0.0f;
                if (gy >= 0 && gy < (int)a.H && gx >= 0 && gx < (int)a.W) {
                    const size_t p = (size_t)gy * a.W + gx;
                    xv = clamp01(a.hwc ? a.image[3 * p + c] : a.image[c * plane + p]);
                    yv = a.target[c * plane + p];
                }
                s_x[r][q] = xv;
                s_y[r][q] = yv;
            }
            __syncthreads();
            // along rows: lane = output column, warps over the staged rows
            for (int r = warp; r < kSH; r += kThreads / 32) {
                float m0 = 0.0f, m1 = 0.0f, m2 = 0.0f, m3 = 0.0f, m4 = 0.0f;
#pragma unroll
                for (int j = 0; j < kWin; ++j) {
                    const float w = a.win.w[j], xv = s_x[r][lane + j], yv = s_y[r][lane + j];
                    m0 = fmaf(w, xv, m0);
                    m1 = fmaf(w, yv, m1);
                    m2 = fmaf(w, xv * xv, m2);
                    m3 = fmaf(w, yv * yv, m3);
                    m4 = fmaf(w, xv * yv, m4);
                }
                s_m[0][r][lane] = m0;
                s_m[1][r][lane] = m1;
                s_m[2][r][lane] = m2;
                s_m[3][r][lane] = m3;
                s_m[4][r][lane] = m4;
            }
            __syncthreads();
            // along columns, then the SSIM map (metrics.cpp:90-113) and the squared error of the tile's pixels
            const int gx = x0 + lane;
            for (int r = warp; r < kTH; r += kThreads / 32) {
                const int gy = y0 + r;
                if (gx >= (int)a.W || gy >= (int)a.H) continue;
                float mu1 = 0.0f, mu2 = 0.0f, e11 = 0.0f, e22 = 0.0f, e12 = 0.0f;
#pragma unroll
                for (int j = 0; j < kWin; ++j) {
                    const float w = a.win.w[j];
                    mu1 = fmaf(w, s_m[0][r + j][lane], mu1);
                    mu2 = fmaf(w, s_m[1][r + j][lane], mu2);
                    e11 = fmaf(w, s_m[2][r + j][lane], e11);
                    e22 = fmaf(w, s_m[3][r + j][lane], e22);
                    e12 = fmaf(w, s_m[4][r + j][lane], e12);
                }
                const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu1_mu2 = mu1 * mu2;
                const float sigma1_sq = e11 - mu1_sq, sigma2_sq = e22 - mu2_sq, sigma12 = e12 - mu1_mu2;
                const float num = (2.0f * mu1_mu2 + kC1) * (2.0f * sigma12 + kC2);
                const float den = (mu1_sq + mu2_sq + kC1) * (sigma1_sq + sigma2_sq + kC2);
                acc_ssim += (double)(num / den);
                const float d = s_x[r + kHalo][lane + kHalo] - s_y[r + kHalo][lane + kHalo];
                acc_se += (double)d * (double)d;
            }
            __syncthreads(); // the next channel overwrites s_x, s_y and s_m
        }
    }

    double tot[2];
    if (!grid_sum_last<kThreads, 2>({acc_se, acc_ssim}, a.partials, a.ticket, tot)) return;
    if (threadIdx.x == 0) {
        const double n = 3.0 * (double)plane;
        const double mse = fmax(tot[0] / n, 1e-10);
        a.out[0] = (float)(20.0 * log10(1.0 / sqrt(mse)));
        a.out[1] = (float)(tot[1] / n);
    }
}

} // namespace metrics
} // namespace gsb

extern "C" size_t gsb_image_metrics_workspace(void) {
    gsb::metrics::Ws w;
    return gsb::metrics::ws_layout(nullptr, w);
}

extern "C" int gsb_image_metrics(uint32_t W, uint32_t H, const float *image, const float *target, uint32_t flags,
                                 float *out, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::metrics;
    if (W == 0 || H == 0 || (uint64_t)W * H * 3 > INT32_MAX) return GSB_E_INVALID;
    if (!image || !target || !out || (flags & ~(uint32_t)GSB_METRICS_IMAGE_HWC)) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_check(workspace, workspace_bytes, ws_layout(workspace, w))) return rc;
    Args a;
    a.W = W;
    a.H = H;
    a.tiles_x = (uint32_t)ceil_div(W, kTW);
    a.n_tiles = a.tiles_x * (uint32_t)ceil_div(H, kTH);
    a.hwc = (flags & GSB_METRICS_IMAGE_HWC) != 0;
    a.image = image;
    a.target = target;
    a.out = out;
    a.partials = w.partials;
    a.ticket = w.ticket;
    static const Window win = make_window();
    a.win = win;
    cudaStream_t s = as_stream(stream);
    ProfScope ps("image_metrics", s);
    GSB_CUDA_TRY(cudaMemsetAsync(w.ticket, 0, sizeof(unsigned int), s));
    metrics_kernel<<<a.n_tiles < kBlocks ? a.n_tiles : kBlocks, kThreads, 0, s>>>(a);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
