// gsb_raster.cu -- a7/a8: front-to-back alpha compositing from world-space rays, and its gradient.
//
// Implements gsplat::rasterize_to_pixels_from_world_3dgs_fwd / _bwd (reference:
// gsplat/RasterizeToPixelsFromWorld3DGSFwd.cu:20-279, ...Bwd.cu:17-373, gsplat/Utils.cuh:80-194)
// for the global-shutter camera models of gsb_camera.cuh.  See gsb_raster.cuh for the math.
//
// Kernel structure (H100):
//   prep      one thread per Gaussian, float64: 64-byte GaussRec (quadratic-form coefficients,
//             log2 opacity, colour).  N x 64 B: 64 MB at 1 M Gaussians, more than the H100's 50 MB L2, so
//             only part of the records stays L2-resident at that size.
//   fwd       one CTA (4 warps, 128 threads) per 16x16 tile; each thread owns two pixels of one
//             column (rows r and r+4) of an 8x8 sub-block, so a warp covers 64 pixels.  The tile's
//             depth-sorted records are gathered by 64-byte TMA bulk copies (cp.async.bulk -> mbarrier
//             complete_tx) into a two-stage shared-memory ring; ids are prefetched one batch ahead so
//             the gather of batch b+1 overlaps the blending of batch b.  Per (record, thread): the
//             column terms of the rejection test once, then two FFMAs per polynomial per pixel
//             (gsb_raster.cuh, eval_pixels); a warp-vote lets only warps with a surviving pixel pay
//             for rcp/ex2 and the colour row.  A warp whose pixels are saturated stops blending; the
//             CTA leaves when all are.
//   bwd       one CTA (2 warps, 64 threads) per tile; each thread owns four pixels of one column
//             (rows r, r+4, r+8, r+12), so a warp covers an 8x16 half tile and the per-event costs
//             (vote, record loads, warp reduction, reds) are paid once per 128 pixels.  Back-to-front
//             from the CTA-wide max(last_ids), three-stage ring released by per-warp mbarrier arrivals
//             (no CTA barrier per batch).  The 15 moments of an event are built on the shared column
//             from per-thread sums  S0 = sum w, S1 = sum w y, S2 = sum w y^2  (slots S0, x S0, S1,
//             x^2 S0, x S1, S2), reduced across the warp with a 16-value butterfly (16 shuffles
//             instead of 15 x 5) and added to a per-Gaussian 64-byte row with one 16-lane
//             red.global.add.f32.  An image too small to fill the GPU with such CTAs runs the same
//             kernel with two pixels per thread (4 warps, 128 threads per tile).
//   finalize  one thread per Gaussian, float32 chain rule from the moments to
//             (v_means, v_quats, v_scales, v_opacities, v_colors); writes every output element.
#include "gsb_raster.cuh"

namespace gsb {

constexpr int kPrepThreads = 128;
// pixels per thread and threads per CTA of the blend kernels; a stage of the record ring holds one record per thread
constexpr int kFwdPix = 2;
constexpr int kFwdThreads = 256 / kFwdPix;
// The backward runs four pixels per thread (64 threads per tile) where the image has enough tiles to fill the GPU,
// else two (128 threads per tile): see launch_bwd.
constexpr int kBwdPix = 4, kBwdPixSmall = 2;

// ------------------------------------------------------------------------------------------
// prep
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPrepThreads) prep_records_kernel(uint32_t N, const float *__restrict__ means,
                                                                     const float *__restrict__ quats,
                                                                     const float *__restrict__ scales,
                                                                     const float *__restrict__ colors,
                                                                     const float *__restrict__ opacities,
                                                                     const float *__restrict__ viewmat,
                                                                     const float *__restrict__ K,
                                                                     GaussRec *__restrict__ recs,
                                                                     float *__restrict__ moments /* nullable */) {
    __shared__ CamConst cam;
    if (threadIdx.x == 0) cam_const_from(viewmat, K, cam);
    __syncthreads();
    const uint32_t g = blockIdx.x * kPrepThreads + threadIdx.x;
    if (g >= N) return;
    if (moments) { // the backward's accumulation rows start at zero (saves a separate 64 B/Gaussian memset pass)
        float4 *m4 = reinterpret_cast<float4 *>(moments + (size_t)g * kMomFloats);
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        m4[0] = z; m4[1] = z; m4[2] = z; m4[3] = z;
    }
    const float mean[3] = {means[(size_t)g * 3], means[(size_t)g * 3 + 1], means[(size_t)g * 3 + 2]};
    const float quat[4] = {quats[(size_t)g * 4], quats[(size_t)g * 4 + 1], quats[(size_t)g * 4 + 2],
                           quats[(size_t)g * 4 + 3]};
    const float scale[3] = {scales[(size_t)g * 3], scales[(size_t)g * 3 + 1], scales[(size_t)g * 3 + 2]};
    const float opac = opacities[g];
    float4 v0, v1, v2, v3;
    const float col[3] = {colors[(size_t)g * 3], colors[(size_t)g * 3 + 1], colors[(size_t)g * 3 + 2]};
    make_record(cam, mean, quat, scale, opac, col, (int32_t)g, v0, v1, v2, v3);
    float4 *dst = reinterpret_cast<float4 *>(recs + g);
    dst[0] = v0; dst[1] = v1; dst[2] = v2; dst[3] = v3;
}

// ------------------------------------------------------------------------------------------
// tile geometry shared by fwd and bwd
// ------------------------------------------------------------------------------------------
struct TileParams {
    uint32_t n_isects;  // end of the last tile's range when the offsets have no closing entry
    uint32_t cap;       // capacity of flatten_ids: every range is clipped to it (== n_isects on the operator path)
    uint32_t closed;    // tile_offsets has tile_w*tile_h + 1 entries, the last one = n_isects (fused path)
    uint32_t chw;       // images are [3,H,W] planes (the fastgs API, SURVEY.md 8 f4) instead of [H,W,3]
    uint32_t W, H, tile_w, tile_h;
    const GaussRec *recs;
    const float *backgrounds; // [3] or null
    const uint8_t *masks;     // [tile_h*tile_w] or null
    const int32_t *tile_offsets;
    const int32_t *flatten_ids;
    // camera (only read by the general-camera instantiation)
    int32_t camera_model;
    const float *Ks, *radial, *tangential, *thin_prism;
    int32_t n_radial, n_tangential, n_thin_prism;
};

// A thread owns kPix pixels of one tile column, rows r, r+4, ..., r+4(kPix-1): a warp covers an 8-wide,
// 4*kPix-tall block and a 16x16 tile takes 256/kPix threads (warp w: column half w & 1, row block w >> 1).
template <int kPix>
struct PixelMap {
    uint32_t x, y[kPix];
    bool in[kPix];
};
template <int kPix>
__device__ __forceinline__ PixelMap<kPix> pixel_map(uint32_t tile_x, uint32_t tile_y, uint32_t W, uint32_t H) {
    const uint32_t w = threadIdx.x >> 5, l = threadIdx.x & 31;
    PixelMap<kPix> m;
    m.x = tile_x * 16 + (w & 1) * 8 + (l & 7);
    const uint32_t y0 = tile_y * 16 + (w >> 1) * (4 * kPix) + (l >> 3);
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        m.y[i] = y0 + 4 * i;
        m.in[i] = (m.x < W) && (m.y[i] < H);
    }
    return m;
}

// Per-thread pixel coordinates in the units of GaussRec (x = px - pcx).  Perfect pinhole: the pixel
// centres themselves, so px[] holds one value.  General camera: the pixel's ray is unprojected through
// the camera model (Newton undistortion / fisheye polynomial inverse) once per pixel and mapped back
// through the ideal pinhole, px = fx * x_n + cx; the warp's cull box is the bounding box of its valid pixels.
template <int kPix>
struct PixelCoords {
    float px[kPix], py[kPix];
    bool ok[kPix];            // ray valid (Fwd.cu:139, Bwd.cu:151)
    float bx0, bx1, by0, by1; // cull box of the warp
};
template <bool kGeneral, int kPix>
__device__ __forceinline__ PixelCoords<kPix> pixel_coords(const PixelMap<kPix> &pm, uint32_t tile_x, uint32_t tile_y,
                                                          const CamModel *cm) {
    PixelCoords<kPix> c;
    const uint32_t w = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        c.px[i] = (float)pm.x + 0.5f;
        c.py[i] = (float)pm.y[i] + 0.5f;
        c.ok[i] = true;
    }
    c.bx0 = (float)(tile_x * 16 + (w & 1) * 8) + 0.5f;
    c.by0 = (float)(tile_y * 16 + (w >> 1) * (4 * kPix)) + 0.5f;
    c.bx1 = c.bx0 + 7.0f;
    c.by1 = c.by0 + (float)(4 * kPix - 1);
    if constexpr (kGeneral) {
        const float BIG = 3.0e38f;
        float lox = BIG, hix = -BIG, loy = BIG, hiy = -BIG;
#pragma unroll
        for (int i = 0; i < kPix; ++i) {
            float xn, yn;
            c.ok[i] = cam_unproject_normalized(*cm, c.px[i], c.py[i], xn, yn);
            c.px[i] = fmaf(cm->fx, xn, cm->cx); c.py[i] = fmaf(cm->fy, yn, cm->cy);
            if (c.ok[i] && pm.in[i]) {
                lox = fminf(lox, c.px[i]); hix = fmaxf(hix, c.px[i]);
                loy = fminf(loy, c.py[i]); hiy = fmaxf(hiy, c.py[i]);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lox = fminf(lox, __shfl_xor_sync(0xffffffffu, lox, o));
            hix = fmaxf(hix, __shfl_xor_sync(0xffffffffu, hix, o));
            loy = fminf(loy, __shfl_xor_sync(0xffffffffu, loy, o));
            hiy = fmaxf(hiy, __shfl_xor_sync(0xffffffffu, hiy, o));
        }
        c.bx0 = lox; c.bx1 = hix; c.by0 = loy; c.by1 = hiy;
    }
    return c;
}

__device__ __forceinline__ void tile_cam_build(const TileParams &p, CamModel &cm) {
    cam_model_build(cm, p.camera_model, p.W, p.H, p.Ks, p.radial, p.n_radial, p.tangential, p.n_tangential, p.thin_prism,
                    p.n_thin_prism);
}


// Thread i gathers the record of Gaussian `gid` into slot i of the stage with one 64-byte bulk
// copy (TMA unit); thread 0 arms the stage's mbarrier with the byte count of the whole batch.
__device__ __forceinline__ void issue_batch(GaussRec *stage, uint64_t *bar, const GaussRec *recs, int32_t gid,
                                            uint32_t cnt) {
    const uint32_t tid = threadIdx.x;
    if (tid == 0) mbar_arrive_expect_tx(bar, cnt * (uint32_t)sizeof(GaussRec));
    if (tid < cnt) bulk_g2s(stage + tid, recs + gid, (uint32_t)sizeof(GaussRec), bar);
}

// ------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------
template <bool kGeneral, bool kEwa = false>
__global__ void __launch_bounds__(kFwdThreads) raster_fwd_kernel(const TileParams p, float *__restrict__ renders,
                                                                  float *__restrict__ alphas,
                                                                  int32_t *__restrict__ last_ids) {
    constexpr int kPix = kFwdPix, kBatch = kFwdThreads, kStages = 2;
    __shared__ __align__(128) GaussRec s_rec[kStages][kBatch];
    __shared__ __align__(8) uint64_t s_full[kStages];
    __shared__ CamModel s_cm;

    const uint32_t tile_id = blockIdx.x;
    const uint32_t tile_y = tile_id / p.tile_w, tile_x = tile_id % p.tile_w;
    const PixelMap<kPix> pm = pixel_map<kPix>(tile_x, tile_y, p.W, p.H);
    const uint32_t tid = threadIdx.x;
    const bool has_bg = p.backgrounds != nullptr;
    const float bg0 = has_bg ? p.backgrounds[0] : 0.f;
    const float bg1 = has_bg ? p.backgrounds[1] : 0.f;
    const float bg2 = has_bg ? p.backgrounds[2] : 0.f;

    if (p.masks != nullptr && !p.masks[tile_id]) { // Fwd.cu:143-150: background only, alpha/last_ids untouched
#pragma unroll
        for (int i = 0; i < kPix; ++i) {
            const size_t pix = (size_t)pm.y[i] * p.W + pm.x;
            if (pm.in[i]) { renders[pix * 3] = bg0; renders[pix * 3 + 1] = bg1; renders[pix * 3 + 2] = bg2; }
        }
        return;
    }

    const int32_t range_start = min(p.tile_offsets[tile_id], (int32_t)p.cap);
    const int32_t range_end = min((!p.closed && tile_id == p.tile_w * p.tile_h - 1) ? (int32_t)p.n_isects
                                                                                     : p.tile_offsets[tile_id + 1],
                                  (int32_t)p.cap);
    const int32_t total = max(range_end - range_start, 0);
    const int32_t n_batches = (total + kBatch - 1) / kBatch;

    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(&s_full[s], 1);
        mbar_fence_init();
        if constexpr (kGeneral) tile_cam_build(p, s_cm);
    }
    __syncthreads();

    const PixelCoords<kPix> pc = pixel_coords<kGeneral, kPix>(pm, tile_x, tile_y, &s_cm);
    // blend state of the thread's pixels
    float T[kPix], CR[kPix], CG[kPix], CB[kPix];
    int32_t last[kPix];
    bool done[kPix];
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        T[i] = 1.0f; CR[i] = CG[i] = CB[i] = 0.0f;
        last[i] = 0;
        done[i] = !pm.in[i] || !pc.ok[i];
    }
    auto all_done = [&]() {
        bool d = true;
#pragma unroll
        for (int i = 0; i < kPix; ++i) d = d && done[i];
        return d;
    };

    // prologue: batch 0 in flight, ids of batch 1 prefetched into a register
    int32_t gid_next = 0;
    if (n_batches > 0) {
        const int32_t idx = range_start + (int32_t)tid;
        const int32_t gid = (idx < range_end) ? p.flatten_ids[idx] : 0;
        issue_batch(s_rec[0], &s_full[0], p.recs, gid, (uint32_t)min(total, kBatch));
        const int32_t idx1 = idx + kBatch;
        gid_next = (idx1 < range_end) ? p.flatten_ids[idx1] : 0;
    }

    int32_t b = 0;
    bool saturated = false;
    for (; b < n_batches; ++b) {
        const int st = b & 1;
        if (b + 1 < n_batches) { // gather batch b+1 while blending batch b
            const int32_t cnt1 = min(total - (b + 1) * kBatch, kBatch);
            issue_batch(s_rec[st ^ 1], &s_full[st ^ 1], p.recs, gid_next, (uint32_t)cnt1);
            const int32_t idx2 = range_start + (b + 2) * kBatch + (int32_t)tid;
            gid_next = (idx2 < range_end) ? p.flatten_ids[idx2] : 0;
        }
        mbar_wait(&s_full[st], (uint32_t)((b >> 1) & 1));

        const int32_t cnt = min(total - b * kBatch, kBatch);
        const int32_t batch_start = range_start + b * kBatch;
        if (!__all_sync(0xffffffffu, all_done())) { // this warp's pixels are not all saturated
            const float4 *rec4 = reinterpret_cast<const float4 *>(s_rec[st]);
            for (int32_t c0 = 0; c0 < cnt; c0 += 32) {
              // lane-parallel culling of 32 records against this warp's pixel block
              const int32_t rl = c0 + (int32_t)(tid & 31);
              bool cand = false;
              if (rl < cnt)
                  cand = block_may_pass<kEwa>(rec4[rl * 4], rec4[rl * 4 + 1], rec4[rl * 4 + 2], pc.bx0, pc.bx1, pc.by0, pc.by1);
              uint32_t cmask = __ballot_sync(0xffffffffu, cand);
              while (cmask) {
                const int32_t t = c0 + __ffs(cmask) - 1;
                cmask &= cmask - 1;
                const float4 q0 = rec4[t * 4], q1 = rec4[t * 4 + 1], q2 = rec4[t * 4 + 2];
                ColTerms c[kGeneral ? kPix : 1];
                PixEval e[kPix];
                eval_pixels<kEwa, !kGeneral, kPix>(q0, q1, q2, pc.px, pc.py, c, e);
                bool pass[kPix], any = false;
#pragma unroll
                for (int i = 0; i < kPix; ++i) { pass[i] = e[i].pass && !done[i]; any = any || pass[i]; }
                if (!__any_sync(0xffffffffu, any)) continue;
                const float4 q3 = rec4[t * 4 + 3];
                // Every pixel branch-free (the warp executes both sides of a per-pixel branch anyway: most pixels
                // pass per event).  A pixel that does not contribute gets alpha = 0: T and colour stay.
#pragma unroll
                for (int i = 0; i < kPix; ++i) {
                    float ex;
                    if constexpr (kEwa) ex = __fadd_rn(e[i].Ns, q2.z);
                    else ex = __fmaf_rn(e[i].Ns, fast_rcp(e[i].Ds), q2.z);
                    const float al = fminf(kMaxAlpha, fast_ex2(ex));
                    const bool ok = pass[i] && al >= kAlphaThreshold;
                    float alpha = ok ? al : 0.0f;
                    const float nT = __fmul_rn(T[i], __fmaf_rn(alpha, -1.0f, 1.0f));
                    // a Gaussian that would push the transmittance to 1e-4 is NOT composited and ends the pixel
                    // (Fwd.cu:244-248)
                    const bool sat = ok && nT <= kMinTransmittance;
                    if (sat) alpha = 0.0f;
                    const float vis = __fmul_rn(alpha, T[i]);
                    CR[i] = __fmaf_rn(q3.x, vis, CR[i]);
                    CG[i] = __fmaf_rn(q3.y, vis, CG[i]);
                    CB[i] = __fmaf_rn(q3.z, vis, CB[i]);
                    if (!sat) T[i] = nT;
                    if (ok && !sat) last[i] = batch_start + t;
                    done[i] = done[i] || sat;
                }
              }
              if (__all_sync(0xffffffffu, all_done())) break;
            }
        }
        // releases stage `st` for batch b+2 and tells every warp whether the tile is saturated
        if (__syncthreads_and(all_done())) { saturated = true; break; }
    }
    // never retire the CTA with a bulk copy still landing in its shared memory
    if (saturated && b + 1 < n_batches) mbar_wait(&s_full[(b + 1) & 1], (uint32_t)(((b + 1) >> 1) & 1));

    // [H,W,3] rows (gsplat operators) or [3,H,W] planes (fastgs API)
    const size_t cs = p.chw ? (size_t)p.W * p.H : 1, ps = p.chw ? 1 : 3;
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        if (!pm.in[i]) continue;
        const size_t pix = (size_t)pm.y[i] * p.W + pm.x;
        alphas[pix] = 1.0f - T[i];
        renders[pix * ps] = has_bg ? CR[i] + T[i] * bg0 : CR[i];
        renders[pix * ps + cs] = has_bg ? CG[i] + T[i] * bg1 : CG[i];
        renders[pix * ps + 2 * cs] = has_bg ? CB[i] + T[i] * bg2 : CB[i];
        last_ids[pix] = last[i];
    }
}

// ------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------

// Per-pixel state of the backward sweep.
struct BwdPixel {
    float T;          // running transmittance (restored front-to-back value at the current Gaussian)
    float bdot;       // (colour accumulated behind) . dL/d(colour)
    float tfva;       // T_final * (dL/d(alpha) - bg . dL/d(colour))
    float vr, vg, vb; // dL/d(render colour)
    int32_t last;
    bool in;
};

// One (record, pixel) event of the backward sweep, branch-free: a pixel that does not contribute gets
// alpha = 0, which leaves its state untouched and yields zero weights.
//   w1 = dL/dNs, w2 = dL/dDs, g = dL/d(power), fac = alpha * T (weight of dL/d(colour))
struct EventWeights {
    float w1, w2, g, fac;
};
template <bool kEwa = false>
__device__ __forceinline__ EventWeights bwd_weights(BwdPixel &s, const PixEval &e, bool pass, float lop, float cr,
                                                    float cg, float cb) {
    float rD, ex; // same rounding as the forward
    if constexpr (kEwa) {
        rD = 1.0f;
        ex = __fadd_rn(e.Ns, lop);
    } else {
        rD = fast_rcp(e.Ds);
        ex = __fmaf_rn(e.Ns, rD, lop);
    }
    const float ar = fast_ex2(ex);
    const float al = fminf(kMaxAlpha, ar);
    const bool ok = pass && al >= kAlphaThreshold;
    const float alpha = ok ? al : 0.0f;
    // Bwd.cu:318: the gradient reaches the Gaussian through alpha only when alpha was not clamped
    // (the fastgs blend differentiates through the clamped value: kernels_backward.cuh:421-426 has no such test)
    const float araw_g = kEwa ? alpha : ((ok && ar <= kMaxAlpha) ? ar : 0.0f);
    const float om = __fmaf_rn(alpha, -1.0f, 1.0f);
    // the reference evaluates 1/(1-alpha) with the fast-math reciprocal too (Bwd.cu:291 under --use_fast_math)
    const float ra = ok ? fast_rcp(om) : 1.0f;
    s.T = __fmul_rn(s.T, ra);
    EventWeights w;
    w.fac = __fmul_rn(alpha, s.T);
    // v_alpha = sum_c (c_c T - behind_c / (1-alpha)) v_c + T_final (...) / (1-alpha)     (Bwd.cu:296-316)
    const float cv = __fmaf_rn(cr, s.vr, __fmaf_rn(cg, s.vg, __fmul_rn(cb, s.vb)));
    const float v_alpha = __fmaf_rn(s.T, cv, __fmul_rn(ra, __fmaf_rn(s.bdot, -1.0f, s.tfva)));
    s.bdot = __fmaf_rn(w.fac, cv, s.bdot);
    w.g = __fmul_rn(araw_g, v_alpha);
    if constexpr (kEwa) {
        w.w1 = w.g; // the moments are sums of g {x, y, x^2, xy, y^2}: the conic's chain rule runs per Gaussian
        w.w2 = 0.0f;
    } else {
        w.w1 = __fmul_rn(__fmul_rn(w.g, rD), kLn2);
        w.w2 = __fmul_rn(-w.w1, __fmul_rn(e.Ns, rD));
    }
    return w;
}

// The five moments  sum w {x, y, x^2, xy, y^2}  and  sum w  of one weight over a thread's pixels.  On a
// shared column they follow from  S0 = sum w, S1 = sum w y, S2 = sum w y^2  and the column's x; a general
// camera gives every pixel its own x.  These sums need not match any other kernel bit for bit: plain
// float arithmetic, which the compiler contracts.
template <bool kSharedX, int kPix>
__device__ __forceinline__ void weight_moments(const float (&w)[kPix], const PixEval (&e)[kPix],
                                               const ColTerms (&c)[kSharedX ? 1 : kPix], float (&m)[6]) {
    float S0 = 0.0f, S1 = 0.0f, S2 = 0.0f, X1 = 0.0f, XX = 0.0f, XY = 0.0f;
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        const float wy = w[i] * e[i].y;
        S0 += w[i];
        S1 += wy;
        S2 += wy * e[i].y;
        if constexpr (!kSharedX) {
            const float wx = w[i] * c[i].x;
            X1 += wx;
            XX += wx * c[i].x;
            XY += wx * e[i].y;
        }
    }
    if constexpr (kSharedX) {
        X1 = c[0].x * S0;
        XX = c[0].xx * S0;
        XY = c[0].x * S1;
    }
    m[0] = S0; m[1] = X1; m[2] = S1; m[3] = XX; m[4] = XY; m[5] = S2;
}

// The 16 registers of an event for the warp reduction, lanes 16..31 pre-swapped (see MomentSlot):
// lane L < 16 holds slot i in R[i], lane L >= 16 holds slot i ^ 8.
template <bool kEwa, bool kSharedX, int kPix>
__device__ __forceinline__ void event_registers(const BwdPixel (&s)[kPix], const EventWeights (&w)[kPix],
                                                const PixEval (&e)[kPix], const ColTerms (&c)[kSharedX ? 1 : kPix],
                                                bool hi16, float (&R)[16]) {
    float mA[6], mB[6], gs;
    if constexpr (kEwa) {
        // six live slots (g, g x, g y, g xx, g xy, g yy): lanes 16..31 hold them in the swapped registers
        float g[kPix];
#pragma unroll
        for (int i = 0; i < kPix; ++i) g[i] = w[i].g;
        float m[6];
        weight_moments<kSharedX, kPix>(g, e, c, m);
        gs = m[0];
#pragma unroll
        for (int k = 0; k < 6; ++k) { mA[k] = hi16 ? 0.0f : m[k]; mB[k] = hi16 ? m[k] : 0.0f; }
    } else {
        // weight A fills slots 1..5 (w1 on lanes 0..15, w2 on lanes 16..31), weight B slots 9..13
        float wA[kPix], wB[kPix];
        gs = 0.0f;
#pragma unroll
        for (int i = 0; i < kPix; ++i) {
            wA[i] = hi16 ? w[i].w2 : w[i].w1;
            wB[i] = hi16 ? w[i].w1 : w[i].w2;
            gs += w[i].g;
        }
        weight_moments<kSharedX, kPix>(wA, e, c, mA);
        weight_moments<kSharedX, kPix>(wB, e, c, mB);
    }
    R[0] = hi16 ? mA[0] : gs; // slot 0 = sum g, slot 8 = sum w2
    R[8] = hi16 ? gs : mB[0];
#pragma unroll
    for (int k = 1; k < 6; ++k) { R[k] = mA[k]; R[k + 8] = mB[k]; }
    float cr = 0.0f, cg = 0.0f, cb = 0.0f;
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        cr += w[i].fac * s[i].vr;
        cg += w[i].fac * s[i].vg;
        cb += w[i].fac * s[i].vb;
    }
    R[6] = hi16 ? cg : cr; R[14] = hi16 ? cr : cg; // slots kS_CR / kS_CG
    R[7] = hi16 ? 0.0f : cb; R[15] = hi16 ? cb : 0.0f; // slots kS_CB / kS_PAD
}

template <bool kGeneral, bool kEwa, int kPix>
__global__ void __launch_bounds__(256 / kPix) raster_bwd_kernel(const TileParams p,
                                                                const float *__restrict__ render_alphas,
                                                                const int32_t *__restrict__ last_ids,
                                                                const float *__restrict__ v_render_colors,
                                                                const float *__restrict__ v_render_alphas,
                                                                float *__restrict__ moments) {
    // Three stages; a stage is filled through its "full" mbarrier (TMA byte count) and released through its "empty"
    // mbarrier (one arrival per warp): no CTA-wide barrier in the loop, a warp with nothing to do in a batch runs ahead
    // of its neighbour instead of waiting at a two-stage / __syncthreads ring.
    constexpr int kBatch = 256 / kPix, kWarps = 256 / kPix / 32, kRing = 3;
    __shared__ __align__(128) GaussRec s_rec[kRing][kBatch];
    __shared__ __align__(8) uint64_t s_full[kRing];
    __shared__ __align__(8) uint64_t s_empty[kRing];
    __shared__ int32_t s_warp_max[kWarps];
    __shared__ CamModel s_cm;
    const uint32_t tile_id = blockIdx.x;
    if (p.masks != nullptr && !p.masks[tile_id]) return; // Bwd.cu:84-86
    const uint32_t tile_y = tile_id / p.tile_w, tile_x = tile_id % p.tile_w;
    const PixelMap<kPix> pm = pixel_map<kPix>(tile_x, tile_y, p.W, p.H);
    const uint32_t tid = threadIdx.x;
    const bool hi16 = (tid & 16) != 0;

    const int32_t range_start = min(p.tile_offsets[tile_id], (int32_t)p.cap);
    const int32_t range_end = min((!p.closed && tile_id == p.tile_w * p.tile_h - 1) ? (int32_t)p.n_isects
                                                                                     : p.tile_offsets[tile_id + 1],
                                  (int32_t)p.cap);

    float bg[3] = {0.f, 0.f, 0.f};
    if (p.backgrounds) { bg[0] = p.backgrounds[0]; bg[1] = p.backgrounds[1]; bg[2] = p.backgrounds[2]; }

    if constexpr (kGeneral) {
        if (tid == 0) tile_cam_build(p, s_cm);
        __syncthreads();
    }
    const PixelCoords<kPix> pc = pixel_coords<kGeneral, kPix>(pm, tile_x, tile_y, &s_cm);
    BwdPixel s[kPix];
    int32_t wmax = -1;
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        BwdPixel &r = s[i];
        r.in = pm.in[i] && pc.ok[i];
        r.bdot = 0.0f;
        if (r.in) {
            const size_t pix = (size_t)pm.y[i] * p.W + pm.x;
            const float Tf = 1.0f - render_alphas[pix];
            r.T = Tf;
            r.last = last_ids[pix];
            const size_t cs = p.chw ? (size_t)p.W * p.H : 1, ps = p.chw ? 1 : 3;
            r.vr = v_render_colors[pix * ps]; r.vg = v_render_colors[pix * ps + cs]; r.vb = v_render_colors[pix * ps + 2 * cs];
            const float va = v_render_alphas[pix];
            const float bgd = bg[0] * r.vr + bg[1] * r.vg + bg[2] * r.vb;
            r.tfva = Tf * va - Tf * bgd; // Bwd.cu:307-316
        } else {
            r.T = 1.f; r.last = -1; r.vr = r.vg = r.vb = 0.f; r.tfva = 0.f;
        }
        wmax = max(wmax, r.last);
    }
    // CTA-wide newest contributor: nothing behind it can receive gradient
    wmax = __reduce_max_sync(0xffffffffu, wmax);
    if ((tid & 31) == 0) s_warp_max[tid >> 5] = wmax;
    if (tid == 0) {
        for (int st = 0; st < kRing; ++st) { mbar_init(&s_full[st], 1); mbar_init(&s_empty[st], kWarps); }
        mbar_fence_init();
    }
    __syncthreads();
    int32_t hi = s_warp_max[0];
#pragma unroll
    for (int w = 1; w < kWarps; ++w) hi = max(hi, s_warp_max[w]);
    hi = min(hi, range_end - 1);
    const int32_t total = hi - range_start + 1;
    if (total <= 0) return;
    const int32_t n_batches = (total + kBatch - 1) / kBatch;
    // this warp only needs records at or before its own newest contributor
    wmax = min(wmax, hi);

    int32_t gid_next = 0;
    {
#pragma unroll
        for (int j = 0; j < kRing - 1; ++j) { // batches 0 .. kRing-2 in flight
            const int32_t idx = hi - j * kBatch - (int32_t)tid;
            const int32_t gid = (idx >= range_start) ? p.flatten_ids[idx] : 0;
            if (j < n_batches) issue_batch(s_rec[j], &s_full[j], p.recs, gid, (uint32_t)min(total - j * kBatch, kBatch));
        }
        const int32_t idx1 = hi - (kRing - 1) * kBatch - (int32_t)tid;
        gid_next = (idx1 >= range_start) ? p.flatten_ids[idx1] : 0;
    }

    for (int32_t b = 0; b < n_batches; ++b) {
        const int st = b % kRing;
        const int32_t nb = b + kRing - 1;
        if (nb < n_batches) {
            const int sn = nb % kRing; // the stage batch b-1 used
            if (b >= 1) mbar_wait(&s_empty[sn], (uint32_t)(((b - 1) / kRing) & 1));
            const int32_t cnt1 = min(total - nb * kBatch, kBatch);
            issue_batch(s_rec[sn], &s_full[sn], p.recs, gid_next, (uint32_t)cnt1);
            const int32_t idx2 = hi - (nb + 1) * kBatch - (int32_t)tid;
            gid_next = (idx2 >= range_start) ? p.flatten_ids[idx2] : 0;
        }
        mbar_wait(&s_full[st], (uint32_t)((b / kRing) & 1));

        const int32_t cnt = min(total - b * kBatch, kBatch);
        const int32_t top = hi - b * kBatch; // sorted index of slot 0
        const float4 *rec4 = reinterpret_cast<const float4 *>(s_rec[st]);
        const int32_t t_first = max(0, top - wmax);
        for (int32_t c0 = t_first & ~31; c0 < cnt; c0 += 32) {
          const int32_t rl = c0 + (int32_t)(tid & 31);
          bool cand = false;
          if (rl >= t_first && rl < cnt)
              cand = block_may_pass<kEwa>(rec4[rl * 4], rec4[rl * 4 + 1], rec4[rl * 4 + 2], pc.bx0, pc.bx1, pc.by0, pc.by1);
          uint32_t cmask = __ballot_sync(0xffffffffu, cand);
          while (cmask) {
            const int32_t t = c0 + __ffs(cmask) - 1;
            cmask &= cmask - 1;
            const int32_t idx = top - t;
            const float4 q0 = rec4[t * 4], q1 = rec4[t * 4 + 1], q2 = rec4[t * 4 + 2];
            ColTerms c[kGeneral ? kPix : 1];
            PixEval e[kPix];
            eval_pixels<kEwa, !kGeneral, kPix>(q0, q1, q2, pc.px, pc.py, c, e);
            bool pass[kPix], any = false;
#pragma unroll
            for (int i = 0; i < kPix; ++i) {
                pass[i] = e[i].pass && s[i].in && idx <= s[i].last;
                any = any || pass[i];
            }
            if (!__any_sync(0xffffffffu, any)) continue;
            const float4 q3 = rec4[t * 4 + 3];
            // A record often covers only part of the warp's 16 rows: a pixel index that no lane passes gets zero
            // weights and keeps its state, exactly what bwd_weights would give it, without the MUFU work.
            EventWeights w[kPix];
#pragma unroll
            for (int i = 0; i < kPix; ++i) {
                if (__any_sync(0xffffffffu, pass[i])) w[i] = bwd_weights<kEwa>(s[i], e[i], pass[i], q2.z, q3.x, q3.y, q3.z);
                else w[i] = EventWeights{0.0f, 0.0f, 0.0f, 0.0f};
            }
            float R[16];
            event_registers<kEwa, !kGeneral, kPix>(s, w, e, c, hi16, R);
            butterfly16_preswapped(R);
            if ((tid & 1) == 0) {
                const uint32_t slot = (tid & 31) >> 1;
                // EWA records: slots 8..13 (the denominator moments) do not exist
                if (slot != (uint32_t)kS_PAD && !(kEwa && slot >= 8u && slot != (uint32_t)kS_CG))
                    red_add_f32(moments + (size_t)__float_as_int(q3.w) * kMomFloats + slot, R[0]);
            }
          }
        }
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(&s_empty[st]); // this warp is done with stage `st`
    }
}

// ------------------------------------------------------------------------------------------
// finalize: moments -> gradients (chain rule once per Gaussian, float32: see FT below)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPrepThreads) finalize_grads_kernel(
    uint32_t N, const float *__restrict__ means, const float *__restrict__ quats, const float *__restrict__ scales,
    const float *__restrict__ opacities, const float *__restrict__ viewmat, const float *__restrict__ K,
    const GaussRec *__restrict__ recs, const float *__restrict__ moments, float *__restrict__ v_means,
    float *__restrict__ v_quats, float *__restrict__ v_scales, float *__restrict__ v_colors,
    float *__restrict__ v_opacities) {
    __shared__ CamConst cam;
    if (threadIdx.x == 0) cam_const_from(viewmat, K, cam);
    __syncthreads();
    const uint32_t g = blockIdx.x * kPrepThreads + threadIdx.x;
    if (g >= N) return;

    float m[16];
    {
        const float4 *m4 = reinterpret_cast<const float4 *>(moments + (size_t)g * kMomFloats);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float4 v = m4[i];
            m[i * 4] = v.x; m[i * 4 + 1] = v.y; m[i * 4 + 2] = v.z; m[i * 4 + 3] = v.w;
        }
    }
    v_colors[(size_t)g * 3] = m[kS_CR]; v_colors[(size_t)g * 3 + 1] = m[kS_CG]; v_colors[(size_t)g * 3 + 2] = m[kS_CB];
    float om[3], oq[4], os[3], oo;
    {
        const float mean[3] = {means[(size_t)g * 3], means[(size_t)g * 3 + 1], means[(size_t)g * 3 + 2]};
        const float quat[4] = {quats[(size_t)g * 4], quats[(size_t)g * 4 + 1], quats[(size_t)g * 4 + 2],
                               quats[(size_t)g * 4 + 3]};
        const float scale[3] = {scales[(size_t)g * 3], scales[(size_t)g * 3 + 1], scales[(size_t)g * 3 + 2]};
        const float4 *r4 = reinterpret_cast<const float4 *>(recs + g);
        finalize_gaussian(cam, mean, quat, scale, opacities[g], r4[0], r4[1], r4[2], m, om, oq, os, oo);
    }
    v_means[(size_t)g * 3] = om[0]; v_means[(size_t)g * 3 + 1] = om[1]; v_means[(size_t)g * 3 + 2] = om[2];
    v_scales[(size_t)g * 3] = os[0]; v_scales[(size_t)g * 3 + 1] = os[1]; v_scales[(size_t)g * 3 + 2] = os[2];
    reinterpret_cast<float4 *>(v_quats)[g] = make_float4(oq[0], oq[1], oq[2], oq[3]);
    v_opacities[g] = oo;
}

static int check_camera(const GsbCamera *cam) {
    if (!cam || !cam->viewmats0 || !cam->Ks) return GSB_E_INVALID;
    if (cam->camera_model != GSB_CAMERA_PINHOLE && cam->camera_model != GSB_CAMERA_FISHEYE)
        return GSB_E_UNSUPPORTED; // orthographic: no such branch in the reference either
    if (cam->shutter_type < GSB_SHUTTER_ROLLING_TOP_TO_BOTTOM || cam->shutter_type > GSB_SHUTTER_GLOBAL) return GSB_E_INVALID;
    return GSB_OK;
}
// A rolling shutter needs the per-pixel-pose kernels of gsb_raster_rs.cu; without an end-of-frame pose the start pose
// serves for both ends (Cameras.cuh:54-56), i.e. a global shutter.
static bool rolling_shutter(const GsbCamera *cam) {
    return cam->viewmats1 != nullptr && cam->shutter_type != GSB_SHUTTER_GLOBAL;
}
int raster_rs_fwd(uint32_t N, uint64_t n_isects, const float *means, const float *quats, const float *scales,
                  const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, uint32_t W,
                  uint32_t H, const GsbCamera *cam, const int32_t *tile_offsets, const int32_t *flatten_ids, float *renders,
                  float *alphas, int32_t *last_ids, void *workspace, cudaStream_t s);
int raster_rs_bwd(uint32_t N, uint64_t n_isects, const float *means, const float *quats, const float *scales,
                  const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, uint32_t W,
                  uint32_t H, const GsbCamera *cam, const int32_t *tile_offsets, const int32_t *flatten_ids,
                  const float *render_alphas, const int32_t *last_ids, const float *v_render_colors,
                  const float *v_render_alphas, float *v_means, float *v_quats, float *v_scales, float *v_colors,
                  float *v_opacities, void *workspace, size_t rec_bytes, cudaStream_t s);

static bool general_camera(const GsbCamera *cam) {
    return cam->camera_model == GSB_CAMERA_FISHEYE || cam->radial_coeffs || cam->tangential_coeffs ||
           cam->thin_prism_coeffs;
}

static void fill_camera(TileParams &p, const GsbCamera *cam) {
    p.camera_model = cam->camera_model;
    p.Ks = cam->Ks;
    p.radial = cam->radial_coeffs; p.tangential = cam->tangential_coeffs; p.thin_prism = cam->thin_prism_coeffs;
    p.n_radial = cam->radial_count; p.n_tangential = cam->tangential_count; p.n_thin_prism = cam->thin_prism_count;
}

} // namespace gsb

extern "C" size_t gsb_raster_fwd_workspace(uint32_t N) { return gsb::align256((size_t)N * sizeof(gsb::GaussRec)) + 256; }

extern "C" size_t gsb_raster_bwd_workspace(uint32_t N) {
    return gsb::align256((size_t)N * sizeof(gsb::GaussRec)) + gsb::align256((size_t)N * gsb::kMomFloats * 4) + 256;
}

namespace gsb {
static void fill_tiles(TileParams &p, uint64_t n_isects, uint32_t cap, int closed, uint32_t image_width,
                       uint32_t image_height, const GaussRec *recs, const float *backgrounds, const uint8_t *masks,
                       const int32_t *tile_offsets, const int32_t *flatten_ids, const GsbCamera *cam) {
    p.n_isects = (uint32_t)n_isects; p.cap = cap; p.closed = closed ? 1u : 0u; p.chw = 0u;
    p.W = image_width; p.H = image_height;
    p.tile_w = (image_width + 15) / 16; p.tile_h = (image_height + 15) / 16;
    p.recs = recs; p.backgrounds = backgrounds; p.masks = masks;
    p.tile_offsets = tile_offsets; p.flatten_ids = flatten_ids;
    fill_camera(p, cam);
}
static int launch_fwd(const TileParams &p, const GsbCamera *cam, float *renders, float *alphas, int32_t *last_ids,
                      cudaStream_t s) {
    {
        ProfScope ps("raster_fwd", s);
        if (general_camera(cam))
            raster_fwd_kernel<true><<<p.tile_w * p.tile_h, kFwdThreads, 0, s>>>(p, renders, alphas, last_ids);
        else
            raster_fwd_kernel<false><<<p.tile_w * p.tile_h, kFwdThreads, 0, s>>>(p, renders, alphas, last_ids);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
// Four pixels per thread pay an event's reduction and REDs once per 128 pixels, but give a tile only two warps.  An
// image with fewer tiles than the GPU holds such CTAs at once (256x256: 256 tiles, against 132 SMs x 14 CTAs on an
// H100 SXM) runs two pixels per thread instead: four warps per tile to hide latency with.
static uint32_t bwd_wide_min_tiles() {
    // immutable after the first call (C++11 thread-safe initialisation)
    static const uint32_t n = [] {
        int sms = 132, per_sm = 14, dev = 0;
        if (cudaGetDevice(&dev) == cudaSuccess) {
            int v = 0;
            if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) sms = v;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, raster_bwd_kernel<false, false, kBwdPix>, 256 / kBwdPix,
                                                              0) == cudaSuccess && v > 0)
                per_sm = v;
        }
        return (uint32_t)(sms * per_sm);
    }();
    return n;
}
template <bool kGeneral, bool kEwa>
static void launch_bwd_kernel(const TileParams &p, const float *render_alphas, const int32_t *last_ids,
                              const float *v_render_colors, const float *v_render_alphas, float *moments,
                              cudaStream_t s) {
    const uint32_t tiles = p.tile_w * p.tile_h;
    if (tiles >= bwd_wide_min_tiles())
        raster_bwd_kernel<kGeneral, kEwa, kBwdPix><<<tiles, 256 / kBwdPix, 0, s>>>(p, render_alphas, last_ids,
                                                                                  v_render_colors, v_render_alphas,
                                                                                  moments);
    else
        raster_bwd_kernel<kGeneral, kEwa, kBwdPixSmall><<<tiles, 256 / kBwdPixSmall, 0, s>>>(
            p, render_alphas, last_ids, v_render_colors, v_render_alphas, moments);
}
static int launch_bwd(const TileParams &p, const GsbCamera *cam, const float *render_alphas, const int32_t *last_ids,
                      const float *v_render_colors, const float *v_render_alphas, float *moments, cudaStream_t s) {
    {
        ProfScope ps("raster_bwd", s);
        if (general_camera(cam))
            launch_bwd_kernel<true, false>(p, render_alphas, last_ids, v_render_colors, v_render_alphas, moments, s);
        else
            launch_bwd_kernel<false, false>(p, render_alphas, last_ids, v_render_colors, v_render_alphas, moments, s);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

// ---- EWA records (SURVEY.md 8 f4, gsb_fastgs.cu): the same two kernels on pure 2-D conics, [3,H,W] images, no
// background, closed tile offsets, flatten_ids of `cap` entries --------------------------------------------------------
static void fill_ewa(TileParams &p, uint32_t cap, uint32_t W, uint32_t H, const GaussRec *recs, const int32_t *tile_offsets,
                     const int32_t *flatten_ids) {
    p.n_isects = 0; p.cap = cap; p.closed = 1u; p.chw = 1u;
    p.W = W; p.H = H; p.tile_w = (W + 15) / 16; p.tile_h = (H + 15) / 16;
    p.recs = recs; p.backgrounds = nullptr; p.masks = nullptr;
    p.tile_offsets = tile_offsets; p.flatten_ids = flatten_ids;
    p.camera_model = GSB_CAMERA_PINHOLE; p.Ks = nullptr; p.radial = p.tangential = p.thin_prism = nullptr;
    p.n_radial = p.n_tangential = p.n_thin_prism = 0;
}
int raster_ewa_fwd(uint32_t cap, const GaussRec *recs, uint32_t W, uint32_t H, const int32_t *tile_offsets,
                   const int32_t *flatten_ids, float *image, float *alpha, int32_t *last_ids, cudaStream_t s) {
    TileParams p;
    fill_ewa(p, cap, W, H, recs, tile_offsets, flatten_ids);
    {
        ProfScope ps("ewa_blend_fwd", s);
        raster_fwd_kernel<false, true><<<p.tile_w * p.tile_h, kFwdThreads, 0, s>>>(p, image, alpha, last_ids);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
int raster_ewa_bwd(uint32_t cap, const GaussRec *recs, uint32_t W, uint32_t H, const int32_t *tile_offsets,
                   const int32_t *flatten_ids, const float *alpha, const int32_t *last_ids, const float *grad_image,
                   const float *grad_alpha, float *moments, cudaStream_t s) {
    TileParams p;
    fill_ewa(p, cap, W, H, recs, tile_offsets, flatten_ids);
    {
        ProfScope ps("ewa_blend_bwd", s);
        launch_bwd_kernel<false, true>(p, alpha, last_ids, grad_image, grad_alpha, moments, s);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

} // namespace gsb

extern "C" int gsb_raster_fwd(uint32_t C, uint32_t N, uint64_t n_isects, const float *means, const float *quats,
                              const float *scales, const float *colors, const float *opacities,
                              const float *backgrounds, const uint8_t *masks, uint32_t image_width,
                              uint32_t image_height, uint32_t tile_size, const GsbCamera *cam,
                              const int32_t *tile_offsets, const int32_t *flatten_ids, float *renders, float *alphas,
                              int32_t *last_ids, void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (int rc = check_camera(cam)) return rc;
    if (image_width == 0 || image_height == 0) return GSB_OK;
    if (C != 1) return GSB_E_UNSUPPORTED;       // the reference's kernels are single-camera too (Fwd.cu:197-200)
    if (tile_size != 16) return GSB_E_UNSUPPORTED; // the reference's callers hard-code 16 (rasterizer.cpp:180)
    if (!renders || !alphas || !last_ids || !tile_offsets) return GSB_E_INVALID;
    if (n_isects > 0 && (!means || !quats || !scales || !colors || !opacities || !flatten_ids)) return GSB_E_INVALID;
    if (n_isects > 0x7fffffffull) return GSB_E_INVALID;
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_raster_fwd_workspace(N))
        return GSB_E_WORKSPACE;
    cudaStream_t s = as_stream(stream);
    if (rolling_shutter(cam))
        return raster_rs_fwd(N, n_isects, means, quats, scales, colors, opacities, backgrounds, masks, image_width,
                             image_height, cam, tile_offsets, flatten_ids, renders, alphas, last_ids, workspace, s);
    GaussRec *recs = reinterpret_cast<GaussRec *>(workspace);
    if (N > 0 && n_isects > 0) {
        {
            ProfScope ps("raster_prep", s);
            prep_records_kernel<<<(N + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, s>>>(
                N, means, quats, scales, colors, opacities, cam->viewmats0, cam->Ks, recs, nullptr);
        }
        GSB_LAUNCH_CHECK();
    }
    TileParams p;
    fill_tiles(p, n_isects, (uint32_t)n_isects, 0, image_width, image_height, recs, backgrounds, masks, tile_offsets,
               flatten_ids, cam);
    return launch_fwd(p, cam, renders, alphas, last_ids, s);
}

extern "C" int gsb_raster_bwd(uint32_t C, uint32_t N, uint64_t n_isects, const float *means, const float *quats,
                              const float *scales, const float *colors, const float *opacities,
                              const float *backgrounds, const uint8_t *masks, uint32_t image_width,
                              uint32_t image_height, uint32_t tile_size, const GsbCamera *cam,
                              const int32_t *tile_offsets, const int32_t *flatten_ids, const float *render_alphas,
                              const int32_t *last_ids, const float *v_render_colors, const float *v_render_alphas,
                              float *v_means, float *v_quats, float *v_scales, float *v_colors, float *v_opacities,
                              void *workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (int rc = check_camera(cam)) return rc;
    if (N == 0) return GSB_OK;
    if (C != 1) return GSB_E_UNSUPPORTED;
    if (tile_size != 16) return GSB_E_UNSUPPORTED;
    if (!v_means || !v_quats || !v_scales || !v_colors || !v_opacities) return GSB_E_INVALID;
    cudaStream_t s = as_stream(stream);
    if (n_isects == 0 || image_width == 0 || image_height == 0) { // Bwd.cu:434-437: gradients stay zero
        GSB_CUDA_TRY(cudaMemsetAsync(v_means, 0, (size_t)N * 12, s));
        GSB_CUDA_TRY(cudaMemsetAsync(v_quats, 0, (size_t)N * 16, s));
        GSB_CUDA_TRY(cudaMemsetAsync(v_scales, 0, (size_t)N * 12, s));
        GSB_CUDA_TRY(cudaMemsetAsync(v_colors, 0, (size_t)N * 12, s));
        GSB_CUDA_TRY(cudaMemsetAsync(v_opacities, 0, (size_t)N * 4, s));
        return GSB_OK;
    }
    if (!means || !quats || !scales || !colors || !opacities || !flatten_ids || !tile_offsets || !render_alphas ||
        !last_ids || !v_render_colors || !v_render_alphas)
        return GSB_E_INVALID;
    if (n_isects > 0x7fffffffull) return GSB_E_INVALID;
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_raster_bwd_workspace(N))
        return GSB_E_WORKSPACE;
    if (rolling_shutter(cam))
        return raster_rs_bwd(N, n_isects, means, quats, scales, colors, opacities, backgrounds, masks, image_width,
                             image_height, cam, tile_offsets, flatten_ids, render_alphas, last_ids, v_render_colors,
                             v_render_alphas, v_means, v_quats, v_scales, v_colors, v_opacities, workspace,
                             align256((size_t)N * sizeof(GaussRec)), s);
    GaussRec *recs = reinterpret_cast<GaussRec *>(workspace);
    float *moments = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + align256((size_t)N * sizeof(GaussRec)));
    {
        ProfScope ps("raster_prep", s);
        prep_records_kernel<<<(N + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, s>>>(
            N, means, quats, scales, colors, opacities, cam->viewmats0, cam->Ks, recs, moments);
    }
    GSB_LAUNCH_CHECK();
    TileParams p;
    fill_tiles(p, n_isects, (uint32_t)n_isects, 0, image_width, image_height, recs, backgrounds, masks, tile_offsets,
               flatten_ids, cam);
    if (int rc = launch_bwd(p, cam, render_alphas, last_ids, v_render_colors, v_render_alphas, moments, s)) return rc;
    {
        ProfScope ps("raster_finalize", s);
        finalize_grads_kernel<<<(N + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, s>>>(
            N, means, quats, scales, opacities, cam->viewmats0, cam->Ks, recs, moments, v_means, v_quats, v_scales,
            v_colors, v_opacities);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

// ---- fused path (SURVEY.md 8f1): blend forward / backward on records made by gsb_fused_front ---------------------------
// `workspace` is the fused workspace ([records][moments], gsb_fused_workspace); tile_offsets has th*tw + 1 entries
// (gsb_isect_plan with tile_offsets_total), so no host-side intersection count is needed: `capacity` is only the size
// of flatten_ids.
extern "C" int gsb_raster_fwd_recs(uint32_t N, uint32_t capacity, const void *workspace, size_t workspace_bytes,
                                   const float *backgrounds, const uint8_t *masks, uint32_t image_width,
                                   uint32_t image_height, const GsbCamera *cam, const int32_t *tile_offsets,
                                   const int32_t *flatten_ids, float *renders, float *alphas, int32_t *last_ids,
                                   gsb_stream_t stream) {
    using namespace gsb;
    if (int rc = check_camera(cam)) return rc;
    if (rolling_shutter(cam)) return GSB_E_UNSUPPORTED; // the fused path is global-shutter only
    if (image_width == 0 || image_height == 0) return GSB_OK;
    if (!renders || !alphas || !last_ids || !tile_offsets) return GSB_E_INVALID;
    if (capacity > 0 && !flatten_ids) return GSB_E_INVALID;
    if (capacity > 0x7fffffffu) return GSB_E_INVALID;
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_raster_bwd_workspace(N))
        return GSB_E_WORKSPACE;
    TileParams p;
    fill_tiles(p, 0, capacity, 1, image_width, image_height, reinterpret_cast<const GaussRec *>(workspace), backgrounds,
               masks, tile_offsets, flatten_ids, cam);
    return launch_fwd(p, cam, renders, alphas, last_ids, as_stream(stream));
}

extern "C" int gsb_raster_bwd_recs(uint32_t N, uint32_t capacity, void *workspace, size_t workspace_bytes,
                                   const float *backgrounds, const uint8_t *masks, uint32_t image_width,
                                   uint32_t image_height, const GsbCamera *cam, const int32_t *tile_offsets,
                                   const int32_t *flatten_ids, const float *render_alphas, const int32_t *last_ids,
                                   const float *v_render_colors, const float *v_render_alphas, gsb_stream_t stream) {
    using namespace gsb;
    if (int rc = check_camera(cam)) return rc;
    if (rolling_shutter(cam)) return GSB_E_UNSUPPORTED;
    if (N == 0 || image_width == 0 || image_height == 0) return GSB_OK;
    if (!tile_offsets || !render_alphas || !last_ids || !v_render_colors || !v_render_alphas) return GSB_E_INVALID;
    if (capacity > 0 && !flatten_ids) return GSB_E_INVALID;
    if (capacity > 0x7fffffffu) return GSB_E_INVALID;
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_raster_bwd_workspace(N))
        return GSB_E_WORKSPACE;
    float *moments = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + align256((size_t)N * sizeof(GaussRec)));
    TileParams p;
    fill_tiles(p, 0, capacity, 1, image_width, image_height, reinterpret_cast<const GaussRec *>(workspace), backgrounds,
               masks, tile_offsets, flatten_ids, cam);
    return launch_bwd(p, cam, render_alphas, last_ids, v_render_colors, v_render_alphas, moments, as_stream(stream));
}

