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
//   fwd       one CTA (4 warps, 128 threads) per 16x16 tile; each thread owns two pixels of an
//             8x8 sub-block so a warp covers 64 pixels.  The tile's depth-sorted records are
//             gathered by 64-byte TMA bulk copies (cp.async.bulk -> mbarrier complete_tx) into a
//             two-stage shared-memory ring; ids are prefetched one batch ahead so the gather of
//             batch b+1 overlaps the blending of batch b.  Per pair: MUFU-free rejection test,
//             then warp-vote: only warps with a surviving lane pay for rcp/ex2 and the colour row.
//             A warp whose 64 pixels are saturated stops blending; the CTA leaves when all are.
//   bwd       same tiling, back-to-front from the CTA-wide max(last_ids), three-stage ring released by per-warp
//             mbarrier arrivals (no CTA barrier per batch); 15 moments per pair are
//             summed over the thread's two pixels, reduced across the warp with a 16-value
//             butterfly (16 shuffles instead of 15 x 5) and added to a per-Gaussian 64-byte row
//             with one 16-lane red.global.add.f32.
//   finalize  one thread per Gaussian, float32 chain rule from the moments to
//             (v_means, v_quats, v_scales, v_opacities, v_colors); writes every output element.
#include "gsb_raster.cuh"

namespace gsb {

constexpr int kPrepThreads = 128;
constexpr int kTileThreads = 128; // 4 warps x 64 pixels
constexpr int kBatch = 128;       // records per pipeline stage (one per thread)
constexpr int kStages = 2;

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

struct PixelMap {
    uint32_t x, y0, y1; // pixel coordinates (two rows, same column)
    bool in0, in1;
};
__device__ __forceinline__ PixelMap pixel_map(uint32_t tile_x, uint32_t tile_y, uint32_t W, uint32_t H) {
    const uint32_t w = threadIdx.x >> 5, l = threadIdx.x & 31;
    PixelMap m;
    m.x = tile_x * 16 + (w & 1) * 8 + (l & 7);
    m.y0 = tile_y * 16 + (w >> 1) * 8 + (l >> 3);
    m.y1 = m.y0 + 4;
    m.in0 = (m.x < W) && (m.y0 < H);
    m.in1 = (m.x < W) && (m.y1 < H);
    return m;
}

// Per-thread pixel coordinates in the units of GaussRec (x = px - pcx).  Perfect pinhole: the pixel
// centres themselves.  General camera: the pixel's ray is unprojected through the camera model
// (Newton undistortion / fisheye polynomial inverse) once per pixel and mapped back through the ideal
// pinhole, px = fx * x_n + cx; the warp's cull box is the bounding box of its valid pixels.
struct PixelCoords {
    float px0, py0, px1, py1;
    bool ok0, ok1;            // ray valid (Fwd.cu:139, Bwd.cu:151)
    float bx0, bx1, by0, by1; // cull box of the warp
};
template <bool kGeneral>
__device__ __forceinline__ PixelCoords pixel_coords(const TileParams &p, const PixelMap &pm, uint32_t tile_x,
                                                    uint32_t tile_y, const CamModel *cm) {
    PixelCoords c;
    const uint32_t tid = threadIdx.x;
    c.px0 = c.px1 = (float)pm.x + 0.5f;
    c.py0 = (float)pm.y0 + 0.5f;
    c.py1 = (float)pm.y1 + 0.5f;
    c.ok0 = c.ok1 = true;
    c.bx0 = (float)(tile_x * 16 + ((tid >> 5) & 1) * 8) + 0.5f;
    c.by0 = (float)(tile_y * 16 + (tid >> 6) * 8) + 0.5f;
    c.bx1 = c.bx0 + 7.0f;
    c.by1 = c.by0 + 7.0f;
    if constexpr (kGeneral) {
        float xn, yn;
        c.ok0 = cam_unproject_normalized(*cm, c.px0, c.py0, xn, yn);
        c.px0 = fmaf(cm->fx, xn, cm->cx); c.py0 = fmaf(cm->fy, yn, cm->cy);
        c.ok1 = cam_unproject_normalized(*cm, c.px1, c.py1, xn, yn);
        c.px1 = fmaf(cm->fx, xn, cm->cx); c.py1 = fmaf(cm->fy, yn, cm->cy);
        const float BIG = 3.0e38f;
        float lox = fminf(c.ok0 && pm.in0 ? c.px0 : BIG, c.ok1 && pm.in1 ? c.px1 : BIG);
        float hix = fmaxf(c.ok0 && pm.in0 ? c.px0 : -BIG, c.ok1 && pm.in1 ? c.px1 : -BIG);
        float loy = fminf(c.ok0 && pm.in0 ? c.py0 : BIG, c.ok1 && pm.in1 ? c.py1 : BIG);
        float hiy = fmaxf(c.ok0 && pm.in0 ? c.py0 : -BIG, c.ok1 && pm.in1 ? c.py1 : -BIG);
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
__global__ void __launch_bounds__(kTileThreads) raster_fwd_kernel(const TileParams p, float *__restrict__ renders,
                                                                   float *__restrict__ alphas,
                                                                   int32_t *__restrict__ last_ids) {
    __shared__ __align__(128) GaussRec s_rec[kStages][kBatch];
    __shared__ __align__(8) uint64_t s_full[kStages];
    __shared__ CamModel s_cm;

    const uint32_t tile_id = blockIdx.x;
    const uint32_t tile_y = tile_id / p.tile_w, tile_x = tile_id % p.tile_w;
    const PixelMap pm = pixel_map(tile_x, tile_y, p.W, p.H);
    const uint32_t tid = threadIdx.x;
    const bool has_bg = p.backgrounds != nullptr;
    const float bg0 = has_bg ? p.backgrounds[0] : 0.f;
    const float bg1 = has_bg ? p.backgrounds[1] : 0.f;
    const float bg2 = has_bg ? p.backgrounds[2] : 0.f;

    const size_t pix0 = (size_t)pm.y0 * p.W + pm.x, pix1 = (size_t)pm.y1 * p.W + pm.x;
    if (p.masks != nullptr && !p.masks[tile_id]) { // Fwd.cu:143-150: background only, alpha/last_ids untouched
        if (pm.in0) { renders[pix0 * 3] = bg0; renders[pix0 * 3 + 1] = bg1; renders[pix0 * 3 + 2] = bg2; }
        if (pm.in1) { renders[pix1 * 3] = bg0; renders[pix1 * 3 + 1] = bg1; renders[pix1 * 3 + 2] = bg2; }
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

    const PixelCoords pc = pixel_coords<kGeneral>(p, pm, tile_x, tile_y, &s_cm);
    // blend state of the thread's two pixels as packed pairs (lo = pixel 0, hi = pixel 1)
    f2 T = f2_bc(1.0f), CR = f2_bc(0.0f), CG = f2_bc(0.0f), CB = f2_bc(0.0f);
    int32_t last0 = 0, last1 = 0;
    bool done0 = !pm.in0 || !pc.ok0, done1 = !pm.in1 || !pc.ok1;
    const f2 PX = f2_make(pc.px0, pc.px1), PY = f2_make(pc.py0, pc.py1);

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
        if (!__all_sync(0xffffffffu, done0 && done1)) { // this warp's 64 pixels are not all saturated
            const float4 *rec4 = reinterpret_cast<const float4 *>(s_rec[st]);
            for (int32_t c0 = 0; c0 < cnt; c0 += 32) {
              // lane-parallel culling of 32 records against this warp's 8x8 pixel block
              const int32_t rl = c0 + (int32_t)(tid & 31);
              bool cand = false;
              if (rl < cnt)
                  cand = block_may_pass<kEwa>(rec4[rl * 4], rec4[rl * 4 + 1], rec4[rl * 4 + 2], pc.bx0, pc.bx1, pc.by0, pc.by1);
              uint32_t cmask = __ballot_sync(0xffffffffu, cand);
              while (cmask) {
                const int32_t t = c0 + __ffs(cmask) - 1;
                cmask &= cmask - 1;
                const float4 q0 = rec4[t * 4], q1 = rec4[t * 4 + 1], q2 = rec4[t * 4 + 2];
                const PairEval2 e = pair_eval2<kEwa>(q0, q1, q2, f2_add(PX, f2_bc(-q0.x)), f2_add(PY, f2_bc(-q0.y)));
                const bool p0 = e.pass0 && !done0, p1 = e.pass1 && !done1;
                if (!__any_sync(0xffffffffu, p0 || p1)) continue;
                const float4 q3 = rec4[t * 4 + 3];
                // Both pixels branch-free on packed pairs (the warp executes both sides of a per-pixel branch anyway:
                // 40 of 64 pixels pass per event).  A pixel that does not contribute gets alpha = 0: T and colour stay.
                f2 ex;
                if constexpr (kEwa) ex = f2_add(e.Ns, f2_bc(q2.z));
                else ex = f2_fma(e.Ns, f2_make(fast_rcp(f2_lo(e.Ds)), fast_rcp(f2_hi(e.Ds))), f2_bc(q2.z));
                const float al0 = fminf(kMaxAlpha, fast_ex2(f2_lo(ex))), al1 = fminf(kMaxAlpha, fast_ex2(f2_hi(ex)));
                const bool ok0 = p0 && al0 >= kAlphaThreshold, ok1 = p1 && al1 >= kAlphaThreshold;
                f2 alpha = f2_make(ok0 ? al0 : 0.0f, ok1 ? al1 : 0.0f);
                const f2 nT = f2_mul(T, f2_fma(alpha, f2_bc(-1.0f), f2_bc(1.0f)));
                // a Gaussian that would push the transmittance to 1e-4 is NOT composited and ends the pixel (Fwd.cu:244-248)
                const bool sat0 = ok0 && f2_lo(nT) <= kMinTransmittance, sat1 = ok1 && f2_hi(nT) <= kMinTransmittance;
                alpha = f2_make(sat0 ? 0.0f : f2_lo(alpha), sat1 ? 0.0f : f2_hi(alpha));
                const f2 vis = f2_mul(alpha, T);
                CR = f2_fma(f2_bc(q3.x), vis, CR); CG = f2_fma(f2_bc(q3.y), vis, CG); CB = f2_fma(f2_bc(q3.z), vis, CB);
                T = f2_make(sat0 ? f2_lo(T) : f2_lo(nT), sat1 ? f2_hi(T) : f2_hi(nT));
                if (ok0 && !sat0) last0 = batch_start + t;
                if (ok1 && !sat1) last1 = batch_start + t;
                done0 = done0 || sat0; done1 = done1 || sat1;
              }
              if (__all_sync(0xffffffffu, done0 && done1)) break;
            }
        }
        // releases stage `st` for batch b+2 and tells every warp whether the tile is saturated
        if (__syncthreads_and(done0 && done1)) { saturated = true; break; }
    }
    // never retire the CTA with a bulk copy still landing in its shared memory
    if (saturated && b + 1 < n_batches) mbar_wait(&s_full[(b + 1) & 1], (uint32_t)(((b + 1) >> 1) & 1));

    // [H,W,3] rows (gsplat operators) or [3,H,W] planes (fastgs API)
    const size_t cs = p.chw ? (size_t)p.W * p.H : 1, ps = p.chw ? 1 : 3;
    const float T0 = f2_lo(T), T1 = f2_hi(T);
    if (pm.in0) {
        alphas[pix0] = 1.0f - T0;
        renders[pix0 * ps] = has_bg ? f2_lo(CR) + T0 * bg0 : f2_lo(CR);
        renders[pix0 * ps + cs] = has_bg ? f2_lo(CG) + T0 * bg1 : f2_lo(CG);
        renders[pix0 * ps + 2 * cs] = has_bg ? f2_lo(CB) + T0 * bg2 : f2_lo(CB);
        last_ids[pix0] = last0;
    }
    if (pm.in1) {
        alphas[pix1] = 1.0f - T1;
        renders[pix1 * ps] = has_bg ? f2_hi(CR) + T1 * bg0 : f2_hi(CR);
        renders[pix1 * ps + cs] = has_bg ? f2_hi(CG) + T1 * bg1 : f2_hi(CG);
        renders[pix1 * ps + 2 * cs] = has_bg ? f2_hi(CB) + T1 * bg2 : f2_hi(CB);
        last_ids[pix1] = last1;
    }
}

// ------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------

// Per-thread state of the backward sweep for the thread's two pixels (lo = pixel 0, hi = pixel 1).
struct BwdState {
    f2 T;      // running transmittance (restored front-to-back value at the current Gaussian)
    f2 bdot;   // (colour accumulated behind) . dL/d(colour)
    f2 tfva;   // T_final * (dL/d(alpha) - bg . dL/d(colour))
    f2 vr, vg, vb; // dL/d(render colour)
    f2 vA, vB, vC, vD; // the colour slots' per-pixel factors, pre-swapped for lanes 16..31 (see MomentSlot)
    int32_t last0, last1;
    bool in0, in1;
};

__device__ __forceinline__ float f2_sum(f2 a) { return f2_lo(a) + f2_hi(a); }

// One (record, pixel pair) event of the backward sweep, branch-free over the two pixels: a pixel that
// does not contribute gets alpha = 0, which leaves its state untouched and yields zero weights.
//   w1 = dL/dNs, w2 = dL/dDs, g = dL/d(power), fac = alpha * T (weight of dL/d(colour))
struct EventWeights {
    f2 w1, w2, g, fac;
};
template <bool kEwa = false>
__device__ __forceinline__ EventWeights bwd_weights(BwdState &s, const PairEval2 &e, bool p0, bool p1, float lop,
                                                    float cr, float cg, float cb) {
    f2 rD, ex; // same rounding as the forward's pair_alpha_raw
    if constexpr (kEwa) {
        rD = f2_bc(1.0f);
        ex = f2_add(e.Ns, f2_bc(lop));
    } else {
        rD = f2_make(fast_rcp(f2_lo(e.Ds)), fast_rcp(f2_hi(e.Ds)));
        ex = f2_fma(e.Ns, rD, f2_bc(lop));
    }
    const float ar0 = fast_ex2(f2_lo(ex)), ar1 = fast_ex2(f2_hi(ex));
    const float al0 = fminf(kMaxAlpha, ar0), al1 = fminf(kMaxAlpha, ar1);
    const bool ok0 = p0 && al0 >= kAlphaThreshold, ok1 = p1 && al1 >= kAlphaThreshold;
    const f2 alpha = f2_make(ok0 ? al0 : 0.0f, ok1 ? al1 : 0.0f);
    // Bwd.cu:318: the gradient reaches the Gaussian through alpha only when alpha was not clamped
    // (the fastgs blend differentiates through the clamped value: kernels_backward.cuh:421-426 has no such test)
    const f2 araw_g = kEwa ? alpha
                           : f2_make((ok0 && ar0 <= kMaxAlpha) ? ar0 : 0.0f, (ok1 && ar1 <= kMaxAlpha) ? ar1 : 0.0f);
    const f2 om = f2_fma(alpha, f2_bc(-1.0f), f2_bc(1.0f));
    // the reference evaluates 1/(1-alpha) with the fast-math reciprocal too (Bwd.cu:291 under --use_fast_math)
    float ra0 = 1.0f, ra1 = 1.0f;
    if (ok0) ra0 = fast_rcp(f2_lo(om));
    if (ok1) ra1 = fast_rcp(f2_hi(om));
    const f2 ra = f2_make(ra0, ra1);
    s.T = f2_mul(s.T, ra);
    EventWeights w;
    w.fac = f2_mul(alpha, s.T);
    // v_alpha = sum_c (c_c T - behind_c / (1-alpha)) v_c + T_final (...) / (1-alpha)     (Bwd.cu:296-316)
    const f2 cv = f2_fma(f2_bc(cr), s.vr, f2_fma(f2_bc(cg), s.vg, f2_mul(f2_bc(cb), s.vb)));
    const f2 v_alpha = f2_fma(s.T, cv, f2_mul(ra, f2_fma(s.bdot, f2_bc(-1.0f), s.tfva)));
    s.bdot = f2_fma(w.fac, cv, s.bdot);
    w.g = f2_mul(araw_g, v_alpha);
    if constexpr (kEwa) {
        w.w1 = w.g; // the moments are sums of g {x, y, x^2, xy, y^2}: the conic's chain rule runs per Gaussian
        w.w2 = f2_bc(0.0f);
    } else {
        const f2 gr = f2_mul(w.g, rD);
        w.w1 = f2_mul(gr, f2_bc(kLn2));
        w.w2 = f2_mul(f2_mul(gr, f2_bc(-kLn2)), f2_mul(e.Ns, rD));
    }
    return w;
}

// Shuffle reduction: the 16 registers of the event, lanes 16..31 pre-swapped (see MomentSlot).
template <bool kEwa = false>
__device__ __forceinline__ void event_registers(const BwdState &s, const EventWeights &w, const PairEval2 &e, f2 x, f2 y,
                                                bool hi16, float (&R)[16]) {
    if constexpr (kEwa) {
        // nine live slots (g, g x, g y, g xx, g xy, g yy, colour): lanes 16..31 hold them in the swapped registers
        const float gs = f2_sum(w.g);
        const float m1 = f2_sum(f2_mul(w.g, x)), m2 = f2_sum(f2_mul(w.g, y));
        const float m3 = f2_sum(f2_mul(w.g, e.xx)), m4 = f2_sum(f2_mul(w.g, e.xy)), m5 = f2_sum(f2_mul(w.g, e.yy));
        R[0] = hi16 ? 0.0f : gs; R[8] = hi16 ? gs : 0.0f;
        R[1] = hi16 ? 0.0f : m1; R[9] = hi16 ? m1 : 0.0f;
        R[2] = hi16 ? 0.0f : m2; R[10] = hi16 ? m2 : 0.0f;
        R[3] = hi16 ? 0.0f : m3; R[11] = hi16 ? m3 : 0.0f;
        R[4] = hi16 ? 0.0f : m4; R[12] = hi16 ? m4 : 0.0f;
        R[5] = hi16 ? 0.0f : m5; R[13] = hi16 ? m5 : 0.0f;
        R[6] = f2_sum(f2_mul(w.fac, s.vA)); R[14] = f2_sum(f2_mul(w.fac, s.vB));
        R[7] = f2_sum(f2_mul(w.fac, s.vC)); R[15] = f2_sum(f2_mul(w.fac, s.vD));
        return;
    }
    const f2 wA = hi16 ? w.w2 : w.w1, wB = hi16 ? w.w1 : w.w2;
    const float gs = f2_sum(w.g), w2s = f2_sum(w.w2);
    R[0] = hi16 ? w2s : gs;
    R[8] = hi16 ? gs : w2s;
    R[1] = f2_sum(f2_mul(wA, x)); R[2] = f2_sum(f2_mul(wA, y));
    R[3] = f2_sum(f2_mul(wA, e.xx)); R[4] = f2_sum(f2_mul(wA, e.xy)); R[5] = f2_sum(f2_mul(wA, e.yy));
    R[9] = f2_sum(f2_mul(wB, x)); R[10] = f2_sum(f2_mul(wB, y));
    R[11] = f2_sum(f2_mul(wB, e.xx)); R[12] = f2_sum(f2_mul(wB, e.xy)); R[13] = f2_sum(f2_mul(wB, e.yy));
    R[6] = f2_sum(f2_mul(w.fac, s.vA)); R[14] = f2_sum(f2_mul(w.fac, s.vB));
    R[7] = f2_sum(f2_mul(w.fac, s.vC)); R[15] = f2_sum(f2_mul(w.fac, s.vD));
}

template <bool kGeneral, bool kEwa = false>
__global__ void __launch_bounds__(kTileThreads) raster_bwd_kernel(const TileParams p,
                                                                   const float *__restrict__ render_alphas,
                                                                   const int32_t *__restrict__ last_ids,
                                                                   const float *__restrict__ v_render_colors,
                                                                   const float *__restrict__ v_render_alphas,
                                                                   float *__restrict__ moments) {
    // Three stages; a stage is filled through its "full" mbarrier (TMA byte count) and released through its "empty"
    // mbarrier (one arrival per warp): no CTA-wide barrier in the loop, a warp with nothing to do in a batch runs ahead
    // of its neighbours instead of waiting at a two-stage / __syncthreads ring.
    constexpr int kRing = 3;
    __shared__ __align__(128) GaussRec s_rec[kRing][kBatch];
    __shared__ __align__(8) uint64_t s_full[kRing];
    __shared__ __align__(8) uint64_t s_empty[kRing];
    __shared__ int32_t s_warp_max[kTileThreads / 32];
    __shared__ CamModel s_cm;
    const uint32_t tile_id = blockIdx.x;
    if (p.masks != nullptr && !p.masks[tile_id]) return; // Bwd.cu:84-86
    const uint32_t tile_y = tile_id / p.tile_w, tile_x = tile_id % p.tile_w;
    const PixelMap pm = pixel_map(tile_x, tile_y, p.W, p.H);
    const uint32_t tid = threadIdx.x;
    const bool hi16 = (tid & 16) != 0;

    const int32_t range_start = min(p.tile_offsets[tile_id], (int32_t)p.cap);
    const int32_t range_end = min((!p.closed && tile_id == p.tile_w * p.tile_h - 1) ? (int32_t)p.n_isects
                                                                                     : p.tile_offsets[tile_id + 1],
                                  (int32_t)p.cap);

    float bg[3] = {0.f, 0.f, 0.f};
    if (p.backgrounds) { bg[0] = p.backgrounds[0]; bg[1] = p.backgrounds[1]; bg[2] = p.backgrounds[2]; }

    struct PixelIn { float T, vr, vg, vb, tfva; int32_t last; };
    auto load_pixel = [&](bool in, uint32_t y) {
        PixelIn r;
        if (in) {
            const size_t pix = (size_t)y * p.W + pm.x;
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
        return r;
    };
    if constexpr (kGeneral) {
        if (tid == 0) tile_cam_build(p, s_cm);
        __syncthreads();
    }
    const PixelCoords pc = pixel_coords<kGeneral>(p, pm, tile_x, tile_y, &s_cm);
    BwdState s;
    s.in0 = pm.in0 && pc.ok0;
    s.in1 = pm.in1 && pc.ok1;
    {
        const PixelIn a = load_pixel(s.in0, pm.y0), b = load_pixel(s.in1, pm.y1);
        s.T = f2_make(a.T, b.T);
        s.bdot = f2_bc(0.0f);
        s.tfva = f2_make(a.tfva, b.tfva);
        s.vr = f2_make(a.vr, b.vr); s.vg = f2_make(a.vg, b.vg); s.vb = f2_make(a.vb, b.vb);
        s.vA = hi16 ? s.vg : s.vr;
        s.vB = hi16 ? s.vr : s.vg;
        s.vC = hi16 ? f2_bc(0.0f) : s.vb;
        s.vD = hi16 ? s.vb : f2_bc(0.0f);
        s.last0 = a.last; s.last1 = b.last;
    }
    const f2 PX = f2_make(pc.px0, pc.px1), PY = f2_make(pc.py0, pc.py1);
    // CTA-wide newest contributor: nothing behind it can receive gradient
    int32_t wmax = __reduce_max_sync(0xffffffffu, max(s.last0, s.last1));
    if ((tid & 31) == 0) s_warp_max[tid >> 5] = wmax;
    if (tid == 0) {
        for (int st = 0; st < kRing; ++st) { mbar_init(&s_full[st], 1); mbar_init(&s_empty[st], kTileThreads / 32); }
        mbar_fence_init();
    }
    __syncthreads();
    int32_t hi = s_warp_max[0];
#pragma unroll
    for (int w = 1; w < kTileThreads / 32; ++w) hi = max(hi, s_warp_max[w]);
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
            const f2 x = f2_add(PX, f2_bc(-q0.x)), y = f2_add(PY, f2_bc(-q0.y));
            const PairEval2 e = pair_eval2<kEwa>(q0, q1, q2, x, y);
            const bool p0 = e.pass0 && s.in0 && idx <= s.last0;
            const bool p1 = e.pass1 && s.in1 && idx <= s.last1;
            if (!__any_sync(0xffffffffu, p0 || p1)) continue;
            const float4 q3 = rec4[t * 4 + 3];
            const EventWeights w = bwd_weights<kEwa>(s, e, p0, p1, q2.z, q3.x, q3.y, q3.z);
            float R[16];
            event_registers<kEwa>(s, w, e, x, y, hi16, R);
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

static inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

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
            raster_fwd_kernel<true><<<p.tile_w * p.tile_h, kTileThreads, 0, s>>>(p, renders, alphas, last_ids);
        else
            raster_fwd_kernel<false><<<p.tile_w * p.tile_h, kTileThreads, 0, s>>>(p, renders, alphas, last_ids);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
static int launch_bwd(const TileParams &p, const GsbCamera *cam, const float *render_alphas, const int32_t *last_ids,
                      const float *v_render_colors, const float *v_render_alphas, float *moments, cudaStream_t s) {
    {
        ProfScope ps("raster_bwd", s);
        if (general_camera(cam))
            raster_bwd_kernel<true><<<p.tile_w * p.tile_h, kTileThreads, 0, s>>>(p, render_alphas, last_ids,
                                                                                v_render_colors, v_render_alphas, moments);
        else
            raster_bwd_kernel<false><<<p.tile_w * p.tile_h, kTileThreads, 0, s>>>(p, render_alphas, last_ids,
                                                                                 v_render_colors, v_render_alphas, moments);
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
        raster_fwd_kernel<false, true><<<p.tile_w * p.tile_h, kTileThreads, 0, s>>>(p, image, alpha, last_ids);
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
        raster_bwd_kernel<false, true><<<p.tile_w * p.tile_h, kTileThreads, 0, s>>>(p, alpha, last_ids, grad_image,
                                                                                   grad_alpha, moments);
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

