// gsb_raster.cuh -- shared definitions of the from-world blend kernels (a7/a8).
//
// ---- the reformulation --------------------------------------------------------------------
// The reference evaluates, per (pixel, Gaussian) pair (RasterizeToPixelsFromWorld3DGSFwd.cu:228-248),
//     gro = M (o - mu),  grd = normalize(M d),  power = -1/2 |grd x gro|^2,   M = S^-1 R_g^T
// with o the camera centre and d the pixel's world ray: two 3x3 mat-vecs, a normalisation, a
// cross product, ~60 FLOP and 13 shared-memory floats per pair.  With a global shutter, o is the
// same for every pixel and d = B c(p) / |c(p)| with B = R_cam^-1 and c(p) = (u, v, 1) the
// pinhole direction of the pixel.  Writing A = M B (3x3 per Gaussian) and p_c = (u_c, v_c, 1)
// the projection of the Gaussian centre (mu_c = B^-1 mu + t = z_c p_c), one gets exactly
//     grd_un = A c(p) = G + du A0 + dv A1,          G = A p_c,  du = u - u_c, dv = v - v_c
//     grd_un x gro = du (A0 x gro) + dv (A1 x gro)  because gro = -z_c G is parallel to G
//     power = -1/2 |du E0 + dv E1|^2 / |G + du A0 + dv A1|^2,   E_i = A_i x gro
// i.e. a ratio of two quadratic forms in the pixel offset from the projected centre:
//     power = -1/2 (n0 du^2 + n1 du dv + n2 dv^2) / (d0 + d1 du + d2 dv + d3 du^2 + d4 du dv + d5 dv^2)
// The numerator is a positive semi-definite form in (du, dv) -- no cancellation, unlike the
// reference's cross product of a ~1000-long vector with a unit vector -- so float32 is enough
// for the per-pair arithmetic while the nine coefficients are computed once per Gaussian in
// float64 (gsb_prep_records_kernel).  Per pair this is ~16 FLOP and 12 shared-memory floats, and
// the alpha < 1/255 rejection needs no MUFU at all (N >= tau * D test).  The backward pass
// accumulates 15 moments  sum w {x, y, x^2, xy, y^2, ...}  per Gaussian instead of running the
// reference's 3x3/quaternion VJP per pair; the chain rule back to (mean, quat, scale) runs once
// per Gaussian in float64 (gsb_finalize_grads_kernel).  Derivation and numerical validation:
// DESIGN.md "Blend kernels".
#pragma once

#include "gsb_camera.cuh"

namespace gsb {

// 64-byte per-Gaussian record consumed by the blend kernels.  Pixel units: x = px - pcx.
//   e(x, y) = Ns / Ds + lop,  alpha_raw = 2^e
//   Ns = n0 x^2 + n1 x y + n2 y^2          (already scaled by -0.5 log2(e) / d0)
//   Ds = 1 + d1 x + d2 y + d3 x^2 + d4 x y + d5 y^2
//   tau: conservative MUFU-free rejection threshold: alpha_raw < 1/255  <=  Ns < tau * Ds
struct __align__(16) GaussRec {
    float pcx, pcy, n0, n1;
    float n2, d1, d2, d3;
    float d4, d5, lop, tau;
    float r, g, b;
    int32_t gid; // index of this Gaussian (row of the gradient-moment buffer)
};
static_assert(sizeof(GaussRec) == 64, "GaussRec must be 64 bytes");

constexpr int kRecFloats = 16;
constexpr int kMomFloats = 16; // 15 moments + pad, one 64-byte row per Gaussian
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kLog2AlphaThr = -7.994353436858858f; // log2(1/255)
constexpr float kTauMargin = 2e-3f;                   // in log2 units; >> float rounding of the test

// Camera constants shared by prep / blend / finalize, computed on the device from the same
// float view matrix the reference reads (Cameras.cuh:33-71,261-265): B = mat3_cast(inverse(q)).
struct CamConst {
    double B[3][3];    // camera->world rotation used for rays (R_inv of the reference)
    double Binv[3][3]; // its exact inverse (NOT the transpose: q is only unit to ~1e-7)
    double t[3];
    double fx, fy, cx, cy;
};

__device__ inline void cam_const_from(const float *viewmat, const float *K, CamConst &c) {
    const CamPose p = cam_pose_from_viewmat(viewmat);
    // glm::inverse(quat) = conjugate / dot, evaluated in float like the reference
    const float d = p.qw * p.qw + p.qx * p.qx + p.qy * p.qy + p.qz * p.qz;
    const float iw = p.qw / d, ix = -p.qx / d, iy = -p.qy / d, iz = -p.qz / d;
    const M3<float> Bf = rotmat_raw(iw, ix, iy, iz);
    M3<double> B;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) B.m[i][j] = (double)Bf.m[i][j];
    const M3<double> Bi = inverse3(B);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { c.B[i][j] = B.m[i][j]; c.Binv[i][j] = Bi.m[i][j]; }
    c.t[0] = p.tx; c.t[1] = p.ty; c.t[2] = p.tz;
    c.fx = K[0]; c.fy = K[4]; c.cx = K[2]; c.cy = K[5];
}

// Geometry of one Gaussian in the camera-relative parametrisation.  T = double in prep (the projected
// centre is cancellation-sensitive), T = float in finalize (the chain rule is not: see DESIGN.md 4.1).
template <typename T>
struct GaussGeom {
    V3<T> A0, A1, A2, G, gro, E0, E1;
    M3<T> Rg;       // rotation of the normalised quaternion (row-major math matrix)
    T inv_s[3];
    T qn[4], inv_qnorm;
    T zc, uc, vc;
    T n[3], d0, d[5];
    bool degenerate;
};

template <typename T>
__device__ inline void gauss_geom(const CamConst &c, const float *mean, const float *quat, const float *scale,
                                  GaussGeom<T> &g) {
    const T qw = quat[0], qx = quat[1], qy = quat[2], qz = quat[3];
    const T nn = qw * qw + qx * qx + qy * qy + qz * qz;
    g.inv_qnorm = T(1) / sqrt(nn);
    g.qn[0] = qw * g.inv_qnorm; g.qn[1] = qx * g.inv_qnorm; g.qn[2] = qy * g.inv_qnorm; g.qn[3] = qz * g.inv_qnorm;
    g.Rg = rotmat_raw<T>(g.qn[0], g.qn[1], g.qn[2], g.qn[3]);
    g.inv_s[0] = T(1) / (T)scale[0]; g.inv_s[1] = T(1) / (T)scale[1]; g.inv_s[2] = T(1) / (T)scale[2];
    // M = diag(1/s) Rg^T ; A = M B
    M3<T> A;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            T s = T(0);
            for (int k = 0; k < 3; ++k) s += g.Rg.m[k][i] * (T)c.B[k][j];
            A.m[i][j] = s * g.inv_s[i];
        }
    g.A0 = col(A, 0); g.A1 = col(A, 1); g.A2 = col(A, 2);
    const T mx = mean[0], my = mean[1], mz = mean[2];
    const T xc = (T)c.Binv[0][0] * mx + (T)c.Binv[0][1] * my + (T)c.Binv[0][2] * mz + (T)c.t[0];
    const T yc = (T)c.Binv[1][0] * mx + (T)c.Binv[1][1] * my + (T)c.Binv[1][2] * mz + (T)c.t[1];
    const T zc = (T)c.Binv[2][0] * mx + (T)c.Binv[2][1] * my + (T)c.Binv[2][2] * mz + (T)c.t[2];
    g.zc = zc;
    g.degenerate = !(fabs((double)zc) > 1e-12 * (fabs((double)xc) + fabs((double)yc) + 1e-300)) || !isfinite((double)zc);
    const T iz = g.degenerate ? T(0) : T(1) / zc;
    g.uc = xc * iz; g.vc = yc * iz;
    g.G = g.A0 * g.uc + g.A1 * g.vc + g.A2;
    g.gro = g.G * (-zc);
    g.E0 = cross(g.A0, g.gro);
    g.E1 = cross(g.A1, g.gro);
    g.n[0] = dot(g.E0, g.E0); g.n[1] = T(2) * dot(g.E0, g.E1); g.n[2] = dot(g.E1, g.E1);
    g.d0 = dot(g.G, g.G);
    g.d[0] = T(2) * dot(g.G, g.A0); g.d[1] = T(2) * dot(g.G, g.A1);
    g.d[2] = dot(g.A0, g.A0); g.d[3] = T(2) * dot(g.A0, g.A1); g.d[4] = dot(g.A1, g.A1);
    if (!(g.d0 > T(0)) || !isfinite((double)g.d0)) g.degenerate = true;
}


// The 64-byte record of one Gaussian (activated parameters in, float64 set-up): see GaussRec.
__device__ __forceinline__ void make_record(const CamConst &cam, const float (&mean)[3], const float (&quat)[4],
                                            const float (&scale)[3], float opac, const float (&col)[3], int32_t gid,
                                            float4 &v0, float4 &v1, float4 &v2, float4 &v3) {
    GaussGeom<double> gg;
    gauss_geom<double>(cam, mean, quat, scale, gg);
    v3 = make_float4(col[0], col[1], col[2], __int_as_float(gid));
    const bool dead = gg.degenerate || !(opac > 0.f);
    if (dead) {
        // never passes the rejection test: Ns (== 0) >= +inf * Ds is false
        v0 = make_float4(0.f, 0.f, 0.f, 0.f);
        v1 = make_float4(0.f, 0.f, 0.f, 0.f);
        v2 = make_float4(0.f, 0.f, 0.f, __int_as_float(0x7f800000));
    } else {
        const double ax = 1.0 / cam.fx, ay = 1.0 / cam.fy;
        const double id0 = 1.0 / gg.d0;
        const double kk = -0.5 * 1.4426950408889634 * id0;
        const float lop = (float)log2((double)opac);
        v0 = make_float4((float)(cam.fx * gg.uc + cam.cx), (float)(cam.fy * gg.vc + cam.cy),
                         (float)(kk * gg.n[0] * ax * ax), (float)(kk * gg.n[1] * ax * ay));
        v1 = make_float4((float)(kk * gg.n[2] * ay * ay), (float)(gg.d[0] * id0 * ax), (float)(gg.d[1] * id0 * ay),
                         (float)(gg.d[2] * id0 * ax * ax));
        v2 = make_float4((float)(gg.d[3] * id0 * ax * ay), (float)(gg.d[4] * id0 * ay * ay), lop,
                         kLog2AlphaThr - kTauMargin - lop);
    }
}

// dL/dq of R = rotmat(q / |q|) from dL/dR (vR[k][i] = dL/dR[k][i], math indices), normalisation included
// (Utils.cuh:104-126): qn = q / |q|, inv_qnorm = 1 / |q|.
__device__ __forceinline__ void quat_vjp_from_rotmat_grad(const float (&qn)[4], float inv_qnorm, const float (&vR)[3][3],
                                                          float (&oq)[4]) {
    const float w = qn[0], x = qn[1], y = qn[2], z = qn[3];
    float vq[4];
    vq[0] = 2.f * (x * (vR[2][1] - vR[1][2]) + y * (vR[0][2] - vR[2][0]) + z * (vR[1][0] - vR[0][1]));
    vq[1] = 2.f * (-2.f * x * (vR[1][1] + vR[2][2]) + y * (vR[1][0] + vR[0][1]) + z * (vR[2][0] + vR[0][2]) +
                   w * (vR[2][1] - vR[1][2]));
    vq[2] = 2.f * (x * (vR[1][0] + vR[0][1]) - 2.f * y * (vR[0][0] + vR[2][2]) + z * (vR[2][1] + vR[1][2]) +
                   w * (vR[0][2] - vR[2][0]));
    vq[3] = 2.f * (x * (vR[2][0] + vR[0][2]) + y * (vR[2][1] + vR[1][2]) - 2.f * z * (vR[0][0] + vR[1][1]) +
                   w * (vR[1][0] - vR[0][1]));
    const float dq = vq[0] * w + vq[1] * x + vq[2] * y + vq[3] * z;
#pragma unroll
    for (int k = 0; k < 4; ++k) oq[k] = (vq[k] - dq * qn[k]) * inv_qnorm;
}

// Sum 16 per-lane values across the warp: after the call lane L holds in v[0] the warp-wide total of
// slot (L >> 1).  16 shuffles (8+4+2+1+1) instead of 16 x 5.  On entry lanes 16..31 hold slot (i ^ 8) in
// v[i] (they built their registers pre-swapped), so stage one needs no lane-dependent selects.
__device__ __forceinline__ void butterfly16_preswapped(float (&v)[16]) {
    const uint32_t lane = threadIdx.x & 31;
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i + 8], 16);
    {
        const bool hi = lane & 8;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float send = hi ? v[i] : v[i + 4];
            const float keep = hi ? v[i + 4] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
    }
    {
        const bool hi = lane & 4;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float send = hi ? v[i] : v[i + 2];
            const float keep = hi ? v[i + 2] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
    }
    {
        const bool hi = lane & 2;
        const float send = hi ? v[0] : v[1];
        const float keep = hi ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
}


// Moment row of a Gaussian (16 floats, kMomFloats), x / y in pixels relative to (pcx, pcy):
//   w1 = dL/dNs, w2 = dL/dDs, g = dL/d(power) summed, c = dL/d(colour).
// Slot s and slot s ^ 8 are partners in the first stage of the warp reduction: they differ only in the
// weight (w1 <-> w2) or in a per-pixel constant, which is what makes that stage select-free.
enum MomentSlot : int {
    kS_G = 0, kS_W1X = 1, kS_W1Y = 2, kS_W1XX = 3, kS_W1XY = 4, kS_W1YY = 5, kS_CR = 6, kS_CB = 7,
    kS_W2 = 8, kS_W2X = 9, kS_W2Y = 10, kS_W2XX = 11, kS_W2XY = 12, kS_W2YY = 13, kS_CG = 14, kS_PAD = 15
};
// Channel counts of the blend (render modes, DESIGN.md 4.16): 3 = RGB, 1 = depth only (colour slot kS_CR), 4 = RGB +
// depth.  The fourth channel's gradient takes the pad slot, the partner of kS_CB in the butterfly's first stage.
constexpr int kS_C4 = kS_PAD;

// chain-rule arithmetic type of the finalize step (float: validated against the f64 oracle by the parity tests)
typedef float FT;

// Chain rule from the 15 moments of one Gaussian to the gradients of its ACTIVATED parameters
// (RasterizeToPixelsFromWorld3DGSBwd.cu:318-370 summed over the pixels): om = v_mean, oq = v_quat w.r.t. the
// quaternion as passed (normalisation included, Utils.cuh:104-126), os = v_scale, oo = v_opacity.
// q0..q2 = the Gaussian's record (normalised coefficients).  The colour gradient is m[kS_CR/CG/CB] itself.
__device__ __forceinline__ void finalize_gaussian(const CamConst &cam, const float (&mean)[3], const float (&quat)[4],
                                                  const float (&scale)[3], float opac, const float4 q0,
                                                  const float4 q1, const float4 q2, const float (&m)[16],
                                                  float (&om)[3], float (&oq)[4], float (&os)[3], float &oo) {
    bool any = false;
#pragma unroll
    for (int i = 0; i < 16; ++i)
        if (i != kS_CR && i != kS_CG && i != kS_CB && i != kS_PAD) any = any || (m[i] != 0.f);
    om[0] = om[1] = om[2] = 0.f; oq[0] = oq[1] = oq[2] = oq[3] = 0.f; os[0] = os[1] = os[2] = 0.f; oo = 0.f;
    if (any) {
        GaussGeom<FT> gg;
        gauss_geom<FT>(cam, mean, quat, scale, gg);
        if (!gg.degenerate) {
            const FT cn0 = q0.z, cn1 = q0.w, cn2 = q1.x;
            const FT cd1 = q1.y, cd2 = q1.z, cd3 = q1.w, cd4 = q2.x, cd5 = q2.y;
            const FT M0 = m[kS_W1X], M1 = m[kS_W1Y], M2 = m[kS_W1XX], M3_ = m[kS_W1XY], M4 = m[kS_W1YY], M5 = m[kS_W2],
                     M6 = m[kS_W2X], M7 = m[kS_W2Y], M8 = m[kS_W2XX], M9 = m[kS_W2XY], M10 = m[kS_W2YY];
            const FT ax = FT(1) / (FT)cam.fx, ay = FT(1) / (FT)cam.fy;
            const FT id0 = FT(1) / gg.d0;
            const FT kk = FT(-0.5 * 1.4426950408889634);
            // gradients w.r.t. the projected centre (pixels -> normalised image coordinates)
            const FT vpcx = -(FT(2) * cn0 * M0 + cn1 * M1 + cd1 * M5 + FT(2) * cd3 * M6 + cd4 * M7);
            const FT vpcy = -(cn1 * M0 + FT(2) * cn2 * M1 + cd2 * M5 + cd4 * M6 + FT(2) * cd5 * M7);
            FT vuc = (FT)cam.fx * vpcx, vvc = (FT)cam.fy * vpcy;
            // gradients w.r.t. the un-normalised quadratic-form coefficients
            const FT vn0 = M2 * kk * ax * ax * id0, vn1 = M3_ * kk * ax * ay * id0, vn2 = M4 * kk * ay * ay * id0;
            const FT vd1 = M6 * ax * id0, vd2 = M7 * ay * id0, vd3 = M8 * ax * ax * id0, vd4 = M9 * ax * ay * id0,
                         vd5 = M10 * ay * ay * id0;
            const FT vd0 = -(cn0 * M2 + cn1 * M3_ + cn2 * M4 + cd1 * M6 + cd2 * M7 + cd3 * M8 + cd4 * M9 + cd5 * M10) * id0;
            // n = (E0.E0, 2 E0.E1, E1.E1), d = (G.G, 2 G.A0, 2 G.A1, A0.A0, 2 A0.A1, A1.A1)
            const V3<FT> vE0 = gg.E0 * (FT(2) * vn0) + gg.E1 * (FT(2) * vn1);
            const V3<FT> vE1 = gg.E1 * (FT(2) * vn2) + gg.E0 * (FT(2) * vn1);
            V3<FT> vG = gg.G * (FT(2) * vd0) + gg.A0 * (FT(2) * vd1) + gg.A1 * (FT(2) * vd2);
            V3<FT> vA0 = gg.G * (FT(2) * vd1) + gg.A0 * (FT(2) * vd3) + gg.A1 * (FT(2) * vd4) + cross(gg.gro, vE0);
            V3<FT> vA1 = gg.G * (FT(2) * vd2) + gg.A1 * (FT(2) * vd5) + gg.A0 * (FT(2) * vd4) + cross(gg.gro, vE1);
            const V3<FT> vgro = cross(vE0, gg.A0) + cross(vE1, gg.A1);
            vG = vG - vgro * gg.zc;
            FT vzc = -dot(gg.G, vgro);
            vA0 = vA0 + vG * gg.uc;
            vA1 = vA1 + vG * gg.vc;
            const V3<FT> vA2 = vG;
            vuc += dot(gg.A0, vG);
            vvc += dot(gg.A1, vG);
            const FT iz = FT(1) / gg.zc;
            const FT vxc = vuc * iz, vyc = vvc * iz;
            vzc += -(gg.uc * vuc + gg.vc * vvc) * iz;
            // mu_c = Binv mu + t
            om[0] = (float)((FT)cam.Binv[0][0] * vxc + (FT)cam.Binv[1][0] * vyc + (FT)cam.Binv[2][0] * vzc);
            om[1] = (float)((FT)cam.Binv[0][1] * vxc + (FT)cam.Binv[1][1] * vyc + (FT)cam.Binv[2][1] * vzc);
            om[2] = (float)((FT)cam.Binv[0][2] * vxc + (FT)cam.Binv[1][2] * vyc + (FT)cam.Binv[2][2] * vzc);
            // A = M B  ->  vM = vA B^T ;  M[i][k] = Rg[k][i] / s_i
            const FT vA[3][3] = {{vA0.x, vA1.x, vA2.x}, {vA0.y, vA1.y, vA2.y}, {vA0.z, vA1.z, vA2.z}};
            FT vRg[3][3];
            for (int i = 0; i < 3; ++i) {
                FT vsi = FT(0);
                for (int k = 0; k < 3; ++k) {
                    const FT vM = vA[i][0] * (FT)cam.B[k][0] + vA[i][1] * (FT)cam.B[k][1] + vA[i][2] * (FT)cam.B[k][2];
                    vsi += vM * gg.Rg.m[k][i];
                    vRg[k][i] = vM * gg.inv_s[i];
                }
                os[i] = (float)(-vsi * gg.inv_s[i] * gg.inv_s[i]);
            }
            // quaternion VJP including the normalisation (Utils.cuh:104-126)
            quat_vjp_from_rotmat_grad(gg.qn, gg.inv_qnorm, vRg, oq);
            oo = (opac > 0.f) ? m[kS_G] / opac : 0.f; // sum vis * v_alpha
        }
    }
}

// Per-pixel evaluation, shared VERBATIM by the forward and backward kernels (explicitly rounded
// operations: the two kernels must agree bit-for-bit on which pairs pass the alpha test):
//   Ns = n0 x^2 + n1 xy + n2 y^2          (pre-scaled by -1/2 log2 e / d0)
//   Ds = 1 + d1 x + d2 y + d3 x^2 + d4 xy + d5 y^2
//   pass <=> Ns >= tau Ds                  (MUFU-free rejection, tau carries a safety margin)
// written as polynomials in y whose coefficients depend on x only:
//   Ns = a + y (b + n2 y),  a = n0 x^2,  b = n1 x
//   Ds = P + y (Q + d5 y),  P = 1 + d1 x + d3 x^2,  Q = d2 + d4 x
// A thread's pixels lie in one column on a pinhole (and EWA) camera, so it computes the column terms
// once per record and two FFMAs per polynomial per pixel.  A pixel's value does not depend on how many
// pixels share its column terms: each pixel runs the same operations in the same order.
// kEwa: the record is a pure 2-D conic (SURVEY.md 8 f4, gsb_fastgs.cu): Ds == 1, no denominator arithmetic.
struct ColTerms {
    float x, xx, a, b, P, Q;
};
template <bool kEwa = false>
__device__ __forceinline__ ColTerms col_terms(const float4 q0, const float4 q1, const float4 q2, float px) {
    ColTerms c;
    c.x = __fadd_rn(px, -q0.x);
    c.xx = __fmul_rn(c.x, c.x);
    c.a = __fmul_rn(q0.z, c.xx);
    c.b = __fmul_rn(q0.w, c.x);
    if constexpr (kEwa) {
        c.P = 1.0f; c.Q = 0.0f;
    } else {
        c.P = __fmaf_rn(q1.w, c.xx, __fmaf_rn(q1.y, c.x, 1.0f));
        c.Q = __fmaf_rn(q2.x, c.x, q1.z);
    }
    return c;
}
struct PixEval {
    float y, Ns, Ds;
    bool pass;
};
template <bool kEwa = false>
__device__ __forceinline__ PixEval pix_eval(const ColTerms &c, const float4 q0, const float4 q1, const float4 q2,
                                            float py) {
    PixEval e;
    e.y = __fadd_rn(py, -q0.y);
    e.Ns = __fmaf_rn(e.y, __fmaf_rn(q1.x, e.y, c.b), c.a);
    if constexpr (kEwa) {
        e.Ds = 1.0f;
        e.pass = e.Ns >= q2.w; // Ns >= tau
    } else {
        e.Ds = __fmaf_rn(e.y, __fmaf_rn(q2.y, e.y, c.Q), c.P);
        e.pass = __fmaf_rn(-q2.w, e.Ds, e.Ns) >= 0.0f; // Ns >= tau * Ds
    }
    return e;
}
// All kPix pixels of a thread against one record.  kSharedX: the pixels share one column (px[0]) and one
// set of column terms c[0]; otherwise (general camera: each pixel's undistorted x differs) c[i] is pixel i's.
template <bool kEwa, bool kSharedX, int kPix>
__device__ __forceinline__ void eval_pixels(const float4 q0, const float4 q1, const float4 q2, const float (&px)[kPix],
                                            const float (&py)[kPix], ColTerms (&c)[kSharedX ? 1 : kPix],
                                            PixEval (&e)[kPix]) {
    if constexpr (kSharedX) c[0] = col_terms<kEwa>(q0, q1, q2, px[0]);
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        if constexpr (!kSharedX) c[i] = col_terms<kEwa>(q0, q1, q2, px[i]);
        e[i] = pix_eval<kEwa>(c[kSharedX ? 0 : i], q0, q1, q2, py[i]);
    }
}
// Warp-level culling: can ANY pixel of the warp's block, whose (undistorted) pixel coordinates lie
// in the box [bx0, bx1] x [by0, by1], pass the rejection test of this record?  The pass region {Ns - tau Ds >= 0} is the interior of an
// ellipse (the form F = A x^2 + B xy + C y^2 + D x + E y + F0 is concave for every realistic
// Gaussian), so the exact answer is max_box F >= 0: the unconstrained maximiser if it lies in the
// box, else the best point on the (at most two) box edges facing it.  One lane tests one record,
// so a warp classifies 32 records per pass; `slack` absorbs the float rounding of both this test
// and pair_eval's, keeping the cull strictly conservative.  Non-concave forms are never culled.
template <bool kEwa = false>
__device__ __forceinline__ bool block_may_pass(const float4 q0, const float4 q1, const float4 q2, float bx0,
                                               float bx1, float by0, float by1) {
    const float tau = q2.w;
    if (!(tau < 3.0e38f)) return false; // dead record (tau = +inf)
    if constexpr (kEwa) {
        // pure conic (the d-slots of the record carry other data): F = Ns - tau, maximal at the box point nearest to
        // the centre in the conic's metric -- the centre itself if it lies inside the box
        const float A = q0.z, B = q0.w, C = q1.x;
        const float x0 = bx0 - q0.x, x1 = bx1 - q0.x, y0 = by0 - q0.y, y1 = by1 - q0.y;
        if (!(A < 0.0f && C < 0.0f && 4.0f * A * C - B * B > 0.0f)) return true;
        const bool xin = x0 <= 0.0f && x1 >= 0.0f, yin = y0 <= 0.0f && y1 >= 0.0f;
        if (xin && yin) return true; // F(0, 0) = -tau >= 0 for every visible primitive
        auto Fv = [&](float x, float y) { return (A * x + B * y) * x + C * y * y - tau; };
        float fmax = -3.0e38f;
        if (!xin) {
            const float xc = fminf(fmaxf(0.0f, x0), x1);
            const float yc = fminf(fmaxf(-(B * xc) / (2.0f * C), y0), y1);
            fmax = fmaxf(fmax, Fv(xc, yc));
        }
        if (!yin) {
            const float yc = fminf(fmaxf(0.0f, y0), y1);
            const float xc = fminf(fmaxf(-(B * yc) / (2.0f * A), x0), x1);
            fmax = fmaxf(fmax, Fv(xc, yc));
        }
        return fmax >= -0.02f;
    }
    const float A = __fmaf_rn(-tau, q1.w, q0.z), B = __fmaf_rn(-tau, q2.x, q0.w), C = __fmaf_rn(-tau, q2.y, q1.x);
    const float D = -tau * q1.y, E = -tau * q1.z, F0 = -tau;
    const float x0 = bx0 - q0.x, x1 = bx1 - q0.x, y0 = by0 - q0.y, y1 = by1 - q0.y;
    const float det = 4.0f * A * C - B * B;
    if (!(A < 0.0f && C < 0.0f && det > 0.0f)) return true;
    const float idet = 1.0f / det;
    const float xs = (B * E - 2.0f * C * D) * idet, ys = (B * D - 2.0f * A * E) * idet;
    const bool xin = (xs >= x0) && (xs <= x1), yin = (ys >= y0) && (ys <= y1);
    auto Fv = [&](float x, float y) { return (A * x + B * y + D) * x + (C * y + E) * y + F0; };
    float fmax;
    if (xin && yin) {
        fmax = Fv(xs, ys);
    } else {
        fmax = -3.0e38f;
        if (!xin) {
            const float xc = fminf(fmaxf(xs, x0), x1);
            const float yc = fminf(fmaxf(-(E + B * xc) / (2.0f * C), y0), y1);
            fmax = fmaxf(fmax, Fv(xc, yc));
        }
        if (!yin) {
            const float yc = fminf(fmaxf(ys, y0), y1);
            const float xc = fminf(fmaxf(-(D + B * yc) / (2.0f * A), x0), x1);
            fmax = fmaxf(fmax, Fv(xc, yc));
        }
    }
    return fmax >= -0.02f;
}

} // namespace gsb
