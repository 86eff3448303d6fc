/*
 * gut_oracle.c -- CPU restatement of the reference's 3DGUT rasterizer hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (the CUDA library, the
 * gsplat:: shim, the python host mirror) may include, link or call this file.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs use it, as the checker / the timed CPU baseline.
 *
 * It is a plain-C, scalar, line-by-line restatement of what the reference's CUDA
 * kernels compute (all file:line citations are relative to /root/reference):
 *
 *   K1 projection (UT)      gsplat/ProjectionUT3DGSFused.cu:47-202,
 *                           gsplat/Cameras.cuh:33-71,228-240,257-320,346-413,
 *                           416-471,1034-1150, gsplat/Utils.cuh:171-179
 *   a2 rolling shutter      gsplat/Cameras.cuh:268-413 (pose interpolation, frame time,
 *                           shutter-pose projection and pixel rays), all four directions
 *   K2/K3 SH fwd/bwd        gsplat/SphericalHarmonicsCUDA.cu:21-371,374-399,445-481
 *   K4-K6 tile intersect    gsplat/IntersectTile.cu:47-113,218-251,
 *                           gsplat/Intersect.cpp:41-121
 *   K7 blend forward        gsplat/RasterizeToPixelsFromWorld3DGSFwd.cu:58-278
 *   K8 blend backward       gsplat/RasterizeToPixelsFromWorld3DGSBwd.cu:63-372,
 *                           gsplat/Utils.cuh:80-158,181-194
 *   K9 quat->rotmat         gsplat/QuatToRotmatCUDA.cu:14-39
 *   K10/K11 MCMC helpers    gsplat/RelocationCUDA.cu:12-43,86-144
 *
 * The device-side vector math of the reference comes from GLM (third-party,
 * vcpkg baseline 4334d8b4, GLM 1.0.x, NOT vendored under /root/reference).  The
 * GLM semantics used here are GLM's published ones: quaternion storage
 * (w,x,y,z); q*v = v + 2(w (u x v) + u x (u x v)); column-major matrices;
 * quat_cast picks the largest of the four 4q^2-1 candidates; slerp falls back to
 * lerp when cos(theta) > 1 - epsilon.
 *
 * Pinning (see DESIGN.md "Oracle"): SH and tile-intersection are pinned against
 * the reference's own torch oracle tests/torch_impl.cpp (tests/golden/, script
 * tests/golden/make_torch_impl_golden.py + .cpp); projection / blend fwd / blend
 * bwd are pinned against the reference's own CUDA kernels compiled from
 * /root/reference/gsplat (oracle/_ref, recipe oracle/build_ref.py) and executed
 * on the GPU box -- fixtures in tests/golden/ref_cuda_*.npz.
 *
 * Precision: compile with -DORC_DOUBLE to get the same algorithm in float64
 * ("truth" for noise-floor measurements).  Interface arrays are float32 either
 * way; gradient outputs are float64 (deterministic summation order).
 *
 * The reference is built with --use_fast_math (approximate div/rsqrt/exp,
 * FTZ, FMA contraction; gsplat/CMakeLists.txt:76) so even a perfect restatement
 * is not bit-identical to it; the float tolerances live in the tests.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef ORC_DOUBLE
typedef double real;
#define R_SQRT sqrt
#define R_EXP exp
#define R_LOG log
#define R_FABS fabs
#define R_CEIL ceil
#define R_FLOOR floor
#define R_ACOS acos
#define R_SIN sin
#define R_POW pow
#define R_EPS 2.220446049250313e-16
#else
typedef float real;
#define R_SQRT sqrtf
#define R_EXP expf
#define R_LOG logf
#define R_FABS fabsf
#define R_CEIL ceilf
#define R_FLOOR floorf
#define R_ACOS acosf
#define R_SIN sinf
#define R_POW powf
#define R_EPS 1.1920929e-07f
#endif

/* The blend's two cut-offs (Fwd.cu:240-248, Bwd.cu:281).  ORC_SMOOTH is a TEST-ONLY build without them: the
 * forward becomes a smooth function of the parameters (for fixed intersection lists), so central differences
 * validate the analytic backward to rounding instead of "up to a threshold crossing". */
#ifdef ORC_SMOOTH
#define ORC_ALPHA_MIN ((real)0)
#define ORC_T_MIN ((real)-1)
#else
#define ORC_ALPHA_MIN ((real)(1.f / 255.f))
#define ORC_T_MIN ((real)1e-4)
#endif


#define ORC_API __attribute__((visibility("default")))

#ifdef _OPENMP
#include <omp.h>
#endif
#define ORC_ATOMIC_ADD(dst, val) do { double _v = (val); _Pragma("omp atomic") (dst) += _v; } while (0)
/* 1 thread (default) = deterministic summation order; bench legs raise it. */
static int g_threads = 1;
ORC_API void orc_set_threads(int n) { g_threads = n > 0 ? n : 1; }
ORC_API int orc_max_threads(void) {
#ifdef _OPENMP
    return omp_get_num_procs();
#else
    return 1;
#endif
}

/* error codes */
#define ORC_OK 0
#define ORC_E_UNSUPPORTED 1

/* gsplat/Common.h:46-50 */
enum { ORC_PINHOLE = 0, ORC_ORTHO = 1, ORC_FISHEYE = 2 };

/* gsplat/Cameras.h:27-44 */
typedef struct {
    float alpha, beta, kappa, in_image_margin_factor;
    int32_t require_all_sigma_points_valid;
} OrcUTParams;

/* ------------------------------------------------------------------ */
/* small vector / matrix helpers.  mat3 is COLUMN-major like GLM:      */
/* m.c[col][row].                                                      */
/* ------------------------------------------------------------------ */
typedef struct { real x, y, z; } v3;
typedef struct { real w, x, y, z; } qt;
typedef struct { real c[3][3]; } m3;

static inline v3 v3_make(real x, real y, real z) { v3 r = {x, y, z}; return r; }
static inline v3 v3_add(v3 a, v3 b) { return v3_make(a.x + b.x, a.y + b.y, a.z + b.z); }
static inline v3 v3_sub(v3 a, v3 b) { return v3_make(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline v3 v3_scale(v3 a, real s) { return v3_make(a.x * s, a.y * s, a.z * s); }
static inline real v3_dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline v3 v3_cross(v3 a, v3 b) {
    /* glm::cross */
    return v3_make(a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y);
}
static inline v3 m3_mulv(const m3 *m, v3 v) {
    return v3_make(m->c[0][0] * v.x + m->c[1][0] * v.y + m->c[2][0] * v.z,
                   m->c[0][1] * v.x + m->c[1][1] * v.y + m->c[2][1] * v.z,
                   m->c[0][2] * v.x + m->c[1][2] * v.y + m->c[2][2] * v.z);
}
static inline m3 m3_transpose(const m3 *m) {
    m3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.c[i][j] = m->c[j][i];
    return r;
}
static inline m3 m3_mul(const m3 *a, const m3 *b) { /* a*b, column-major */
    m3 r;
    for (int col = 0; col < 3; ++col)
        for (int row = 0; row < 3; ++row) {
            real s = 0;
            for (int k = 0; k < 3; ++k) s += a->c[k][row] * b->c[col][k];
            r.c[col][row] = s;
        }
    return r;
}

/* GLM quat_cast(mat3) -- glm/gtc/quaternion.inl */
static qt quat_cast(const m3 *m) {
    real fourXSquaredMinus1 = m->c[0][0] - m->c[1][1] - m->c[2][2];
    real fourYSquaredMinus1 = m->c[1][1] - m->c[0][0] - m->c[2][2];
    real fourZSquaredMinus1 = m->c[2][2] - m->c[0][0] - m->c[1][1];
    real fourWSquaredMinus1 = m->c[0][0] + m->c[1][1] + m->c[2][2];
    int biggestIndex = 0;
    real fourBiggestSquaredMinus1 = fourWSquaredMinus1;
    if (fourXSquaredMinus1 > fourBiggestSquaredMinus1) { fourBiggestSquaredMinus1 = fourXSquaredMinus1; biggestIndex = 1; }
    if (fourYSquaredMinus1 > fourBiggestSquaredMinus1) { fourBiggestSquaredMinus1 = fourYSquaredMinus1; biggestIndex = 2; }
    if (fourZSquaredMinus1 > fourBiggestSquaredMinus1) { fourBiggestSquaredMinus1 = fourZSquaredMinus1; biggestIndex = 3; }
    real biggestVal = R_SQRT(fourBiggestSquaredMinus1 + (real)1) * (real)0.5;
    real mult = (real)0.25 / biggestVal;
    qt q;
    switch (biggestIndex) {
    case 0:
        q.w = biggestVal;
        q.x = (m->c[1][2] - m->c[2][1]) * mult;
        q.y = (m->c[2][0] - m->c[0][2]) * mult;
        q.z = (m->c[0][1] - m->c[1][0]) * mult;
        break;
    case 1:
        q.w = (m->c[1][2] - m->c[2][1]) * mult;
        q.x = biggestVal;
        q.y = (m->c[0][1] + m->c[1][0]) * mult;
        q.z = (m->c[2][0] + m->c[0][2]) * mult;
        break;
    case 2:
        q.w = (m->c[2][0] - m->c[0][2]) * mult;
        q.x = (m->c[0][1] + m->c[1][0]) * mult;
        q.y = biggestVal;
        q.z = (m->c[1][2] + m->c[2][1]) * mult;
        break;
    default:
        q.w = (m->c[0][1] - m->c[1][0]) * mult;
        q.x = (m->c[2][0] + m->c[0][2]) * mult;
        q.y = (m->c[1][2] + m->c[2][1]) * mult;
        q.z = biggestVal;
        break;
    }
    return q;
}

/* GLM mat3_cast(quat) */
static m3 mat3_cast(qt q) {
    m3 r;
    real qxx = q.x * q.x, qyy = q.y * q.y, qzz = q.z * q.z;
    real qxz = q.x * q.z, qxy = q.x * q.y, qyz = q.y * q.z;
    real qwx = q.w * q.x, qwy = q.w * q.y, qwz = q.w * q.z;
    r.c[0][0] = (real)1 - (real)2 * (qyy + qzz);
    r.c[0][1] = (real)2 * (qxy + qwz);
    r.c[0][2] = (real)2 * (qxz - qwy);
    r.c[1][0] = (real)2 * (qxy - qwz);
    r.c[1][1] = (real)1 - (real)2 * (qxx + qzz);
    r.c[1][2] = (real)2 * (qyz + qwx);
    r.c[2][0] = (real)2 * (qxz + qwy);
    r.c[2][1] = (real)2 * (qyz - qwx);
    r.c[2][2] = (real)1 - (real)2 * (qxx + qyy);
    return r;
}

/* GLM operator*(quat, vec3) == glm::rotate(quat, vec3) */
static v3 quat_rotate(qt q, v3 v) {
    v3 u = v3_make(q.x, q.y, q.z);
    v3 uv = v3_cross(u, v);
    v3 uuv = v3_cross(u, uv);
    return v3_add(v, v3_scale(v3_add(v3_scale(uv, q.w), uuv), (real)2));
}

/* GLM inverse(quat) = conjugate / dot */
static qt quat_inverse(qt q) {
    real d = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    qt r = {q.w / d, -q.x / d, -q.y / d, -q.z / d};
    return r;
}

/* GLM normalize(quat) */
static qt quat_normalize(qt q) {
    real len = R_SQRT(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    if (len <= (real)0) { qt id = {1, 0, 0, 0}; return id; }
    real ool = (real)1 / len;
    qt r = {q.w * ool, q.x * ool, q.y * ool, q.z * ool};
    return r;
}

/* GLM slerp(x, y, a) */
static qt quat_slerp(qt x, qt y, real a) {
    qt z = y;
    real cosTheta = x.w * y.w + x.x * y.x + x.y * y.y + x.z * y.z;
    if (cosTheta < (real)0) {
        z.w = -y.w; z.x = -y.x; z.y = -y.y; z.z = -y.z;
        cosTheta = -cosTheta;
    }
    qt r;
    if (cosTheta > (real)1 - (real)R_EPS) {
        r.w = x.w * ((real)1 - a) + z.w * a;
        r.x = x.x * ((real)1 - a) + z.x * a;
        r.y = x.y * ((real)1 - a) + z.y * a;
        r.z = x.z * ((real)1 - a) + z.z * a;
    } else {
        real angle = R_ACOS(cosTheta);
        real s0 = R_SIN(((real)1 - a) * angle), s1 = R_SIN(a * angle), sd = R_SIN(angle);
        r.w = (s0 * x.w + s1 * z.w) / sd;
        r.x = (s0 * x.x + s1 * z.x) / sd;
        r.y = (s0 * x.y + s1 * z.y) / sd;
        r.z = (s0 * x.z + s1 * z.z) / sd;
    }
    return r;
}

/* Cameras.cuh:33-71 -- pose (t, q) from a row-major [4,4] view matrix */
typedef struct { v3 t; qt q; } Pose;
static Pose pose_from_viewmat(const float *se3) {
    m3 m; /* glm::mat3(se3[0],se3[4],se3[8], se3[1],se3[5],se3[9], se3[2],se3[6],se3[10]) */
    m.c[0][0] = se3[0]; m.c[0][1] = se3[4]; m.c[0][2] = se3[8];
    m.c[1][0] = se3[1]; m.c[1][1] = se3[5]; m.c[1][2] = se3[9];
    m.c[2][0] = se3[2]; m.c[2][1] = se3[6]; m.c[2][2] = se3[10];
    Pose p;
    p.q = quat_cast(&m);
    p.t = v3_make(se3[3], se3[7], se3[11]);
    return p;
}
/* Cameras.cuh:33-71: the end pose is the start pose when viewmats1 == nullptr (:54-56) */
static void shutter_poses(const float *viewmats0, const float *viewmats1, uint32_t cid, Pose *start, Pose *end) {
    *start = pose_from_viewmat(viewmats0 + cid * 16);
    *end = viewmats1 ? pose_from_viewmat(viewmats1 + cid * 16) : *start;
}

/* Cameras.cuh:268-280: lerp of t, GLM slerp of q */
static Pose interpolate_pose(Pose s, Pose e, real tau) {
    Pose r;
    r.t = v3_add(v3_scale(s.t, (real)1 - tau), v3_scale(e.t, tau));
    r.q = quat_slerp(s.q, e.q, tau);
    return r;
}

/* gsplat/Common.h ShutterType */
enum { ORC_ROLLING_TOP_TO_BOTTOM = 0, ORC_ROLLING_LEFT_TO_RIGHT = 1, ORC_ROLLING_BOTTOM_TO_TOP = 2,
       ORC_ROLLING_RIGHT_TO_LEFT = 3, ORC_GLOBAL = 4 };

/* Cameras.cuh:288-320: relative frame time of an image point (0 for a global shutter).  The resolution is
 * unsigned there, so (resolution - 1) is the integer W - 1 / H - 1 converted to floating point. */
static real shutter_relative_frame_time(int rs_type, real px, real py, uint32_t W, uint32_t H) {
    switch (rs_type) {
    case ORC_ROLLING_TOP_TO_BOTTOM: return R_FLOOR(py) / (real)(H - 1);
    case ORC_ROLLING_LEFT_TO_RIGHT: return R_FLOOR(px) / (real)(W - 1);
    case ORC_ROLLING_BOTTOM_TO_TOP: return ((real)H - R_CEIL(py)) / (real)(H - 1);
    case ORC_ROLLING_RIGHT_TO_LEFT: return ((real)W - R_CEIL(px)) / (real)(W - 1);
    default: return 0;
    }
}

/* Utils.cuh:80-102 quat_to_rotmat (normalising; rsqrt) -> column-major */
static m3 quat_to_rotmat(const real q4[4]) {
    real w = q4[0], x = q4[1], y = q4[2], z = q4[3];
    real inv_norm = (real)1 / R_SQRT(x * x + y * y + z * z + w * w);
    x *= inv_norm; y *= inv_norm; z *= inv_norm; w *= inv_norm;
    real x2 = x * x, y2 = y * y, z2 = z * z;
    real xy = x * y, xz = x * z, yz = y * z;
    real wx = w * x, wy = w * y, wz = w * z;
    m3 r;
    r.c[0][0] = (real)1 - (real)2 * (y2 + z2);
    r.c[0][1] = (real)2 * (xy + wz);
    r.c[0][2] = (real)2 * (xz - wy);
    r.c[1][0] = (real)2 * (xy - wz);
    r.c[1][1] = (real)1 - (real)2 * (x2 + z2);
    r.c[1][2] = (real)2 * (yz + wx);
    r.c[2][0] = (real)2 * (xz + wy);
    r.c[2][1] = (real)2 * (yz - wx);
    r.c[2][2] = (real)1 - (real)2 * (x2 + y2);
    return r;
}

/* ------------------------------------------------------------------ */
/* K1: UT projection (global and rolling shutter)                      */
/* ------------------------------------------------------------------ */

/* Cameras.cuh:228-240 */
static int in_bounds_margin(real px, real py, uint32_t W, uint32_t H, real margin_factor) {
    const real MX = (real)W * margin_factor;
    const real MY = (real)H * margin_factor;
    int valid = 1;
    valid &= (-MX) <= px && px < ((real)W + MX);
    valid &= (-MY) <= py && py < ((real)H + MY);
    return valid;
}

/* ---- camera models (Cameras.cuh:416-1001) ----------------------------------------------- */
enum { CM_PERFECT_PINHOLE = 0, CM_OPENCV_PINHOLE = 1, CM_OPENCV_FISHEYE = 2 };
typedef struct {
    int kind;
    uint32_t W, H;
    real fx, fy, cx, cy;
    real k[6], p[2], s[4];    /* OpenCV pinhole: radial, tangential, thin prism (Cameras.cuh:481-487) */
    real fk[4];               /* fisheye radial (Cameras.cuh:824-828) */
    real fwd[5], dfwd[5];     /* fisheye forward polynomial (odd) and its derivative (even) */
    real bwd0, bwd1;          /* fisheye linear approximation of the inverse */
    real max_angle, min_2d_norm;
} CamModel;

/* Cameras.cuh:759-815 */
static real fisheye_max_angle_cubic(real a, real b, real c) {
    const real INF = (real)3.402823466e+38;
    if (c == (real)0) {
        if (b == (real)0) return a >= (real)0 ? INF : (real)-1 / a;
        real delta = a * a - (real)4 * b;
        if (delta >= (real)0) {
            delta = R_SQRT(delta) - a;
            if (delta > (real)0) return (real)2 / delta;
        }
    } else {
        real boc = b / c, boc2 = boc * boc;
        real t1 = ((real)9 * a * boc - (real)2 * b * boc2 - (real)27) / c;
        real t2 = (real)3 * a / c - boc2;
        real delta = t1 * t1 + (real)4 * t2 * t2 * t2;
        if (delta >= (real)0) {
            real d2 = R_SQRT(delta);
            real cube_root = (real)cbrt((double)((d2 + t1) / (real)2));
            if (cube_root != (real)0) {
                real soln = (cube_root - (t2 / cube_root) - boc) / (real)3;
                if (soln > (real)0) return soln;
            }
        } else {
            real theta = (real)atan2((double)R_SQRT(-delta), (double)t1) / (real)3;
            const real two_third_pi = (real)2 * (real)3.14159265358979323846 / (real)3;
            real t3 = (real)2 * R_SQRT(-t2);
            real soln = INF;
            for (int i = -1; i <= 1; ++i) {
                real angle = theta + (real)i * two_third_pi;
                real sv = (t3 * (real)cos((double)angle) - boc) / (real)3;
                if (sv > (real)0 && sv < soln) soln = sv;
            }
            return soln;
        }
    }
    return INF;
}

static real poly_horner(const real *c, int n, real x) { /* c0 + c1 x + ... (Cameras.cuh:91-107) */
    real y = 0;
    for (int i = n - 1; i >= 0; --i) y = x * y + c[i];
    return y;
}

/* nr / nt / ns = number of floats behind each pointer (missing coefficients are zero) */
static CamModel cam_model_make(int camera_model, uint32_t W, uint32_t H, const float *K, const float *radial, int nr,
                               const float *tangential, int nt, const float *thin_prism, int ns) {
    CamModel m;
    memset(&m, 0, sizeof(m));
    m.W = W; m.H = H;
    m.fx = K[0]; m.fy = K[4]; m.cx = K[2]; m.cy = K[5];
    if (camera_model == ORC_FISHEYE) { /* Cameras.cuh:830-885 */
        m.kind = CM_OPENCV_FISHEYE;
        for (int i = 0; i < 4 && radial && i < nr; ++i) m.fk[i] = radial[i];
        const real k1 = m.fk[0], k2 = m.fk[1], k3 = m.fk[2], k4 = m.fk[3];
        m.fwd[0] = 1; m.fwd[1] = k1; m.fwd[2] = k2; m.fwd[3] = k3; m.fwd[4] = k4;
        m.dfwd[0] = 1; m.dfwd[1] = 3 * k1; m.dfwd[2] = 5 * k2; m.dfwd[3] = 7 * k3; m.dfwd[4] = 9 * k4;
        m.min_2d_norm = (real)1e-6;
        real mdx = ((real)W - m.cx) > m.cx ? ((real)W - m.cx) : m.cx;
        real mdy = ((real)H - m.cy) > m.cy ? ((real)H - m.cy) : m.cy;
        real max_radius_pixels = R_SQRT(mdx * mdx + mdy * mdy);
        if (k4 == (real)0) {
            m.max_angle = R_SQRT(fisheye_max_angle_cubic((real)3 * k1, (real)5 * k2, (real)7 * k3));
        } else { /* Newton on the derivative polynomial from 1.57 (Cameras.cuh:857-870, 174-206) */
            const real dd[4] = {6 * k1, 20 * k2, 42 * k3, 72 * k4};
            real x = (real)1.57;
            int converged = 0;
            for (int j = 0; j < 20; ++j) {
                real dfdx = x * poly_horner(dd, 4, x * x);
                real residual = poly_horner(m.dfwd, 5, x * x) - (real)0;
                real dx = residual / dfdx;
                x -= dx;
                if (R_FABS(dx) < (real)1e-6) { converged = 1; break; }
            }
            m.max_angle = (!converged || x <= (real)0) ? (real)3.402823466e+38 : x;
        }
        real a = max_radius_pixels / m.fx, b = max_radius_pixels / m.fy;
        real lim = a > b ? a : b;
        if (lim < m.max_angle) m.max_angle = lim;
        real nx = (real)W / (real)2 / m.fx, ny = (real)H / (real)2 / m.fy;
        real max_normalized_dist = nx > ny ? nx : ny;
        m.bwd0 = 0; m.bwd1 = m.max_angle / max_normalized_dist;
    } else if (radial || tangential || thin_prism) { /* ProjectionUT3DGSFused.cu:98-115 */
        m.kind = CM_OPENCV_PINHOLE;
        for (int i = 0; i < 6 && radial && i < nr; ++i) m.k[i] = radial[i];
        for (int i = 0; i < 2 && tangential && i < nt; ++i) m.p[i] = tangential[i];
        for (int i = 0; i < 4 && thin_prism && i < ns; ++i) m.s[i] = thin_prism[i];
    } else {
        m.kind = CM_PERFECT_PINHOLE;
    }
    return m;
}

/* Cameras.cuh:504-533 */
static void opencv_distortion(const CamModel *m, real u, real v, real *icD, real *dx, real *dy) {
    const real u2 = u * u, v2 = v * v, r2 = u2 + v2;
    const real a1 = (real)2 * u * v, a2 = r2 + (real)2 * u2, a3 = r2 + (real)2 * v2;
    const real num = (real)1 + r2 * (m->k[0] + r2 * (m->k[1] + r2 * m->k[2]));
    const real den = (real)1 + r2 * (m->k[3] + r2 * (m->k[4] + r2 * m->k[5]));
    *icD = num / den;
    *dx = m->p[0] * a1 + m->p[1] * a2 + r2 * (m->s[0] + r2 * m->s[1]);
    *dy = m->p[0] * a3 + m->p[1] * a1 + r2 * (m->s[2] + r2 * m->s[3]);
}

/* camera_ray_to_image_point of the three models (Cameras.cuh:431-455, 535-597, 894-959) */
static int cam_project(const CamModel *m, v3 cam, real margin, real *ox, real *oy) {
    *ox = 0; *oy = 0;
    if (cam.z <= (real)0) return 0;
    if (m->kind == CM_PERFECT_PINHOLE) {
        *ox = (cam.x / cam.z) * m->fx + m->cx;
        *oy = (cam.y / cam.z) * m->fy + m->cy;
        return in_bounds_margin(*ox, *oy, m->W, m->H, margin);
    }
    if (m->kind == CM_OPENCV_PINHOLE) {
        const real u = cam.x / cam.z, v = cam.y / cam.z;
        real icD, dx, dy;
        opencv_distortion(m, u, v, &icD, &dx, &dy);
        const int valid_radial = icD > (real)0.8;
        *ox = (icD * u + dx) * m->fx + m->cx;
        *oy = (icD * v + dy) * m->fy + m->cy;
        return valid_radial && in_bounds_margin(*ox, *oy, m->W, m->H, margin);
    }
    /* fisheye; numerically_stable_norm2 (Cameras.cuh:77-89) */
    real ax = R_FABS(cam.x), ay = R_FABS(cam.y);
    real mn = ax < ay ? ax : ay, mx = ax < ay ? ay : ax;
    real xy_norm = 0;
    if (mx > (real)0) { real r = mn / mx; xy_norm = mx * R_SQRT((real)1 + r * r); }
    if (xy_norm <= (real)0) xy_norm = (real)R_EPS;
    const real theta_full = (real)atan2((double)xy_norm, (double)cam.z);
    const real theta = theta_full < m->max_angle ? theta_full : m->max_angle;
    const real delta = theta * poly_horner(m->fwd, 5, theta * theta) / xy_norm;
    if (delta <= (real)0) return 0;
    *ox = m->fx * delta * cam.x + m->cx;
    *oy = m->fy * delta * cam.y + m->cy;
    return in_bounds_margin(*ox, *oy, m->W, m->H, margin) && (theta <= m->max_angle);
}

/* world_point_to_image_point_shutter_pose (Cameras.cuh:346-413).  Global shutter: the start-pose projection.
 * Rolling: project with the start and the end pose; seed from the start point if it is valid, else from the end
 * point; if neither is valid, return the end point as invalid; else ten rounds of "row / column time of the current
 * point -> interpolated pose -> projection", whose result is valid whatever the last projection says. */
static int project_shutter_pose(const CamModel *cm, int rs_type, Pose s, Pose e, v3 pt, real margin, real *ox,
                                real *oy) {
    real sx, sy;
    const int valid_start = cam_project(cm, v3_add(quat_rotate(s.q, pt), s.t), margin, &sx, &sy);
    if (rs_type == ORC_GLOBAL) { *ox = sx; *oy = sy; return valid_start; }
    real ex, ey;
    const int valid_end = cam_project(cm, v3_add(quat_rotate(e.q, pt), e.t), margin, &ex, &ey);
    real px, py;
    if (valid_start) { px = sx; py = sy; }
    else if (valid_end) { px = ex; py = ey; }
    else { *ox = ex; *oy = ey; return 0; }
    for (int j = 0; j < 10; ++j) {
        const real tau = shutter_relative_frame_time(rs_type, px, py, cm->W, cm->H);
        const Pose p = interpolate_pose(s, e, tau);
        real nx, ny;
        cam_project(cm, v3_add(quat_rotate(p.q, pt), p.t), margin, &nx, &ny);
        px = nx; py = ny;
    }
    *ox = px; *oy = py;
    return 1;
}

/* image_point_to_camera_ray (Cameras.cuh:457-470, 698-754, 961-1000): unit camera-space ray */
static int cam_unproject(const CamModel *m, real px, real py, v3 *ray) {
    const real u0 = (px - m->cx) / m->fx, v0 = (py - m->cy) / m->fy;
    if (m->kind == CM_PERFECT_PINHOLE) {
        real len = R_SQRT(u0 * u0 + v0 * v0 + (real)1);
        *ray = v3_make(u0 / len, v0 / len, (real)1 / len);
        return 1;
    }
    if (m->kind == CM_OPENCV_PINHOLE) { /* Newton, at most 5 iterations (:698-740) */
        real x = u0, y = v0;
        int converged = 0;
        for (int iter = 0; iter < 5; ++iter) {
            const real k1 = m->k[0], k2 = m->k[1], k3 = m->k[2], k4 = m->k[3], k5 = m->k[4], k6 = m->k[5];
            const real p1 = m->p[0], p2 = m->p[1], s1 = m->s[0], s2 = m->s[1], s3 = m->s[2], s4 = m->s[3];
            const real r = x * x + y * y, r2 = r * r;
            const real alpha = (real)1 + r * (k1 + r * (k2 + r * k3));
            const real beta = (real)1 + r * (k4 + r * (k5 + r * k6));
            const real d = alpha / beta;
            if (d <= (real)0) break;
            real fx_ = d * x + 2 * p1 * x * y + p2 * (r + 2 * x * x) + s1 * r + s2 * r2 - u0;
            real fy_ = d * y + 2 * p2 * x * y + p1 * (r + 2 * y * y) + s3 * r + s4 * r2 - v0;
            const real alpha_r = k1 + r * ((real)2 * k2 + r * ((real)3 * k3));
            const real beta_r = k4 + r * ((real)2 * k5 + r * ((real)3 * k6));
            const real d_r = (alpha_r * beta - alpha * beta_r) / (beta * beta);
            const real d_x = (real)2 * x * d_r, d_y = (real)2 * y * d_r;
            real fx_x = d + d_x * x + (real)2 * p1 * y + (real)6 * p2 * x;
            fx_x += (real)2 * x * (s1 + (real)2 * s2 * r);
            real fx_y = d_y * x + (real)2 * p1 * x + (real)2 * p2 * y;
            fx_y += (real)2 * y * (s1 + (real)2 * s2 * r);
            real fy_x = d_x * y + (real)2 * p2 * y + (real)2 * p1 * x;
            fy_x += (real)2 * x * (s3 + (real)2 * s4 * r);
            real fy_y = d + d_y * y + (real)2 * p2 * x + (real)6 * p1 * y;
            fy_y += (real)2 * y * (s3 + (real)2 * s4 * r);
            const real det = fx_y * fy_x - fx_x * fy_y;
            if (R_FABS(det) < (real)1e-6) break;
            const real dx = (fx_ * fy_y - fy_ * fx_y) / det;
            const real dy = (fy_ * fx_x - fx_ * fy_x) / det;
            x += dx; y += dy;
            if (R_FABS(dx) < (real)1e-6 && R_FABS(dy) < (real)1e-6) { converged = 1; break; }
        }
        real len = R_SQRT(x * x + y * y + (real)1);
        *ray = v3_make(x / len, y / len, (real)1 / len);
        return converged;
    }
    /* fisheye: invert theta * P(theta^2) = delta by Newton from the linear guess (:961-1000, 174-206) */
    const real delta = R_SQRT(u0 * u0 + v0 * v0);
    real th = m->bwd0 + m->bwd1 * delta;
    int converged = 0;
    for (int j = 0; j < 20; ++j) {
        const real dfdx = poly_horner(m->dfwd, 5, th * th);
        const real residual = th * poly_horner(m->fwd, 5, th * th) - delta;
        const real dx = residual / dfdx;
        th -= dx;
        if (R_FABS(dx) < (real)1e-6) { converged = 1; break; }
    }
    if (th < (real)0 || th >= m->max_angle || !converged) { *ray = v3_make(0, 0, 1); return 0; }
    if (delta >= m->min_2d_norm) {
        const real sf = R_SIN(th) / delta;
        *ray = v3_make(sf * u0, sf * v0, (real)cos((double)th));
    } else {
        *ray = v3_make(0, 0, 1);
    }
    return 1;
}

/*
 * ProjectionUT3DGSFused.cu:17-203.  Outputs for culled Gaussians: radii = 0,
 * everything else UNTOUCHED (the reference leaves at::empty garbage there,
 * Projection.cpp:70-73) -- compare under the radii>0 mask.
 * viewmats1 (nullable) is the end-of-frame pose and rs_type the ShutterType; the centre-of-shutter pose
 * (tau = 0.5) gives the near / far cull and the depth (:73-80), every sigma point goes through
 * project_shutter_pose.
 */
ORC_API int orc_projection_ut(
    uint32_t C, uint32_t N,
    const float *means, const float *quats, const float *scales, const float *opacities /*nullable*/,
    const float *viewmats0, const float *viewmats1 /*nullable*/, const float *Ks,
    uint32_t image_width, uint32_t image_height,
    float eps2d_f, float near_plane, float far_plane, float radius_clip,
    int camera_model, OrcUTParams ut, int rs_type,
    const float *radial, int n_radial, const float *tangential, int n_tangential, const float *thin_prism,
    int n_thin_prism,
    int32_t *radii, float *means2d, float *depths, float *conics, float *compensations /*nullable*/) {
    if ((camera_model != ORC_PINHOLE && camera_model != ORC_FISHEYE) || rs_type < 0 || rs_type > ORC_GLOBAL)
        return ORC_E_UNSUPPORTED; /* ortho: not restated */
    const real eps2d = eps2d_f;
    for (uint32_t cid = 0; cid < C; ++cid) {
        Pose start, end;
        shutter_poses(viewmats0, viewmats1, cid, &start, &end);
        const Pose mid = interpolate_pose(start, end, (real)0.5);
        const CamModel cm = cam_model_make(camera_model, image_width, image_height, Ks + cid * 9,
                                           radial ? radial + cid * n_radial : NULL, n_radial,
                                           tangential ? tangential + cid * n_tangential : NULL, n_tangential,
                                           thin_prism ? thin_prism + cid * n_thin_prism : NULL, n_thin_prism);
#pragma omp parallel for num_threads(g_threads) schedule(static)
        for (uint32_t gid = 0; gid < N; ++gid) {
            const uint64_t idx = (uint64_t)cid * N + gid;
            v3 mean = v3_make(means[gid * 3], means[gid * 3 + 1], means[gid * 3 + 2]);
            v3 scale = v3_make(scales[gid * 3], scales[gid * 3 + 1], scales[gid * 3 + 2]);
            qt quat = {quats[gid * 4], quats[gid * 4 + 1], quats[gid * 4 + 2], quats[gid * 4 + 3]};
            quat = quat_normalize(quat);

            v3 mean_c = v3_add(quat_rotate(mid.q, mean), mid.t);
            if (mean_c.z < (real)near_plane || mean_c.z > (real)far_plane) {
                radii[idx * 2] = 0; radii[idx * 2 + 1] = 0;
                continue;
            }
            /* sigma points, Cameras.cuh:1034-1083 */
            const real alpha = ut.alpha, beta = ut.beta, kappa = ut.kappa;
            const real D = 3;
            const real lambda = alpha * alpha * (D + kappa) - D;
            m3 R = mat3_cast(quat);
            v3 pts[7];
            real w_mean[7], w_cov[7];
            pts[0] = mean;
            const real sq = R_SQRT(D + lambda);
            const real sc[3] = {scale.x, scale.y, scale.z};
            for (int i = 0; i < 3; ++i) {
                v3 col = v3_make(R.c[i][0], R.c[i][1], R.c[i][2]);
                v3 delta = v3_scale(col, sq * sc[i]);
                pts[i + 1] = v3_add(mean, delta);
                pts[i + 4] = v3_sub(mean, delta);
            }
            w_mean[0] = lambda / (D + lambda);
            w_cov[0] = lambda / (D + lambda) + ((real)1 - alpha * alpha + beta);
            for (int i = 0; i < 6; ++i) {
                w_mean[i + 1] = (real)1 / ((real)2 * (D + lambda));
                w_cov[i + 1] = (real)1 / ((real)2 * (D + lambda));
            }
            /* Cameras.cuh:1107-1149 */
            int valid = ut.require_all_sigma_points_valid ? 1 : 0;
            real ipx[7], ipy[7];
            real mx = 0, my = 0;
            int early = 0;
            for (int i = 0; i < 7; ++i) {
                real px, py;
                int pv = project_shutter_pose(&cm, rs_type, start, end, pts[i], (real)ut.in_image_margin_factor, &px,
                                              &py);
                if (ut.require_all_sigma_points_valid) {
                    valid &= pv;
                    if (!pv) { early = 1; break; }
                } else {
                    valid |= pv;
                }
                ipx[i] = px; ipy[i] = py;
                mx += w_mean[i] * px;
                my += w_mean[i] * py;
            }
            if (early || !valid) {
                radii[idx * 2] = 0; radii[idx * 2 + 1] = 0;
                continue;
            }
            real cxx = 0, cxy = 0, cyy = 0;
            for (int i = 0; i < 7; ++i) {
                real dx = ipx[i] - mx, dy = ipy[i] - my;
                cxx += w_cov[i] * (dx * dx);
                cxy += w_cov[i] * (dx * dy);
                cyy += w_cov[i] * (dy * dy);
            }
            /* add_blur, Utils.cuh:171-179 */
            real det_orig = cxx * cyy - cxy * cxy;
            cxx += eps2d; cyy += eps2d;
            real det = cxx * cyy - cxy * cxy;
            real q0 = det_orig / det;
            real compensation = R_SQRT(q0 > 0 ? q0 : (real)0);
            if (det <= (real)0) {
                radii[idx * 2] = 0; radii[idx * 2 + 1] = 0;
                continue;
            }
            /* glm::inverse(mat2) */
            real ood = (real)1 / (cxx * cyy - cxy * cxy);
            real i00 = cyy * ood, i01 = -cxy * ood, i11 = cxx * ood;

            real extend = (real)3.33;
            if (opacities != NULL) {
                real opacity = opacities[gid];
                opacity *= compensation;
                if (opacity < (real)(1.f / 255.f)) {
                    radii[idx * 2] = 0; radii[idx * 2 + 1] = 0;
                    continue;
                }
                real e2 = R_SQRT((real)2 * R_LOG(opacity / (real)(1.f / 255.f)));
                if (e2 < extend) extend = e2;
            }
            real b = (real)0.5 * (cxx + cyy);
            real bb = b * b - det;
            real tmp = R_SQRT(bb > (real)0.01 ? bb : (real)0.01);
            real v1 = b + tmp;
            real r1 = extend * R_SQRT(v1);
            real rx0 = extend * R_SQRT(cxx), ry0 = extend * R_SQRT(cyy);
            real radius_x = R_CEIL(rx0 < r1 ? rx0 : r1);
            real radius_y = R_CEIL(ry0 < r1 ? ry0 : r1);
            if (radius_x <= (real)radius_clip && radius_y <= (real)radius_clip) {
                radii[idx * 2] = 0; radii[idx * 2 + 1] = 0;
                continue;
            }
            if (mx + radius_x <= 0 || mx - radius_x >= (real)image_width ||
                my + radius_y <= 0 || my - radius_y >= (real)image_height) {
                radii[idx * 2] = 0; radii[idx * 2 + 1] = 0;
                continue;
            }
            radii[idx * 2] = (int32_t)radius_x;
            radii[idx * 2 + 1] = (int32_t)radius_y;
            means2d[idx * 2] = (float)mx;
            means2d[idx * 2 + 1] = (float)my;
            depths[idx] = (float)mean_c.z;
            conics[idx * 3] = (float)i00;
            conics[idx * 3 + 1] = (float)i01;
            conics[idx * 3 + 2] = (float)i11;
            if (compensations) compensations[idx] = (float)compensation;
        }
    }
    return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* K2/K3: spherical harmonics                                          */
/* ------------------------------------------------------------------ */

/* SH basis values (Sloan ordering), SphericalHarmonicsCUDA.cu:29-103.
 * Also returns d(basis)/d(x,y,z) of the UNIT direction (:171-352). */
static void sh_bases(uint32_t degree, real x, real y, real z, real *b /*25*/,
                     real *bx, real *by, real *bz /*25 each, may be NULL*/) {
    const int want = bx != NULL;
    for (int i = 0; i < 25; ++i) { b[i] = 0; if (want) { bx[i] = by[i] = bz[i] = 0; } }
    b[0] = (real)0.2820947917738781;
    if (degree < 1) return;
    b[1] = (real)-0.48860251190292 * y;
    b[2] = (real)0.48860251190292 * z;
    b[3] = (real)-0.48860251190292 * x;
    if (want) { by[1] = (real)-0.48860251190292; bz[2] = (real)0.48860251190292; bx[3] = (real)-0.48860251190292; }
    if (degree < 2) return;
    real z2 = z * z;
    real fTmp0B = (real)-1.092548430592079 * z;
    real fC1 = x * x - y * y;
    real fS1 = (real)2 * x * y;
    b[6] = (real)0.9461746957575601 * z2 - (real)0.3153915652525201;
    b[7] = fTmp0B * x;
    b[5] = fTmp0B * y;
    b[8] = (real)0.5462742152960395 * fC1;
    b[4] = (real)0.5462742152960395 * fS1;
    real fTmp0B_z = (real)-1.092548430592079;
    real fC1_x = (real)2 * x, fC1_y = (real)-2 * y, fS1_x = (real)2 * y, fS1_y = (real)2 * x;
    real pSH6_z = (real)2 * (real)0.9461746957575601 * z;
    if (want) {
        bz[6] = pSH6_z;
        bx[7] = fTmp0B; bz[7] = fTmp0B_z * x;
        by[5] = fTmp0B; bz[5] = fTmp0B_z * y;
        bx[8] = (real)0.5462742152960395 * fC1_x; by[8] = (real)0.5462742152960395 * fC1_y;
        bx[4] = (real)0.5462742152960395 * fS1_x; by[4] = (real)0.5462742152960395 * fS1_y;
    }
    if (degree < 3) return;
    real fTmp0C = (real)-2.285228997322329 * z2 + (real)0.4570457994644658;
    real fTmp1B = (real)1.445305721320277 * z;
    real fC2 = x * fC1 - y * fS1;
    real fS2 = x * fS1 + y * fC1;
    real pSH12 = z * ((real)1.865881662950577 * z2 - (real)1.119528997770346);
    b[12] = pSH12;
    b[13] = fTmp0C * x;
    b[11] = fTmp0C * y;
    b[14] = fTmp1B * fC1;
    b[10] = fTmp1B * fS1;
    b[15] = (real)-0.5900435899266435 * fC2;
    b[9] = (real)-0.5900435899266435 * fS2;
    real fTmp0C_z = (real)-2.285228997322329 * (real)2 * z;
    real fTmp1B_z = (real)1.445305721320277;
    real fC2_x = fC1 + x * fC1_x - y * fS1_x;
    real fC2_y = x * fC1_y - fS1 - y * fS1_y;
    real fS2_x = fS1 + x * fS1_x + y * fC1_x;
    real fS2_y = x * fS1_y + fC1 + y * fC1_y;
    real pSH12_z = (real)3 * (real)1.865881662950577 * z2 - (real)1.119528997770346;
    if (want) {
        bz[12] = pSH12_z;
        bx[13] = fTmp0C; bz[13] = fTmp0C_z * x;
        by[11] = fTmp0C; bz[11] = fTmp0C_z * y;
        bx[14] = fTmp1B * fC1_x; by[14] = fTmp1B * fC1_y; bz[14] = fTmp1B_z * fC1;
        bx[10] = fTmp1B * fS1_x; by[10] = fTmp1B * fS1_y; bz[10] = fTmp1B_z * fS1;
        bx[15] = (real)-0.5900435899266435 * fC2_x; by[15] = (real)-0.5900435899266435 * fC2_y;
        bx[9] = (real)-0.5900435899266435 * fS2_x; by[9] = (real)-0.5900435899266435 * fS2_y;
    }
    if (degree < 4) return;
    real fTmp0D = z * ((real)-4.683325804901025 * z2 + (real)2.007139630671868);
    real fTmp1C = (real)3.31161143515146 * z2 - (real)0.47308734787878;
    real fTmp2B = (real)-1.770130769779931 * z;
    real fC3 = x * fC2 - y * fS2;
    real fS3 = x * fS2 + y * fC2;
    b[20] = (real)1.984313483298443 * z * pSH12 + (real)-1.006230589874905 * b[6];
    b[21] = fTmp0D * x;
    b[19] = fTmp0D * y;
    b[22] = fTmp1C * fC1;
    b[18] = fTmp1C * fS1;
    b[23] = fTmp2B * fC2;
    b[17] = fTmp2B * fS2;
    b[24] = (real)0.6258357354491763 * fC3;
    b[16] = (real)0.6258357354491763 * fS3;
    if (want) {
        real fTmp0D_z = (real)3 * (real)-4.683325804901025 * z2 + (real)2.007139630671868;
        real fTmp1C_z = (real)2 * (real)3.31161143515146 * z;
        real fTmp2B_z = (real)-1.770130769779931;
        real fC3_x = fC2 + x * fC2_x - y * fS2_x;
        real fC3_y = x * fC2_y - fS2 - y * fS2_y;
        real fS3_x = fS2 + y * fC2_x + x * fS2_x;
        real fS3_y = x * fS2_y + fC2 + y * fC2_y;
        bz[20] = (real)1.984313483298443 * (pSH12 + z * pSH12_z) + (real)-1.006230589874905 * pSH6_z;
        bx[21] = fTmp0D; bz[21] = fTmp0D_z * x;
        by[19] = fTmp0D; bz[19] = fTmp0D_z * y;
        bx[22] = fTmp1C * fC1_x; by[22] = fTmp1C * fC1_y; bz[22] = fTmp1C_z * fC1;
        bx[18] = fTmp1C * fS1_x; by[18] = fTmp1C * fS1_y; bz[18] = fTmp1C_z * fS1;
        bx[23] = fTmp2B * fC2_x; by[23] = fTmp2B * fC2_y; bz[23] = fTmp2B_z * fC2;
        bx[17] = fTmp2B * fS2_x; by[17] = fTmp2B * fS2_y; bz[17] = fTmp2B_z * fS2;
        bx[24] = (real)0.6258357354491763 * fC3_x; by[24] = (real)0.6258357354491763 * fC3_y;
        bx[16] = (real)0.6258357354491763 * fS3_x; by[16] = (real)0.6258357354491763 * fS3_y;
    }
}

/* SphericalHarmonicsCUDA.cu:374-399.  Masked-out rows are left untouched. */
ORC_API int orc_sh_fwd(uint32_t n, uint32_t K, uint32_t degree, const float *dirs,
                       const float *coeffs, const uint8_t *masks /*nullable*/, float *colors) {
    const uint32_t nb = (degree + 1) * (degree + 1);
    if (degree > 4 || nb > K) return ORC_E_UNSUPPORTED;
#pragma omp parallel for num_threads(g_threads) schedule(static)
    for (uint32_t e = 0; e < n; ++e) {
        if (masks && !masks[e]) continue;
        real b[25];
        real x = dirs[e * 3], y = dirs[e * 3 + 1], z = dirs[e * 3 + 2];
        if (degree >= 1) {
            real inorm = (real)1 / R_SQRT(x * x + y * y + z * z);
            x *= inorm; y *= inorm; z *= inorm;
        }
        sh_bases(degree, x, y, z, b, NULL, NULL, NULL);
        const float *c = coeffs + (uint64_t)e * K * 3;
        for (int ch = 0; ch < 3; ++ch) {
            real r = 0;
            for (uint32_t k = 0; k < nb; ++k) r += b[k] * (real)c[k * 3 + ch];
            colors[e * 3 + ch] = (float)r;
        }
    }
    return ORC_OK;
}

/* SphericalHarmonicsCUDA.cu:445-481.  v_coeffs / v_dirs must be zero-initialised
 * by the caller (SphericalHarmonics.cpp:58-62). */
ORC_API int orc_sh_bwd(uint32_t n, uint32_t K, uint32_t degree, const float *dirs,
                       const float *coeffs, const uint8_t *masks /*nullable*/,
                       const float *v_colors, float *v_coeffs, float *v_dirs /*nullable*/) {
    const uint32_t nb = (degree + 1) * (degree + 1);
    if (degree > 4 || nb > K) return ORC_E_UNSUPPORTED;
#pragma omp parallel for num_threads(g_threads) schedule(static)
    for (uint32_t e = 0; e < n; ++e) {
        if (masks && !masks[e]) continue;
        real b[25], bx[25], by[25], bz[25];
        real dx = dirs[e * 3], dy = dirs[e * 3 + 1], dz = dirs[e * 3 + 2];
        real inorm = 1, x = dx, y = dy, z = dz;
        if (degree >= 1) {
            inorm = (real)1 / R_SQRT(dx * dx + dy * dy + dz * dz);
            x = dx * inorm; y = dy * inorm; z = dz * inorm;
        }
        sh_bases(degree, x, y, z, b, bx, by, bz);
        const float *c = coeffs + (uint64_t)e * K * 3;
        float *vc = v_coeffs + (uint64_t)e * K * 3;
        real vx = 0, vy = 0, vz = 0;
        for (int ch = 0; ch < 3; ++ch) {
            real vcol = v_colors[e * 3 + ch];
            for (uint32_t k = 0; k < nb; ++k) {
                vc[k * 3 + ch] = (float)(b[k] * vcol);
                vx += vcol * bx[k] * (real)c[k * 3 + ch];
                vy += vcol * by[k] * (real)c[k * 3 + ch];
                vz += vcol * bz[k] * (real)c[k * 3 + ch];
            }
        }
        if (v_dirs && degree >= 1) {
            real dot = vx * x + vy * y + vz * z;
            v_dirs[e * 3 + 0] += (float)((vx - dot * x) * inorm);
            v_dirs[e * 3 + 1] += (float)((vy - dot * y) * inorm);
            v_dirs[e * 3 + 2] += (float)((vz - dot * z) * inorm);
        }
    }
    return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* K4-K6: tile intersection                                            */
/* ------------------------------------------------------------------ */

/* (uint32_t)floorf(x) under CUDA's saturating cvt.rzi.u32.f32 (IntersectTile.cu:72-76;
 * negatives -> 0, NaN -> 0, overflow -> UINT32_MAX). */
static uint32_t sat_u32(float x) {
    if (!(x > 0.0f)) return 0;
    if (x >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)x;
}
static uint32_t umin32(uint32_t a, uint32_t b) { return a < b ? a : b; }

static void tile_bbox(const float *means2d, const int32_t *radii, uint64_t idx, uint32_t tile_size,
                      uint32_t tile_width, uint32_t tile_height, uint32_t *x0, uint32_t *x1,
                      uint32_t *y0, uint32_t *y1, int *active) {
    const float radius_x = (float)radii[idx * 2], radius_y = (float)radii[idx * 2 + 1];
    if (radius_x <= 0 || radius_y <= 0) { *active = 0; return; }
    *active = 1;
    const float ts = (float)tile_size;
    const float trx = radius_x / ts, try_ = radius_y / ts;
    const float tx = means2d[idx * 2] / ts, ty = means2d[idx * 2 + 1] / ts;
    *x0 = umin32(sat_u32(floorf(tx - trx)), tile_width);
    *y0 = umin32(sat_u32(floorf(ty - try_)), tile_height);
    *x1 = umin32(sat_u32(ceilf(tx + trx)), tile_width);
    *y1 = umin32(sat_u32(ceilf(ty + try_)), tile_height);
}

static uint32_t bit_width_u32(uint32_t n) { /* floor(log2(n)) + 1, Intersect.cpp:46-47 */
    uint32_t b = 0;
    while (n) { ++b; n >>= 1; }
    return b;
}

ORC_API uint32_t orc_tile_n_bits(uint32_t n_tiles) { return bit_width_u32(n_tiles); }

/* pass 1: tiles_per_gauss [C*N]; returns n_isects. IntersectTile.cu:47-84 */
ORC_API int64_t orc_isect_count(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii,
                                uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
                                int32_t *tiles_per_gauss) {
    int64_t total = 0;
    for (uint64_t idx = 0; idx < (uint64_t)C * N; ++idx) {
        uint32_t x0, x1, y0, y1; int active;
        tile_bbox(means2d, radii, idx, tile_size, tile_width, tile_height, &x0, &x1, &y0, &y1, &active);
        int32_t cnt = active ? (int32_t)((y1 - y0) * (x1 - x0)) : 0;
        tiles_per_gauss[idx] = cnt;
        total += cnt;
    }
    return total;
}

typedef struct { uint64_t key; int32_t val; } kv_t;

/* stable LSD radix sort on the low `bits` bits (== cub::DeviceRadixSort::SortPairs
 * begin_bit=0,end_bit=bits; IntersectTile.cu:307-314) */
static void radix_sort_kv(uint64_t *keys, int32_t *vals, int64_t n, uint32_t bits) {
    if (n <= 1) return;
    uint64_t *k2 = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)n);
    int32_t *v2 = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    uint64_t *ks = keys, *kd = k2;
    int32_t *vs = vals, *vd = v2;
    for (uint32_t shift = 0; shift < bits; shift += 8) {
        uint32_t nb = bits - shift < 8 ? bits - shift : 8;
        uint64_t mask = ((uint64_t)1 << nb) - 1;
        int64_t hist[257];
        memset(hist, 0, sizeof(hist));
        for (int64_t i = 0; i < n; ++i) hist[((ks[i] >> shift) & mask) + 1]++;
        for (int i = 0; i < 256; ++i) hist[i + 1] += hist[i];
        for (int64_t i = 0; i < n; ++i) {
            int64_t p = hist[(ks[i] >> shift) & mask]++;
            kd[p] = ks[i]; vd[p] = vs[i];
        }
        uint64_t *tk = ks; ks = kd; kd = tk;
        int32_t *tv = vs; vs = vd; vd = tv;
    }
    if (ks != keys) {
        memcpy(keys, ks, sizeof(uint64_t) * (size_t)n);
        memcpy(vals, vs, sizeof(int32_t) * (size_t)n);
    }
    free(k2); free(v2);
}

/* pass 2 + sort: isect_ids [n_isects] int64, flatten_ids [n_isects] int32.
 * IntersectTile.cu:86-113, Intersect.cpp:75-121 */
ORC_API int orc_isect_emit_sort(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii,
                                const float *depths, uint32_t tile_size, uint32_t tile_width,
                                uint32_t tile_height, int sort, int64_t n_isects,
                                int64_t *isect_ids, int32_t *flatten_ids) {
    const uint32_t n_tiles = tile_width * tile_height;
    const uint32_t tile_n_bits = bit_width_u32(n_tiles);
    const uint32_t cam_n_bits = bit_width_u32(C);
    int64_t cur = 0;
    for (uint64_t idx = 0; idx < (uint64_t)C * N; ++idx) {
        uint32_t x0, x1, y0, y1; int active;
        tile_bbox(means2d, radii, idx, tile_size, tile_width, tile_height, &x0, &x1, &y0, &y1, &active);
        if (!active) continue;
        const int64_t cid = (int64_t)(idx / N);
        const int64_t cid_enc = cid << (32 + tile_n_bits);
        uint32_t dbits;
        memcpy(&dbits, depths + idx, 4);
        const int64_t depth_enc = (int64_t)dbits; /* zero-extended */
        for (uint32_t i = y0; i < y1; ++i)
            for (uint32_t j = x0; j < x1; ++j) {
                int64_t tile_id = (int64_t)i * tile_width + j;
                if (cur >= n_isects) return ORC_E_UNSUPPORTED;
                isect_ids[cur] = cid_enc | (tile_id << 32) | depth_enc;
                flatten_ids[cur] = (int32_t)idx;
                ++cur;
            }
    }
    if (cur != n_isects) return ORC_E_UNSUPPORTED;
    if (sort) radix_sort_kv((uint64_t *)isect_ids, flatten_ids, n_isects, 32 + tile_n_bits + cam_n_bits);
    return ORC_OK;
}

/* IntersectTile.cu:206-252 / :268-271 */
ORC_API int orc_isect_offsets(int64_t n_isects, const int64_t *isect_ids, uint32_t C,
                              uint32_t tile_width, uint32_t tile_height, int32_t *offsets) {
    const uint32_t n_tiles = tile_width * tile_height;
    const uint32_t tile_n_bits = bit_width_u32(n_tiles);
    const int64_t total = (int64_t)C * n_tiles;
    if (n_isects == 0) {
        for (int64_t i = 0; i < total; ++i) offsets[i] = 0;
        return ORC_OK;
    }
    for (int64_t idx = 0; idx < n_isects; ++idx) {
        int64_t cur = isect_ids[idx] >> 32;
        int64_t cid_curr = cur >> tile_n_bits;
        int64_t tid_curr = cur & (((int64_t)1 << tile_n_bits) - 1);
        int64_t id_curr = cid_curr * n_tiles + tid_curr;
        if (idx == 0)
            for (int64_t i = 0; i < id_curr + 1 && i < total; ++i) offsets[i] = 0;
        if (idx == n_isects - 1)
            for (int64_t i = id_curr + 1; i < total; ++i) offsets[i] = (int32_t)n_isects;
        if (idx > 0) {
            int64_t prev = isect_ids[idx - 1] >> 32;
            if (prev == cur) continue;
            int64_t cid_prev = prev >> tile_n_bits;
            int64_t tid_prev = prev & (((int64_t)1 << tile_n_bits) - 1);
            int64_t id_prev = cid_prev * n_tiles + tid_prev;
            for (int64_t i = id_prev + 1; i < id_curr + 1 && i < total; ++i) offsets[i] = (int32_t)idx;
        }
    }
    return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* K7/K8: from-world blend                                             */
/* ------------------------------------------------------------------ */

typedef struct { v3 o, d; int valid; } Ray;

/* Cameras.cuh:322-339,261-265: the pose of the frame time of (px, py) itself, the pixel centre */
static Ray pixel_ray(real px, real py, const CamModel *cm, Pose start, Pose end, int rs_type) {
    v3 cam;
    Ray r;
    r.valid = cam_unproject(cm, px, py, &cam);
    if (!r.valid) { r.o = v3_make(0, 0, 0); r.d = v3_make(0, 0, 0); return r; }
    Pose p = interpolate_pose(start, end, shutter_relative_frame_time(rs_type, px, py, cm->W, cm->H));
    m3 R_inv = mat3_cast(quat_inverse(p.q));
    r.o = m3_mulv(&R_inv, v3_scale(p.t, (real)-1));
    r.d = m3_mulv(&R_inv, cam);
    return r;
}

/* Utils.cuh:181-184 */
static v3 safe_normalize(v3 v) {
    real l = v.x * v.x + v.y * v.y + v.z * v.z;
    return l > (real)0 ? v3_scale(v, (real)1 / R_SQRT(l)) : v;
}
/* Utils.cuh:186-194 */
static v3 safe_normalize_bw(v3 v, v3 d_out) {
    real l = v.x * v.x + v.y * v.y + v.z * v.z;
    if (l > (real)0) {
        real il = (real)1 / R_SQRT(l);
        real il3 = il * il * il;
        real dd = v3_dot(d_out, v);
        return v3_sub(v3_scale(d_out, il), v3_scale(v, il3 * dd));
    }
    return d_out;
}

/* S^-1 R^T for one Gaussian (Fwd.cu:204-219) */
static m3 iscl_rot_of(const float *quat4, const float *scale3) {
    real q4[4] = {quat4[0], quat4[1], quat4[2], quat4[3]};
    m3 R = quat_to_rotmat(q4);
    m3 S;
    memset(&S, 0, sizeof(S));
    S.c[0][0] = (real)1 / (real)scale3[0];
    S.c[1][1] = (real)1 / (real)scale3[1];
    S.c[2][2] = (real)1 / (real)scale3[2];
    m3 Rt = m3_transpose(&R);
    return m3_mul(&S, &Rt);
}

/*
 * RasterizeToPixelsFromWorld3DGSFwd.cu:20-279 (CDIM == 3, C == 1 per call is
 * what the reference supports: flatten_ids index means[] directly, :197-200).
 * masks: [C, th, tw] bytes or NULL; backgrounds [C,3] or NULL.
 * viewmats1 (nullable): end-of-frame poses; rs_type: ShutterType (Fwd.cu:80-127).
 * Outputs for masked-out tiles: only render_colors written (:143-150).
 */
ORC_API int orc_raster_fwd(
    uint32_t C, uint32_t N, int64_t n_isects,
    const float *means, const float *quats, const float *scales, const float *colors,
    const float *opacities, const float *backgrounds, const uint8_t *masks,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size,
    const float *viewmats0, const float *viewmats1, const float *Ks, int camera_model, int rs_type,
    const float *radial, int n_radial, const float *tangential, int n_tangential, const float *thin_prism,
    int n_thin_prism,
    const int32_t *tile_offsets, const int32_t *flatten_ids,
    float *render_colors, float *render_alphas, int32_t *last_ids) {
    if (camera_model != ORC_PINHOLE && camera_model != ORC_FISHEYE) return ORC_E_UNSUPPORTED;
    if (rs_type < 0 || rs_type > ORC_GLOBAL) return ORC_E_UNSUPPORTED;
    (void)N;
    const uint32_t tile_width = (image_width + tile_size - 1) / tile_size;
    const uint32_t tile_height = (image_height + tile_size - 1) / tile_size;
    for (uint32_t cid = 0; cid < C; ++cid) {
        Pose start, end;
        shutter_poses(viewmats0, viewmats1, cid, &start, &end);
        const CamModel cm = cam_model_make(camera_model, image_width, image_height, Ks + cid * 9,
                                           radial ? radial + cid * n_radial : NULL, n_radial,
                                           tangential ? tangential + cid * n_tangential : NULL, n_tangential,
                                           thin_prism ? thin_prism + cid * n_thin_prism : NULL, n_thin_prism);
        const int32_t *toff = tile_offsets + (uint64_t)cid * tile_height * tile_width;
        float *rc = render_colors + (uint64_t)cid * image_height * image_width * 3;
        float *ra = render_alphas + (uint64_t)cid * image_height * image_width;
        int32_t *li = last_ids + (uint64_t)cid * image_height * image_width;
        const float *bg = backgrounds ? backgrounds + cid * 3 : NULL;
        const uint8_t *mk = masks ? masks + (uint64_t)cid * tile_height * tile_width : NULL;
#pragma omp parallel for num_threads(g_threads) schedule(dynamic, 1)
        for (uint32_t tile_id = 0; tile_id < tile_height * tile_width; ++tile_id) {
            {
                const uint32_t ty = tile_id / tile_width, tx = tile_id % tile_width;
                int32_t range_start = toff[tile_id];
                int32_t range_end = (cid == C - 1 && tile_id == tile_width * tile_height - 1)
                                        ? (int32_t)n_isects : toff[tile_id + 1];
                const int32_t cnt = range_end > range_start ? range_end - range_start : 0;
                /* per-tile staging of S^-1 R^T (:192-220) */
                m3 *isr = (m3 *)malloc(sizeof(m3) * (size_t)(cnt > 0 ? cnt : 1));
                for (int32_t k = 0; k < cnt; ++k) {
                    int32_t g = flatten_ids[range_start + k];
                    isr[k] = iscl_rot_of(quats + (uint64_t)g * 4, scales + (uint64_t)g * 3);
                }
                for (uint32_t iy = 0; iy < tile_size; ++iy)
                    for (uint32_t ix = 0; ix < tile_size; ++ix) {
                        const uint32_t i = ty * tile_size + iy, j = tx * tile_size + ix;
                        if (!(i < image_height && j < image_width)) continue;
                        const uint64_t pix = (uint64_t)i * image_width + j;
                        if (mk && !mk[tile_id]) {
                            for (int k = 0; k < 3; ++k) rc[pix * 3 + k] = bg ? bg[k] : 0.0f;
                            continue;
                        }
                        const Ray ray = pixel_ray((real)j + (real)0.5, (real)i + (real)0.5, &cm, start, end, rs_type);
                        real T = 1;
                        uint32_t cur_idx = 0;
                        real pix_out[3] = {0, 0, 0};
                        for (int32_t k = 0; k < cnt && ray.valid; ++k) { /* done = !inside || !ray.valid (:139) */
                            const int32_t g = flatten_ids[range_start + k];
                            const real opac = opacities[g];
                            const v3 xyz = v3_make(means[g * 3], means[g * 3 + 1], means[g * 3 + 2]);
                            const v3 gro = m3_mulv(&isr[k], v3_sub(ray.o, xyz));
                            const v3 grd = safe_normalize(m3_mulv(&isr[k], ray.d));
                            const v3 gcrod = v3_cross(grd, gro);
                            const real grayDist = v3_dot(gcrod, gcrod);
                            const real power = (real)-0.5 * grayDist;
                            real alpha = opac * R_EXP(power);
                            if (alpha > (real)0.999) alpha = (real)0.999;
                            if (alpha < ORC_ALPHA_MIN) continue;
                            const real next_T = T * ((real)1 - alpha);
                            if (next_T <= ORC_T_MIN) break;
                            const real vis = alpha * T;
                            for (int c = 0; c < 3; ++c) pix_out[c] += (real)colors[(uint64_t)g * 3 + c] * vis;
                            cur_idx = (uint32_t)(range_start + k);
                            T = next_T;
                        }
                        ra[pix] = (float)((real)1 - T);
                        for (int c = 0; c < 3; ++c)
                            rc[pix * 3 + c] = (float)(bg ? pix_out[c] + T * (real)bg[c] : pix_out[c]);
                        li[pix] = (int32_t)cur_idx;
                    }
                free(isr);
            }
        }
    }
    return ORC_OK;
}

/* Utils.cuh:104-126 */
static void quat_to_rotmat_vjp(const real q4[4], const m3 *v_R, real v_quat[4]) {
    real w = q4[0], x = q4[1], y = q4[2], z = q4[3];
    real inv_norm = (real)1 / R_SQRT(x * x + y * y + z * z + w * w);
    x *= inv_norm; y *= inv_norm; z *= inv_norm; w *= inv_norm;
#define VR(i, j) (v_R->c[i][j])
    real vq[4];
    vq[0] = (real)2 * (x * (VR(1, 2) - VR(2, 1)) + y * (VR(2, 0) - VR(0, 2)) + z * (VR(0, 1) - VR(1, 0)));
    vq[1] = (real)2 * ((real)-2 * x * (VR(1, 1) + VR(2, 2)) + y * (VR(0, 1) + VR(1, 0)) +
                       z * (VR(0, 2) + VR(2, 0)) + w * (VR(1, 2) - VR(2, 1)));
    vq[2] = (real)2 * (x * (VR(0, 1) + VR(1, 0)) - (real)2 * y * (VR(0, 0) + VR(2, 2)) +
                       z * (VR(1, 2) + VR(2, 1)) + w * (VR(2, 0) - VR(0, 2)));
    vq[3] = (real)2 * (x * (VR(0, 2) + VR(2, 0)) + y * (VR(1, 2) + VR(2, 1)) -
                       (real)2 * z * (VR(0, 0) + VR(1, 1)) + w * (VR(0, 1) - VR(1, 0)));
#undef VR
    real qn[4] = {w, x, y, z};
    real dot = vq[0] * qn[0] + vq[1] * qn[1] + vq[2] * qn[2] + vq[3] * qn[3];
    for (int k = 0; k < 4; ++k) v_quat[k] += (vq[k] - dot * qn[k]) * inv_norm;
}

/* Utils.cuh:128-158 */
static void quat_scale_to_preci_half_vjp(const real q4[4], const real s3[3], const m3 *R,
                                         const m3 *v_M, real v_quat[4], real v_scale[3]) {
    real sx = (real)1 / s3[0], sy = (real)1 / s3[1], sz = (real)1 / s3[2];
    m3 S;
    memset(&S, 0, sizeof(S));
    S.c[0][0] = sx; S.c[1][1] = sy; S.c[2][2] = sz;
    m3 v_R = m3_mul(v_M, &S);
    quat_to_rotmat_vjp(q4, &v_R, v_quat);
    v_scale[0] += -sx * sx * (R->c[0][0] * v_M->c[0][0] + R->c[0][1] * v_M->c[0][1] + R->c[0][2] * v_M->c[0][2]);
    v_scale[1] += -sy * sy * (R->c[1][0] * v_M->c[1][0] + R->c[1][1] * v_M->c[1][1] + R->c[1][2] * v_M->c[1][2]);
    v_scale[2] += -sz * sz * (R->c[2][0] * v_M->c[2][0] + R->c[2][1] * v_M->c[2][1] + R->c[2][2] * v_M->c[2][2]);
}

/*
 * RasterizeToPixelsFromWorld3DGSBwd.cu:17-373.  Gradient outputs are float64
 * and must be zero-initialised by the caller (Rasterization.cpp:190-194).
 * The per-pixel walk from last_ids[pix] down to range_start is equivalent to
 * the reference's batch/warp schedule (:196-233): lanes whose index is above
 * their own bin_final are invalid there and contribute nothing.
 */
ORC_API int orc_raster_bwd(
    uint32_t C, uint32_t N, int64_t n_isects,
    const float *means, const float *quats, const float *scales, const float *colors,
    const float *opacities, const float *backgrounds, const uint8_t *masks,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size,
    const float *viewmats0, const float *viewmats1, const float *Ks, int camera_model, int rs_type,
    const float *radial, int n_radial, const float *tangential, int n_tangential, const float *thin_prism,
    int n_thin_prism,
    const int32_t *tile_offsets, const int32_t *flatten_ids,
    const float *render_alphas, const int32_t *last_ids,
    const float *v_render_colors, const float *v_render_alphas,
    double *v_means, double *v_quats, double *v_scales, double *v_colors, double *v_opacities) {
    if (camera_model != ORC_PINHOLE && camera_model != ORC_FISHEYE) return ORC_E_UNSUPPORTED;
    if (rs_type < 0 || rs_type > ORC_GLOBAL) return ORC_E_UNSUPPORTED;
    (void)N;
    if (n_isects == 0) return ORC_OK;
    const uint32_t tile_width = (image_width + tile_size - 1) / tile_size;
    const uint32_t tile_height = (image_height + tile_size - 1) / tile_size;
    for (uint32_t cid = 0; cid < C; ++cid) {
        Pose start, end;
        shutter_poses(viewmats0, viewmats1, cid, &start, &end);
        const CamModel cm = cam_model_make(camera_model, image_width, image_height, Ks + cid * 9,
                                           radial ? radial + cid * n_radial : NULL, n_radial,
                                           tangential ? tangential + cid * n_tangential : NULL, n_tangential,
                                           thin_prism ? thin_prism + cid * n_thin_prism : NULL, n_thin_prism);
        const int32_t *toff = tile_offsets + (uint64_t)cid * tile_height * tile_width;
        const float *ra_ = render_alphas + (uint64_t)cid * image_height * image_width;
        const int32_t *li = last_ids + (uint64_t)cid * image_height * image_width;
        const float *vrc = v_render_colors + (uint64_t)cid * image_height * image_width * 3;
        const float *vra = v_render_alphas + (uint64_t)cid * image_height * image_width;
        const float *bg = backgrounds ? backgrounds + cid * 3 : NULL;
        const uint8_t *mk = masks ? masks + (uint64_t)cid * tile_height * tile_width : NULL;
#pragma omp parallel for num_threads(g_threads) schedule(dynamic, 1)
        for (uint32_t tile_id = 0; tile_id < tile_height * tile_width; ++tile_id) {
            {
                const uint32_t ty = tile_id / tile_width, tx = tile_id % tile_width;
                if (mk && !mk[tile_id]) continue;
                const int32_t range_start = toff[tile_id];
                const int32_t range_end = (cid == C - 1 && tile_id == tile_width * tile_height - 1)
                                              ? (int32_t)n_isects : toff[tile_id + 1];
                for (uint32_t iy = 0; iy < tile_size; ++iy)
                    for (uint32_t ix = 0; ix < tile_size; ++ix) {
                        const uint32_t i = ty * tile_size + iy, j = tx * tile_size + ix;
                        if (!(i < image_height && j < image_width)) continue;
                        const uint64_t pix = (uint64_t)i * image_width + j;
                        const Ray ray = pixel_ray((real)j + (real)0.5, (real)i + (real)0.5, &cm, start, end, rs_type);
                        if (!ray.valid) continue; /* Bwd.cu:151: such pixels are never valid */
                        const real T_final = (real)1 - (real)ra_[pix];
                        real T = T_final;
                        real buffer[3] = {0, 0, 0};
                        const int32_t bin_final = li[pix];
                        const real v_render_c[3] = {vrc[pix * 3], vrc[pix * 3 + 1], vrc[pix * 3 + 2]};
                        const real v_render_a = vra[pix];
                        for (int32_t idx = (bin_final < range_end - 1 ? bin_final : range_end - 1); idx >= range_start; --idx) {
                            const int32_t g = flatten_ids[idx];
                            const real opac = opacities[g];
                            const v3 xyz = v3_make(means[g * 3], means[g * 3 + 1], means[g * 3 + 2]);
                            const real s3[3] = {scales[g * 3], scales[g * 3 + 1], scales[g * 3 + 2]};
                            const real q4[4] = {quats[g * 4], quats[g * 4 + 1], quats[g * 4 + 2], quats[g * 4 + 3]};
                            m3 R = quat_to_rotmat(q4);
                            m3 S;
                            memset(&S, 0, sizeof(S));
                            S.c[0][0] = (real)1 / s3[0]; S.c[1][1] = (real)1 / s3[1]; S.c[2][2] = (real)1 / s3[2];
                            m3 RS = m3_mul(&R, &S);
                            m3 Mt = m3_transpose(&RS);
                            const v3 o_minus_mu = v3_sub(ray.o, xyz);
                            const v3 gro = m3_mulv(&Mt, o_minus_mu);
                            const v3 grd = m3_mulv(&Mt, ray.d);
                            const v3 grd_n = safe_normalize(grd);
                            const v3 gcrod = v3_cross(grd_n, gro);
                            const real grayDist = v3_dot(gcrod, gcrod);
                            const real power = (real)-0.5 * grayDist;
                            const real vis = R_EXP(power);
                            real alpha = opac * vis;
                            if (alpha > (real)0.999) alpha = (real)0.999;
                            if (power > (real)0 || alpha < ORC_ALPHA_MIN) continue;

                            const real ra = (real)1 / ((real)1 - alpha);
                            T *= ra;
                            const real fac = alpha * T;
                            real v_alpha = 0;
                            for (int c = 0; c < 3; ++c) {
                                ORC_ATOMIC_ADD(v_colors[(uint64_t)g * 3 + c], (double)(fac * v_render_c[c]));
                                v_alpha += ((real)colors[(uint64_t)g * 3 + c] * T - buffer[c] * ra) * v_render_c[c];
                            }
                            v_alpha += T_final * ra * v_render_a;
                            if (bg) {
                                real accum = 0;
                                for (int c = 0; c < 3; ++c) accum += (real)bg[c] * v_render_c[c];
                                v_alpha += -T_final * ra * accum;
                            }
                            if (opac * vis <= (real)0.999) {
                                const real v_vis = opac * v_alpha;
                                const real v_gradDist = (real)-0.5 * vis * v_vis;
                                const v3 v_gcrod = v3_scale(gcrod, (real)2 * v_gradDist);
                                const v3 v_grd_n = v3_scale(v3_cross(v_gcrod, gro), (real)-1);
                                const v3 v_gro = v3_cross(v_gcrod, grd_n);
                                const v3 v_grd = safe_normalize_bw(grd, v_grd_n);
                                /* v_Mt = outer(v_grd, ray_d) + outer(v_gro, o_minus_mu); [col j][row i] = a_i b_j */
                                m3 v_Mt;
                                const real a1[3] = {v_grd.x, v_grd.y, v_grd.z}, b1[3] = {ray.d.x, ray.d.y, ray.d.z};
                                const real a2[3] = {v_gro.x, v_gro.y, v_gro.z}, b2[3] = {o_minus_mu.x, o_minus_mu.y, o_minus_mu.z};
                                for (int col = 0; col < 3; ++col)
                                    for (int row = 0; row < 3; ++row)
                                        v_Mt.c[col][row] = a1[row] * b1[col] + a2[row] * b2[col];
                                m3 Mtt = m3_transpose(&Mt);
                                const v3 v_o_minus_mu = m3_mulv(&Mtt, v_gro);
                                ORC_ATOMIC_ADD(v_means[(uint64_t)g * 3 + 0], (double)(-v_o_minus_mu.x));
                                ORC_ATOMIC_ADD(v_means[(uint64_t)g * 3 + 1], (double)(-v_o_minus_mu.y));
                                ORC_ATOMIC_ADD(v_means[(uint64_t)g * 3 + 2], (double)(-v_o_minus_mu.z));
                                real vq[4] = {0, 0, 0, 0}, vs[3] = {0, 0, 0};
                                m3 v_M = m3_transpose(&v_Mt);
                                quat_scale_to_preci_half_vjp(q4, s3, &R, &v_M, vq, vs);
                                for (int k = 0; k < 4; ++k) ORC_ATOMIC_ADD(v_quats[(uint64_t)g * 4 + k], (double)vq[k]);
                                for (int k = 0; k < 3; ++k) ORC_ATOMIC_ADD(v_scales[(uint64_t)g * 3 + k], (double)vs[k]);
                                ORC_ATOMIC_ADD(v_opacities[g], (double)(vis * v_alpha));
                            }
                            for (int c = 0; c < 3; ++c) buffer[c] += (real)colors[(uint64_t)g * 3 + c] * fac;
                        }
                    }
            }
        }
    }
    return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* K9-K11: link-surface helpers                                        */
/* ------------------------------------------------------------------ */

/* QuatToRotmatCUDA.cu:14-39: row-major [N,3,3] */
ORC_API int orc_quat_to_rotmat(uint32_t N, const float *quats, float *rotmats) {
    for (uint32_t n = 0; n < N; ++n) {
        real q4[4] = {quats[n * 4], quats[n * 4 + 1], quats[n * 4 + 2], quats[n * 4 + 3]};
        m3 R = quat_to_rotmat(q4);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) rotmats[n * 9 + i * 3 + j] = (float)R.c[j][i];
    }
    return ORC_OK;
}

/* RelocationCUDA.cu:12-43 */
ORC_API int orc_relocation(uint32_t N, const float *opacities, const float *scales, const int32_t *ratios,
                           const float *binoms, int n_max, float *new_opacities, float *new_scales) {
    for (uint32_t idx = 0; idx < N; ++idx) {
        int n_idx = ratios[idx];
        real denom_sum = 0;
        real no = (real)1 - R_POW((real)1 - (real)opacities[idx], (real)1 / (real)n_idx);
        new_opacities[idx] = (float)no;
        no = (real)new_opacities[idx];
        for (int i = 1; i <= n_idx; ++i)
            for (int k = 0; k <= i - 1; ++k) {
                real bin_coeff = binoms[(i - 1) * n_max + k];
                real term = (R_POW((real)-1, (real)k) / R_SQRT((real)(k + 1))) * R_POW(no, (real)(k + 1));
                denom_sum += bin_coeff * term;
            }
        real coeff = (real)opacities[idx] / denom_sum;
        for (int i = 0; i < 3; ++i) new_scales[idx * 3 + i] = (float)(coeff * (real)scales[idx * 3 + i]);
    }
    return ORC_OK;
}

/* RelocationCUDA.cu:86-144 (means updated in place) */
ORC_API int orc_add_noise(uint32_t N, const float *raw_opacities, const float *raw_scales,
                          const float *raw_quats, const float *noise, float *means, float current_lr) {
    for (uint32_t idx = 0; idx < N; ++idx) {
        real e[3];
        for (int i = 0; i < 3; ++i) e[i] = R_EXP((real)2 * (real)raw_scales[idx * 3 + i]);
        real w = raw_quats[idx * 4], x = raw_quats[idx * 4 + 1], y = raw_quats[idx * 4 + 2], z = raw_quats[idx * 4 + 3];
        real inv_norm = (real)1 / R_SQRT(x * x + y * y + z * z + w * w);
        if (inv_norm > (real)1e12) inv_norm = (real)1e12;
        real q4[4] = {w * inv_norm, x * inv_norm, y * inv_norm, z * inv_norm};
        /* already unit (up to the 1e12 clamp); quat_to_rotmat renormalises harmlessly */
        real x2 = q4[1] * q4[1], y2 = q4[2] * q4[2], z2 = q4[3] * q4[3];
        real xy = q4[1] * q4[2], xz = q4[1] * q4[3], yz = q4[2] * q4[3];
        real wx = q4[0] * q4[1], wy = q4[0] * q4[2], wz = q4[0] * q4[3];
        m3 R;
        R.c[0][0] = (real)1 - (real)2 * (y2 + z2); R.c[0][1] = (real)2 * (xy + wz); R.c[0][2] = (real)2 * (xz - wy);
        R.c[1][0] = (real)2 * (xy - wz); R.c[1][1] = (real)1 - (real)2 * (x2 + z2); R.c[1][2] = (real)2 * (yz + wx);
        R.c[2][0] = (real)2 * (xz + wy); R.c[2][1] = (real)2 * (yz - wx); R.c[2][2] = (real)1 - (real)2 * (x2 + y2);
        m3 S2;
        memset(&S2, 0, sizeof(S2));
        S2.c[0][0] = e[0]; S2.c[1][1] = e[1]; S2.c[2][2] = e[2];
        m3 RS = m3_mul(&R, &S2);
        m3 Rt = m3_transpose(&R);
        m3 cov = m3_mul(&RS, &Rt);
        v3 nz = v3_make(noise[idx * 3], noise[idx * 3 + 1], noise[idx * 3 + 2]);
        v3 tn = m3_mulv(&cov, nz);
        real opacity = (real)1 / ((real)1 + R_EXP(-(real)raw_opacities[idx]));
        real op_sigmoid = (real)1 / ((real)1 + R_EXP((real)100 * opacity - (real)0.5));
        real nf = (real)current_lr * op_sigmoid;
        means[idx * 3 + 0] = (float)((real)means[idx * 3 + 0] + nf * tn.x);
        means[idx * 3 + 1] = (float)((real)means[idx * 3 + 1] + nf * tn.y);
        means[idx * 3 + 2] = (float)((real)means[idx * 3 + 2] + nf * tn.z);
    }
    return ORC_OK;
}

ORC_API int orc_real_bytes(void) { return (int)sizeof(real); }
