/*
 * fastgs_oracle.c -- CPU restatement of the reference's "fastgs" (EWA splatting) rasterizer, SURVEY.md 8 f4.
 *
 * TEST INFRASTRUCTURE ONLY (same rule as gut_oracle.c): nothing in the product path may include, link or call
 * this file; only tests/, __graft_entry__.smoke() and bench.py's CPU legs use it, as the checker.
 *
 * What it restates (file:line relative to /root/reference/fastgs/rasterization):
 *   per-primitive set-up      include/kernels_forward.cuh:19-226   (cull, covariance, EWA projection, conic, tile bounds)
 *   SH colour and its VJP     include/kernel_utils.cuh:16-102
 *   exact tile test           include/kernel_utils.cuh:105-139     (closest point of the tile rectangle to the ellipse)
 *   depth order, tile lists   src/forward.cu:99-146                (radix sort on the depth bits, instances per tile)
 *   blend                     include/kernels_forward.cuh:357-459
 *   blend gradient            include/kernels_backward.cuh:260-448
 *   set-up gradient           include/kernels_backward.cuh:18-257
 * Constants: include/rasterization_config.h:15-30 (dilation 0.3, 1/255, 0.999, 1e-4, 16x16 tiles).
 *
 * Differences that are not observable in the outputs: the reference orders equal depths by the arrival order of an
 * atomicAdd (non-deterministic); here ties go by index.  The reference's backward walks 32-primitive buckets with
 * the blend state stored at bucket boundaries; here every pixel walks its own list front to back -- the same
 * arithmetic per (pixel, primitive) pair.
 *
 * Pinning: the reference has no test for this path; the pin is the reference's own kernels, compiled unmodified from
 * where they lie (oracle/build_ref.py -> oracle/_ref/libfastgs_ref.so): their outputs on a seeded scene, dumped on the GPU
 * by tests/test_gpu_fastgs.py::test_dump_reference_fastgs_golden, are committed as tests/golden/ref_fastgs_small.npz and
 * checked in the no-GPU suite (tests/test_oracle_fastgs.py::test_oracle_vs_reference_fastgs_golden: image 1e-4, every
 * gradient 1e-3, w2c gradient, densification statistics); on the GPU box tests/test_gpu_fastgs.py compares reference
 * kernels, this oracle and this library's kernels on the same inputs.
 *
 * Precision: -DORC_DOUBLE builds the same algorithm in float64.  Gradients are accumulated in float64 either way.
 * -DORC_SMOOTH (test only) drops the three cut-offs (tile bounds / tile test, alpha < 1/255, transmittance < 1e-4) so
 * that the forward is a smooth function of the parameters and central differences validate the backward.
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
#define R_FLOOR floor
#define R_CEIL ceil
#else
typedef float real;
#define R_SQRT sqrtf
#define R_EXP expf
#define R_LOG logf
#define R_FLOOR floorf
#define R_CEIL ceilf
#endif

#define FGO_API __attribute__((visibility("default")))

#define DILATION ((real)0.3)
#define ALPHA_MIN ((real)(1.0 / 255.0))
#define ALPHA_MIN_RCP ((real)255.0)
#define ALPHA_MAX ((real)0.999)
#define T_MIN ((real)1e-4)
#define TILE 16

typedef struct {
    int visible;
    uint32_t depth_bits;
    real mx, my;        /* screen-space centre */
    real ca, cb, cc;    /* conic (inverse 2-D covariance): ca dx^2 + 2 cb dx dy + cc dy^2 */
    real opacity;
    real col[3];        /* unclamped SH colour */
    uint32_t x0, x1, y0, y1; /* tile bounds, half open */
} Prim;

static real clampr(real v, real lo, real hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* SH colour of the view direction, degree by active_bases (1, 4, 9, 16): kernel_utils.cuh:16-40 */
static void sh_basis(int active, real x, real y, real z, real *b /* [16] */) {
    for (int i = 0; i < 16; ++i) b[i] = 0;
    b[0] = (real)0.28209479177387814;
    if (active > 1) {
        b[1] = (real)-0.48860251190291987 * y;
        b[2] = (real)0.48860251190291987 * z;
        b[3] = (real)-0.48860251190291987 * x;
    }
    if (active > 4) {
        const real xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
        b[4] = (real)1.0925484305920792 * xy;
        b[5] = (real)-1.0925484305920792 * yz;
        b[6] = (real)0.94617469575755997 * zz - (real)0.31539156525251999;
        b[7] = (real)-1.0925484305920792 * xz;
        b[8] = (real)0.54627421529603959 * xx - (real)0.54627421529603959 * yy;
        if (active > 9) {
            b[9] = (real)0.59004358992664352 * y * ((real)-3.0 * xx + yy);
            b[10] = (real)2.8906114426405538 * xy * z;
            b[11] = (real)0.45704579946446572 * y * ((real)1.0 - (real)5.0 * zz);
            b[12] = (real)0.3731763325901154 * z * ((real)5.0 * zz - (real)3.0);
            b[13] = (real)0.45704579946446572 * x * ((real)1.0 - (real)5.0 * zz);
            b[14] = (real)1.4453057213202769 * z * (xx - yy);
            b[15] = (real)0.59004358992664352 * x * (-xx + (real)3.0 * yy);
        }
    }
}

/* d basis_k / d(x, y, z) for the unit direction: the polynomial derivatives used by kernel_utils.cuh:57-88 */
static void sh_basis_grad(int active, real x, real y, real z, real (*g)[3] /* [16][3] */) {
    for (int i = 0; i < 16; ++i) g[i][0] = g[i][1] = g[i][2] = 0;
    if (active > 1) {
        g[1][1] = (real)-0.48860251190291987;
        g[2][2] = (real)0.48860251190291987;
        g[3][0] = (real)-0.48860251190291987;
    }
    if (active > 4) {
        const real c = (real)1.0925484305920792;
        g[4][0] = c * y; g[4][1] = c * x;
        g[5][1] = -c * z; g[5][2] = -c * y;
        g[6][2] = (real)1.8923493915151202 * z;
        g[7][0] = -c * z; g[7][2] = -c * x;
        g[8][0] = c * x; g[8][1] = -c * y;
        if (active > 9) {
            const real xx = x * x, yy = y * y, zz = z * z, xy = x * y, xz = x * z, yz = y * z;
            g[9][0] = (real)-3.5402615395598609 * xy;
            g[9][1] = (real)-1.7701307697799304 * xx + (real)1.7701307697799304 * yy;
            g[10][0] = (real)2.8906114426405538 * yz; g[10][1] = (real)2.8906114426405538 * xz;
            g[10][2] = (real)2.8906114426405538 * xy;
            g[11][1] = (real)0.45704579946446572 - (real)2.2852289973223288 * zz;
            g[11][2] = (real)-4.5704579946446566 * yz;
            g[12][2] = (real)5.597644988851731 * zz - (real)1.1195289977703462;
            g[13][0] = (real)0.45704579946446572 - (real)2.2852289973223288 * zz;
            g[13][2] = (real)-4.5704579946446566 * xz;
            g[14][0] = (real)2.8906114426405538 * xz; g[14][1] = (real)-2.8906114426405538 * yz;
            g[14][2] = (real)1.4453057213202769 * xx - (real)1.4453057213202769 * yy;
            g[15][0] = (real)-1.7701307697799304 * xx + (real)1.7701307697799304 * yy;
            g[15][1] = (real)3.5402615395598609 * xy;
        }
    }
}

/* kernel_utils.cuh:105-139: does the ellipse {sigma/2 <= thr} reach the tile's pixel-centre rectangle?  `mx, my` are
 * the centre shifted by -0.5 (pixel centres become integers). */
static int tile_contributes(real mx, real my, real ca, real cb, real cc, uint32_t tx, uint32_t ty, real thr) {
#ifdef ORC_SMOOTH
    (void)mx; (void)my; (void)ca; (void)cb; (void)cc; (void)tx; (void)ty; (void)thr;
    return 1;
#endif
    const real lo_x = (real)(tx * TILE), lo_y = (real)(ty * TILE);
    const real hi_x = (real)((tx + 1) * TILE - 1), hi_y = (real)((ty + 1) * TILE - 1);
    const int left = lo_x > mx, right = mx > hi_x, above = lo_y > my, below = my > hi_y;
    const int out_x = left + right, out_y = above + below;
    if (out_x + out_y == 0) return 1;
    /* nearest corner, then slide along the two edges that leave it */
    const real cx = left ? lo_x : hi_x, cy = above ? lo_y : hi_y;
    const real dfx = mx - cx, dfy = my - cy;
    const real ex = (lo_x - mx) < 0 ? (real)-(TILE - 1) : (real)(TILE - 1);
    const real ey = (lo_y - my) < 0 ? (real)-(TILE - 1) : (real)(TILE - 1);
    real tx_ = (ex * ca * dfx + ex * cb * dfy) / (ex * ca * ex);
    real ty_ = (ey * cb * dfx + ey * cc * dfy) / (ey * cc * ey);
    tx_ = (real)out_y * clampr(tx_, 0, 1);
    ty_ = (real)out_x * clampr(ty_, 0, 1);
    const real px = cx + tx_ * ex, py = cy + ty_ * ey;
    const real dx = mx - px, dy = my - py;
    const real power = (real)0.5 * (ca * dx * dx + cc * dy * dy) + cb * dx * dy;
    return power <= thr;
}

typedef struct {
    real R[3][3];
    real var[3];
    real cov[6]; /* m11 m12 m13 m22 m23 m33 */
    real qn2;
} Cov3;

/* kernels_forward.cuh:78-104: Sigma = R diag(exp(2 s)) R^T with R from the un-normalised quaternion (w, x, y, z) */
static void cov3_build(const float *s, const float *q, Cov3 *c) {
    for (int i = 0; i < 3; ++i) c->var[i] = R_EXP((real)2.0 * (real)s[i]);
    const real w = q[0], x = q[1], y = q[2], z = q[3];
    c->qn2 = w * w + x * x + y * y + z * z;
    const real n = c->qn2;
    const real xx = (real)2 * x * x / n, yy = (real)2 * y * y / n, zz = (real)2 * z * z / n;
    const real xy = (real)2 * x * y / n, xz = (real)2 * x * z / n, yz = (real)2 * y * z / n;
    const real wx = (real)2 * w * x / n, wy = (real)2 * w * y / n, wz = (real)2 * w * z / n;
    c->R[0][0] = (real)1 - (yy + zz); c->R[0][1] = xy - wz; c->R[0][2] = wy + xz;
    c->R[1][0] = wz + xy; c->R[1][1] = (real)1 - (xx + zz); c->R[1][2] = yz - wx;
    c->R[2][0] = xz - wy; c->R[2][1] = wx + yz; c->R[2][2] = (real)1 - (xx + yy);
    int k = 0;
    for (int i = 0; i < 3; ++i)
        for (int j = i; j < 3; ++j) {
            real acc = 0;
            for (int m = 0; m < 3; ++m) acc += c->R[i][m] * c->var[m] * c->R[j][m];
            c->cov[k++] = acc;
        }
}

typedef struct {
    real depth, x, y;         /* camera-space depth, normalised image coordinates */
    real tx, ty;              /* x, y clamped to the 15 % guard band */
    real j11, j13, j22, j23;
    real r1[3], r2[3];        /* rows of J W */
    real c1[3], c2[3];        /* rows of J W Sigma */
    real a, b, c;             /* dilated 2-D covariance */
} Ewa;

static void ewa_project(const float *mean, const float *w2c, const Cov3 *cv, real W, real H, real fx, real fy, real cx,
                        real cy, Ewa *e) {
    const float *r1 = w2c, *r2 = w2c + 4, *r3 = w2c + 8;
    e->depth = (real)r3[0] * mean[0] + (real)r3[1] * mean[1] + (real)r3[2] * mean[2] + (real)r3[3];
    e->x = ((real)r1[0] * mean[0] + (real)r1[1] * mean[1] + (real)r1[2] * mean[2] + (real)r1[3]) / e->depth;
    e->y = ((real)r2[0] * mean[0] + (real)r2[1] * mean[1] + (real)r2[2] * mean[2] + (real)r2[3]) / e->depth;
    e->tx = clampr(e->x, ((real)-0.15 * W - cx) / fx, ((real)1.15 * W - cx) / fx);
    e->ty = clampr(e->y, ((real)-0.15 * H - cy) / fy, ((real)1.15 * H - cy) / fy);
    e->j11 = fx / e->depth; e->j13 = -e->j11 * e->tx;
    e->j22 = fy / e->depth; e->j23 = -e->j22 * e->ty;
    for (int k = 0; k < 3; ++k) {
        e->r1[k] = e->j11 * (real)r1[k] + e->j13 * (real)r3[k];
        e->r2[k] = e->j22 * (real)r2[k] + e->j23 * (real)r3[k];
    }
    const real *S = cv->cov;
    const real M[3][3] = {{S[0], S[1], S[2]}, {S[1], S[3], S[4]}, {S[2], S[4], S[5]}};
    for (int k = 0; k < 3; ++k) {
        e->c1[k] = e->r1[0] * M[0][k] + e->r1[1] * M[1][k] + e->r1[2] * M[2][k];
        e->c2[k] = e->r2[0] * M[0][k] + e->r2[1] * M[1][k] + e->r2[2] * M[2][k];
    }
    e->a = e->c1[0] * e->r1[0] + e->c1[1] * e->r1[1] + e->c1[2] * e->r1[2] + DILATION;
    e->b = e->c1[0] * e->r2[0] + e->c1[1] * e->r2[1] + e->c1[2] * e->r2[2];
    e->c = e->c2[0] * e->r2[0] + e->c2[1] * e->r2[1] + e->c2[2] * e->r2[2] + DILATION;
}

static uint32_t tile_lo(real v, uint32_t lim) {
    const long t = (long)R_FLOOR(v / (real)TILE);
    const long c = t < 0 ? 0 : t;
    return (uint32_t)(c > (long)lim ? (long)lim : c);
}
static uint32_t tile_hi(real v, uint32_t lim) {
    const long t = (long)R_CEIL(v / (real)TILE);
    const long c = t < 0 ? 0 : t;
    return (uint32_t)(c > (long)lim ? (long)lim : c);
}

typedef struct { uint32_t key, idx; } SortRec;
static int cmp_sort(const void *a, const void *b) {
    const SortRec *x = (const SortRec *)a, *y = (const SortRec *)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx ? 1 : 0);
}

/*
 * Forward, and when grad_image != NULL the backward as well.
 *   means [n,3], scales_raw [n,3], rotations_raw [n,4] (w,x,y,z), opacities_raw [n], sh0 [n,3], shN [n,total_rest,3]
 *   w2c [4,4] row-major, cam_position [3]
 *   image [3,H,W], alpha [H,W], n_touched [n] (tiles per primitive; 0 = culled), n_instances (sum)
 *   grad_image [3,H,W], grad_alpha [H,W]
 *   g_* : float64 gradients (caller-zeroed not required), g_w2c [4,4] or NULL, densification [2,n] float or NULL (+=)
 */
FGO_API int fgo_render(uint32_t n, const float *means, const float *scales_raw, const float *rotations_raw,
                       const float *opacities_raw, const float *sh0, const float *shN, uint32_t total_rest,
                       uint32_t active_bases, const float *w2c, const float *cam_position, uint32_t W, uint32_t H,
                       float fx_, float fy_, float cx_, float cy_, float near_, float far_, float *image, float *alpha,
                       int32_t *n_touched, int64_t *n_instances, const float *grad_image, const float *grad_alpha,
                       double *g_means, double *g_scales, double *g_rot, double *g_opac, double *g_sh0, double *g_shN,
                       double *g_w2c, float *densification) {
    const real fx = fx_, fy = fy_, cx = cx_, cy = cy_;
    const uint32_t gw = (W + TILE - 1) / TILE, gh = (H + TILE - 1) / TILE, n_tiles = gw * gh;
    Prim *P = (Prim *)calloc(n ? n : 1, sizeof(Prim));
    SortRec *order = (SortRec *)malloc((n ? n : 1) * sizeof(SortRec));
    uint32_t n_vis = 0;
    int64_t total = 0;

    for (uint32_t i = 0; i < n; ++i) {
        Prim *p = &P[i];
        n_touched[i] = 0;
        const float *mean = means + 3 * (size_t)i;
        Cov3 cv;
        Ewa e;
        cov3_build(scales_raw + 3 * (size_t)i, rotations_raw + 4 * (size_t)i, &cv);
        ewa_project(mean, w2c, &cv, (real)W, (real)H, fx, fy, cx, cy, &e);
        if (e.depth < (real)near_ || e.depth > (real)far_) continue;
        const real opacity = (real)1 / ((real)1 + R_EXP(-(real)opacities_raw[i]));
        if (opacity < ALPHA_MIN) continue;
        if (cv.qn2 < (real)1e-8) continue;
        const real det = e.a * e.c - e.b * e.b;
        if (det < (real)1e-8) continue;
        p->ca = e.c / det; p->cb = -e.b / det; p->cc = e.a / det;
        p->mx = e.x * fx + cx; p->my = e.y * fy + cy;
        p->opacity = opacity;
        const real thr = R_LOG(opacity * ALPHA_MIN_RCP);
        const real fac = R_SQRT((real)2 * thr);
        real ext_x = fac * R_SQRT(e.a) - (real)0.5, ext_y = fac * R_SQRT(e.c) - (real)0.5;
        if (ext_x < 0) ext_x = 0;
        if (ext_y < 0) ext_y = 0;
        p->x0 = tile_lo(p->mx - ext_x, gw); p->x1 = tile_hi(p->mx + ext_x, gw);
        p->y0 = tile_lo(p->my - ext_y, gh); p->y1 = tile_hi(p->my + ext_y, gh);
#ifdef ORC_SMOOTH
        p->x0 = 0; p->x1 = gw; p->y0 = 0; p->y1 = gh;
#endif
        if ((p->x1 - p->x0) * (p->y1 - p->y0) == 0) continue;
        uint32_t cnt = 0;
        for (uint32_t ty = p->y0; ty < p->y1; ++ty)
            for (uint32_t tx = p->x0; tx < p->x1; ++tx)
                cnt += (uint32_t)tile_contributes(p->mx - (real)0.5, p->my - (real)0.5, p->ca, p->cb, p->cc, tx, ty, thr);
        if (cnt == 0) continue;
        /* colour */
        real dx = (real)mean[0] - cam_position[0], dy = (real)mean[1] - cam_position[1], dz = (real)mean[2] - cam_position[2];
        const real inv = (real)1 / R_SQRT(dx * dx + dy * dy + dz * dz);
        real b[16];
        sh_basis((int)active_bases, dx * inv, dy * inv, dz * inv, b);
        for (int ch = 0; ch < 3; ++ch) {
            real acc = (real)0.5 + b[0] * (real)sh0[3 * (size_t)i + ch];
            for (uint32_t k = 1; k < active_bases; ++k) acc += b[k] * (real)shN[((size_t)i * total_rest + (k - 1)) * 3 + ch];
            p->col[ch] = acc;
        }
        p->visible = 1;
        n_touched[i] = (int32_t)cnt;
        total += cnt;
        float df = (float)e.depth;
        memcpy(&p->depth_bits, &df, 4);
        order[n_vis].key = p->depth_bits; order[n_vis].idx = i;
        ++n_vis;
    }
    if (n_instances) *n_instances = total;
    qsort(order, n_vis, sizeof(SortRec), cmp_sort);

    /* per-tile lists in depth order */
    uint32_t *t_cnt = (uint32_t *)calloc(n_tiles + 1, sizeof(uint32_t));
    for (uint32_t s = 0; s < n_vis; ++s) {
        const Prim *p = &P[order[s].idx];
        const real thr = R_LOG(p->opacity * ALPHA_MIN_RCP);
        for (uint32_t ty = p->y0; ty < p->y1; ++ty)
            for (uint32_t tx = p->x0; tx < p->x1; ++tx)
                if (tile_contributes(p->mx - (real)0.5, p->my - (real)0.5, p->ca, p->cb, p->cc, tx, ty, thr)) ++t_cnt[ty * gw + tx + 1];
    }
    for (uint32_t t = 0; t < n_tiles; ++t) t_cnt[t + 1] += t_cnt[t];
    uint32_t *t_fill = (uint32_t *)malloc((n_tiles ? n_tiles : 1) * sizeof(uint32_t));
    memcpy(t_fill, t_cnt, n_tiles * sizeof(uint32_t));
    uint32_t *lists = (uint32_t *)malloc((size_t)(total ? total : 1) * sizeof(uint32_t));
    for (uint32_t s = 0; s < n_vis; ++s) {
        const Prim *p = &P[order[s].idx];
        const real thr = R_LOG(p->opacity * ALPHA_MIN_RCP);
        for (uint32_t ty = p->y0; ty < p->y1; ++ty)
            for (uint32_t tx = p->x0; tx < p->x1; ++tx)
                if (tile_contributes(p->mx - (real)0.5, p->my - (real)0.5, p->ca, p->cb, p->cc, tx, ty, thr))
                    lists[t_fill[ty * gw + tx]++] = order[s].idx;
    }

    /* per-primitive accumulators of the blend gradient */
    const int bwd = grad_image != NULL;
    double *acc = bwd ? (double *)calloc((size_t)(n ? n : 1) * 9, sizeof(double)) : NULL; /* m2d.xy conic.abc opac col.rgb */
    const size_t HW = (size_t)W * H;

#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t t = 0; t < (int64_t)n_tiles; ++t) {
        const uint32_t tx = (uint32_t)t % gw, ty = (uint32_t)t / gw;
        const uint32_t lo = t_cnt[t], hi = t_cnt[t + 1];
        for (uint32_t py = ty * TILE; py < (ty + 1) * TILE && py < H; ++py)
            for (uint32_t px = tx * TILE; px < (tx + 1) * TILE && px < W; ++px) {
                const real fxp = (real)px + (real)0.5, fyp = (real)py + (real)0.5;
                real T = 1, C[3] = {0, 0, 0};
                uint32_t last = 0;
                for (uint32_t j = lo; j < hi; ++j) {
                    const Prim *p = &P[lists[j]];
                    const real dx = p->mx - fxp, dy = p->my - fyp;
                    const real s2 = (real)0.5 * (p->ca * dx * dx + p->cc * dy * dy) + p->cb * dx * dy;
                    if (s2 < 0) continue;
                    real a = p->opacity * R_EXP(-s2);
                    if (a > ALPHA_MAX) a = ALPHA_MAX;
#ifndef ORC_SMOOTH
                    if (a < ALPHA_MIN) continue;
#endif
                    const real nT = T * ((real)1 - a);
#ifndef ORC_SMOOTH
                    if (nT < T_MIN) break;
#endif
                    for (int ch = 0; ch < 3; ++ch) C[ch] += T * a * (p->col[ch] > 0 ? p->col[ch] : 0);
                    T = nT;
                    last = j - lo + 1;
                }
                const size_t pix = (size_t)py * W + px;
                image[pix] = (float)C[0]; image[HW + pix] = (float)C[1]; image[2 * HW + pix] = (float)C[2];
                alpha[pix] = (float)((real)1 - T);
                if (!bwd) continue;
                /* kernels_backward.cuh:391-430, front to back */
                const real gc[3] = {grad_image[pix], grad_image[HW + pix], grad_image[2 * HW + pix]};
                const real ga = (real)grad_alpha[pix] * T; /* grad_alpha (1 - alpha_pixel) */
                real Tr = 1, after[3] = {C[0], C[1], C[2]};
                for (uint32_t j = lo; j < lo + last; ++j) {
                    const uint32_t id = lists[j];
                    const Prim *p = &P[id];
                    const real dx = p->mx - fxp, dy = p->my - fyp;
                    const real s2 = (real)0.5 * (p->ca * dx * dx + p->cc * dy * dy) + p->cb * dx * dy;
                    if (s2 < 0) continue;
                    real a = p->opacity * R_EXP(-s2);
                    if (a > ALPHA_MAX) a = ALPHA_MAX;
#ifndef ORC_SMOOTH
                    if (a < ALPHA_MIN) continue;
#endif
                    const real om = (real)1 - a, w = Tr * a;
                    real col[3], dA = 0;
                    double dcol[3];
                    for (int ch = 0; ch < 3; ++ch) {
                        col[ch] = p->col[ch] > 0 ? p->col[ch] : 0;
                        dcol[ch] = p->col[ch] >= 0 ? (double)(w * gc[ch]) : 0.0;
                        after[ch] -= w * col[ch];
                        dA += (Tr * col[ch] - after[ch] / om) * gc[ch];
                    }
                    dA += ga / om;
                    const real h = -a * dA;
                    double *A = acc + (size_t)id * 9;
                    const double v[9] = {(double)(h * (p->ca * dx + p->cb * dy)), (double)(h * (p->cb * dx + p->cc * dy)),
                                         (double)((real)0.5 * h * dx * dx), (double)((real)0.5 * h * dx * dy),
                                         (double)((real)0.5 * h * dy * dy), (double)(a * dA), dcol[0], dcol[1], dcol[2]};
                    for (int k = 0; k < 9; ++k) {
#pragma omp atomic
                        A[k] += v[k];
                    }
                    Tr *= om;
                }
            }
    }

    if (bwd) {
        if (g_w2c) memset(g_w2c, 0, 16 * sizeof(double));
        for (uint32_t i = 0; i < n; ++i) {
            double *gm = g_means + 3 * (size_t)i, *gs = g_scales + 3 * (size_t)i, *gq = g_rot + 4 * (size_t)i;
            gm[0] = gm[1] = gm[2] = gs[0] = gs[1] = gs[2] = gq[0] = gq[1] = gq[2] = gq[3] = 0;
            g_opac[i] = 0;
            g_sh0[3 * (size_t)i] = g_sh0[3 * (size_t)i + 1] = g_sh0[3 * (size_t)i + 2] = 0;
            for (uint32_t k = 0; k < total_rest * 3; ++k) g_shN[(size_t)i * total_rest * 3 + k] = 0;
            if (!P[i].visible) continue;
            const Prim *p = &P[i];
            const double *A = acc + (size_t)i * 9;
            const float *mean = means + 3 * (size_t)i;
            g_opac[i] = A[5] * (1.0 - (double)p->opacity);
            /* SH: kernel_utils.cuh:42-102 */
            const real gcol[3] = {(real)A[6], (real)A[7], (real)A[8]};
            real ddir[3] = {0, 0, 0};
            {
                const real rx = (real)mean[0] - cam_position[0], ry = (real)mean[1] - cam_position[1], rz = (real)mean[2] - cam_position[2];
                const real n2 = rx * rx + ry * ry + rz * rz, inv = (real)1 / R_SQRT(n2);
                const real x = rx * inv, y = ry * inv, z = rz * inv;
                real b[16], g[16][3];
                sh_basis((int)active_bases, x, y, z, b);
                sh_basis_grad((int)active_bases, x, y, z, g);
                for (int ch = 0; ch < 3; ++ch) g_sh0[3 * (size_t)i + ch] = (double)(b[0] * gcol[ch]);
                real gd[3] = {0, 0, 0};
                for (uint32_t k = 1; k < active_bases; ++k) {
                    real dotc = 0;
                    for (int ch = 0; ch < 3; ++ch) {
                        g_shN[((size_t)i * total_rest + (k - 1)) * 3 + ch] = (double)(b[k] * gcol[ch]);
                        dotc += (real)shN[((size_t)i * total_rest + (k - 1)) * 3 + ch] * gcol[ch];
                    }
                    for (int a = 0; a < 3; ++a) gd[a] += g[k][a] * dotc;
                }
                if (active_bases > 1) {
                    /* through the normalisation: (|r|^2 I - r r^T) gd / |r|^3 */
                    const real dotrg = rx * gd[0] + ry * gd[1] + rz * gd[2];
                    const real s = (real)1 / (n2 * R_SQRT(n2));
                    ddir[0] = (n2 * gd[0] - rx * dotrg) * s;
                    ddir[1] = (n2 * gd[1] - ry * dotrg) * s;
                    ddir[2] = (n2 * gd[2] - rz * dotrg) * s;
                }
            }
            Cov3 cv;
            Ewa e;
            cov3_build(scales_raw + 3 * (size_t)i, rotations_raw + 4 * (size_t)i, &cv);
            ewa_project(mean, w2c, &cv, (real)W, (real)H, fx, fy, cx, cy, &e);
            const real a = e.a, b = e.b, c = e.c;
            const real det = a * c - b * b, idet2 = ((real)1 / det) * ((real)1 / det);
            /* accumulated conic gradient: gA, (1/2) gB, gC  (kernels_backward.cuh:120-130) */
            const real gA = (real)A[2], gBh = (real)A[3], gC = (real)A[4];
            const real dca = idet2 * ((real)2 * b * c * gBh - c * c * gA - b * b * gC);
            const real dcb = idet2 * (b * c * gA - (a * c + b * b) * gBh + a * b * gC); /* half of dL/db */
            const real dcc = idet2 * ((real)2 * a * b * gBh - b * b * gA - a * a * gC);
            /* Sigma gradient (symmetric, upper triangle holds the sum of both halves) */
            real dS[3][3];
            for (int r = 0; r < 3; ++r)
                for (int s = 0; s < 3; ++s)
                    dS[r][s] = e.r1[r] * e.r1[s] * dca + (e.r1[r] * e.r2[s] + e.r1[s] * e.r2[r]) * dcb + e.r2[r] * e.r2[s] * dcc;
            real dr1[3], dr2[3];
            for (int k = 0; k < 3; ++k) {
                dr1[k] = (real)2 * (e.c1[k] * dca + e.c2[k] * dcb);
                dr2[k] = (real)2 * (e.c1[k] * dcb + e.c2[k] * dcc);
            }
            const float *w1 = w2c, *w2 = w2c + 4, *w3 = w2c + 8;
            real dj11 = 0, dj22 = 0, dj13 = 0, dj23 = 0;
            for (int k = 0; k < 3; ++k) {
                dj11 += (real)w1[k] * dr1[k]; dj22 += (real)w2[k] * dr2[k];
                dj13 += (real)w3[k] * dr1[k]; dj23 += (real)w3[k] * dr2[k];
            }
            const real h1 = dj11 - (real)2 * e.tx * dj13, h2 = dj22 - (real)2 * e.ty * dj23;
            const real gmx = (real)A[0], gmy = (real)A[1];
            const real dcam[3] = {e.j11 * (gmx - dj13 / e.depth), e.j22 * (gmy - dj23 / e.depth),
                                  -e.j11 * (e.x * gmx + h1 / e.depth) - e.j22 * (e.y * gmy + h2 / e.depth)};
            if (g_w2c)
                for (int r = 0; r < 3; ++r) {
                    for (int k = 0; k < 3; ++k) g_w2c[r * 4 + k] += (double)(dcam[r] * (real)mean[k]);
                    g_w2c[r * 4 + 3] += (double)dcam[r];
                }
            for (int k = 0; k < 3; ++k)
                gm[k] = (double)((real)w1[k] * dcam[0] + (real)w2[k] * dcam[1] + (real)w3[k] * dcam[2] + ddir[k]);
            /* Sigma = R V R^T:  dL/dV_m = R[:,m]^T dS R[:,m];  dL/dR = 2 dS R V */
            real dR[3][3];
            for (int m = 0; m < 3; ++m) {
                real q = 0;
                for (int r = 0; r < 3; ++r)
                    for (int s = 0; s < 3; ++s) q += cv.R[r][m] * dS[r][s] * cv.R[s][m];
                gs[m] = (double)((real)2 * cv.var[m] * q);
                for (int r = 0; r < 3; ++r) {
                    real v = 0;
                    for (int s = 0; s < 3; ++s) v += dS[r][s] * cv.R[s][m];
                    dR[r][m] = (real)2 * v * cv.var[m];
                }
            }
            /* R(q / |q|): the nine products 2 q_i q_j / |q|^2 (kernels_backward.cuh:228-243) */
            const float *q = rotations_raw + 4 * (size_t)i;
            const real qw = q[0], qx = q[1], qy = q[2], qz = q[3], nn = cv.qn2;
            const real dxx = -dR[1][1] - dR[2][2], dyy = -dR[0][0] - dR[2][2], dzz = -dR[0][0] - dR[1][1];
            const real dxy = dR[0][1] + dR[1][0], dxz = dR[0][2] + dR[2][0], dyz = dR[1][2] + dR[2][1];
            const real dwx = dR[2][1] - dR[1][2], dwy = dR[0][2] - dR[2][0], dwz = dR[1][0] - dR[0][1];
            const real pxx = (real)2 * qx * qx / nn, pyy = (real)2 * qy * qy / nn, pzz = (real)2 * qz * qz / nn;
            const real pxy = (real)2 * qx * qy / nn, pxz = (real)2 * qx * qz / nn, pyz = (real)2 * qy * qz / nn;
            const real pwx = (real)2 * qw * qx / nn, pwy = (real)2 * qw * qy / nn, pwz = (real)2 * qw * qz / nn;
            const real hn = pxx * dxx + pyy * dyy + pzz * dzz + pxy * dxy + pxz * dxz + pyz * dyz + pwx * dwx + pwy * dwy + pwz * dwz;
            gq[0] = (double)((real)2 * (qx * dwx + qy * dwy + qz * dwz - qw * hn) / nn);
            gq[1] = (double)((real)2 * ((real)2 * qx * dxx + qy * dxy + qz * dxz + qw * dwx - qx * hn) / nn);
            gq[2] = (double)((real)2 * ((real)2 * qy * dyy + qx * dxy + qz * dyz + qw * dwy - qy * hn) / nn);
            gq[3] = (double)((real)2 * ((real)2 * qz * dzz + qx * dxz + qy * dyz + qw * dwz - qz * hn) / nn);
            if (densification) {
                densification[i] += 1.0f;
                const real sx = gmx * (real)0.5 * (real)W, sy = gmy * (real)0.5 * (real)H;
                densification[(size_t)n + i] += (float)R_SQRT(sx * sx + sy * sy);
            }
        }
    }
    free(acc); free(lists); free(t_fill); free(t_cnt); free(order); free(P);
    return 0;
}
