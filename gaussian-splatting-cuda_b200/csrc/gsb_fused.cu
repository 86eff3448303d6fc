// gsb_fused.cu -- SURVEY.md 8(f1): the L3 glue of the hot path folded into two kernels over the RAW SplatData
// tensors (means, sh0, shN, log-scales, unnormalised quaternions, logit opacities).
//
// What the reference does around the gsplat:: operators every step with ~10 torch kernels and three host
// synchronisations (activations  src/core/splat_data.cpp:267-286; cat(sh0, shN), dirs, masks, inverse(viewmat),
// clamp_min(+0.5)  src/training/rasterization/rasterizer.cpp:250-266; their autograd backward) becomes:
//
//   fused_front_kernel   one thread per Gaussian: exp / sigmoid activations -> unscented-transform projection
//                        (gsb_projection.cuh, same arithmetic as the a1 operator) -> SH colour of the view
//                        direction straight from sh0 / shN (no concatenated copy) + 0.5, clamp -> the 64-byte
//                        blend record (gsb_raster.cuh).  Writes radii / means2d / depths for the intersect stage,
//                        the record, and zeroes the backward's moment row.
//   fused_back_kernel    one thread per Gaussian: moments -> gradients of the activated parameters
//                        (finalize_gaussian) -> chained through exp / sigmoid / normalise to the RAW parameters,
//                        clamp mask recomputed, SH backward written directly into the sh0 / shN gradient
//                        layouts, the direction gradient added to the position gradient.
//
// Per Gaussian the front reads 236 B and writes 84 (+64) B, the back reads ~364 B and writes 236 B: both are
// HBM streaming kernels.  The shN rows (180 B at K = 16, 4-byte aligned only) are moved per 128-Gaussian slab with
// one TMA bulk copy each way (23 KB per 128-Gaussian slab, 16-byte aligned as a whole) and read from shared memory at an odd word stride.
// Compiled with -fmad=false like gsb_projection.cu: the radii must be the a1 operator's, bit for bit.
#include "gsb_projection.cuh"
#include "gsb_raster.cuh"
#include "gsb_sh.cuh"

namespace gsb {

constexpr int kFusedThreads = 128; // 110-128 registers per thread: four 128-thread CTAs per SM (five would spill)

struct FusedParams {
    uint32_t N, K; // K = SH coefficients per Gaussian including sh0
    const float *means, *sh0, *shN, *scaling_raw, *rotation_raw, *opacity_raw;
    float scaling_modifier;
    const float *viewmat, *Ks; // one camera
    int32_t camera_model;
    const float *radial, *tangential, *thin_prism;
    int32_t n_radial, n_tangential, n_thin_prism;
    ProjConsts pk;
    // front outputs
    int32_t *radii;
    float *means2d, *depths;
    GaussRec *recs;
    float *moments; // front: zeroed when non-null; back: input
    // back outputs
    float *v_means, *v_sh0, *v_shN, *v_scaling, *v_rotation, *v_opacity;
};

struct FusedCam {
    CamModel cm;
    CamConst cc;
    ProjPose pp;
    float campos[3];
};

__device__ inline void fused_cam_build(const FusedParams &p, FusedCam &c) {
    cam_model_build(c.cm, p.camera_model, p.pk.W, p.pk.H, p.Ks, p.radial, p.n_radial, p.tangential, p.n_tangential,
                    p.thin_prism, p.n_thin_prism);
    cam_const_from(p.viewmat, p.Ks, c.cc);
    c.pp = proj_pose_from_viewmat(p.viewmat);
    // camera centre = inverse(viewmat)[:3, 3] (rasterizer.cpp:250-251) = -R^-1 t, in double from the float matrix
    M3<double> R;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R.m[i][j] = (double)p.viewmat[i * 4 + j];
    const M3<double> Ri = inverse3(R);
    const V3<double> t = {(double)p.viewmat[3], (double)p.viewmat[7], (double)p.viewmat[11]};
    const V3<double> cpos = mulv(Ri, t);
    c.campos[0] = (float)(-cpos.x); c.campos[1] = (float)(-cpos.y); c.campos[2] = (float)(-cpos.z);
}

// activations of splat_data.cpp:267-286 (torch.exp, torch.sigmoid in float)
__device__ __forceinline__ float act_scale(float raw, float modifier) { return expf(raw) * modifier; }
__device__ __forceinline__ float act_opacity(float raw) { return 1.0f / (1.0f + expf(-raw)); }

// Stages the slab's shN rows in shared memory (one bulk copy when the slab is 16-byte aligned as a whole).
__device__ __forceinline__ void stage_rows_in(float *s_rows, const float *g_rows, uint32_t n_floats, uint64_t *bar,
                                              bool bulk) {
    if (n_floats == 0) return;
    if (bulk) {
        if (threadIdx.x == 0) {
            mbar_init(bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(bar, n_floats * 4);
            // cp.async.bulk moves at most 2^20-ish bytes per instruction comfortably; a slab is <= 74 KB
            bulk_g2s(s_rows, g_rows, n_floats * 4, bar);
        }
    } else {
        for (uint32_t i = threadIdx.x; i < n_floats; i += kFusedThreads) s_rows[i] = g_rows[i];
        __syncthreads();
    }
}

// kColour: the record's channels are the SH colour (RGB, and RGB_D / RGB_ED, whose fourth channel the blend reads from
// `depths`); otherwise the camera-space depth alone (D / ED: one channel, no SH evaluation).
template <int DEG, bool kColour>
__device__ __forceinline__ void fused_front_impl(const FusedParams &p) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    extern __shared__ __align__(128) float s_rows[]; // [kFusedThreads][(K-1)*3]
    __shared__ FusedCam s_cam;
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t tid = threadIdx.x;
    const uint32_t g0 = blockIdx.x * kFusedThreads;
    const uint32_t cnt = min((uint32_t)kFusedThreads, p.N - g0);
    const uint32_t g = g0 + tid;
    const uint32_t rowf = (p.K - 1) * 3; // floats per shN row
    const float *g_rows = p.shN ? p.shN + (size_t)g0 * rowf : nullptr;
    const bool want_rows = (DEG >= 1) && rowf > 0 && g_rows != nullptr;
    const uint32_t n_floats = want_rows ? cnt * rowf : 0u;
    const bool bulk = want_rows && ((reinterpret_cast<uintptr_t>(g_rows) & 15) == 0) && ((n_floats & 3u) == 0);

    if (tid == 0) fused_cam_build(p, s_cam);
    stage_rows_in(s_rows, g_rows, n_floats, &s_bar, bulk);
    __syncthreads();

    bool keep = false;
    ProjResult pr;
    float mean[3] = {0.f, 0.f, 0.f}, quat[4] = {1.f, 0.f, 0.f, 0.f}, scale[3] = {1.f, 1.f, 1.f};
    float opac = 0.f;
    if (tid < cnt) {
        mean[0] = p.means[(size_t)g * 3]; mean[1] = p.means[(size_t)g * 3 + 1]; mean[2] = p.means[(size_t)g * 3 + 2];
        const float4 q = reinterpret_cast<const float4 *>(p.rotation_raw)[g];
        quat[0] = q.x; quat[1] = q.y; quat[2] = q.z; quat[3] = q.w;
        scale[0] = act_scale(p.scaling_raw[(size_t)g * 3], p.scaling_modifier);
        scale[1] = act_scale(p.scaling_raw[(size_t)g * 3 + 1], p.scaling_modifier);
        scale[2] = act_scale(p.scaling_raw[(size_t)g * 3 + 2], p.scaling_modifier);
        opac = act_opacity(p.opacity_raw[g]);
        const V3<float> m = {mean[0], mean[1], mean[2]};
        pr = project_gaussian<false>(p.pk, s_cam.cm, s_cam.pp, m, scale, quat[0], quat[1], quat[2], quat[3], true, opac);
        keep = pr.keep;
        reinterpret_cast<int2 *>(p.radii)[g] = make_int2(pr.rx, pr.ry);
        reinterpret_cast<float2 *>(p.means2d)[g] = make_float2(pr.mx, pr.my);
        p.depths[g] = pr.depth;
        if (p.moments) {
            float4 *m4 = reinterpret_cast<float4 *>(p.moments + (size_t)g * kMomFloats);
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            m4[0] = z; m4[1] = z; m4[2] = z; m4[3] = z;
        }
    }
    if (bulk) mbar_wait(&s_bar, 0);
    if (!keep) return;
    if constexpr (!kColour) {
        const float col[3] = {pr.depth, 0.f, 0.f};
        float4 v0, v1, v2, v3;
        make_record(s_cam.cc, mean, quat, scale, opac, col, (int32_t)g, v0, v1, v2, v3);
        float4 *dst = reinterpret_cast<float4 *>(p.recs + g);
        dst[0] = v0; dst[1] = v1; dst[2] = v2; dst[3] = v3;
        return;
    }

    // view-dependent colour (SphericalHarmonicsCUDA.cu:374-481 on dirs = mean - campos; +0.5, clamp: rasterizer.cpp:266)
    float b[NB];
    float x = mean[0] - s_cam.campos[0], y = mean[1] - s_cam.campos[1], z = mean[2] - s_cam.campos[2];
    if constexpr (DEG >= 1) {
        const float inorm = rsqrtf(x * x + y * y + z * z);
        x *= inorm; y *= inorm; z *= inorm;
    }
    sh_basis<DEG>(x, y, z, b);
    float col[3];
    col[0] = b[0] * p.sh0[(size_t)g * 3]; col[1] = b[0] * p.sh0[(size_t)g * 3 + 1]; col[2] = b[0] * p.sh0[(size_t)g * 3 + 2];
    if constexpr (DEG >= 1) {
        const float *row = s_rows + (size_t)tid * rowf;
#pragma unroll
        for (int k = 1; k < NB; ++k) {
            col[0] += b[k] * row[(k - 1) * 3];
            col[1] += b[k] * row[(k - 1) * 3 + 1];
            col[2] += b[k] * row[(k - 1) * 3 + 2];
        }
    }
    col[0] = fmaxf(col[0] + 0.5f, 0.f); col[1] = fmaxf(col[1] + 0.5f, 0.f); col[2] = fmaxf(col[2] + 0.5f, 0.f);

    float4 v0, v1, v2, v3;
    make_record(s_cam.cc, mean, quat, scale, opac, col, (int32_t)g, v0, v1, v2, v3);
    float4 *dst = reinterpret_cast<float4 *>(p.recs + g);
    dst[0] = v0; dst[1] = v1; dst[2] = v2; dst[3] = v3;
}
template <int DEG>
__global__ void __launch_bounds__(kFusedThreads, 5) fused_front_kernel(const FusedParams p) {
    fused_front_impl<DEG, true>(p);
}
__global__ void __launch_bounds__(kFusedThreads, 5) fused_front_depth_kernel(const FusedParams p) {
    fused_front_impl<0, false>(p);
}

// kColour: the colour slots of the moment row route into sh0 / shN (RGB, RGB_D, RGB_ED: the fourth channel's slot,
// kS_C4, is the depth's and is dropped); otherwise they hold the depth's gradient, which is dropped with sh0 / shN = 0.
template <int DEG, bool kColour>
__device__ __forceinline__ void fused_back_impl(const FusedParams &p) {
    constexpr int NB = (DEG + 1) * (DEG + 1);
    extern __shared__ __align__(128) float s_rows[]; // shN rows in, v_shN rows out (each thread owns its row)
    __shared__ FusedCam s_cam;
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t tid = threadIdx.x;
    const uint32_t g0 = blockIdx.x * kFusedThreads;
    const uint32_t cnt = min((uint32_t)kFusedThreads, p.N - g0);
    const uint32_t g = g0 + tid;
    const uint32_t rowf = (p.K - 1) * 3;
    const float *g_rows = p.shN ? p.shN + (size_t)g0 * rowf : nullptr;
    float *g_out = p.v_shN ? p.v_shN + (size_t)g0 * rowf : nullptr;
    const bool have_rows = rowf > 0 && g_rows != nullptr && g_out != nullptr;
    const bool read_rows = have_rows && DEG >= 1;
    const uint32_t n_floats = have_rows ? cnt * rowf : 0u;
    const bool al = have_rows && ((n_floats & 3u) == 0);
    const bool bulk_in = read_rows && al && ((reinterpret_cast<uintptr_t>(g_rows) & 15) == 0);
    const bool bulk_out = al && ((reinterpret_cast<uintptr_t>(g_out) & 15) == 0);

    if (tid == 0) fused_cam_build(p, s_cam);
    stage_rows_in(s_rows, g_rows, read_rows ? n_floats : 0u, &s_bar, bulk_in);
    __syncthreads();

    float m[16];
    float mean[3] = {0.f, 0.f, 0.f}, quat[4] = {1.f, 0.f, 0.f, 0.f}, scale[3] = {1.f, 1.f, 1.f};
    float opac = 0.5f;
    bool visible = false;
    float om[3] = {0.f, 0.f, 0.f}, oq[4] = {0.f, 0.f, 0.f, 0.f}, os[3] = {0.f, 0.f, 0.f}, oo = 0.f;
    if (tid < cnt) {
        const float4 *m4 = reinterpret_cast<const float4 *>(p.moments + (size_t)g * kMomFloats);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float4 v = m4[i];
            m[i * 4] = v.x; m[i * 4 + 1] = v.y; m[i * 4 + 2] = v.z; m[i * 4 + 3] = v.w;
        }
        const int2 r = reinterpret_cast<const int2 *>(p.radii)[g];
        visible = r.x > 0 && r.y > 0;
        mean[0] = p.means[(size_t)g * 3]; mean[1] = p.means[(size_t)g * 3 + 1]; mean[2] = p.means[(size_t)g * 3 + 2];
        if (visible) {
            const float4 q = reinterpret_cast<const float4 *>(p.rotation_raw)[g];
            quat[0] = q.x; quat[1] = q.y; quat[2] = q.z; quat[3] = q.w;
            scale[0] = act_scale(p.scaling_raw[(size_t)g * 3], p.scaling_modifier);
            scale[1] = act_scale(p.scaling_raw[(size_t)g * 3 + 1], p.scaling_modifier);
            scale[2] = act_scale(p.scaling_raw[(size_t)g * 3 + 2], p.scaling_modifier);
            opac = act_opacity(p.opacity_raw[g]);
            const float4 *r4 = reinterpret_cast<const float4 *>(p.recs + g);
            finalize_gaussian(s_cam.cc, mean, quat, scale, opac, r4[0], r4[1], r4[2], m, om, oq, os, oo);
        }
    }
    if (bulk_in) mbar_wait(&s_bar, 0);

    // SH backward with the clamp mask recomputed from the forward colour
    float vsh0[3] = {0.f, 0.f, 0.f};
    float *row = s_rows + (size_t)tid * rowf;
    if (tid < cnt) {
        if (visible && kColour) {
            float b[NB];
            const float dx = mean[0] - s_cam.campos[0], dy = mean[1] - s_cam.campos[1], dz = mean[2] - s_cam.campos[2];
            float x = dx, y = dy, z = dz, inorm = 1.f;
            if constexpr (DEG >= 1) {
                inorm = rsqrtf(dx * dx + dy * dy + dz * dz);
                x *= inorm; y *= inorm; z *= inorm;
            }
            sh_basis<DEG>(x, y, z, b);
            float col[3];
            col[0] = b[0] * p.sh0[(size_t)g * 3]; col[1] = b[0] * p.sh0[(size_t)g * 3 + 1];
            col[2] = b[0] * p.sh0[(size_t)g * 3 + 2];
            if constexpr (DEG >= 1) {
#pragma unroll
                for (int k = 1; k < NB; ++k) {
                    col[0] += b[k] * row[(k - 1) * 3];
                    col[1] += b[k] * row[(k - 1) * 3 + 1];
                    col[2] += b[k] * row[(k - 1) * 3 + 2];
                }
            }
            // clamp_min(colour + 0.5, 0) backward: the gradient passes where the argument is >= 0 (torch)
            const float g0c = (col[0] + 0.5f >= 0.f) ? m[kS_CR] : 0.f;
            const float g1c = (col[1] + 0.5f >= 0.f) ? m[kS_CG] : 0.f;
            const float g2c = (col[2] + 0.5f >= 0.f) ? m[kS_CB] : 0.f;
            vsh0[0] = b[0] * g0c; vsh0[1] = b[0] * g1c; vsh0[2] = b[0] * g2c;
            if constexpr (DEG >= 1) {
                float w[NB];
                w[0] = 0.f;
#pragma unroll
                for (int k = 1; k < NB; ++k) {
                    const float c0 = row[(k - 1) * 3], c1 = row[(k - 1) * 3 + 1], c2 = row[(k - 1) * 3 + 2];
                    w[k] = g0c * c0 + g1c * c1 + g2c * c2;
                    row[(k - 1) * 3] = b[k] * g0c; row[(k - 1) * 3 + 1] = b[k] * g1c; row[(k - 1) * 3 + 2] = b[k] * g2c;
                }
                float vx = 0.f, vy = 0.f, vz = 0.f;
                sh_basis_vjp<DEG>(x, y, z, w, vx, vy, vz);
                const float d = vx * x + vy * y + vz * z;
                om[0] += (vx - d * x) * inorm; om[1] += (vy - d * y) * inorm; om[2] += (vz - d * z) * inorm;
            }
            if (have_rows)
                for (uint32_t i = (NB - 1) * 3; i < rowf; ++i) row[i] = 0.f; // inactive degrees
        } else if (have_rows) {
            for (uint32_t i = 0; i < rowf; ++i) row[i] = 0.f;
        }
        // raw-parameter chain: d exp(s) m / ds = activated scale; d sigmoid / dx = o (1 - o)
        p.v_means[(size_t)g * 3] = om[0]; p.v_means[(size_t)g * 3 + 1] = om[1]; p.v_means[(size_t)g * 3 + 2] = om[2];
        p.v_scaling[(size_t)g * 3] = os[0] * scale[0]; p.v_scaling[(size_t)g * 3 + 1] = os[1] * scale[1];
        p.v_scaling[(size_t)g * 3 + 2] = os[2] * scale[2];
        reinterpret_cast<float4 *>(p.v_rotation)[g] = make_float4(oq[0], oq[1], oq[2], oq[3]);
        p.v_opacity[g] = visible ? oo * (opac * (1.0f - opac)) : 0.f;
        p.v_sh0[(size_t)g * 3] = vsh0[0]; p.v_sh0[(size_t)g * 3 + 1] = vsh0[1]; p.v_sh0[(size_t)g * 3 + 2] = vsh0[2];
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
        for (uint32_t i = tid; i < n_floats; i += kFusedThreads) g_out[i] = s_rows[i];
    }
}
template <int DEG>
__global__ void __launch_bounds__(kFusedThreads, 4) fused_back_kernel(const FusedParams p) {
    fused_back_impl<DEG, true>(p);
}
__global__ void __launch_bounds__(kFusedThreads, 4) fused_back_depth_kernel(const FusedParams p) {
    fused_back_impl<0, false>(p);
}

static int check_fused(const GsbSplatRaw *sp, const GsbCamera *cam) {
    if (!sp || !cam || !cam->viewmats0 || !cam->Ks) return GSB_E_INVALID;
    if ((cam->camera_model != GSB_CAMERA_PINHOLE && cam->camera_model != GSB_CAMERA_FISHEYE) || cam->viewmats1 ||
        cam->shutter_type != GSB_SHUTTER_GLOBAL)
        return GSB_E_UNSUPPORTED;
    if (sp->N == 0) return GSB_OK;
    if (!sp->means || !sp->sh0 || !sp->scaling_raw || !sp->rotation_raw || !sp->opacity_raw) return GSB_E_INVALID;
    if (sp->sh_coeffs < 1 || sp->sh_degree > 4) return GSB_E_INVALID;
    if ((sp->sh_degree + 1) * (sp->sh_degree + 1) > sp->sh_coeffs) return GSB_E_INVALID;
    if (sp->sh_coeffs > 1 && sp->sh_degree >= 1 && !sp->shN) return GSB_E_INVALID;
    if (reinterpret_cast<uintptr_t>(sp->rotation_raw) & 15) return GSB_E_INVALID;
    return GSB_OK;
}

static void fill_fused(FusedParams &p, const GsbSplatRaw *sp, const GsbCamera *cam, uint32_t W, uint32_t H, float eps2d,
                       float near_plane, float far_plane, float radius_clip) {
    p.N = sp->N; p.K = sp->sh_coeffs;
    p.means = sp->means; p.sh0 = sp->sh0; p.shN = sp->shN; p.scaling_raw = sp->scaling_raw;
    p.rotation_raw = sp->rotation_raw; p.opacity_raw = sp->opacity_raw;
    p.scaling_modifier = sp->scaling_modifier;
    p.viewmat = cam->viewmats0; p.Ks = cam->Ks;
    p.camera_model = cam->camera_model;
    p.radial = cam->radial_coeffs; p.tangential = cam->tangential_coeffs; p.thin_prism = cam->thin_prism_coeffs;
    p.n_radial = cam->radial_count; p.n_tangential = cam->tangential_count; p.n_thin_prism = cam->thin_prism_count;
    p.pk.W = W; p.pk.H = H; p.pk.eps2d = eps2d; p.pk.near_plane = near_plane; p.pk.far_plane = far_plane;
    p.pk.radius_clip = radius_clip; p.pk.ut = cam->ut;
    p.radii = nullptr; p.means2d = nullptr; p.depths = nullptr; p.recs = nullptr; p.moments = nullptr;
    p.v_means = p.v_sh0 = p.v_shN = p.v_scaling = p.v_rotation = p.v_opacity = nullptr;
}

#define GSB_FUSED_LAUNCH(KERNEL)                                                                                       \
    switch (sp->sh_degree) {                                                                                           \
        case 0: GSB_FUSED_ONE(KERNEL, 0); break;                                                                       \
        case 1: GSB_FUSED_ONE(KERNEL, 1); break;                                                                       \
        case 2: GSB_FUSED_ONE(KERNEL, 2); break;                                                                       \
        case 3: GSB_FUSED_ONE(KERNEL, 3); break;                                                                       \
        default: GSB_FUSED_ONE(KERNEL, 4); break;                                                                      \
    }
#define GSB_FUSED_ONE(KERNEL, D)                                                                                       \
    do {                                                                                                               \
        if (smem > 48 * 1024)                                                                                          \
            GSB_CUDA_TRY(cudaFuncSetAttribute(KERNEL<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));     \
        KERNEL<D><<<grid, kFusedThreads, smem, s>>>(p);                                                                \
    } while (0)

} // namespace gsb

extern "C" size_t gsb_fused_workspace(uint32_t N) {
    // [records N x 64 B][moments N x 64 B]
    return ((size_t)N * sizeof(gsb::GaussRec) + 255) / 256 * 256 + ((size_t)N * gsb::kMomFloats * 4 + 255) / 256 * 256 + 256;
}

namespace gsb {
static bool valid_render_mode(int render_mode) { return render_mode >= GSB_RENDER_RGB && render_mode <= GSB_RENDER_RGB_ED; }
// D / ED blend the depth alone: their records and moment rows carry no colour
static bool depth_only(int render_mode) { return render_mode == GSB_RENDER_D || render_mode == GSB_RENDER_ED; }

static int fused_front(const GsbSplatRaw *sp, const GsbCamera *cam, uint32_t image_width, uint32_t image_height,
                       float eps2d, float near_plane, float far_plane, float radius_clip, int zero_moments,
                       int render_mode, int32_t *radii, float *means2d, float *depths, void *workspace,
                       size_t workspace_bytes, cudaStream_t s) {
    if (int rc = check_fused(sp, cam)) return rc;
    if (sp->N == 0) return GSB_OK;
    if (!radii || !means2d || !depths) return GSB_E_INVALID;
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_fused_workspace(sp->N))
        return GSB_E_WORKSPACE;
    FusedParams p;
    fill_fused(p, sp, cam, image_width, image_height, eps2d, near_plane, far_plane, radius_clip);
    p.radii = radii; p.means2d = means2d; p.depths = depths;
    p.recs = reinterpret_cast<GaussRec *>(workspace);
    float *moments = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) +
                                               ((size_t)sp->N * sizeof(GaussRec) + 255) / 256 * 256);
    p.moments = zero_moments ? moments : nullptr;
    const uint32_t grid = (sp->N + kFusedThreads - 1) / kFusedThreads;
    {
        ProfScope ps("fused_front", s);
        if (depth_only(render_mode)) {
            fused_front_depth_kernel<<<grid, kFusedThreads, 0, s>>>(p);
        } else {
            const size_t smem = sp->sh_degree >= 1 ? (size_t)kFusedThreads * (sp->sh_coeffs - 1) * 12 : 0;
            GSB_FUSED_LAUNCH(fused_front_kernel);
        }
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

static int fused_back(const GsbSplatRaw *sp, const GsbCamera *cam, uint32_t image_width, uint32_t image_height,
                      int render_mode, const int32_t *radii, const void *workspace, size_t workspace_bytes,
                      float *v_means, float *v_sh0, float *v_shN, float *v_scaling, float *v_rotation,
                      float *v_opacity, cudaStream_t s) {
    if (int rc = check_fused(sp, cam)) return rc;
    if (sp->N == 0) return GSB_OK;
    if (!radii || !v_means || !v_sh0 || !v_scaling || !v_rotation || !v_opacity) return GSB_E_INVALID;
    if (sp->sh_coeffs > 1 && !v_shN) return GSB_E_INVALID;
    if (reinterpret_cast<uintptr_t>(v_rotation) & 15) return GSB_E_INVALID;
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_fused_workspace(sp->N))
        return GSB_E_WORKSPACE;
    FusedParams p;
    fill_fused(p, sp, cam, image_width, image_height, 0.f, 0.f, 0.f, 0.f);
    p.radii = const_cast<int32_t *>(radii);
    p.recs = reinterpret_cast<GaussRec *>(const_cast<void *>(workspace));
    p.moments = reinterpret_cast<float *>(reinterpret_cast<char *>(const_cast<void *>(workspace)) +
                                          ((size_t)sp->N * sizeof(GaussRec) + 255) / 256 * 256);
    p.v_means = v_means; p.v_sh0 = v_sh0; p.v_shN = v_shN; p.v_scaling = v_scaling; p.v_rotation = v_rotation;
    p.v_opacity = v_opacity;
    const uint32_t grid = (sp->N + kFusedThreads - 1) / kFusedThreads;
    // the shN gradient rows are staged through shared memory even when they are all zero (D / ED)
    const size_t smem = sp->sh_coeffs > 1 ? (size_t)kFusedThreads * (sp->sh_coeffs - 1) * 12 : 0;
    {
        ProfScope ps("fused_back", s);
        if (depth_only(render_mode)) {
            if (smem > 48 * 1024)
                GSB_CUDA_TRY(cudaFuncSetAttribute(fused_back_depth_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  (int)smem));
            fused_back_depth_kernel<<<grid, kFusedThreads, smem, s>>>(p);
        } else {
            GSB_FUSED_LAUNCH(fused_back_kernel);
        }
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
} // namespace gsb

extern "C" int gsb_fused_front(const GsbSplatRaw *sp, const GsbCamera *cam, uint32_t image_width, uint32_t image_height,
                               float eps2d, float near_plane, float far_plane, float radius_clip, int zero_moments,
                               int32_t *radii, float *means2d, float *depths, void *workspace, size_t workspace_bytes,
                               gsb_stream_t stream) {
    return gsb::fused_front(sp, cam, image_width, image_height, eps2d, near_plane, far_plane, radius_clip, zero_moments,
                            GSB_RENDER_RGB, radii, means2d, depths, workspace, workspace_bytes, gsb::as_stream(stream));
}

extern "C" int gsb_fused_front_mode(const GsbSplatRaw *sp, const GsbCamera *cam, uint32_t image_width,
                                    uint32_t image_height, float eps2d, float near_plane, float far_plane,
                                    float radius_clip, int zero_moments, int render_mode, int32_t *radii,
                                    float *means2d, float *depths, void *workspace, size_t workspace_bytes,
                                    gsb_stream_t stream) {
    if (!gsb::valid_render_mode(render_mode)) return GSB_E_UNSUPPORTED;
    return gsb::fused_front(sp, cam, image_width, image_height, eps2d, near_plane, far_plane, radius_clip, zero_moments,
                            render_mode, radii, means2d, depths, workspace, workspace_bytes, gsb::as_stream(stream));
}

extern "C" int gsb_fused_back(const GsbSplatRaw *sp, const GsbCamera *cam, uint32_t image_width, uint32_t image_height,
                              const int32_t *radii, const void *workspace, size_t workspace_bytes, float *v_means,
                              float *v_sh0, float *v_shN, float *v_scaling, float *v_rotation, float *v_opacity,
                              gsb_stream_t stream) {
    return gsb::fused_back(sp, cam, image_width, image_height, GSB_RENDER_RGB, radii, workspace, workspace_bytes,
                           v_means, v_sh0, v_shN, v_scaling, v_rotation, v_opacity, gsb::as_stream(stream));
}

extern "C" int gsb_fused_back_mode(const GsbSplatRaw *sp, const GsbCamera *cam, uint32_t image_width,
                                   uint32_t image_height, int render_mode, const int32_t *radii, const void *workspace,
                                   size_t workspace_bytes, float *v_means, float *v_sh0, float *v_shN,
                                   float *v_scaling, float *v_rotation, float *v_opacity, gsb_stream_t stream) {
    if (!gsb::valid_render_mode(render_mode)) return GSB_E_UNSUPPORTED;
    return gsb::fused_back(sp, cam, image_width, image_height, render_mode, radii, workspace, workspace_bytes, v_means,
                           v_sh0, v_shN, v_scaling, v_rotation, v_opacity, gsb::as_stream(stream));
}
