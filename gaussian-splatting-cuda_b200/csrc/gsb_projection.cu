// gsb_projection.cu -- a1: unscented-transform projection of world Gaussians to image Gaussians.
//
// Implements gsplat::projection_ut_3dgs_fused (reference: gsplat/ProjectionUT3DGSFused.cu:17-203,
// gsplat/Cameras.cuh:1034-1150, gsplat/Utils.cuh:171-179) for the perfect-pinhole / global-shutter
// camera, the only configuration the reference's callers reach (rasterizer_autograd.cpp:217-237).
//
// H100 notes: the kernel is a pure stream (44 B in, <= 36 B out per Gaussian, ~500 FLOP), so the
// design goal is full-sector HBM traffic: a CTA stages its 256-Gaussian slab of the AoS inputs
// (means/scales 12 B rows, quats 16 B rows, opacities) into shared memory with TMA bulk copies
// (cp.async.bulk, one per array) and writes the 12-byte conic rows back through shared memory
// with a bulk store, so every global transaction is a full 128-byte line.
//
// This file is compiled with -fmad=false: radii come out of ceilf() and feed the bit-exact tile
// intersection, so the arithmetic deliberately follows the reference's operation order without
// FMA contraction (the CPU oracle is built with -ffp-contract=off for the same reason).
#include "gsb_projection.cuh"

namespace gsb {

constexpr int kProjThreads = 256;

struct ProjParams {
    uint32_t C, N;
    const float *means, *quats, *scales, *opacities;
    const float *viewmats0, *viewmats1, *Ks;
    int32_t shutter;
    uint32_t W, H;
    float eps2d, near_plane, far_plane, radius_clip;
    GsbUTParams ut;
    int32_t camera_model;
    const float *radial, *tangential, *thin_prism; // per-camera coefficient rows, nullable
    int32_t n_radial, n_tangential, n_thin_prism;
    int32_t *radii;
    float *means2d, *depths, *conics, *compensations;
    uint32_t inputs_aligned16; // every input base pointer is 16-byte aligned: full slabs may use bulk copies
};

template <bool kRolling>
__global__ void __launch_bounds__(kProjThreads) projection_ut_kernel(const ProjParams p) {
    __shared__ __align__(128) float s_means[kProjThreads * 3];
    __shared__ __align__(128) float s_scales[kProjThreads * 3];
    __shared__ __align__(128) float s_quats[kProjThreads * 4];
    __shared__ __align__(128) float s_opac[kProjThreads];
    __shared__ __align__(128) float s_conics[kProjThreads * 3];
    __shared__ __align__(8) uint64_t s_bar;

    const uint32_t cid = blockIdx.y;
    const uint32_t g0 = blockIdx.x * kProjThreads;
    const uint32_t cnt = min((uint32_t)kProjThreads, p.N - g0);
    const uint32_t tid = threadIdx.x;
    // cp.async.bulk needs 16-byte aligned global addresses: true for every full slab when the base pointers
    // are (256 rows x 12 / 16 / 4 bytes), not for a contiguous view such as means[1:] -- the reference accepts
    // those, so they take the plain staging loop instead of faulting
    const bool full = (cnt == kProjThreads);
    const bool bulk_in = full && p.inputs_aligned16;

    // ---- stage the slab ------------------------------------------------------------------
    if (bulk_in) {
        if (tid == 0) {
            mbar_init(&s_bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (tid == 0) {
            const uint32_t bytes = kProjThreads * (12 + 12 + 16) + (p.opacities ? kProjThreads * 4 : 0);
            mbar_arrive_expect_tx(&s_bar, bytes);
            bulk_g2s(s_means, p.means + (size_t)g0 * 3, kProjThreads * 12, &s_bar);
            bulk_g2s(s_scales, p.scales + (size_t)g0 * 3, kProjThreads * 12, &s_bar);
            bulk_g2s(s_quats, p.quats + (size_t)g0 * 4, kProjThreads * 16, &s_bar);
            if (p.opacities) bulk_g2s(s_opac, p.opacities + g0, kProjThreads * 4, &s_bar);
        }
        mbar_wait(&s_bar, 0);
    } else {
        for (uint32_t i = tid; i < cnt * 3; i += kProjThreads) {
            s_means[i] = p.means[(size_t)g0 * 3 + i];
            s_scales[i] = p.scales[(size_t)g0 * 3 + i];
        }
        for (uint32_t i = tid; i < cnt * 4; i += kProjThreads) s_quats[i] = p.quats[(size_t)g0 * 4 + i];
        if (p.opacities)
            for (uint32_t i = tid; i < cnt; i += kProjThreads) s_opac[i] = p.opacities[g0 + i];
        __syncthreads();
    }

    // ---- camera (Cameras.cuh:33-71, 268-280) -----------------------------------------------
    __shared__ CamModel s_cm;
    if (tid == 0)
        cam_model_build(s_cm, p.camera_model, p.W, p.H, p.Ks + cid * 9,
                        p.radial ? p.radial + (size_t)cid * p.n_radial : nullptr, p.n_radial,
                        p.tangential ? p.tangential + (size_t)cid * p.n_tangential : nullptr, p.n_tangential,
                        p.thin_prism ? p.thin_prism + (size_t)cid * p.n_thin_prism : nullptr, p.n_thin_prism);
    __syncthreads();
    const ProjPose pp = proj_pose_from_viewmat(p.viewmats0 + cid * 16, p.viewmats1 ? p.viewmats1 + cid * 16 : nullptr, p.shutter);
    ProjConsts pk;
    pk.W = p.W; pk.H = p.H; pk.eps2d = p.eps2d; pk.near_plane = p.near_plane; pk.far_plane = p.far_plane;
    pk.radius_clip = p.radius_clip; pk.ut = p.ut;

    // ---- per-Gaussian work -----------------------------------------------------------------
    int32_t rx_i = 0, ry_i = 0;
    float o_mx = 0.f, o_my = 0.f, o_depth = 0.f, o_c0 = 0.f, o_c1 = 0.f, o_c2 = 0.f, o_comp = 0.f;
    bool keep = false;
    if (tid < cnt) {
        const V3<float> mean = {s_means[tid * 3], s_means[tid * 3 + 1], s_means[tid * 3 + 2]};
        const float sc[3] = {s_scales[tid * 3], s_scales[tid * 3 + 1], s_scales[tid * 3 + 2]};
        const ProjResult r = project_gaussian<kRolling>(pk, s_cm, pp, mean, sc, s_quats[tid * 4], s_quats[tid * 4 + 1],
                                              s_quats[tid * 4 + 2], s_quats[tid * 4 + 3], p.opacities != nullptr,
                                              p.opacities ? s_opac[tid] : 0.f);
        keep = r.keep;
        rx_i = r.rx; ry_i = r.ry;
        o_mx = r.mx; o_my = r.my; o_depth = r.depth; o_c0 = r.c0; o_c1 = r.c1; o_c2 = r.c2; o_comp = r.comp;
    }

    // ---- outputs ---------------------------------------------------------------------------
    const size_t idx = (size_t)cid * p.N + g0 + tid;
    if (tid < cnt) {
        reinterpret_cast<int2 *>(p.radii)[idx] = make_int2(rx_i, ry_i);
        if (keep) {
            reinterpret_cast<float2 *>(p.means2d)[idx] = make_float2(o_mx, o_my);
            p.depths[idx] = o_depth;
            if (p.compensations) p.compensations[idx] = o_comp;
        }
    }
    // conics: culled rows must stay untouched (Projection.cpp:70-73), so the full-line bulk store
    // is only used when every Gaussian of the slab survived; otherwise scalar stores.
    const bool all_keep = __syncthreads_and(keep || tid >= cnt) != 0;
    float *cdst = p.conics + ((size_t)cid * p.N + g0) * 3;
    if (all_keep && full && ((reinterpret_cast<uintptr_t>(cdst) & 15) == 0)) {
        s_conics[tid * 3] = o_c0; s_conics[tid * 3 + 1] = o_c1; s_conics[tid * 3 + 2] = o_c2;
        fence_proxy_async();
        __syncthreads();
        if (tid == 0) {
            bulk_s2g(cdst, s_conics, kProjThreads * 12);
            bulk_commit();
            bulk_wait_read_all();
        }
    } else if (keep) {
        cdst[tid * 3] = o_c0; cdst[tid * 3 + 1] = o_c1; cdst[tid * 3 + 2] = o_c2;
    }
}

} // namespace gsb

extern "C" int gsb_projection_ut(
    uint32_t C, uint32_t N, const float *means, const float *quats, const float *scales,
    const float *opacities, const GsbCamera *cam, uint32_t image_width, uint32_t image_height,
    float eps2d, float near_plane, float far_plane, float radius_clip, int32_t *radii, float *means2d,
    float *depths, float *conics, float *compensations, gsb_stream_t stream) {
    if (!cam || !cam->viewmats0 || !cam->Ks) return GSB_E_INVALID;
    if (C == 0 || N == 0) return GSB_OK; // ProjectionUT3DGSFused.cu:242-245
    if (!means || !quats || !scales || !radii || !means2d || !depths || !conics) return GSB_E_INVALID;
    if (cam->camera_model != GSB_CAMERA_PINHOLE && cam->camera_model != GSB_CAMERA_FISHEYE)
        return GSB_E_UNSUPPORTED; // orthographic: the reference has no such branch either (ProjectionUT3DGSFused.cu:130-134)
    if (cam->shutter_type < GSB_SHUTTER_ROLLING_TOP_TO_BOTTOM || cam->shutter_type > GSB_SHUTTER_GLOBAL) return GSB_E_INVALID;
    gsb::ProjParams p;
    p.C = C; p.N = N;
    p.means = means; p.quats = quats; p.scales = scales; p.opacities = opacities;
    p.viewmats0 = cam->viewmats0; p.Ks = cam->Ks;
    // without an end-of-frame pose the start pose is used for both ends (Cameras.cuh:54-56): a global shutter
    p.viewmats1 = cam->viewmats1; p.shutter = cam->viewmats1 ? cam->shutter_type : GSB_SHUTTER_GLOBAL;
    p.W = image_width; p.H = image_height;
    p.eps2d = eps2d; p.near_plane = near_plane; p.far_plane = far_plane; p.radius_clip = radius_clip;
    p.ut = cam->ut;
    p.camera_model = cam->camera_model;
    p.radial = cam->radial_coeffs; p.tangential = cam->tangential_coeffs; p.thin_prism = cam->thin_prism_coeffs;
    p.n_radial = cam->radial_count; p.n_tangential = cam->tangential_count; p.n_thin_prism = cam->thin_prism_count;
    p.radii = radii; p.means2d = means2d; p.depths = depths; p.conics = conics; p.compensations = compensations;
    const uintptr_t bits = reinterpret_cast<uintptr_t>(means) | reinterpret_cast<uintptr_t>(quats) |
                           reinterpret_cast<uintptr_t>(scales) | reinterpret_cast<uintptr_t>(opacities);
    p.inputs_aligned16 = (bits & 15) == 0 ? 1u : 0u;
    dim3 grid((N + gsb::kProjThreads - 1) / gsb::kProjThreads, C);
    {
        gsb::ProfScope ps("projection_ut", gsb::as_stream(stream));
        if (p.shutter != GSB_SHUTTER_GLOBAL)
            gsb::projection_ut_kernel<true><<<grid, gsb::kProjThreads, 0, gsb::as_stream(stream)>>>(p);
        else
            gsb::projection_ut_kernel<false><<<grid, gsb::kProjThreads, 0, gsb::as_stream(stream)>>>(p);
    }
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
