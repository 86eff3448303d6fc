/*
 * gsb200.h -- C ABI of the H100-native (sm_90a) 3DGUT rasterizer hot path.
 *
 * This is the drop-in boundary underneath the reference's C++ operator API
 * (namespace gsplat, /root/reference/gsplat/Ops.h:12-165).  Every entry point
 * below states which reference operator it implements; the thin libtorch shim
 * in gaussian-splatting-cuda_b200/shim/Ops.cpp exports the identical gsplat::
 * signatures on top of it, so the reference's src/training and src/rendering
 * link against it unchanged (see INTEGRATION.md).
 *
 * Conventions
 *  - plain C: raw DEVICE pointers, sizes, POD structs, a cudaStream_t.  No torch
 *    types, no exceptions.  All tensors are contiguous row-major float32 unless
 *    stated; layouts are exactly the reference's (Ops.h comments).
 *  - nothing here allocates device memory: outputs and workspaces are provided
 *    by the caller (the shim allocates them through the torch caching allocator,
 *    like gsplat/Common.h:23-30 does for CUB).  Workspace sizes come from the
 *    *_workspace() queries; workspaces need 256-byte alignment.
 *  - every call is asynchronous on `stream` and re-entrant (no static mutable
 *    state) -- the reference calls these ops from the training thread and the
 *    viewer thread (SURVEY.md section 8b).
 *  - return value: GSB_OK (0), a negative GSB_E_* code, or a positive
 *    cudaError_t from a failed launch.  gsb_error_string() names them.
 *  - there is NO CPU fallback: on a machine without an sm_90 device every
 *    compute entry point returns a CUDA error.
 */
#ifndef GSB200_H_
#define GSB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef GSB_API
#define GSB_API __attribute__((visibility("default")))
#endif

/* Opaque to C callers that do not include cuda_runtime.h. */
typedef struct CUstream_st *gsb_stream_t;

enum {
    GSB_OK = 0,
    GSB_E_INVALID = -1,     /* bad argument (null pointer, zero size where not allowed) */
    GSB_E_UNSUPPORTED = -2, /* valid in the reference but not implemented here (see DESIGN.md) */
    GSB_E_WORKSPACE = -3    /* workspace too small / misaligned */
};

/* gsplat::CameraModelType, gsplat/Common.h:46-50 */
enum { GSB_CAMERA_PINHOLE = 0, GSB_CAMERA_ORTHO = 1, GSB_CAMERA_FISHEYE = 2 };

/* ShutterType, gsplat/Cameras.h:16-22 */
enum {
    GSB_SHUTTER_ROLLING_TOP_TO_BOTTOM = 0,
    GSB_SHUTTER_ROLLING_LEFT_TO_RIGHT = 1,
    GSB_SHUTTER_ROLLING_BOTTOM_TO_TOP = 2,
    GSB_SHUTTER_ROLLING_RIGHT_TO_LEFT = 3,
    GSB_SHUTTER_GLOBAL = 4
};

/* UnscentedTransformParameters, gsplat/Cameras.h:27-44 */
typedef struct GsbUTParams {
    float alpha;
    float beta;
    float kappa;
    float in_image_margin_factor;
    int32_t require_all_sigma_points_valid;
} GsbUTParams;

/* Camera block shared by projection and the from-world rasterizer.
 * viewmats1 / distortion pointers are nullable; *_count gives the number of
 * floats per camera behind each distortion pointer (the reference reads a fixed
 * 6/2/4 regardless of what the caller allocated, SURVEY.md section 7; here the
 * count is explicit and missing coefficients are zero-filled). */
typedef struct GsbCamera {
    const float *viewmats0; /* [C,4,4] world->camera, row-major */
    const float *viewmats1; /* [C,4,4] end-of-frame pose for rolling shutter, or NULL */
    const float *Ks;        /* [C,3,3] */
    int32_t camera_model;   /* GSB_CAMERA_* */
    int32_t shutter_type;   /* GSB_SHUTTER_* */
    const float *radial_coeffs;
    int32_t radial_count;
    const float *tangential_coeffs;
    int32_t tangential_count;
    const float *thin_prism_coeffs;
    int32_t thin_prism_count;
    GsbUTParams ut;
} GsbCamera;

GSB_API const char *gsb_error_string(int code);
GSB_API int gsb_version(void);

/* Diagnostics (no effect on results).  gsb_launch_count: number of this library's own kernel
 * launches so far in the process (CUB / memset launches are not counted).  gsb_profile_enable(1)
 * makes the hot kernels record CUDA events on their launch stream; gsb_profile_read sums the
 * recorded durations of one kernel ("projection_ut", "sh_fwd", "sh_bwd", "isect_count",
 * "isect_emit", "isect_sort", "isect_offsets", "raster_prep", "raster_fwd", "raster_bwd",
 * "raster_finalize") and returns how many launches were found. */
GSB_API uint64_t gsb_launch_count(void);
GSB_API void gsb_profile_enable(int on);
GSB_API int gsb_profile_read(const char *kernel, double *total_ms);

/* ---- a1: gsplat::projection_ut_3dgs_fused (Ops.h:69-98, Projection.cpp:16-110,
 *      ProjectionUT3DGSFused.cu:17-203) ------------------------------------------
 * radii [C,N,2] int32 (0,0 = culled), means2d [C,N,2], depths [C,N], conics [C,N,3],
 * compensations [C,N] or NULL.  Culled rows of means2d/depths/conics are left
 * untouched, like the reference (Projection.cpp:70-73).  Inputs need only their natural 4-byte
 * alignment (e.g. a contiguous view means[1:]); 16-byte aligned base pointers get the TMA staging path. */
GSB_API int gsb_projection_ut(
    uint32_t C, uint32_t N,
    const float *means, const float *quats, const float *scales, const float *opacities /*nullable*/,
    const GsbCamera *cam, uint32_t image_width, uint32_t image_height,
    float eps2d, float near_plane, float far_plane, float radius_clip,
    int32_t *radii, float *means2d, float *depths, float *conics, float *compensations /*nullable*/,
    gsb_stream_t stream);

/* ---- a3/a4: gsplat::spherical_harmonics_fwd / _bwd (Ops.h:12-25,
 *      SphericalHarmonics.cpp:15-75, SphericalHarmonicsCUDA.cu:374-481) -----------
 * M = number of (camera, Gaussian) elements, K = coefficients per element.
 * masks: [M] bytes (bool) or NULL.  fwd leaves masked-out rows of `colors`
 * untouched.  bwd writes EVERY element of v_coeffs (zeros for masked rows and for
 * k >= (degree+1)^2) and of v_dirs -- the caller need not zero-fill them
 * (the reference memsets 192 B/Gaussian first, SphericalHarmonics.cpp:58). */
GSB_API int gsb_sh_fwd(uint32_t M, uint32_t K, uint32_t degrees_to_use, const float *dirs,
                       const float *coeffs, const uint8_t *masks, float *colors, gsb_stream_t stream);
GSB_API int gsb_sh_bwd(uint32_t M, uint32_t K, uint32_t degrees_to_use, const float *dirs,
                       const float *coeffs, const uint8_t *masks, const float *v_colors,
                       float *v_coeffs, float *v_dirs /*nullable*/, gsb_stream_t stream);

/* ---- (e) multi-GPU exchange step: SH backward of V views at once ------------------------------
 * The reference has no distributed mode (SURVEY.md 2.1); this entry point belongs to the view-sharded
 * data-parallel step of SURVEY.md 8(e).  Per view the SH gradient row is the outer product of the basis
 * at that view's direction and a 12-byte colour gradient, so ranks all-gather the colour gradients
 * (v_colors [V, M, 3], zero where a Gaussian was not blended) and each expands and sums all views:
 *   v_coeffs [M, K, 3]  = sum_v Y(normalize(means - campos[v])) (x) v_colors[v]      (fully written)
 *   v_means  [M, 3]    += sum_v d(colour_v)/d(mean)                                   (accumulated)
 * Equal to summing gsb_sh_bwd over the views with dirs = means - campos[v]. */
GSB_API int gsb_sh_bwd_views(uint32_t M, uint32_t K, uint32_t degrees_to_use, uint32_t V,
                             const float *means, const float *campos /* [V,3] */, const float *coeffs,
                             const float *v_colors /* [V,M,3] */, float *v_coeffs, float *v_means,
                             gsb_stream_t stream);
/* The same step with the all-gather INSIDE the kernel: view v's colour gradients [M,3] and camera position [3] are
 * read through per-view device pointers (host arrays of V <= 16 pointers), which may point into PEER memory --
 * NVLink-mapped buffers of the other ranks (CUDA IPC / symmetric memory).  The remote reads overlap the expansion
 * and the gathered [V,M,3] tensor is never materialised.  The caller orders the kernel after every rank's write of
 * its buffer (a device-side barrier) and must not overwrite its buffer before all ranks have finished reading. */
GSB_API int gsb_sh_bwd_views_peer(uint32_t M, uint32_t K, uint32_t degrees_to_use, uint32_t V, const float *means,
                                  const float *const *campos_views /* host array [V] of device ptrs to [3] */,
                                  const float *coeffs,
                                  const float *const *v_colors_views /* host array [V] of device ptrs to [M,3] */,
                                  float *v_coeffs, float *v_means, gsb_stream_t stream);

/* ---- a5: gsplat::intersect_tile (Ops.h:28-38, Intersect.cpp:15-122,
 *      IntersectTile.cu:24-114,290-328) ----------------------------------------------
 * Three device steps around the one host read-back the API forces (the op
 * returns exactly-sized tensors):
 *   gsb_isect_count      tiles_per_gauss [C*N] int32 and its inclusive int64 scan
 *                        cum_tiles [C*N]; n_isects = cum_tiles[C*N-1].
 *   gsb_isect_emit       unsorted isect_ids [I] int64 / flatten_ids [I] int32.
 *   gsb_isect_sort       stable LSD radix sort (own kernels) by the low 32+tile_bits+cam_bits
 *                        key bits; equal keys keep emission order, like the reference's CUB sort.
 * Non-packed ([C,N,...]) layout only; packed mode is rejected by the reference's
 * caller too (rasterizer.cpp:56). */
GSB_API size_t gsb_isect_count_workspace(uint64_t n_elements);
GSB_API int gsb_isect_count(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii,
                            uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
                            int32_t *tiles_per_gauss, int64_t *cum_tiles,
                            void *workspace, size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_isect_emit(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii,
                           const float *depths, const int64_t *cum_tiles,
                           uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
                           int64_t *isect_ids, int32_t *flatten_ids, gsb_stream_t stream);
GSB_API size_t gsb_isect_sort_workspace(uint64_t n_isects);
GSB_API int gsb_isect_sort(uint64_t n_isects, uint32_t C, uint32_t tile_width, uint32_t tile_height,
                           const int64_t *isect_ids_in, const int32_t *flatten_ids_in,
                           int64_t *isect_ids_out, int32_t *flatten_ids_out,
                           void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* Planned sorted path for sort == true: same outputs as gsb_isect_emit + gsb_isect_sort, bit for bit,
 * without sorting any intersection.  The Gaussians are ordered by depth once (N elements, own radix
 * sort), the runs in that order are cut into chunks, a per-(chunk, tile) histogram is scanned, and every
 * intersection is written DIRECTLY to its final position, each (chunk, tile) group being filled in depth
 * order (csrc/gsb_intersect.cu).  It is arranged around the one host read-back the
 * operator API forces: everything that does not need the host to know n_isects runs in the PLAN.
 *   gsb_isect_plan          tiles_per_gauss [C*N]; *n_isects_out (device OR pinned host int64,
 *                           written asynchronously on `stream`); tile_offsets_out [C*th*tw] int32 or
 *                           NULL -- the a6 result, a by-product of the plan's scan (with
 *                           tile_offsets_total != 0 one more entry, [C*th*tw] = n_isects, so a
 *                           consumer needs no host-side count); plan_workspace keeps the run table
 *                           and the per-chunk first slots for the emit.
 *   gsb_isect_emit_planned  flatten_ids and, unless NULL, isect_ids, sorted.  `n_isects` is the CAPACITY
 *                           of those arrays: the true count is read on the device, slots beyond the
 *                           capacity are dropped (a caller that allocates from a guess checks the
 *                           count afterwards) -- with the exact count it is the reference's behaviour.
 * Limits: C*N < 2^31, C*th*tw < 2^31, tile grid sides <= 65535, n_isects < 2^31. */
GSB_API size_t gsb_isect_plan_workspace(uint32_t C, uint32_t N, uint32_t tile_width, uint32_t tile_height);
GSB_API int gsb_isect_plan(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii,
                           const float *depths, uint32_t tile_size, uint32_t tile_width,
                           uint32_t tile_height, int32_t *tiles_per_gauss, int64_t *n_isects_out,
                           int32_t *tile_offsets_out /*nullable*/, int tile_offsets_total,
                           void *plan_workspace, size_t plan_workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_isect_emit_planned(uint32_t C, uint32_t N, const float *depths,
                                   uint32_t tile_width, uint32_t tile_height,
                                   uint64_t n_isects, const void *plan_workspace,
                                   size_t plan_workspace_bytes, int64_t *isect_ids /*nullable*/,
                                   int32_t *flatten_ids, gsb_stream_t stream);

/* ---- a6: gsplat::intersect_offset (Ops.h:39-43, IntersectTile.cu:206-288) --------
 * offsets [C,tile_height,tile_width] int32; all zero when n_isects == 0. */
GSB_API int gsb_isect_offsets(uint64_t n_isects, const int64_t *isect_ids_sorted, uint32_t C,
                              uint32_t tile_width, uint32_t tile_height, int32_t *offsets,
                              gsb_stream_t stream);

/* ---- a7: gsplat::rasterize_to_pixels_from_world_3dgs_fwd (Ops.h:100-129,
 *      Rasterization.cpp:20-132, RasterizeToPixelsFromWorld3DGSFwd.cu:20-279) ---------
 * colors [C,N,3] (3 channels only, as the reference asserts), opacities [C,N],
 * backgrounds [C,3] or NULL, masks [C,th,tw] bytes or NULL, tile_offsets [C,th,tw],
 * flatten_ids [I].  C must be 1 (the reference's kernels index means[] with the
 * flattened id, Fwd.cu:197-200).  Outputs: renders [C,H,W,3], alphas [C,H,W,1],
 * last_ids [C,H,W] int32. */
GSB_API size_t gsb_raster_fwd_workspace(uint32_t N);
GSB_API int gsb_raster_fwd(
    uint32_t C, uint32_t N, uint64_t n_isects,
    const float *means, const float *quats, const float *scales, const float *colors,
    const float *opacities, const float *backgrounds, const uint8_t *masks,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, const GsbCamera *cam,
    const int32_t *tile_offsets, const int32_t *flatten_ids,
    float *renders, float *alphas, int32_t *last_ids,
    void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* ---- a8: gsplat::rasterize_to_pixels_from_world_3dgs_bwd (Ops.h:131-165,
 *      Rasterization.cpp:134-261, RasterizeToPixelsFromWorld3DGSBwd.cu:17-373) --------
 * Writes every element of v_means [N,3], v_quats [N,4], v_scales [N,3],
 * v_colors [C,N,3], v_opacities [C,N] (zeros for untouched Gaussians): the caller
 * need not zero-fill (the reference does, Rasterization.cpp:190-194). */
GSB_API size_t gsb_raster_bwd_workspace(uint32_t N);
GSB_API int gsb_raster_bwd(
    uint32_t C, uint32_t N, uint64_t n_isects,
    const float *means, const float *quats, const float *scales, const float *colors,
    const float *opacities, const float *backgrounds, const uint8_t *masks,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, const GsbCamera *cam,
    const int32_t *tile_offsets, const int32_t *flatten_ids,
    const float *render_alphas, const int32_t *last_ids,
    const float *v_render_colors, const float *v_render_alphas,
    float *v_means, float *v_quats, float *v_scales, float *v_colors, float *v_opacities,
    void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* ---- a7 / a8 at 1, 3 or 4 channels: the blend of the reference's render modes (rasterizer.cpp:272-298) -----------
 * The same operators with `channels` colour channels per Gaussian: colors [C,N,channels], backgrounds
 * [C,channels] or NULL, renders [C,H,W,channels], v_colors [C,N,channels]; everything else as above, and the same
 * workspaces.  channels = 1 blends the depth alone (RenderMode D / ED), 4 colour + depth (RGB_D / RGB_ED);
 * channels = 3 is exactly gsb_raster_fwd / gsb_raster_bwd.  Checked before any launch:
 *   channels not in {1, 3, 4}                          -> GSB_E_UNSUPPORTED
 *   channels != 3 with a rolling shutter              -> GSB_E_UNSUPPORTED (the rolling-shutter blend is RGB only)
 *   a NULL camera or argument pointer                  -> GSB_E_INVALID, as for the 3-channel calls. */
GSB_API int gsb_raster_fwd_nc(
    uint32_t C, uint32_t N, uint64_t n_isects, uint32_t channels,
    const float *means, const float *quats, const float *scales, const float *colors,
    const float *opacities, const float *backgrounds, const uint8_t *masks,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, const GsbCamera *cam,
    const int32_t *tile_offsets, const int32_t *flatten_ids,
    float *renders, float *alphas, int32_t *last_ids,
    void *workspace, size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_raster_bwd_nc(
    uint32_t C, uint32_t N, uint64_t n_isects, uint32_t channels,
    const float *means, const float *quats, const float *scales, const float *colors,
    const float *opacities, const float *backgrounds, const uint8_t *masks,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, const GsbCamera *cam,
    const int32_t *tile_offsets, const int32_t *flatten_ids,
    const float *render_alphas, const int32_t *last_ids,
    const float *v_render_colors, const float *v_render_alphas,
    float *v_means, float *v_quats, float *v_scales, float *v_colors, float *v_opacities,
    void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* ---- SURVEY.md 8(f1): the L3 glue folded into the path -- an EXTENDED operator set over the raw SplatData --------
 * The reference's caller activates the parameters and builds SH inputs with ~10 torch kernels around the
 * operators every step (src/core/splat_data.cpp:267-286: exp / sigmoid / normalize / cat(sh0, shN);
 * src/training/rasterization/rasterizer.cpp:250-266: inverse(viewmat), dirs, masks, clamp_min(SH + 0.5)) and
 * their autograd backward.  These entry points take the RAW tensors instead (fastgs already does,
 * fastgs/rasterization/include/rasterization_api.h:25-75) and keep the unfused operators above untouched:
 *
 *   gsb_fused_front   activations -> UT projection (bit-identical radii / means2d / depths to a1) -> SH colour of
 *                     the view direction (+0.5, clamp) -> blend record; zeroes the backward's moment rows.
 *   gsb_isect_plan / gsb_isect_emit_planned          (above; tile_offsets_total = 1, isect_ids = NULL)
 *   gsb_raster_fwd_recs / gsb_raster_bwd_recs        a7 / a8 on the records of gsb_fused_front
 *   gsb_fused_back    moments -> gradients of the RAW parameters: finalize chain rule, exp / sigmoid /
 *                     normalise backward, clamp mask, SH backward straight into the sh0 / shN layouts,
 *                     direction gradient added to the position gradient.  Every output element is written.
 *
 * No step of this sequence needs a host-side value: flatten_ids may be allocated from a capacity guess
 * (intersections beyond it are dropped; compare *n_isects_out with the capacity afterwards), so a whole
 * training step can be enqueued -- or captured in a CUDA graph -- without a synchronisation. */
typedef struct GsbSplatRaw {
    uint32_t N;
    uint32_t sh_coeffs;       /* K: coefficients per Gaussian, sh0 included (shN holds K - 1) */
    uint32_t sh_degree;       /* active degree, (degree + 1)^2 <= K */
    float scaling_modifier;
    const float *means;        /* [N,3] */
    const float *sh0;          /* [N,1,3] */
    const float *shN;          /* [N,K-1,3], may be NULL when K == 1 */
    const float *scaling_raw;  /* [N,3] log-scales */
    const float *rotation_raw; /* [N,4] (w,x,y,z), not normalised; 16-byte aligned */
    const float *opacity_raw;  /* [N] logits */
} GsbSplatRaw;

GSB_API size_t gsb_fused_workspace(uint32_t N); /* [records][moments]; == gsb_raster_bwd_workspace(N) */
GSB_API int gsb_fused_front(const GsbSplatRaw *splats, const GsbCamera *cam, uint32_t image_width,
                            uint32_t image_height, float eps2d, float near_plane, float far_plane,
                            float radius_clip, int zero_moments,
                            int32_t *radii /*[N,2]*/, float *means2d /*[N,2]*/, float *depths /*[N]*/,
                            void *workspace, size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_raster_fwd_recs(uint32_t N, uint32_t capacity, const void *workspace, size_t workspace_bytes,
                                const float *backgrounds, const uint8_t *masks, uint32_t image_width,
                                uint32_t image_height, const GsbCamera *cam,
                                const int32_t *tile_offsets /*[th*tw + 1]*/, const int32_t *flatten_ids,
                                float *renders, float *alphas, int32_t *last_ids, gsb_stream_t stream);
GSB_API int gsb_raster_bwd_recs(uint32_t N, uint32_t capacity, void *workspace, size_t workspace_bytes,
                                const float *backgrounds, const uint8_t *masks, uint32_t image_width,
                                uint32_t image_height, const GsbCamera *cam,
                                const int32_t *tile_offsets /*[th*tw + 1]*/, const int32_t *flatten_ids,
                                const float *render_alphas, const int32_t *last_ids,
                                const float *v_render_colors, const float *v_render_alphas, gsb_stream_t stream);
GSB_API int gsb_fused_back(const GsbSplatRaw *splats, const GsbCamera *cam, uint32_t image_width,
                           uint32_t image_height, const int32_t *radii, const void *workspace,
                           size_t workspace_bytes, float *v_means, float *v_sh0, float *v_shN /*NULL iff K == 1*/,
                           float *v_scaling, float *v_rotation /*16-byte aligned*/, float *v_opacity,
                           gsb_stream_t stream);

/* Render modes on the fused path (gs::training::RenderMode, rasterizer.hpp:25-31; POINT_CLOUD is not a blend).
 *   gsb_fused_front_mode   RGB / RGB_D / RGB_ED: the records of gsb_fused_front (SH colour); D / ED: the record's
 *                          one channel is the camera-space depth written to depths[].
 *   gsb_raster_fwd_recs_nc / gsb_raster_bwd_recs_nc   the blend at `channels` = 1 (D / ED), 3 (RGB) or 4 (RGB_D /
 *                          RGB_ED: the fourth channel is read from the front's depths [N]; NULL -> GSB_E_INVALID).
 *                          backgrounds [channels] or NULL, renders / v_render_colors [H,W,channels].
 *   gsb_fused_back_mode    as gsb_fused_back; the depth channel's gradient is dropped (the depth is not
 *                          differentiable, Ops.h:67): D / ED give sh0 / shN gradients of zero.
 * A render_mode outside GSB_RENDER_* or channels outside {1, 3, 4} -> GSB_E_UNSUPPORTED, checked first.  The
 * mode passed to the front, the blend's channel count and the mode passed to the back must agree. */
enum GsbRenderMode {
    GSB_RENDER_RGB = 0,
    GSB_RENDER_D = 1,     /* accumulated depth */
    GSB_RENDER_ED = 2,    /* expected depth: accumulated depth / alpha, divided by the caller */
    GSB_RENDER_RGB_D = 3,
    GSB_RENDER_RGB_ED = 4
};
GSB_API int gsb_fused_front_mode(const GsbSplatRaw *splats, const GsbCamera *cam, uint32_t image_width,
                                 uint32_t image_height, float eps2d, float near_plane, float far_plane,
                                 float radius_clip, int zero_moments, int render_mode,
                                 int32_t *radii /*[N,2]*/, float *means2d /*[N,2]*/, float *depths /*[N]*/,
                                 void *workspace, size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_raster_fwd_recs_nc(uint32_t N, uint32_t capacity, uint32_t channels, const void *workspace,
                                   size_t workspace_bytes, const float *depths /*[N]*/, const float *backgrounds,
                                   const uint8_t *masks, uint32_t image_width, uint32_t image_height,
                                   const GsbCamera *cam, const int32_t *tile_offsets /*[th*tw + 1]*/,
                                   const int32_t *flatten_ids, float *renders, float *alphas, int32_t *last_ids,
                                   gsb_stream_t stream);
GSB_API int gsb_raster_bwd_recs_nc(uint32_t N, uint32_t capacity, uint32_t channels, void *workspace,
                                   size_t workspace_bytes, const float *depths /*[N]*/, const float *backgrounds,
                                   const uint8_t *masks, uint32_t image_width, uint32_t image_height,
                                   const GsbCamera *cam, const int32_t *tile_offsets /*[th*tw + 1]*/,
                                   const int32_t *flatten_ids, const float *render_alphas, const int32_t *last_ids,
                                   const float *v_render_colors, const float *v_render_alphas, gsb_stream_t stream);
GSB_API int gsb_fused_back_mode(const GsbSplatRaw *splats, const GsbCamera *cam, uint32_t image_width,
                                uint32_t image_height, int render_mode, const int32_t *radii, const void *workspace,
                                size_t workspace_bytes, float *v_means, float *v_sh0,
                                float *v_shN /*NULL iff K == 1*/, float *v_scaling,
                                float *v_rotation /*16-byte aligned*/, float *v_opacity, gsb_stream_t stream);

/* ---- SURVEY.md 8(f2): photometric loss of the training step and its gradient, one kernel -------------------------
 * loss = (1 - lambda) * mean|clamp(render,0,1) - target| + lambda * (1 - mean SSIM_valid)
 * (src/training/trainer.cpp:103-126; fused_ssim(..., "valid"): 11x11 Gaussian window, zero padding, map cropped by 5
 * per side: src/training/kernels/ssim.cu:64-420, include/kernels/fused_ssim.cuh:27-117).
 * renders [H,W,3] is the blend's output (unclamped); target is [3,H,W] (the reference's layout) or [H,W,3].
 * target_chw is a bit set: GSB_LOSS_TARGET_CHW (1) = target is [3,H,W]; GSB_LOSS_RENDERS_CHW (2) = renders AND v_renders
 * are [3,H,W] planes (the fastgs path's image, SURVEY.md 8 f4).
 * v_renders (laid out like renders) = grad_scale * dLoss/d(renders) including the clamp mask, or NULL to evaluate only.
 * loss_out: DEVICE float[3] = (loss, l1 mean, ssim mean).  workspace: gsb_ssim_l1_workspace() bytes, 256-aligned.
 * GSB_LOSS_NO_CLAMP (4): the renders are used as they are -- no clamp and no clamp mask -- as the reference's loss
 * treats an image that went through the bilateral grid (trainer.cpp:662-665 -> 103-126).
 * NaN propagates: a NaN render makes the loss NaN (the clamp keeps NaN, as torch::clamp does).  Its own gradient is 0
 * with the clamp (the mask 0 <= render <= 1 is false there) and NaN with GSB_LOSS_NO_CLAMP. */
enum { GSB_LOSS_TARGET_CHW = 1, GSB_LOSS_RENDERS_CHW = 2, GSB_LOSS_NO_CLAMP = 4 };
GSB_API size_t gsb_ssim_l1_workspace(void);
GSB_API int gsb_ssim_l1(uint32_t image_width, uint32_t image_height, const float *renders, const float *target,
                        int target_chw, float lambda_dssim, float grad_scale, float *v_renders /*nullable*/,
                        float *loss_out, void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* ---- SURVEY.md 8(f3): Adam over all parameter groups in one launch ---------------------------------------------------
 * The update of fastgs/optimizer/include/adam_kernels.cuh:13-36 (param -= lr * bc1_rcp * m / (sqrt(v) * bc2_sqrt_rcp
 * + eps)); the caller keeps the step counts and learning-rate schedule (src/training/optimizers/fused_adam.cpp:22-95,
 * strategies/strategy_utils.cpp:27-55).  Up to 8 groups; groups with n == 0 are skipped. */
typedef struct GsbAdamGroup {
    float *param;
    const float *grad;
    float *exp_avg;
    float *exp_avg_sq;
    uint64_t n; /* elements */
    float lr, beta1, beta2, eps;
    float bias_correction1_rcp;      /* 1 / (1 - beta1^t) */
    float bias_correction2_sqrt_rcp; /* 1 / sqrt(1 - beta2^t) */
} GsbAdamGroup;
GSB_API int gsb_adam_step(const GsbAdamGroup *groups, uint32_t n_groups, gsb_stream_t stream);
/* Same, with the step-dependent scalars read from DEVICE memory at run time: dynamic_scalars [n_groups][4] floats =
 * (lr, bias_correction1_rcp, bias_correction2_sqrt_rcp, enabled != 0), 16-byte aligned; the lr / bias fields of
 * `groups` are ignored.  Lets a whole training iteration be captured once in a CUDA graph and replayed. */
GSB_API int gsb_adam_step_dynamic(const GsbAdamGroup *groups, uint32_t n_groups, const float *dynamic_scalars,
                                  gsb_stream_t stream);

/* ---- SURVEY.md 8(f4): the reference's default rasterizer ("fastgs", EWA splatting of 2-D conics) ----------------------
 * fast_gs::rasterization::forward / backward (fastgs/rasterization/src/forward.cu:15-199, src/backward.cu:14-116;
 * API fastgs/rasterization/include/rasterization_api.h:25-75 -> include/fastgs/rasterization_api.h + shim/FastGs.cpp).
 * RAW parameters in (log-scales, un-normalised (w,x,y,z) quaternions, logit opacities, sh0 [N,1,3], shN [N,rest,3]),
 * image [3,H,W] and alpha [1,H,W] out (no background: the caller composites it, fast_rasterizer.cpp:71).
 * The three opaque buffers play the role of the reference's per_primitive / per_tile / per_instance blobs: the caller
 * allocates them (sizes below; the instance buffer holds n_instances int32), keeps them from forward to backward and
 * never looks inside.  Forward is two calls because the instance count sizes the third buffer:
 *   gsb_fastgs_forward_plan   per-primitive set-up, depth order, tile histogram; *n_instances_out (DEVICE or PINNED HOST
 *                             int64, written asynchronously on `stream`) = number of (primitive, tile) instances
 *   gsb_fastgs_forward_blend  instances placed in (tile, depth) order, blended; `capacity` = entries of `instances`
 *                             (>= n_instances for an exact result; smaller capacities drop the farthest-sorted slots)
 *   gsb_fastgs_backward       blend gradient + the set-up's chain rule; writes EVERY element of the six gradients
 *                             (the reference zero-fills them first), grad_w2c [4,4] if non-NULL, and adds to
 *                             densification_info [2,N] if non-NULL (kernels_backward.cuh:252-255). */
typedef struct GsbFastgsView {
    const float *w2c;          /* [4,4] world->camera, row-major, DEVICE */
    const float *cam_position; /* [3] DEVICE */
    uint32_t width, height;
    float focal_x, focal_y, center_x, center_y, near_plane, far_plane;
    uint32_t active_sh_bases;     /* 1, 4, 9 or 16 */
    uint32_t total_bases_sh_rest; /* rows of shN per primitive */
} GsbFastgsView;
GSB_API size_t gsb_fastgs_primitive_bytes(uint32_t N, uint32_t width, uint32_t height);
GSB_API size_t gsb_fastgs_tile_bytes(uint32_t width, uint32_t height);
GSB_API int gsb_fastgs_forward_plan(uint32_t N, const float *means, const float *scales_raw,
                                    const float *rotations_raw /*16-byte aligned*/, const float *opacities_raw,
                                    const float *sh0, const float *shN, const GsbFastgsView *view, void *per_primitive,
                                    size_t per_primitive_bytes, void *per_tile, size_t per_tile_bytes,
                                    int64_t *n_instances_out, gsb_stream_t stream);
GSB_API int gsb_fastgs_forward_blend(uint32_t N, const GsbFastgsView *view, void *per_primitive,
                                     size_t per_primitive_bytes, void *per_tile, size_t per_tile_bytes, int32_t *instances,
                                     uint64_t capacity, float *image, float *alpha, gsb_stream_t stream);
GSB_API int gsb_fastgs_backward(uint32_t N, const float *means, const float *scales_raw, const float *rotations_raw,
                                const float *shN, const GsbFastgsView *view,
                                void *per_primitive, size_t per_primitive_bytes, const void *per_tile,
                                size_t per_tile_bytes, const int32_t *instances, uint64_t capacity, const float *alpha,
                                const float *grad_image, const float *grad_alpha, float *grad_means,
                                float *grad_scales_raw, float *grad_rotations_raw /*16-byte aligned*/,
                                float *grad_opacities_raw, float *grad_sh0, float *grad_shN, float *grad_w2c /*nullable*/,
                                float *densification_info /*nullable*/, gsb_stream_t stream);

/* ---- SURVEY.md 8(f5): the bilateral grid of the training iteration (appearance correction per image) ---------------
 * src/training/components/bilateral_grid.cpp:94-127 and src/training/kernels/bilateral_grid_{forward,backward,tv}.cu.
 * grids: [n_images, 12, grid_l, grid_h, grid_w] float32 (grid_w = bilateral_grid_X, grid_h = _Y, grid_l = _W, the
 * guidance depth).  image_idx: DEVICE int32 scalar selecting the grid (NULL = 0), so a captured CUDA graph can slice a
 * different image per replay; an index outside [0, n_images) writes NaN into the output / input gradient.
 * The image is [H,W,3] or, with GSB_BILAGRID_CHW in `layout`, [3,H,W]; the output / gradients have the input's layout.
 * The slice clamps the input to [0,1] first (bilateral_grid.cpp:110); the backward returns the gradient with respect
 * to the UNCLAMPED input (zero where input < 0 or > 1) and ADDS the grid gradient into v_grids (only image_idx's grid
 * is touched).  Image width and height must be >= 2 (the grid coordinates divide by width-1 and height-1).
 * gsb_bilagrid_tv: loss_out (DEVICE float) = (1 / (12 n_images)) * sum over (n, c) of the means of the squared
 * neighbour differences along x, y and z; if v_grids is non-NULL it is WRITTEN in full with *grad_weight (DEVICE float,
 * NULL = 1) times the loss's gradient.  Deterministic; workspace: gsb_bilagrid_tv_workspace() bytes, 256-aligned. */
enum { GSB_BILAGRID_CHW = 1 };
GSB_API int gsb_bilagrid_slice_fwd(uint32_t grid_w, uint32_t grid_h, uint32_t grid_l, uint32_t n_images,
                                   const float *grids, const int32_t *image_idx /*DEVICE, nullable*/, uint32_t image_width,
                                   uint32_t image_height, int layout, const float *input, float *output,
                                   gsb_stream_t stream);
GSB_API int gsb_bilagrid_slice_bwd(uint32_t grid_w, uint32_t grid_h, uint32_t grid_l, uint32_t n_images,
                                   const float *grids, const int32_t *image_idx /*DEVICE, nullable*/, uint32_t image_width,
                                   uint32_t image_height, int layout, const float *input, const float *v_output,
                                   float *v_grids /*added into*/, float *v_input, gsb_stream_t stream);
GSB_API size_t gsb_bilagrid_tv_workspace(void);
GSB_API int gsb_bilagrid_tv(uint32_t grid_w, uint32_t grid_h, uint32_t grid_l, uint32_t n_images, const float *grids,
                            const float *grad_weight /*DEVICE, nullable*/, float *loss_out, float *v_grids /*nullable*/,
                            void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* ---- link-surface ops used by the densification strategies -------------------------
 * gsplat::quats_to_rotmats (Ops.h:46-48, QuatToRotmatCUDA.cu:14-39): [N,4] -> [N,3,3] */
GSB_API int gsb_quat_to_rotmat(uint32_t N, const float *quats, float *rotmats, gsb_stream_t stream);
/* gsplat::relocation (Ops.h:52-57, RelocationCUDA.cu:12-43) */
GSB_API int gsb_relocation(uint32_t N, const float *opacities, const float *scales, const int32_t *ratios,
                           const float *binoms, int32_t n_max, float *new_opacities, float *new_scales,
                           gsb_stream_t stream);
/* gsplat::add_noise (Ops.h:59-65, RelocationCUDA.cu:113-144): means updated in place */
GSB_API int gsb_add_noise(uint32_t N, const float *raw_opacities, const float *raw_scales,
                          const float *raw_quats, const float *noise, float *means, float current_lr,
                          gsb_stream_t stream);

/* ---- SURVEY.md 8(f6): MCMC densification (src/training/strategies/mcmc.cpp:112-393, trainer.cpp:132-158) -------------
 * All counts that depend on the data stay in DEVICE memory: a refine never synchronises with the host.  Indices are
 * int32.  rotation_raw / raw_quats are read as float4: they must be 16-byte aligned (GSB_E_INVALID otherwise).  The four compute calls share one workspace of gsb_mcmc_workspace(N) bytes, 256-aligned.
 *
 * gsb_mcmc_dead: a Gaussian is dead when sigmoid(opacity_raw) <= min_opacity or |rotation_raw|^2 < 1e-8.  Writes the
 *   ascending dead indices to dead_idx[0 .. *n_dead) (dead_idx holds N entries, *n_dead is a DEVICE uint32) and the
 *   sampling weights: sigmoid(opacity_raw) where alive, 0 where dead.
 * gsb_mcmc_sample: draws with replacement, weighted; sample j is the first i with C[i] > u_j * C[N-1], C the float64
 *   inclusive prefix of the weights (or of sigmoid(weights) with weights_are_logits), so a zero weight is never drawn.
 *   Draws min(n_samples, *n_samples_dev) samples (n_samples_dev: DEVICE uint32, nullable).  u_j in [0, 1) is
 *   uniforms[j] (DEVICE float64, the test hook) or comes from the Philox state `philox` (torch's generator state; under
 *   CUDA-graph capture its seed and offset are device pointers).  A sample is -1 when every weight is 0; a sample that
 *   rounding of the prefix would put on a zero weight moves to the nearest positive one.
 * gsb_mcmc_apply: targets non-NULL -- relocation (mcmc.cpp:112-190): sample j is copied onto row targets[j];
 *   targets NULL -- growth (:192-347): onto row N + j (the caller's storage holds the rows).  ratio = min(copies of the
 *   sample + 1, n_max) (binoms: [n_max][n_max] float), relocation's opacity clamped to [min_opacity, 1 - 1e-7]; the
 *   sampled row and the target receive logit(opacity) and log(scale), the target a copy of means, sh0, shN and
 *   rotation.  Adam moments: zeroed at the sampled rows when relocating (the targets keep theirs, as the reference's
 *   update_optimizer_for_relocate does) and at the new rows when growing.  Samples < 0 are skipped. */
typedef struct GsbPhilox {
    uint64_t seed;
    uint64_t offset;
    const uint64_t *seed_ptr;   /* non-NULL under graph capture: the seed is read from the device */
    const int64_t *offset_ptr;  /* non-NULL under graph capture: offset = *offset_ptr + offset_intragraph */
    uint64_t offset_intragraph;
} GsbPhilox;
typedef struct GsbMcmcRows {
    float *means;         /* [rows,3] */
    float *sh0;           /* [rows,1,3] */
    float *shN;           /* [rows,shN_rows,3]; NULL iff shN_rows == 0 */
    float *scaling_raw;   /* [rows,3] */
    float *rotation_raw;  /* [rows,4], 16-byte aligned */
    float *opacity_raw;   /* [rows] */
    uint32_t shN_rows;
    /* Adam moments in the order means, sh0, shN, scaling_raw, rotation_raw, opacity_raw; NULL entries are skipped */
    float *exp_avg[6];
    float *exp_avg_sq[6];
} GsbMcmcRows;
GSB_API size_t gsb_mcmc_workspace(uint32_t N);
GSB_API int gsb_mcmc_dead(uint32_t N, const float *opacity_raw, const float *rotation_raw, float min_opacity,
                          int32_t *dead_idx, uint32_t *n_dead, float *weights, void *workspace, size_t workspace_bytes,
                          gsb_stream_t stream);
GSB_API int gsb_mcmc_sample(uint32_t N, const float *weights, int weights_are_logits, uint32_t n_samples,
                            const uint32_t *n_samples_dev /*nullable*/, const double *uniforms /*nullable*/,
                            const GsbPhilox *philox /*nullable iff uniforms*/, int32_t *samples, void *workspace,
                            size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_mcmc_apply(uint32_t N, const GsbMcmcRows *rows, const int32_t *samples, uint32_t n_samples,
                           const uint32_t *n_samples_dev /*nullable*/, const int32_t *targets /*NULL: growth*/,
                           const float *binoms, int32_t n_max, float min_opacity, void *workspace,
                           size_t workspace_bytes, gsb_stream_t stream);
/* gsb_add_noise with the rate read on the device: current_lr = *lr * lr_scale (e.g. the means group's learning rate
 * from the graphed step's scalars times the strategy's 5e5), so that the noise can be captured in a CUDA graph. */
GSB_API int gsb_mcmc_add_noise(uint32_t N, const float *raw_opacities, const float *raw_scales,
                               const float *raw_quats, const float *noise, float *means, const float *lr /*DEVICE*/,
                               float lr_scale, gsb_stream_t stream);
/* The trainer's regularisers: adds scale_reg * exp(s) / (3N) into v_scaling and opacity_reg * sigmoid(o) (1 -
 * sigmoid(o)) / N into v_opacity (either nullable: that term is skipped) and writes loss_out (DEVICE float[2]) =
 * (scale_reg * mean(exp(scaling_raw)), opacity_reg * mean(sigmoid(opacity_raw))).  Deterministic. */
GSB_API int gsb_mcmc_regularize(uint32_t N, const float *scaling_raw, const float *opacity_raw, float scale_reg,
                                float opacity_reg, float *v_scaling, float *v_opacity, float *loss_out,
                                void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* ---- Adaptive density control, the default densification strategy (src/training/strategies/default_strategy.cpp:
 * 164-290) --------------------------------------------------------------------------------------------------------------
 * A refine -- grow_gs (duplicate, then split) followed by prune_gs -- is one compaction into freshly allocated rows:
 *   gsb_adc_classify: per row, with g = info[1] / max(info[0], 1) (densification_info [2,N]; NULL: no row is high):
 *     duplicate = g > grad_threshold and max(exp(scaling_raw)) <= grow_scale3d * scene_scale; split = g >
 *     grad_threshold and not small.  prune_gs then removes a row (original, duplicate copy or split copy) when
 *     sigmoid(opacity_raw) < prune_opacity, |rotation_raw|^2 < 1e-8 or, when prune_too_big, max(exp(scaling_raw)) >
 *     prune_scale3d * scene_scale.  Writes counts (DEVICE int32[8]): [0] duplicated, [1] split, [2] pruned from the
 *     grown set, [3] final rows, [4..6] kept rest rows / duplicate copies / split rows, [7] 0.  The flags and ranks stay
 *     in the workspace for gsb_adc_apply.  N must be at most INT32_MAX / 2 (the grown set of N + n_dup + n_split <= 2N
 *     rows is indexed in int32).
 *   gsb_adc_apply: writes the final rows into dst (which holds n_final = counts[3] rows; n_split = counts[1], both read
 *     back by the caller) in the reference's order: kept rows that were not split, kept duplicate copies, copy 0 of
 *     every kept split row, copy 1 of every kept split row.  Copy b of split row i takes means + R(normalize(q))
 *     (exp(scaling_raw) * z[b, rank of i among split rows]) (z: [2, n_split, 3], torch::randn's draw), scaling_raw =
 *     log(exp(scaling_raw) * (1.0f / 1.6f)) and, with revised_opacity, opacity_raw = logit(1 - sqrt(1 -
 *     sigmoid(opacity_raw))).  Adam moments: copied for kept original rows, zero for new rows (NULL entries skipped).
 *     densification_info (nullable) receives zeros [2, n_final].  Same workspace and params as the classify call.
 *   gsb_adc_reset_opacity: opacity_raw = min(opacity_raw, logit(2 prune_opacity)) (the logit in float), the opacity
 *     group's moments (nullable) zeroed.
 * rotation_raw is read as float4: 16-byte aligned (GSB_E_INVALID otherwise).  Workspace: gsb_adc_workspace(N) bytes,
 * 256-aligned. */
typedef struct GsbAdcParams {
    float grad_threshold;
    float grow_scale3d;
    float prune_scale3d;
    float scene_scale;
    float prune_opacity;
    int32_t prune_too_big;   /* iter > reset_every */
    int32_t revised_opacity;
} GsbAdcParams;
GSB_API size_t gsb_adc_workspace(uint32_t N);
GSB_API int gsb_adc_classify(uint32_t N, const float *densification_info /*nullable*/, const float *scaling_raw,
                             const float *rotation_raw, const float *opacity_raw, const GsbAdcParams *params,
                             int32_t *counts /*DEVICE [8]*/, void *workspace, size_t workspace_bytes,
                             gsb_stream_t stream);
GSB_API int gsb_adc_apply(uint32_t N, const GsbMcmcRows *src, const GsbMcmcRows *dst, uint32_t n_split,
                          uint32_t n_final, const float *z /*nullable iff n_split == 0*/, const GsbAdcParams *params,
                          const int32_t *counts /*DEVICE, from gsb_adc_classify*/, float *densification_info /*nullable*/,
                          void *workspace, size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_adc_reset_opacity(uint32_t N, float *opacity_raw, float prune_opacity, float *exp_avg /*nullable*/,
                                  float *exp_avg_sq /*nullable*/, gsb_stream_t stream);

/* ---- ADMM opacity sparsification (src/training/components/sparsity_optimizer.cpp) ------------------------------------
 * s = sigmoid(opacity_raw) in float; k = (int)(prune_ratio * N) as the caller forms it (a float product); prune_z(x) =
 * (x > x_(k)) * x with x_(k) the k-th smallest of x (NaN sorts last), and 0 when k == 0.  The k-th value is found by
 * radix passes on the device and never read back: every call below is stream-ordered and graph-capturable.
 *   gsb_sparsity_update: initialize != 0: u = 0, z = prune_z(s + u); otherwise zt = s + u, z = prune_z(zt),
 *     u += s - z.  z, u: [N] float, bit for bit as torch computes them.  k must be at most N.
 *   gsb_sparsity_loss: loss_out (DEVICE float[1]) = 0.5 * rho * ||s - z + u||^2 (reduced deterministically) and
 *     rho (s - z + u) s (1 - s) added into v_opacity [N].  rho is DEVICE float[1]; rho == 0 writes 0 and leaves
 *     v_opacity alone.
 *   Workspace: gsb_sparsity_workspace(N) bytes, 256-aligned.
 *   gsb_adc_prune_classify: the final prune as a compaction for gsb_adc_apply.  Removes exactly n_prune rows: every
 *     row with s below v, the n_prune-th smallest s, then the first rows in index order with s == v.  Writes counts
 *     (DEVICE int32[8]) as gsb_adc_classify does -- [2] = n_prune, [3] = [4] = N - n_prune, the rest 0 -- and the
 *     flags and ranks that gsb_adc_apply(N, src, dst, 0, N - n_prune, NULL, ...) reads.  Workspace:
 *     gsb_adc_workspace(N) bytes, 256-aligned; N at most INT32_MAX / 2. */
GSB_API size_t gsb_sparsity_workspace(uint32_t N);
GSB_API int gsb_sparsity_update(uint32_t N, const float *opacity_raw, float *z, float *u, uint32_t k, int initialize,
                                void *workspace, size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_sparsity_loss(uint32_t N, const float *opacity_raw, const float *z, const float *u,
                              const float *rho /*DEVICE*/, float *v_opacity, float *loss_out /*DEVICE*/,
                              void *workspace, size_t workspace_bytes, gsb_stream_t stream);
GSB_API int gsb_adc_prune_classify(uint32_t N, const float *opacity_raw, uint32_t n_prune,
                                   int32_t *counts /*DEVICE [8]*/, void *workspace, size_t workspace_bytes,
                                   gsb_stream_t stream);

/* ---- Evaluation metrics (src/training/metrics/metrics.cpp:17-116, PSNR::compute and SSIM::compute) -------------------
 * gsb_image_metrics: one view's (psnr, ssim) as float32 into out (DEVICE float[2]), in one launch and with no host
 * read-back, so a caller can fill [V,2] for V views and read it once.  x = clamp(image, 0, 1), y = target:
 *   psnr = 20 log10(1 / sqrt(max(mean((x - y)^2), 1e-10))) over all 3 H W values (100 for identical images);
 *   ssim = mean of the SSIM map over all 3 H W values: 11 x 11 window with zero padding 5 ("same" size, no crop),
 *          per channel, C1 = 0.01^2, C2 = 0.03^2, sigma^2 = E[x^2] - mu^2.  The window is the reference's gaussian(11,
 *          1.5), whose float32 taps are exp(-d^2 * 1.125) normalised (its inv_denom evaluates to 1.125).
 * target is [3,H,W]; image is [3,H,W], or [H,W,3] with GSB_METRICS_IMAGE_HWC in flags.  W, H >= 1 and 3 W H at most
 * INT32_MAX; images smaller than the window are fine.  The sums are float64 and reduced in an order fixed by W and H:
 * repeated calls give the same bits.  Workspace: gsb_image_metrics_workspace() bytes, 256-aligned; its ticket is zeroed
 * on the stream, so the call can be captured in a CUDA graph. */
enum { GSB_METRICS_IMAGE_HWC = 1 };
GSB_API size_t gsb_image_metrics_workspace(void);
GSB_API int gsb_image_metrics(uint32_t W, uint32_t H, const float *image, const float *target, uint32_t flags,
                              float *out /*DEVICE [2]*/, void *workspace, size_t workspace_bytes, gsb_stream_t stream);

/* ---- Model set-up: initial scales (src/core/splat_data.cpp:63-111, compute_mean_neighbor_distances) ------------------
 * gsb_knn_mean_dist: for each of the N points (DEVICE float[N,3]) the mean distance to its nearest neighbours, into out
 * (DEVICE float[N]), computed exactly (the reference's nanoflann query uses eps = 10 and is approximate):
 *   the k = min(4, N) smallest squared distances over all points, the point itself and its duplicates included, each
 *   ((dx*dx) + (dy*dy)) + (dz*dz) in float32 without FMA, dx = q.x - p.x; walked in ascending order, the first (at most
 *   3) with d2 > 1e-8f are averaged as sqrtf values summed in float32 in that order; 0.01f when none qualifies.
 * status (DEVICE uint32[1]) is written on the stream: 0, or GSB_KNN_NONFINITE when a coordinate is NaN or infinite (out
 * is then unspecified).  N == 0 only writes status.  N at most GSB_KNN_MAX_POINTS.  Workspace:
 * gsb_knn_mean_dist_workspace(N) bytes, 256-aligned; its counters are reset on the stream, so the call can be captured
 * in a CUDA graph.  Each value depends only on the point set, not on the search order: repeated calls give the same
 * bits. */
enum { GSB_KNN_NONFINITE = 1 };
#define GSB_KNN_MAX_POINTS (1u << 28)
GSB_API size_t gsb_knn_mean_dist_workspace(uint32_t N);
GSB_API int gsb_knn_mean_dist(uint32_t N, const float *points, float *out, void *workspace, size_t workspace_bytes,
                              uint32_t *status /*DEVICE [1]*/, gsb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GSB200_H_ */
