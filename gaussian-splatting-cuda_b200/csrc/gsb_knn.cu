// gsb_knn.cu -- mean distance to the nearest neighbours of every point of a cloud: the initial scale of
// SplatData::init_model_from_pointcloud (src/core/splat_data.cpp:63-111, compute_mean_neighbor_distances), computed
// EXACTLY.  For each point i:
//   d2 = the min(4, N) smallest squared distances over all points, i itself and its duplicates included
//        (KNNResultSet(4)); each is ((dx*dx) + (dy*dy)) + (dz*dz) in float32, dx = q.x - p.x (L2_Simple_Adaptor), with
//        no FMA (this file is built with -fmad=false and spells the operations out);
//   out[i] = the mean of sqrtf of the first (at most 3) of them, in ascending order, with d2 > 1e-8f, summed in float32
//            in that order; 0.01f when none qualifies (so for every point when N == 1).
// The result is a function of the sorted distance multiset, so ties and the order of equal candidates change nothing.
// The reference's nanoflann search runs with eps = 10 (SearchParameters(10)) and is approximate; see DESIGN.md 4.17.
//
// Algorithm: a uniform grid over a sigma-clipped box, searched in growing Chebyshev shells.
//   1. stats_kernel / plan_kernel: the bounding box and (in two more passes) the mean and deviation of the points
//      inside the current box; the grid box is mean +- 4 sigma clipped twice, so a few far outliers do not stretch the
//      cells over the bulk.  The cell size is the smallest that keeps the cell count at most 2 N.  A point outside the
//      box goes to the nearest boundary cell; the shell bound below stays valid for it (its cell index along an axis
//      still says on which side of every inner cell boundary it lies).  These statistics only shape the grid: the
//      result is exact whatever they are.
//   2. key_kernel + gsb_devsort.cuh: points sorted by cell; gsb_scan.cuh: inclusive scan of the cell counts = the end
//      of every cell's run.  A row of cells along x is one contiguous run of sorted points.
//   3. query_kernel: one thread per sorted point.  Shell r visits the cells at Chebyshev distance r from the query's
//      cell.  After shell r every unvisited point lies beyond one of the six planes bounding the visited cube, so its
//      distance is at least g = the query's distance to the nearest such plane (infinite where the cube reaches the
//      grid's side).  The search stops once the k-th best squared distance is <= g^2 (1 - 1e-6): the computed float
//      distance of any unvisited point is at least that (the cell coordinates are float64, the float32 distance's
//      relative error is below 2^-21), so it cannot change the k smallest values.  Past kMaxShell shells the query
//      is handed on, so a far outlier costs a bounded number of shells here.
//   4. fallback_kernel: those queries scan all points, eight per CTA over points staged in shared memory, each lane
//      keeping its own four best, merged across the warp by a butterfly.
// Non-finite coordinates set GSB_KNN_NONFINITE in the status word and leave `out` unspecified.  Every buffer lives
// in the caller's workspace; the status word and counters are reset on the stream, so the call can be captured in a
// CUDA graph.
#include <cfloat>
#include <cmath>

#include "gsb_common.cuh"
#include "gsb_devsort.cuh"
#include "gsb_scan.cuh"

namespace gsb {
namespace knn {

constexpr int kThreads = 256;
constexpr uint32_t kStatBlocks = 1056; // 8 CTAs of 256 threads on each of the H100's 132 SMs
constexpr uint32_t kFallbackBlocks = 264;
constexpr int kClipPasses = 2;         // sigma-clipping passes after the bounding box
constexpr double kClipSigmas = 4.0;
constexpr int kMaxShell = 10;
constexpr uint32_t kScanBlocks = 264;
constexpr int kStage = 1024;           // points staged per round of fallback_kernel

struct Grid {
    double lo[3];
    double inv_h, h;
    int dims[3];
    uint32_t pad;
};

struct Ctl {
    uint32_t status;
    uint32_t n_fallback;
    uint32_t mn[3], mx[3];             // order-preserving encodings of the bounding box
    double stats[kClipPasses + 1][7];  // count, sum x y z, sum x^2 y^2 z^2 of the points inside box[pass]
    double box[kClipPasses + 1][2][3]; // box[pass] is set by plan_kernel(pass - 1); box[0] is the bounding box
    Grid grid;
};

struct Ws {
    Ctl *ctl;
    uint32_t *k0, *k1, *v0, *v1, *hist;
    int32_t *cnt, *cell_end;
    long long *bsum;
    float4 *spts;
    uint32_t *fb;
};

static uint64_t max_cells(uint32_t N) { return N ? 2ull * N : 1ull; }

static size_t ws_layout(uint32_t N, void *base, Ws &w) {
    const uint64_t C = max_cells(N);
    const ScanPlan sort = scan_plan(N, kScanBlocks), cells = scan_plan(C, kScanBlocks);
    WsLayout l{static_cast<char *>(base)};
    w.ctl = l.carve<Ctl>(1);
    w.k0 = l.carve<uint32_t>(N);
    w.k1 = l.carve<uint32_t>(N);
    w.v0 = l.carve<uint32_t>(N);
    w.v1 = l.carve<uint32_t>(N);
    w.hist = l.carve<uint32_t>((size_t)sort.nblocks * kRadixBins);
    w.cnt = l.carve<int32_t>(C);
    w.cell_end = l.carve<int32_t>(C);
    w.bsum = l.carve<long long>(cells.nblocks);
    w.spts = l.carve<float4>(N);
    w.fb = l.carve<uint32_t>(N);
    return l.bytes;
}

// float <-> an unsigned key with the same order (atomicMin / atomicMax on the bounding box)
__device__ __forceinline__ uint32_t ord_key(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord_val(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void init_kernel(Ctl *c) {
    uint32_t *w = reinterpret_cast<uint32_t *>(c);
    for (uint32_t i = threadIdx.x; i < sizeof(Ctl) / 4; i += blockDim.x) w[i] = 0u;
    __syncthreads();
    if (threadIdx.x < 3) c->mn[threadIdx.x] = 0xffffffffu;
}

__device__ __forceinline__ bool in_box(const Ctl *c, int pass, float x, float y, float z) {
    const double p[3] = {x, y, z};
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (p[a] < c->box[pass][0][a] || p[a] > c->box[pass][1][a]) return false;
    return true;
}

// pass 0: finiteness, bounding box and moments of every point; pass > 0: moments of the points inside box[pass]
__global__ void __launch_bounds__(kThreads) stats_kernel(const float *__restrict__ pts, uint32_t N, int pass, Ctl *c) {
    double s[7] = {0, 0, 0, 0, 0, 0, 0};
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    bool bad = false;
    for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < N; i += gridDim.x * kThreads) {
        const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) {
            bad = true;
            continue;
        }
        if (pass == 0) {
            mn[0] = fminf(mn[0], x); mn[1] = fminf(mn[1], y); mn[2] = fminf(mn[2], z);
            mx[0] = fmaxf(mx[0], x); mx[1] = fmaxf(mx[1], y); mx[2] = fmaxf(mx[2], z);
        } else if (!in_box(c, pass, x, y, z)) {
            continue;
        }
        s[0] += 1.0;
        s[1] += x; s[2] += y; s[3] += z;
        s[4] += (double)x * x; s[5] += (double)y * y; s[6] += (double)z * z;
    }
    // the sums only shape the grid, so their order does not matter: warp butterflies, then one atomic per warp
#pragma unroll
    for (int k = 0; k < 7; ++k)
        for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
    if (pass == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
            for (int o = 16; o > 0; o >>= 1) {
                mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
                mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
            }
    }
    bad = __any_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) {
        if (bad) atomicOr(&c->status, (uint32_t)GSB_KNN_NONFINITE);
        if (s[0] > 0.0) {
#pragma unroll
            for (int k = 0; k < 7; ++k) atomicAdd(&c->stats[pass][k], s[k]);
            if (pass == 0) {
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    atomicMin(&c->mn[a], ord_key(mn[a]));
                    atomicMax(&c->mx[a], ord_key(mx[a]));
                }
            }
        }
    }
}

// one thread: box[pass + 1] from the moments of pass `pass`; after the last pass, the grid
__global__ void plan_kernel(Ctl *c, int pass, uint64_t max_cells) {
    if (pass == 0) {
        for (int a = 0; a < 3; ++a) {
            const bool any = c->stats[0][0] > 0.0;
            c->box[0][0][a] = any ? (double)ord_val(c->mn[a]) : 0.0;
            c->box[0][1][a] = any ? (double)ord_val(c->mx[a]) : 0.0;
        }
    }
    const double *s = c->stats[pass];
    for (int a = 0; a < 3; ++a) {
        double lo = c->box[pass][0][a], hi = c->box[pass][1][a];
        if (s[0] > 0.0) {
            const double mean = s[1 + a] / s[0];
            const double sd = sqrt(fmax(s[4 + a] / s[0] - mean * mean, 0.0));
            lo = fmax(lo, mean - kClipSigmas * sd);
            hi = fmin(hi, mean + kClipSigmas * sd);
            if (!(lo <= hi)) lo = hi = mean; // rounding in a degenerate axis
        }
        c->box[pass + 1][0][a] = lo;
        c->box[pass + 1][1][a] = hi;
    }
    if (pass + 1 < kClipPasses) return;

    Grid &g = c->grid;
    double ext[3], emax = 0.0;
    for (int a = 0; a < 3; ++a) {
        g.lo[a] = c->box[kClipPasses][0][a];
        ext[a] = c->box[kClipPasses][1][a] - g.lo[a];
        emax = fmax(emax, ext[a]);
    }
    if (!(emax > 0.0)) { // one cell
        g.inv_h = 0.0;
        g.h = 1.0;
        g.dims[0] = g.dims[1] = g.dims[2] = 1;
        return;
    }
    // the smallest cell size h with prod(floor(ext / h) + 1) <= max_cells, by bisection on log h
    auto cells = [&](double h, int *d) {
        double n = 1.0;
        for (int a = 0; a < 3; ++a) {
            const double k = floor(ext[a] / h) + 1.0;
            if (d) d[a] = (int)k;
            n *= k;
        }
        return n;
    };
    double hlo = emax / (double)max_cells, hhi = 2.0 * emax; // cells(hlo) > max_cells >= cells(hhi) = 1
    for (int it = 0; it < 64; ++it) {
        const double mid = sqrt(hlo * hhi);
        if (cells(mid, nullptr) <= (double)max_cells) hhi = mid; else hlo = mid;
    }
    cells(hhi, g.dims);
    g.h = hhi;
    g.inv_h = 1.0 / hhi;
}

__device__ __forceinline__ int cell_coord(double t, int dim) {
    return (int)fmin(fmax(floor(t), 0.0), (double)(dim - 1));
}

__device__ __forceinline__ void coords(const Grid &g, float x, float y, float z, double t[3], int cc[3]) {
    const float p[3] = {x, y, z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        t[a] = ((double)p[a] - g.lo[a]) * g.inv_h;
        cc[a] = cell_coord(t[a], g.dims[a]);
    }
}

__device__ __forceinline__ uint32_t cell_id(const Grid &g, const int cc[3]) {
    return (uint32_t)(((uint64_t)cc[2] * g.dims[1] + cc[1]) * g.dims[0] + cc[0]);
}

__global__ void __launch_bounds__(kThreads) key_kernel(const float *__restrict__ pts, uint32_t N, const Ctl *__restrict__ c,
                                                       uint32_t *__restrict__ keys, uint32_t *__restrict__ vals,
                                                       int32_t *__restrict__ cnt) {
    const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= N) return;
    const Grid g = c->grid;
    double t[3];
    int cc[3];
    coords(g, pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], t, cc);
    const uint32_t key = cell_id(g, cc);
    keys[i] = key;
    vals[i] = i;
    atomicAdd(&cnt[key], 1);
}

__global__ void __launch_bounds__(kThreads) gather_kernel(const float *__restrict__ pts, uint32_t N,
                                                          const uint32_t *__restrict__ order, float4 *__restrict__ spts) {
    const uint32_t j = blockIdx.x * kThreads + threadIdx.x;
    if (j >= N) return;
    const size_t i = order[j];
    spts[j] = make_float4(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 0.0f);
}

// the four smallest squared distances seen so far, ascending; +inf where none yet
struct Best4 {
    float d[4];
    __device__ __forceinline__ void init() { d[0] = d[1] = d[2] = d[3] = INFINITY; }
    __device__ __forceinline__ float kth(uint32_t k) const { // d[k - 1] without dynamic indexing
        return k >= 4 ? d[3] : k == 3 ? d[2] : k == 2 ? d[1] : d[0];
    }
    __device__ __forceinline__ void insert(float v) {
        if (!(v < d[3])) return; // equal values leave the multiset of the four smallest unchanged
        d[3] = v;
        if (d[3] < d[2]) { const float t = d[2]; d[2] = d[3]; d[3] = t; }
        if (d[2] < d[1]) { const float t = d[1]; d[1] = d[2]; d[2] = t; }
        if (d[1] < d[0]) { const float t = d[0]; d[0] = d[1]; d[1] = t; }
    }
};

// L2_Simple_Adaptor's accumulation, without contraction
__device__ __forceinline__ float dist2(float qx, float qy, float qz, float4 p) {
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// compute_mean_neighbor_distances' loop over the k = min(4, N) results
__device__ __forceinline__ float mean_of_best(const Best4 &b, uint32_t k) {
    float sum = 0.0f;
    int valid = 0;
#pragma unroll
    for (uint32_t j = 0; j < 4; ++j) {
        if (j < k && valid < 3 && b.d[j] > 1e-8f) {
            sum = __fadd_rn(sum, __fsqrt_rn(b.d[j]));
            ++valid;
        }
    }
    return valid > 0 ? __fdiv_rn(sum, (float)valid) : 0.01f;
}

__global__ void __launch_bounds__(kThreads) query_kernel(uint32_t N, const float4 *__restrict__ spts,
                                                         const uint32_t *__restrict__ order,
                                                         const int32_t *__restrict__ cell_end, Ctl *__restrict__ c,
                                                         uint32_t *__restrict__ fb, float *__restrict__ out) {
    const uint32_t j = blockIdx.x * kThreads + threadIdx.x;
    if (j >= N || c->status) return;
    const Grid g = c->grid;
    const uint32_t k = N < 4 ? N : 4;
    const float4 q = spts[j];
    double t[3];
    int cc[3];
    coords(g, q.x, q.y, q.z, t, cc);
    Best4 b;
    b.init();
    for (int r = 0;; ++r) {
        const int z0 = max(cc[2] - r, 0), z1 = min(cc[2] + r, g.dims[2] - 1);
        const int y0 = max(cc[1] - r, 0), y1 = min(cc[1] + r, g.dims[1] - 1);
        const int x0 = max(cc[0] - r, 0), x1 = min(cc[0] + r, g.dims[0] - 1);
        for (int z = z0; z <= z1; ++z) {
            for (int y = y0; y <= y1; ++y) {
                const bool shell = abs(z - cc[2]) == r || abs(y - cc[1]) == r;
                const uint32_t row = ((uint32_t)z * g.dims[1] + y) * g.dims[0];
                // a row on the shell is scanned whole; inside it, only its two end cells are on the shell
                for (int part = 0; part < 2; ++part) {
                    int xa, xb;
                    if (shell) {
                        if (part) break;
                        xa = x0; xb = x1;
                    } else {
                        xa = xb = part ? cc[0] + r : cc[0] - r;
                        if (xa < 0 || xa >= g.dims[0]) continue;
                    }
                    const uint32_t ca = row + xa, cb = row + xb;
                    const int32_t lo = ca ? cell_end[ca - 1] : 0, hi = cell_end[cb];
                    for (int32_t p = lo; p < hi; ++p) b.insert(dist2(q.x, q.y, q.z, spts[p]));
                }
            }
        }
        // distance from q to the nearest face of the visited cube that has unvisited cells beyond it
        double gap = INFINITY;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (cc[a] - r > 0) gap = fmin(gap, t[a] - (double)(cc[a] - r));
            if (cc[a] + r < g.dims[a] - 1) gap = fmin(gap, (double)(cc[a] + r + 1) - t[a]);
        }
        if (gap == INFINITY) break; // every cell visited
        const double lb = gap * g.h;
        if (lb > 0.0 && (double)b.kth(k) <= lb * lb * (1.0 - 1e-6)) break;
        if (r == kMaxShell) {
            fb[atomicAdd(&c->n_fallback, 1u)] = j;
            return;
        }
    }
    out[order[j]] = mean_of_best(b, k);
}

__device__ __forceinline__ void merge_warp(Best4 &b) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float other[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) other[m] = __shfl_xor_sync(0xffffffffu, b.d[m], o);
#pragma unroll
        for (int m = 0; m < 4; ++m) b.insert(other[m]);
    }
}

// the handed-on queries against every point: warp w of a CTA takes query (round * 8 + w) of the CTA's share
__global__ void __launch_bounds__(kThreads) fallback_kernel(uint32_t N, const float4 *__restrict__ spts,
                                                            const uint32_t *__restrict__ order, const Ctl *__restrict__ c,
                                                            const uint32_t *__restrict__ fb, float *__restrict__ out) {
    __shared__ float4 s_pts[kStage];
    if (c->status) return;
    const uint32_t nq = c->n_fallback;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t k = N < 4 ? N : 4;
    constexpr uint32_t kWarps = kThreads / 32;
    for (uint32_t base = blockIdx.x * kWarps; base < nq; base += gridDim.x * kWarps) {
        const uint32_t qi = base + warp;
        const bool active = qi < nq;
        const uint32_t j = active ? fb[qi] : 0u;
        const float4 q = spts[j];
        Best4 b;
        b.init();
        for (uint32_t p0 = 0; p0 < N; p0 += kStage) {
            const uint32_t n = N - p0 < (uint32_t)kStage ? N - p0 : (uint32_t)kStage;
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < n; i += kThreads) s_pts[i] = spts[p0 + i];
            __syncthreads();
            if (active)
                for (uint32_t i = lane; i < n; i += 32) b.insert(dist2(q.x, q.y, q.z, s_pts[i]));
        }
        merge_warp(b);
        if (active && lane == 0) out[order[j]] = mean_of_best(b, k);
    }
}

} // namespace knn
} // namespace gsb

extern "C" size_t gsb_knn_mean_dist_workspace(uint32_t N) {
    gsb::knn::Ws w;
    return gsb::knn::ws_layout(N, nullptr, w);
}

extern "C" int gsb_knn_mean_dist(uint32_t N, const float *points, float *out, void *workspace, size_t workspace_bytes,
                                 uint32_t *status, gsb_stream_t stream) {
    using namespace gsb;
    using namespace gsb::knn;
    if (N > GSB_KNN_MAX_POINTS || !status || (N && (!points || !out))) return GSB_E_INVALID;
    Ws w;
    if (int rc = ws_check(workspace, workspace_bytes, ws_layout(N, workspace, w))) return rc;
    cudaStream_t s = as_stream(stream);
    ProfScope ps("knn_mean_dist", s);
    init_kernel<<<1, 256, 0, s>>>(w.ctl);
    GSB_LAUNCH_CHECK();
    if (N) {
        const uint32_t sb = (uint32_t)ceil_div(N, kThreads) < kStatBlocks ? (uint32_t)ceil_div(N, kThreads) : kStatBlocks;
        const uint64_t C = max_cells(N);
        for (int pass = 0; pass < kClipPasses; ++pass) {
            stats_kernel<<<sb, kThreads, 0, s>>>(points, N, pass, w.ctl);
            GSB_LAUNCH_CHECK();
            plan_kernel<<<1, 1, 0, s>>>(w.ctl, pass, C);
            GSB_LAUNCH_CHECK();
        }
        GSB_CUDA_TRY(cudaMemsetAsync(w.cnt, 0, C * sizeof(int32_t), s));
        const uint32_t nb = (uint32_t)ceil_div(N, kThreads);
        key_kernel<<<nb, kThreads, 0, s>>>(points, N, w.ctl, w.k0, w.v0, w.cnt);
        GSB_LAUNCH_CHECK();
        if (int rc = scan_launch(LoadI32{w.cnt}, C, scan_plan(C, kScanBlocks), w.bsum, w.cell_end, s)) return rc;
        const uint32_t key_bits = bit_width_u32((uint32_t)(C - 1));
        const int passes = (int)ceil_div(key_bits, 8);
        if (int rc = radix_sort_launch<uint32_t>(w.k0, w.k1, w.v0, w.v1, N, scan_plan(N, kScanBlocks), passes, 0,
                                                 key_bits, nullptr, w.hist, s))
            return rc;
        const uint32_t *order = (passes & 1) ? w.v1 : w.v0;
        gather_kernel<<<nb, kThreads, 0, s>>>(points, N, order, w.spts);
        GSB_LAUNCH_CHECK();
        query_kernel<<<nb, kThreads, 0, s>>>(N, w.spts, order, w.cell_end, w.ctl, w.fb, out);
        GSB_LAUNCH_CHECK();
        fallback_kernel<<<kFallbackBlocks, kThreads, 0, s>>>(N, w.spts, order, w.ctl, w.fb, out);
        GSB_LAUNCH_CHECK();
    }
    GSB_CUDA_TRY(cudaMemcpyAsync(status, &w.ctl->status, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
    return GSB_OK;
}
