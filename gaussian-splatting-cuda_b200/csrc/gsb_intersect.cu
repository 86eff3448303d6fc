// gsb_intersect.cu -- a5/a6: Gaussian -> tile expansion, (camera, tile, depth) sort, tile offsets.
//
// Implements gsplat::intersect_tile / intersect_offset (reference: gsplat/IntersectTile.cu:24-114
// count+emit, :206-252 offsets, :290-328 radix sort; gsplat/Intersect.cpp:15-137 host side).
// All results are integer functions of (means2d, radii, depths) and are bit-exact with the
// reference: same float tile-bbox arithmetic (division by the tile size, floor/ceil, CUDA's
// saturating float->uint32 conversion), same 64-bit key layout
//      cam_id << (32 + tile_bits) | tile_id << 32 | float_bits(depth)
// and the same final order: ascending (camera, tile, depth bits), ties in emission order
// (ascending flattened Gaussian index), which is what the reference's stable
// cub::DeviceRadixSort::SortPairs over 32+tile_bits+cam_bits key bits produces.
//
// How the sorted lists are built (gsb_isect_plan + gsb_isect_emit_planned).  The reference radix-sorts
// all I intersections on 46 bits (six 8-bit passes over 12-byte pairs, ~150 B of HBM traffic per
// intersection).  Here no intersection is ever sorted:
//   1. plan      one thread per Gaussian: tile box, tile count, depth key.
//   2. depth     stable LSD radix sort of the C*N Gaussians by depth bits (N elements, not I;
//                gsb_devsort.cuh), passes whose digit is constant are skipped.
//   3. runs      scan of the tile counts in depth order -> compact run table (Gaussians with >= 1 tile:
//                cumulative end slot, index, box, depth key); n_isects goes to the host here.
//   4. histogram the runs are cut into P chunks of ~I/P intersections; one CTA per chunk counts its intersections per
//                tile with shared-memory atomics: matrix M[P][tiles].
//   5. column scan over (tile, chunk): M[p][t] becomes the first output slot of chunk p in tile t;
//                the tile offsets (a6) fall out of the same scan.
//   -- host reads n_isects, allocates the outputs --
//   6. place     the same pass again, each intersection taking the next slot of its (chunk, tile) group in run order:
//                4 bytes written per intersection DIRECTLY to its final position, nothing read back; the 64-bit keys,
//                when the caller wants them, are written by a coalesced pass.
// Chunks are in depth order and groups are filled in run order, which is (depth bits, index) order: every tile's list
// is ordered by (depth, index) -- the same permutation as the reference's single 46-bit sort, ties included.
#include "gsb_devsort.cuh"
#include "gsb_ewa.cuh"
#include "gsb_scan.cuh"

namespace gsb {

constexpr int kIsectThreads = 256;

struct TileBox {
    uint32_t x0, y0, x1, y1;
    bool active;
};

// IntersectTile.cu:54-76.  This file is compiled with -fmad=false and uses IEEE division so the
// tile bounds are a pure function of the inputs (the reference's fast-math `x / 16.f` is exact
// for power-of-two tile sizes, which is what its callers use: rasterizer.cpp:180).
__device__ __forceinline__ TileBox tile_box(const float *__restrict__ means2d, const int32_t *__restrict__ radii,
                                            size_t idx, uint32_t tile_size, uint32_t tile_width,
                                            uint32_t tile_height) {
    TileBox b;
    const int2 r = reinterpret_cast<const int2 *>(radii)[idx];
    const float radius_x = (float)r.x, radius_y = (float)r.y;
    b.active = !(radius_x <= 0 || radius_y <= 0);
    if (!b.active) { b.x0 = b.x1 = b.y0 = b.y1 = 0; return b; }
    const float2 m = reinterpret_cast<const float2 *>(means2d)[idx];
    const float ts = (float)tile_size;
    const float trx = __fdiv_rn(radius_x, ts), try_ = __fdiv_rn(radius_y, ts);
    const float tx = __fdiv_rn(m.x, ts), ty = __fdiv_rn(m.y, ts);
    // (uint32_t) of a negative float saturates to 0 on the GPU (cvt.rzi.u32.f32)
    b.x0 = min((uint32_t)floorf(tx - trx), tile_width);
    b.y0 = min((uint32_t)floorf(ty - try_), tile_height);
    b.x1 = min((uint32_t)ceilf(tx + trx), tile_width);
    b.y1 = min((uint32_t)ceilf(ty + try_), tile_height);
    return b;
}

__global__ void __launch_bounds__(kIsectThreads) isect_count_kernel(uint64_t n, const float *__restrict__ means2d,
                                                                     const int32_t *__restrict__ radii,
                                                                     uint32_t tile_size, uint32_t tile_width,
                                                                     uint32_t tile_height,
                                                                     int32_t *__restrict__ tiles_per_gauss) {
    const uint64_t idx = (uint64_t)blockIdx.x * kIsectThreads + threadIdx.x;
    if (idx >= n) return;
    const TileBox b = tile_box(means2d, radii, idx, tile_size, tile_width, tile_height);
    tiles_per_gauss[idx] = b.active ? (int32_t)((b.y1 - b.y0) * (b.x1 - b.x0)) : 0;
}

// Unsorted path (sort == false): Gaussian i writes its intersections at cum[i-1], row-major over its box.
__global__ void __launch_bounds__(kIsectThreads) isect_emit_kernel(uint64_t n, uint32_t N,
                                                                    const float *__restrict__ means2d,
                                                                    const int32_t *__restrict__ radii,
                                                                    const float *__restrict__ depths,
                                                                    const int64_t *__restrict__ cum_tiles,
                                                                    uint32_t tile_size, uint32_t tile_width,
                                                                    uint32_t tile_height, uint32_t tile_n_bits,
                                                                    int64_t *__restrict__ isect_ids,
                                                                    int32_t *__restrict__ flatten_ids) {
    const uint64_t idx = (uint64_t)blockIdx.x * kIsectThreads + threadIdx.x;
    if (idx >= n) return;
    const TileBox b = tile_box(means2d, radii, idx, tile_size, tile_width, tile_height);
    if (!b.active) return;
    const int64_t cid_enc = (int64_t)(idx / N) << (32 + tile_n_bits);
    const int64_t depth_enc = (int64_t)__float_as_uint(depths[idx]); // zero-extended bit pattern (:98-99)
    int64_t cur = (idx == 0) ? 0 : cum_tiles[idx - 1];
    for (uint32_t y = b.y0; y < b.y1; ++y)
        for (uint32_t x = b.x0; x < b.x1; ++x) {
            const int64_t tile_id = (int64_t)y * tile_width + x;
            isect_ids[cur] = cid_enc | (tile_id << 32) | depth_enc;
            flatten_ids[cur] = (int32_t)idx;
            ++cur;
        }
}

// ---- planned path, step 1: tile box, count and depth key of every Gaussian ---------------------------------
// boxes[idx] = (x0 | y0 << 16, w | h << 16) in tiles.  Gaussians without tiles get the key 0xffffffff: they
// end up behind every Gaussian that has tiles and never enter the run table.  vals[idx] = idx is the depth
// sort's initial permutation: the sort skips every pass whose digit is constant over the Gaussians with tiles,
// possibly all four, so the first pass that runs -- or the run table, when none does -- reads it.
__global__ void __launch_bounds__(kIsectThreads) isect_plan_kernel(uint64_t n, const float *__restrict__ means2d,
                                                                    const int32_t *__restrict__ radii,
                                                                    const float *__restrict__ depths,
                                                                    uint32_t tile_size, uint32_t tile_width,
                                                                    uint32_t tile_height,
                                                                    int32_t *__restrict__ tiles_per_gauss,
                                                                    uint32_t *__restrict__ keys,
                                                                    uint32_t *__restrict__ vals,
                                                                    uint2 *__restrict__ boxes,
                                                                    SortCtl *__restrict__ ctl) {
    __shared__ uint32_t s_or[kIsectThreads / 32], s_nor[kIsectThreads / 32];
    const uint64_t idx = (uint64_t)blockIdx.x * kIsectThreads + threadIdx.x;
    uint32_t k_or = 0u, k_nor = 0u;
    if (idx < n) {
        const TileBox b = tile_box(means2d, radii, idx, tile_size, tile_width, tile_height);
        const uint32_t w = b.x1 - b.x0, h = b.y1 - b.y0;
        const int32_t cnt = b.active ? (int32_t)(w * h) : 0;
        tiles_per_gauss[idx] = cnt;
        uint32_t key = 0xffffffffu;
        if (cnt > 0) {
            key = __float_as_uint(depths[idx]);
            k_or = key;
            k_nor = ~key;
        }
        keys[idx] = key;
        vals[idx] = (uint32_t)idx;
        boxes[idx] = make_uint2(b.x0 | (b.y0 << 16), w | (h << 16));
    }
    k_or = __reduce_or_sync(0xffffffffu, k_or);
    k_nor = __reduce_or_sync(0xffffffffu, k_nor);
    if ((threadIdx.x & 31) == 0) { s_or[threadIdx.x >> 5] = k_or; s_nor[threadIdx.x >> 5] = k_nor; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kIsectThreads / 32; ++w) { k_or |= s_or[w]; k_nor |= s_nor[w]; }
        if (k_or | k_nor) { // at least one Gaussian of this CTA touches a tile
            atomicOr(&ctl->key_or, k_or);
            atomicOr(&ctl->key_nor, k_nor);
        }
    }
}

// EWA path (SURVEY.md 8 f4): the front kernel of gsb_fastgs.cu has already computed every primitive's tile box and its
// EXACT tile count; this step only derives the sort keys (depth bits, 0xffffffff for primitives without tiles) and the
// initial permutation.
__global__ void __launch_bounds__(kIsectThreads) isect_plan_boxes_kernel(uint64_t n, const int32_t *__restrict__ counts,
                                                                          const float *__restrict__ depths,
                                                                          uint32_t *__restrict__ keys,
                                                                          uint32_t *__restrict__ vals,
                                                                          SortCtl *__restrict__ ctl) {
    __shared__ uint32_t s_or[kIsectThreads / 32], s_nor[kIsectThreads / 32];
    const uint64_t idx = (uint64_t)blockIdx.x * kIsectThreads + threadIdx.x;
    uint32_t k_or = 0u, k_nor = 0u;
    if (idx < n) {
        uint32_t key = 0xffffffffu;
        if (counts[idx] > 0) {
            key = __float_as_uint(depths[idx]);
            k_or = key;
            k_nor = ~key;
        }
        keys[idx] = key;
        vals[idx] = (uint32_t)idx;
    }
    k_or = __reduce_or_sync(0xffffffffu, k_or);
    k_nor = __reduce_or_sync(0xffffffffu, k_nor);
    if ((threadIdx.x & 31) == 0) { s_or[threadIdx.x >> 5] = k_or; s_nor[threadIdx.x >> 5] = k_nor; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kIsectThreads / 32; ++w) { k_or |= s_or[w]; k_nor |= s_nor[w]; }
        if (k_or | k_nor) {
            atomicOr(&ctl->key_or, k_or);
            atomicOr(&ctl->key_nor, k_nor);
        }
    }
}

// ---- step 3: run table ---------------------------------------------------------------------------------------
// One scan over the Gaussians in depth order of the pair (has tiles ? 1 : 0, tile count).
struct RunAcc {
    unsigned long long cnt;
    uint32_t runs;
    RunAcc() = default;
    __device__ __forceinline__ RunAcc(int v) : cnt(v), runs(v) {}
    __device__ __forceinline__ RunAcc &operator+=(const RunAcc &o) { cnt += o.cnt; runs += o.runs; return *this; }
    __device__ __forceinline__ RunAcc operator+(const RunAcc &o) const { RunAcc r = *this; return r += o; }
    // found by argument-dependent lookup from block_scan_inclusive
    friend __device__ __forceinline__ RunAcc __shfl_up_sync(unsigned mask, const RunAcc &v, int delta) {
        RunAcc r;
        r.cnt = ::__shfl_up_sync(mask, v.cnt, delta);
        r.runs = ::__shfl_up_sync(mask, v.runs, delta);
        return r;
    }
};

struct RunTable {
    uint32_t *end;  // cumulative number of intersections up to and including this run
    uint32_t *idx;  // flattened Gaussian index (camera * N + gaussian)
    uint2 *box;
    uint32_t *key;  // depth bits
    // EWA path only (SURVEY.md 8 f4): the run covers the tiles of its box that pass ewa_tile_contributes.  For boxes of
    // up to 32 tiles the front kernel has already evaluated the test: bit j of `mask` = tile j of the box (row-major)
    // passes.  Larger boxes (rare) evaluate the test again from the per-primitive parameters.
    uint32_t *mask;
    const float4 *f0;     // per primitive: (mx, my, ca, cb)
    const float2 *f1;     // per primitive: (cc, thr)
};
__device__ __forceinline__ EwaFilter prim_filter(const RunTable &rt, uint32_t idx) {
    const float4 a = rt.f0[idx];
    const float2 b = rt.f1[idx];
    return EwaFilter{a.x, a.y, a.z, a.w, b.x, b.y};
}

__device__ __forceinline__ const uint32_t *sorted_vals(const SortCtl *ctl, const uint32_t *v0, const uint32_t *v1) {
    return (radix_passes_done(ctl, 4) & 1) ? v1 : v0;
}

__global__ void __launch_bounds__(kScanThreads) runs_blocksum_kernel(const SortCtl *__restrict__ ctl,
                                                                     const uint32_t *__restrict__ v0,
                                                                     const uint32_t *__restrict__ v1,
                                                                     const int32_t *__restrict__ counts, uint64_t n,
                                                                     uint32_t seg, RunAcc *__restrict__ bsum) {
    __shared__ RunAcc s_warp[kScanWarps];
    const uint32_t *perm = sorted_vals(ctl, v0, v1);
    const SegRange r = cta_segment(n, seg);
    RunAcc acc = 0;
    for (uint64_t i = r.lo + threadIdx.x; i < r.hi; i += kScanThreads) {
        const int32_t c = counts[perm[i]];
        acc.cnt += (unsigned long long)c;
        acc.runs += c > 0 ? 1u : 0u;
    }
    RunAcc tot;
    block_scan_inclusive<RunAcc, kScanWarps>(acc, s_warp, tot);
    if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kScanThreads) runs_build_kernel(SortCtl *__restrict__ ctl,
                                                                  const uint32_t *__restrict__ v0,
                                                                  const uint32_t *__restrict__ v1,
                                                                  const uint32_t *__restrict__ k0,
                                                                  const uint32_t *__restrict__ k1,
                                                                  const int32_t *__restrict__ counts,
                                                                  const uint2 *__restrict__ boxes, uint64_t n,
                                                                  uint32_t seg, uint32_t nblocks,
                                                                  const RunAcc *__restrict__ bsum, RunTable rt,
                                                                  const uint32_t *__restrict__ masks) {
    __shared__ RunAcc s_warp[kScanWarps];
    const bool odd = (radix_passes_done(ctl, 4) & 1) != 0;
    const uint32_t *perm = odd ? v1 : v0;
    const uint32_t *keys = odd ? k1 : k0;
    RunAcc carry;
    {
        RunAcc part = 0;
        for (uint32_t bb = threadIdx.x; bb < blockIdx.x; bb += kScanThreads) part += bsum[bb];
        block_scan_inclusive<RunAcc, kScanWarps>(part, s_warp, carry);
    }
    const SegRange r = cta_segment(n, seg);
    for (uint64_t i0 = r.lo; i0 < r.hi; i0 += kScanThreads) {
        const uint64_t i = i0 + threadIdx.x;
        RunAcc v = 0;
        uint32_t idx = 0;
        if (i < r.hi) {
            idx = perm[i];
            const int32_t c = counts[idx];
            v.cnt = (unsigned long long)c;
            v.runs = c > 0 ? 1u : 0u;
        }
        RunAcc tot;
        const RunAcc inc = block_scan_inclusive<RunAcc, kScanWarps>(v, s_warp, tot);
        if (v.runs) {
            const uint32_t k = carry.runs + inc.runs - 1u;
            rt.end[k] = (uint32_t)(carry.cnt + inc.cnt);
            rt.idx[k] = idx;
            rt.box[k] = boxes[idx];
            rt.key[k] = keys[i];
            if (masks) rt.mask[k] = masks[idx];
        }
        carry += tot;
    }
    if (blockIdx.x == nblocks - 1 && threadIdx.x == 0) {
        ctl->n_runs = carry.runs;
        ctl->n_isects = carry.cnt;
    }
}

// ---- steps 4 and 6: per-chunk tile counters, ordered placement ------------------------------------------------
// The runs (Gaussians with tiles, in depth order) are cut into P chunks of about I / P intersections each, at run
// boundaries.  One CTA per chunk keeps one counter per tile in shared memory.
//   hist   every intersection of the chunk does an atomicAdd on its tile's counter -> M[p][tile] (any order);
//   place  the counters start at the chunk's first slot in each tile (column scan of M) and every intersection takes
//          the next slot of its tile IN RUN ORDER, so each (chunk, tile) group lands in its final range already in
//          (depth bits, index) order: the runs are in that order (stable depth sort) and a run covers a tile at most
//          once.
// How place keeps run order without a CTA-wide handshake: warp w owns the tile rows y with y % 8 == w (of every
// camera), so no two warps share a counter and a tile's order is decided inside ONE warp.  Every warp walks all the
// chunk's runs, 32 per step (one per lane), and expands only its rows of their boxes; the expanded intersections are
// laid out flat in run order and taken 32 per round, so the lanes of a round are in run order and rounds follow
// each other.  Inside a round every lane takes a slot with a shared atomic; when a tile has several members in the
// round (the atomic tells), the members are re-ranked by lane.
struct BinArgs {
    RunTable rt;
    const SortCtl *ctl;
    uint32_t N;          // Gaussians per camera
    uint32_t n_tiles;    // tiles per camera
    uint32_t tile_width;
    uint32_t multi_cam;
    uint32_t t_lo, t_cnt; // window of global tile ids (camera * n_tiles + tile) handled by this launch
    uint32_t T_total, P;
    uint32_t *M;          // [P][T_total]
    uint32_t *chunk_run;  // [P + 1] first run of every chunk (written by hist)
    int32_t *flatten_ids;
    uint32_t cap;         // capacity of flatten_ids (>= n_isects unless the caller under-allocated)
};

constexpr int kBinThreads = 256;
constexpr uint32_t kBinWarps = kBinThreads / 32; // place: warp w owns the tile rows y % kBinWarps == w

// first r in [0, n_runs) with end[r] > s (exists: s < end[n_runs - 1]); one probe per lane and round
__device__ __forceinline__ uint32_t first_run_after(const uint32_t *__restrict__ end, uint32_t n_runs, uint32_t s) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t lo = 0, hi = n_runs; // answer in [lo, hi)
    while (hi - lo > 1) {
        const uint32_t len = hi - lo;
        const uint32_t step = (len + 32) / 33;
        const uint32_t p = lo + (lane + 1) * step - 1;
        const bool le = (p < hi - 1) ? (end[p] <= s) : false; // position hi-1 is known to be > s
        const uint32_t k = __popc(__ballot_sync(0xffffffffu, le));
        const uint32_t nlo = (k == 0) ? lo : lo + k * step;
        const uint32_t nhi = (k == 32) ? hi : min(hi, lo + (k + 1) * step);
        lo = nlo; hi = nhi;
    }
    return lo;
}

// chunk p = runs [first run whose end exceeds p I / P, the same for p + 1)
__device__ __forceinline__ uint32_t chunk_first_run(const BinArgs &a, uint32_t p, unsigned long long I, uint32_t n_runs) {
    if (p >= a.P || n_runs == 0) return n_runs;
    const uint32_t s = (uint32_t)(((unsigned long long)p * I) / a.P);
    if (I == 0 || s >= I) return n_runs;
    return first_run_after(a.rt.end, n_runs, s);
}

template <bool kFilter = false>
__global__ void __launch_bounds__(kBinThreads) tile_hist_kernel(const BinArgs a) {
    extern __shared__ uint32_t s_cnt[]; // [t_cnt]
    __shared__ uint32_t s_range[2];
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint32_t p = blockIdx.x;
    uint32_t *row = a.M + (size_t)p * a.T_total + a.t_lo;
    const unsigned long long I = a.ctl->n_isects;
    const uint32_t n_runs = a.ctl->n_runs;
    if (tid < 32) {
        const uint32_t ra = chunk_first_run(a, p, I, n_runs);
        const uint32_t rb = chunk_first_run(a, p + 1, I, n_runs);
        if (tid == 0) {
            s_range[0] = ra; s_range[1] = rb;
            a.chunk_run[p] = ra;
            if (p == a.P - 1) a.chunk_run[a.P] = n_runs;
        }
    }
    for (uint32_t t = tid; t < a.t_cnt; t += kBinThreads) s_cnt[t] = 0;
    __syncthreads();
    const uint32_t ra = s_range[0], rb = s_range[1];

    for (uint32_t r0 = ra + (tid & ~31u); r0 < rb; r0 += kBinThreads) { // warp-uniform trip count
        const uint32_t r = r0 + lane;
        uint32_t idx = 0, bx = 0, by = 0, tmask = 0xffffffffu;
        if (r < rb) {
            idx = a.rt.idx[r];
            const uint2 b = a.rt.box[r];
            bx = b.x; by = b.y;
            if constexpr (kFilter) tmask = a.rt.mask[r];
        }
        const uint32_t w = by & 0xffffu, h = by >> 16, n = w * h; // 0 for the lanes past the chunk
        const uint32_t x0 = bx & 0xffffu, y0 = bx >> 16;
        const uint32_t cam_base = a.multi_cam ? (idx / a.N) * a.n_tiles : 0u;
        // runs of up to 32 tiles: one lane each
        if (n > 0 && n <= 32) {
            // four tiles per trip: the four shared-memory atomics are in flight together
            uint32_t x = x0, y = y0;
            for (uint32_t j = 0; j < n; j += 4) {
                uint32_t g[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    bool take = j + u < n;
                    if constexpr (kFilter) take = take && ((tmask >> (j + u)) & 1u);
                    g[u] = take ? cam_base + y * a.tile_width + x - a.t_lo : 0xffffffffu;
                    if (++x == x0 + w) { x = x0; ++y; }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (g[u] < a.t_cnt) atomicAdd(&s_cnt[g[u]], 1u);
            }
        }
        // larger runs: the whole warp strides over the box
        uint32_t big = __ballot_sync(0xffffffffu, n > 32);
        while (big) {
            const int src = __ffs(big) - 1;
            big &= big - 1;
            const uint32_t bidx = __shfl_sync(0xffffffffu, idx, src), bcam = __shfl_sync(0xffffffffu, cam_base, src);
            const uint32_t bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
            const uint32_t bw = __shfl_sync(0xffffffffu, w, src), bn = __shfl_sync(0xffffffffu, n, src);
            EwaFilter bf = {0.f, 0.f, 1.f, 0.f, 1.f, 0.f};
            if constexpr (kFilter) bf = prim_filter(a.rt, bidx); // one broadcast load per warp
            for (uint32_t j = lane; j < bn; j += 32) {
                const uint32_t dy = j / bw, dx = j - dy * bw;
                if constexpr (kFilter) {
                    if (!ewa_tile_contributes(bf, bx0 + dx, by0 + dy)) continue;
                }
                const uint32_t g = bcam + (by0 + dy) * a.tile_width + bx0 + dx - a.t_lo;
                if (g < a.t_cnt) atomicAdd(&s_cnt[g], 1u);
            }
        }
    }
    __syncthreads();
    for (uint32_t t = tid; t < a.t_cnt; t += kBinThreads) row[t] = s_cnt[t];
}

template <bool kFilter = false>
__global__ void __launch_bounds__(kBinThreads) tile_place_kernel(const BinArgs a) {
    extern __shared__ uint32_t s_cnt[]; // [t_cnt]: next slot of every tile of the window
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t p = blockIdx.x;
    const uint32_t *row = a.M + (size_t)p * a.T_total + a.t_lo;
    const uint32_t ra = a.chunk_run[p], rb = a.chunk_run[p + 1];
    for (uint32_t t = tid; t < a.t_cnt; t += kBinThreads) s_cnt[t] = row[t];
    __syncthreads();

    for (uint32_t r0 = ra; r0 < rb; r0 += 32) { // every warp walks every run
        const uint32_t r = r0 + lane;
        uint32_t idx = 0, bx = 0, by = 0, tmask = 0xffffffffu;
        if (r < rb) {
            idx = a.rt.idx[r];
            const uint2 b = a.rt.box[r];
            bx = b.x; by = b.y;
            if constexpr (kFilter) tmask = a.rt.mask[r];
        }
        const uint32_t w = by & 0xffffu, h = by >> 16; // 0 for the lanes past the chunk
        const uint32_t x0 = bx & 0xffffu, y0 = bx >> 16;
        const uint32_t y1 = y0 + ((warp - y0) & (kBinWarps - 1)); // this warp's first row of the box
        const uint32_t n = y1 < y0 + h ? ((y0 + h - 1 - y1) / kBinWarps + 1) * w : 0u;
        const uint32_t cam = a.multi_cam ? idx / a.N : 0u;
        // inclusive scan of n: the lane's intersections are [end - n, end) of the step's flat sequence
        uint32_t end = n;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, end, o);
            if (lane >= (uint32_t)o) end += t;
        }
        const uint32_t first = end - n, total = __shfl_sync(0xffffffffu, end, 31);
        for (uint32_t e0 = 0; e0 < total; e0 += 32) { // warp-uniform
            const uint32_t e = e0 + lane;
            // owner: the last lane whose first intersection is <= e (a lane without intersections in this warp's rows
            // shares its `first` with the next lane, so the last such lane has intersections)
            uint32_t src = 0;
#pragma unroll
            for (uint32_t s = 16; s; s >>= 1)
                if (__shfl_sync(0xffffffffu, first, src + s) <= e) src += s;
            const uint32_t j = e - __shfl_sync(0xffffffffu, first, src);
            const uint32_t ridx = __shfl_sync(0xffffffffu, idx, src);
            const uint32_t rx0 = __shfl_sync(0xffffffffu, x0, src), ry1 = __shfl_sync(0xffffffffu, y1, src);
            const uint32_t rw = max(__shfl_sync(0xffffffffu, w, src), 1u), rcam = __shfl_sync(0xffffffffu, cam, src);
            const uint32_t k = j / rw, dx = j - k * rw;
            const uint32_t x = rx0 + dx, y = ry1 + k * kBinWarps;
            bool take = e < total;
            if constexpr (kFilter) {
                const uint32_t rmask = __shfl_sync(0xffffffffu, tmask, src), ry0 = __shfl_sync(0xffffffffu, y0, src);
                const uint32_t rh = __shfl_sync(0xffffffffu, h, src);
                if (take)
                    take = (rw * rh <= 32u) ? ((rmask >> ((y - ry0) * rw + dx)) & 1u) != 0u
                                            : ewa_tile_contributes(prim_filter(a.rt, ridx), x, y);
            }
            const uint32_t g = take ? rcam * a.n_tiles + y * a.tile_width + x - a.t_lo : 0xffffffffu;
            take = g < a.t_cnt;
            // the lanes of a round are in run order: a tile's members are ranked by lane.  Most rounds have no tile
            // twice, which the atomic tells: every lane read its tile's counter before any lane advanced it.
            uint32_t slot = take ? s_cnt[g] : 0u;
            __syncwarp();
            const uint32_t got = take ? atomicAdd(&s_cnt[g], 1u) : slot;
            if (__any_sync(0xffffffffu, got != slot)) {
                uint32_t rank = 0;
                for (uint32_t l = 0; l < 32; ++l) {
                    const uint32_t gl = __shfl_sync(0xffffffffu, g, l);
                    rank += (l < lane && gl == g) ? 1u : 0u;
                }
                slot += rank;
            }
            __syncwarp();
            if (take && slot < a.cap) a.flatten_ids[slot] = (int32_t)ridx;
        }
    }
}

// isect_ids of the sorted list, written in order (coalesced) instead of scattered with the values:
//   key[pos] = cam << (32 + tile_bits) | tile << 32 | depth bits of flatten_ids[pos]
// One warp per tile: its positions are the contiguous range tile_off[t] .. tile_off[t + 1] of the closed offsets table, so
// the tile needs no search and loads / stores are coalesced; the warps of a CTA take consecutive tiles.
constexpr int kKeyWarps = kIsectThreads / 32;
__global__ void __launch_bounds__(kIsectThreads) isect_keys_kernel(uint32_t n, const uint32_t *__restrict__ tile_off,
                                                                   uint32_t T, uint32_t n_tiles, uint32_t tile_n_bits,
                                                                   const int32_t *__restrict__ flatten_ids,
                                                                   const float *__restrict__ depths,
                                                                   int64_t *__restrict__ isect_ids) {
    const uint32_t t = blockIdx.x * kKeyWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (t >= T) return;
    const uint32_t lo = min(__ldg(tile_off + t), n), hi = min(__ldg(tile_off + t + 1), n);
    const uint32_t cam = t / n_tiles, tile = t - cam * n_tiles;
    const int64_t head = ((int64_t)cam << (32 + tile_n_bits)) | ((int64_t)tile << 32);
    for (uint32_t p0 = lo + lane; p0 < hi; p0 += 128) { // four positions per lane in flight (ids, then depths, then stores)
        uint32_t idx[4], key[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) idx[u] = (p0 + 32u * u < hi) ? (uint32_t)flatten_ids[p0 + 32u * u] : 0u;
#pragma unroll
        for (int u = 0; u < 4; ++u) key[u] = (p0 + 32u * u < hi) ? __float_as_uint(depths[idx[u]]) : 0u;
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (p0 + 32u * u < hi) isect_ids[p0 + 32u * u] = head | (int64_t)key[u];
    }
}

// ---- step 5: exclusive scan of M over (tile, chunk) ----------------------------------------------------------
// col_segsum: seg[s][t] = sum of M[p][t] over the chunks p of segment s.
__global__ void __launch_bounds__(kIsectThreads) col_segsum_kernel(const uint32_t *__restrict__ M, uint32_t T,
                                                                   uint32_t P, uint32_t seg_len,
                                                                   uint32_t *__restrict__ seg,
                                                                   uint32_t *__restrict__ tot) {
    const uint32_t t = blockIdx.x * kIsectThreads + threadIdx.x;
    if (t >= T) return;
    const uint32_t s = blockIdx.y;
    const uint32_t p0 = s * seg_len, p1 = min(P, p0 + seg_len);
    uint32_t acc = 0;
    uint32_t p = p0;
    for (; p + 4 <= p1; p += 4) { // four independent loads in flight
        const uint32_t v0 = M[(size_t)p * T + t], v1 = M[(size_t)(p + 1) * T + t];
        const uint32_t v2 = M[(size_t)(p + 2) * T + t], v3 = M[(size_t)(p + 3) * T + t];
        acc += (v0 + v1) + (v2 + v3);
    }
    for (; p < p1; ++p) acc += M[(size_t)p * T + t];
    seg[(size_t)s * T + t] = acc;
    if (acc) atomicAdd(&tot[t], acc); // the tile's intersection count (zeroed before the launch)
}
// col_tilescan (one CTA): exclusive scan of the tiles' counts -> first slot of every tile (the tile offsets, a6).
__global__ void __launch_bounds__(kScanThreads) col_tilescan_kernel(const uint32_t *__restrict__ tot, uint32_t T,
                                                                    uint32_t *__restrict__ toff /* [T + 1] */,
                                                                    int32_t *__restrict__ tile_offsets /*nullable*/,
                                                                    int write_total) {
    __shared__ uint32_t s_warp[kScanWarps];
    uint32_t carry = 0;
    for (uint32_t t0 = 0; t0 < T; t0 += kScanThreads) {
        const uint32_t t = t0 + threadIdx.x;
        const uint32_t v = t < T ? tot[t] : 0u;
        uint32_t all;
        const uint32_t inc = block_scan_inclusive<uint32_t>(v, s_warp, all);
        if (t < T) {
            const uint32_t first = carry + inc - v;
            toff[t] = first;
            if (tile_offsets) tile_offsets[t] = (int32_t)first;
        }
        carry += all;
    }
    if (threadIdx.x == 0) {
        toff[T] = carry; // = n_isects
        if (tile_offsets && write_total) tile_offsets[T] = (int32_t)carry;
    }
}
// col_apply: M[p][t] = first output slot of chunk p in tile t.
__global__ void __launch_bounds__(kIsectThreads) col_apply_kernel(uint32_t *__restrict__ M, uint32_t T, uint32_t P,
                                                                  uint32_t seg_len, const uint32_t *__restrict__ seg,
                                                                  const uint32_t *__restrict__ toff) {
    const uint32_t t = blockIdx.x * kIsectThreads + threadIdx.x;
    if (t >= T) return;
    const uint32_t s = blockIdx.y;
    const uint32_t p0 = s * seg_len, p1 = min(P, p0 + seg_len);
    uint32_t run = toff[t]; // first slot of the tile + what the earlier segments of this column hold
#pragma unroll 8
    for (uint32_t s2 = 0; s2 < s; ++s2) run += seg[(size_t)s2 * T + t];
    uint32_t p = p0;
    for (; p + 4 <= p1; p += 4) { // loads first: a store to M would otherwise fence the next load
        const uint32_t v0 = M[(size_t)p * T + t], v1 = M[(size_t)(p + 1) * T + t];
        const uint32_t v2 = M[(size_t)(p + 2) * T + t], v3 = M[(size_t)(p + 3) * T + t];
        M[(size_t)p * T + t] = run;
        M[(size_t)(p + 1) * T + t] = run + v0;
        M[(size_t)(p + 2) * T + t] = run + v0 + v1;
        M[(size_t)(p + 3) * T + t] = run + v0 + v1 + v2;
        run += (v0 + v1) + (v2 + v3);
    }
    for (; p < p1; ++p) {
        const uint32_t v = M[(size_t)p * T + t];
        M[(size_t)p * T + t] = run;
        run += v;
    }
}

// IntersectTile.cu:206-252, restated as "first sorted position whose (cam, tile) >= id": the reference streams over all
// n_isects keys and lets the position where the tile changes write the offsets in between; on keys that are sorted (the
// operator's contract) that is lower_bound(keys >> 32, id) per tile -- one binary search per tile, ~23 probes each, instead
// of a pass over 8 bytes per intersection (0.037 -> 0.004 ms at config B).
__global__ void __launch_bounds__(kIsectThreads) isect_offsets_kernel(uint64_t n_isects,
                                                                       const int64_t *__restrict__ isect_ids,
                                                                       uint32_t total_tiles, uint32_t n_tiles,
                                                                       uint32_t tile_n_bits,
                                                                       int32_t *__restrict__ offsets) {
    const uint32_t id = blockIdx.x * kIsectThreads + threadIdx.x;
    if (id >= total_tiles) return;
    const int64_t cam = id / n_tiles, tile = id - cam * n_tiles;
    const int64_t want = (cam << tile_n_bits) | tile; // the key's bits above the depth
    uint64_t lo = 0, hi = n_isects;                   // first position whose (cam, tile) >= want, in [0, n_isects]
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if ((isect_ids[mid] >> 32) < want) lo = mid + 1; else hi = mid;
    }
    offsets[id] = (int32_t)lo;
}

// ---- host-side geometry ------------------------------------------------------------------------------------------

struct DeviceShape {
    int sms;
    int smem_optin; // max dynamic shared memory per block
    int smem_sm;    // shared memory per SM
};
static const DeviceShape &device_shape() {
    // immutable after the first call (C++11 thread-safe initialisation); sm_90a (H100 SXM): 132 SMs, 227 KB / 228 KB
    static const DeviceShape s = [] {
        DeviceShape d{132, 227 * 1024, 228 * 1024};
        int dev = 0;
        if (cudaGetDevice(&dev) == cudaSuccess) {
            int v = 0;
            if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) d.sms = v;
            if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess && v > 0)
                d.smem_optin = v;
            if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) == cudaSuccess && v > 0)
                d.smem_sm = v;
        }
        return d;
    }();
    return s;
}

// segments of the 1024-thread sort and scan kernels: at most one CTA per SM
static ScanPlan seg_plan(uint64_t n) { return scan_plan(n, (uint32_t)device_shape().sms); }

constexpr uint32_t kMaxWindowTiles = 36 * 1024; // 144 KB of counters at most

struct BinPlan {
    uint32_t T_total, t_win, n_win, P, S, seg_len;
    size_t smem; // counters of the histogram and placement passes
};
static BinPlan bin_plan(uint32_t C, uint32_t N, uint32_t tile_width, uint32_t tile_height) {
    const DeviceShape &d = device_shape();
    BinPlan b;
    b.T_total = C * tile_width * tile_height;
    b.t_win = b.T_total < kMaxWindowTiles ? b.T_total : kMaxWindowTiles;
    if (b.t_win == 0) b.t_win = 1;
    b.n_win = (b.T_total + b.t_win - 1) / b.t_win;
    if (b.n_win == 0) b.n_win = 1;
    b.smem = (size_t)b.t_win * 4;
    uint32_t per_sm = (uint32_t)((size_t)d.smem_sm / (b.smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8; // 8 x 256 threads fill an SM
    uint64_t P = (uint64_t)d.sms * per_sm;
    const uint64_t n = (uint64_t)C * N;
    // a (chunk, tile) group should hold one or two intersections: more Gaussians -> more waves of chunks, as long as
    // the P x tiles matrix stays below 128 MB
    uint64_t waves = (n + 2500000 - 1) / 2500000;
    if (waves < 1) waves = 1;
    if (waves > 4) waves = 4;
    while (waves > 1 && P * waves * b.T_total * 4 > (128ull << 20)) --waves;
    P *= waves;
    const uint64_t cap = (n + 255) / 256; // no point in chunks of a handful of Gaussians
    if (P > cap) P = cap;
    if (P < 1) P = 1;
    b.P = (uint32_t)P;
    // column scan: S segments of chunks per tile column, about a quarter of a million threads
    uint32_t S = b.T_total ? (262144u + b.T_total - 1) / b.T_total : 1u;
    if (S > 64) S = 64;
    if (S > b.P) S = b.P;
    if (S < 1) S = 1;
    b.seg_len = (b.P + S - 1) / S;
    b.S = (b.P + b.seg_len - 1) / b.seg_len;
    return b;
}

// Workspace of the plan; everything the emit needs afterwards lives here too.
struct PlanWs {
    size_t ctl, keys0, keys1, vals0, vals1, boxes, hist, bsum, rt_end, rt_idx, rt_box, rt_key, rt_mask, M, seg, tot, toff,
        chunk_run, total;
};
static PlanWs plan_ws(uint64_t n, const BinPlan &b, const ScanPlan &sp, bool filter = false) {
    PlanWs w;
    WsLayout l;
    w.ctl = l.take(sizeof(SortCtl));
    w.keys0 = l.take(n * 4); w.keys1 = l.take(n * 4);
    w.vals0 = l.take(n * 4); w.vals1 = l.take(n * 4);
    w.boxes = l.take(n * 8);
    w.hist = l.take((size_t)sp.nblocks * kRadixBins * 4);
    w.bsum = l.take((size_t)sp.nblocks * sizeof(RunAcc));
    w.rt_end = l.take(n * 4); w.rt_idx = l.take(n * 4); w.rt_box = l.take(n * 8); w.rt_key = l.take(n * 4);
    w.rt_mask = filter ? l.take(n * 4) : 0;
    w.M = l.take((size_t)b.P * b.T_total * 4);
    w.seg = l.take((size_t)b.S * b.T_total * 4);
    w.tot = l.take((size_t)b.T_total * 4);
    w.toff = l.take(((size_t)b.T_total + 1) * 4);
    w.chunk_run = l.take(((size_t)b.P + 1) * 4);
    w.total = align256(l.bytes) + 256;
    return w;
}

} // namespace gsb

extern "C" size_t gsb_isect_count_workspace(uint64_t n_elements) {
    const gsb::ScanPlan sp = gsb::seg_plan(n_elements);
    return gsb::align256((size_t)sp.nblocks * sizeof(long long)) + 256;
}

extern "C" int gsb_isect_count(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii,
                               uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
                               int32_t *tiles_per_gauss, int64_t *cum_tiles, void *workspace,
                               size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    const uint64_t n = (uint64_t)C * N;
    if (n == 0) return GSB_OK;
    if (!means2d || !radii || !tiles_per_gauss || !cum_tiles || tile_size == 0) return GSB_E_INVALID;
    if (!workspace || workspace_bytes < gsb_isect_count_workspace(n)) return GSB_E_WORKSPACE;
    cudaStream_t s = as_stream(stream);
    const uint32_t grid = (uint32_t)((n + kIsectThreads - 1) / kIsectThreads);
    ProfScope ps("isect_count", s); // count kernel + scan
    isect_count_kernel<<<grid, kIsectThreads, 0, s>>>(n, means2d, radii, tile_size, tile_width, tile_height,
                                                      tiles_per_gauss);
    GSB_LAUNCH_CHECK();
    long long *bsum = reinterpret_cast<long long *>(workspace);
    return scan_launch(LoadI32{tiles_per_gauss}, n, seg_plan(n), bsum, cum_tiles, s);
}

extern "C" int gsb_isect_emit(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii,
                              const float *depths, const int64_t *cum_tiles, uint32_t tile_size,
                              uint32_t tile_width, uint32_t tile_height, int64_t *isect_ids,
                              int32_t *flatten_ids, gsb_stream_t stream) {
    const uint64_t n = (uint64_t)C * N;
    if (n == 0) return GSB_OK;
    if (!means2d || !radii || !depths || !cum_tiles || !isect_ids || !flatten_ids) return GSB_E_INVALID;
    const uint32_t tile_n_bits = gsb::bit_width_u32(tile_width * tile_height);
    const uint32_t cam_n_bits = gsb::bit_width_u32(C);
    if (tile_n_bits + cam_n_bits > 32) return GSB_E_INVALID; // Intersect.cpp:50
    const uint32_t grid = (uint32_t)((n + gsb::kIsectThreads - 1) / gsb::kIsectThreads);
    gsb::ProfScope ps("isect_emit", gsb::as_stream(stream));
    gsb::isect_emit_kernel<<<grid, gsb::kIsectThreads, 0, gsb::as_stream(stream)>>>(
        n, N, means2d, radii, depths, cum_tiles, tile_size, tile_width, tile_height, tile_n_bits, isect_ids,
        flatten_ids);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}

// Generic stable sort of unsorted (isect_id, flatten_id) pairs on the low 32+tile_bits+cam_bits key bits
// (IntersectTile.cu:290-328): ceil(bits / 8) passes of the radix kernels of gsb_devsort.cuh.
extern "C" size_t gsb_isect_sort_workspace(uint64_t n_isects) {
    const gsb::ScanPlan sp = gsb::seg_plan(n_isects);
    return gsb::align256(n_isects * 8) + gsb::align256(n_isects * 4) +
           gsb::align256((size_t)sp.nblocks * gsb::kRadixBins * 4) + 256;
}

extern "C" int gsb_isect_sort(uint64_t n_isects, uint32_t C, uint32_t tile_width, uint32_t tile_height,
                              const int64_t *isect_ids_in, const int32_t *flatten_ids_in,
                              int64_t *isect_ids_out, int32_t *flatten_ids_out, void *workspace,
                              size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (n_isects == 0) return GSB_OK;
    if (!isect_ids_in || !flatten_ids_in || !isect_ids_out || !flatten_ids_out) return GSB_E_INVALID;
    if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255) || workspace_bytes < gsb_isect_sort_workspace(n_isects))
        return GSB_E_WORKSPACE;
    const uint32_t tile_n_bits = bit_width_u32(tile_width * tile_height);
    const uint32_t cam_n_bits = bit_width_u32(C);
    const uint32_t end_bit = 32 + tile_n_bits + cam_n_bits;
    if (end_bit > 64) return GSB_E_INVALID;
    const int passes = (int)((end_bit + 7) / 8);
    cudaStream_t s = as_stream(stream);
    ProfScope ps("isect_sort", s);
    const ScanPlan sp = seg_plan(n_isects);
    char *base = reinterpret_cast<char *>(workspace);
    unsigned long long *tmp_k = reinterpret_cast<unsigned long long *>(base);
    uint32_t *tmp_v = reinterpret_cast<uint32_t *>(base + align256(n_isects * 8));
    uint32_t *H = reinterpret_cast<uint32_t *>(base + align256(n_isects * 8) + align256(n_isects * 4));
    unsigned long long *out_k = reinterpret_cast<unsigned long long *>(isect_ids_out);
    uint32_t *out_v = reinterpret_cast<uint32_t *>(flatten_ids_out);
    // The input is read-only: copy it into the buffer from which `passes` alternations end in the outputs.
    unsigned long long *k0 = (passes & 1) ? tmp_k : out_k, *k1 = (passes & 1) ? out_k : tmp_k;
    uint32_t *v0 = (passes & 1) ? tmp_v : out_v, *v1 = (passes & 1) ? out_v : tmp_v;
    GSB_CUDA_TRY(cudaMemcpyAsync(k0, isect_ids_in, n_isects * 8, cudaMemcpyDeviceToDevice, s));
    GSB_CUDA_TRY(cudaMemcpyAsync(v0, flatten_ids_in, n_isects * 4, cudaMemcpyDeviceToDevice, s));
    return radix_sort_launch<unsigned long long>(k0, k1, v0, v1, n_isects, sp, passes, 0, end_bit, nullptr, H, s);
}

extern "C" size_t gsb_isect_plan_workspace(uint32_t C, uint32_t N, uint32_t tile_width, uint32_t tile_height) {
    const uint64_t n = (uint64_t)C * N;
    return gsb::plan_ws(n, gsb::bin_plan(C, N, tile_width, tile_height), gsb::seg_plan(n)).total;
}

namespace gsb {
// Source of step 1: either the gsplat operator inputs (means2d / radii -> tile boxes here) or the EWA front kernel's
// precomputed boxes, exact counts and tile-test parameters.
struct PlanSource {
    const float *means2d = nullptr;
    const int32_t *radii = nullptr;
    uint32_t tile_size = 16;
    const uint2 *boxes = nullptr;   // EWA
    const uint32_t *masks = nullptr; // EWA: tile-test results of boxes of up to 32 tiles
    const float4 *filt0 = nullptr;   // EWA: test parameters (for the larger boxes)
    const float2 *filt1 = nullptr;   // EWA
    bool ewa() const { return boxes != nullptr; }
};

static int plan_impl(uint32_t C, uint32_t N, const PlanSource &src, const float *depths, uint32_t tile_width,
                     uint32_t tile_height, int32_t *tiles_per_gauss, int64_t *n_isects_out, int32_t *tile_offsets_out,
                     int tile_offsets_total, void *plan_workspace, size_t plan_workspace_bytes, cudaStream_t s) {
    const uint64_t n = (uint64_t)C * N;
    if (!n_isects_out) return GSB_E_INVALID;
    const uint64_t T64 = (uint64_t)C * tile_width * tile_height;
    if (n == 0 || T64 == 0) {
        GSB_CUDA_TRY(cudaMemsetAsync(n_isects_out, 0, sizeof(int64_t), s));
        if (tile_offsets_out && T64)
            GSB_CUDA_TRY(cudaMemsetAsync(tile_offsets_out, 0, (T64 + (tile_offsets_total ? 1 : 0)) * 4, s));
        if (n && tiles_per_gauss && !src.ewa()) GSB_CUDA_TRY(cudaMemsetAsync(tiles_per_gauss, 0, n * 4, s));
        return GSB_OK;
    }
    if (!depths || !tiles_per_gauss) return GSB_E_INVALID;
    if (src.ewa() ? (!src.filt0 || !src.filt1 || !src.masks) : (!src.means2d || !src.radii || src.tile_size == 0))
        return GSB_E_INVALID;
    const uint32_t tile_n_bits = bit_width_u32(tile_width * tile_height);
    const uint32_t cam_n_bits = bit_width_u32(C);
    if (tile_n_bits + cam_n_bits > 32) return GSB_E_INVALID; // Intersect.cpp:50
    if (tile_width > 0xffffu || tile_height > 0xffffu || n > 0x7fffffffull || T64 > 0x7fffffffull) return GSB_E_INVALID;
    const BinPlan bp = bin_plan(C, N, tile_width, tile_height);
    const ScanPlan sp = seg_plan(n);
    const PlanWs w = plan_ws(n, bp, sp, src.ewa());
    if (int rc = ws_check(plan_workspace, plan_workspace_bytes, w.total)) return rc;
    char *base = reinterpret_cast<char *>(plan_workspace);
    SortCtl *ctl = reinterpret_cast<SortCtl *>(base + w.ctl);
    uint32_t *k0 = reinterpret_cast<uint32_t *>(base + w.keys0), *k1 = reinterpret_cast<uint32_t *>(base + w.keys1);
    uint32_t *v0 = reinterpret_cast<uint32_t *>(base + w.vals0), *v1 = reinterpret_cast<uint32_t *>(base + w.vals1);
    uint2 *boxes = reinterpret_cast<uint2 *>(base + w.boxes);
    uint32_t *H = reinterpret_cast<uint32_t *>(base + w.hist);
    RunAcc *bsum = reinterpret_cast<RunAcc *>(base + w.bsum);
    RunTable rt{reinterpret_cast<uint32_t *>(base + w.rt_end), reinterpret_cast<uint32_t *>(base + w.rt_idx),
                reinterpret_cast<uint2 *>(base + w.rt_box), reinterpret_cast<uint32_t *>(base + w.rt_key),
                src.ewa() ? reinterpret_cast<uint32_t *>(base + w.rt_mask) : nullptr, src.filt0, src.filt1};
    uint32_t *M = reinterpret_cast<uint32_t *>(base + w.M);
    uint32_t *seg = reinterpret_cast<uint32_t *>(base + w.seg);
    {
        ProfScope ps("isect_count", s);
        GSB_CUDA_TRY(cudaMemsetAsync(ctl, 0, sizeof(SortCtl), s));
        const uint32_t grid = (uint32_t)((n + kIsectThreads - 1) / kIsectThreads);
        if (src.ewa())
            isect_plan_boxes_kernel<<<grid, kIsectThreads, 0, s>>>(n, tiles_per_gauss, depths, k0, v0, ctl);
        else
            isect_plan_kernel<<<grid, kIsectThreads, 0, s>>>(n, src.means2d, src.radii, depths, src.tile_size, tile_width,
                                                            tile_height, tiles_per_gauss, k0, v0, boxes, ctl);
        GSB_LAUNCH_CHECK();
    }
    {
        ProfScope ps("isect_depth_sort", s);
        if (int rc = radix_sort_launch<uint32_t>(k0, k1, v0, v1, n, sp, 4, 0, 32, ctl, H, s)) return rc;
    }
    {
        ProfScope ps("isect_runs", s);
        runs_blocksum_kernel<<<sp.nblocks, kScanThreads, 0, s>>>(ctl, v0, v1, tiles_per_gauss, n, sp.seg, bsum);
        GSB_LAUNCH_CHECK();
        runs_build_kernel<<<sp.nblocks, kScanThreads, 0, s>>>(ctl, v0, v1, k0, k1, tiles_per_gauss,
                                                             src.ewa() ? src.boxes : boxes, n, sp.seg, sp.nblocks, bsum,
                                                             rt, src.masks);
        GSB_LAUNCH_CHECK();
    }
    // device or pinned-host destination alike
    GSB_CUDA_TRY(cudaMemcpyAsync(n_isects_out, &ctl->n_isects, sizeof(int64_t), cudaMemcpyDefault, s));
    {
        ProfScope ps("isect_tile_hist", s);
        BinArgs a;
        a.rt = rt; a.ctl = ctl; a.N = N; a.n_tiles = tile_width * tile_height; a.tile_width = tile_width;
        a.multi_cam = C > 1 ? 1u : 0u;
        a.T_total = bp.T_total; a.P = bp.P; a.M = M; a.flatten_ids = nullptr; a.cap = 0;
        a.chunk_run = reinterpret_cast<uint32_t *>(base + w.chunk_run);
        if (bp.smem > 48 * 1024) {
            GSB_CUDA_TRY(cudaFuncSetAttribute(tile_hist_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)bp.smem));
            GSB_CUDA_TRY(cudaFuncSetAttribute(tile_hist_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              (int)bp.smem));
        }
        for (uint32_t wnd = 0; wnd < bp.n_win; ++wnd) {
            a.t_lo = wnd * bp.t_win;
            a.t_cnt = min(bp.t_win, bp.T_total - a.t_lo);
            if (src.ewa())
                tile_hist_kernel<true><<<bp.P, kBinThreads, bp.smem, s>>>(a);
            else
                tile_hist_kernel<false><<<bp.P, kBinThreads, bp.smem, s>>>(a);
            GSB_LAUNCH_CHECK();
        }
    }
    {
        ProfScope ps("isect_colscan", s);
        const dim3 cgrid((bp.T_total + kIsectThreads - 1) / kIsectThreads, bp.S);
        uint32_t *tot = reinterpret_cast<uint32_t *>(base + w.tot), *toff = reinterpret_cast<uint32_t *>(base + w.toff);
        GSB_CUDA_TRY(cudaMemsetAsync(tot, 0, (size_t)bp.T_total * 4, s));
        col_segsum_kernel<<<cgrid, kIsectThreads, 0, s>>>(M, bp.T_total, bp.P, bp.seg_len, seg, tot);
        GSB_LAUNCH_CHECK();
        col_tilescan_kernel<<<1, kScanThreads, 0, s>>>(tot, bp.T_total, toff, tile_offsets_out, tile_offsets_total);
        GSB_LAUNCH_CHECK();
        col_apply_kernel<<<cgrid, kIsectThreads, 0, s>>>(M, bp.T_total, bp.P, bp.seg_len, seg, toff);
        GSB_LAUNCH_CHECK();
    }
    return GSB_OK;
}

static int emit_impl(uint32_t C, uint32_t N, bool filter, const float4 *filt0, const float2 *filt1, const float *depths,
                     uint32_t tile_width, uint32_t tile_height,
                     uint64_t n_isects, const void *plan_workspace, size_t plan_workspace_bytes, int64_t *isect_ids,
                     int32_t *flatten_ids, cudaStream_t s) {
    const uint64_t n = (uint64_t)C * N;
    if (n == 0 || n_isects == 0) return GSB_OK;
    if (!plan_workspace || !flatten_ids || !depths) return GSB_E_INVALID;
    if (n_isects > 0x7fffffffull) return GSB_E_INVALID;
    const BinPlan bp = bin_plan(C, N, tile_width, tile_height);
    const ScanPlan sp = seg_plan(n);
    const PlanWs w = plan_ws(n, bp, sp, filter);
    if ((reinterpret_cast<uintptr_t>(plan_workspace) & 255) || plan_workspace_bytes < w.total) return GSB_E_WORKSPACE;
    char *base = const_cast<char *>(reinterpret_cast<const char *>(plan_workspace));
    BinArgs a;
    a.rt = RunTable{reinterpret_cast<uint32_t *>(base + w.rt_end), reinterpret_cast<uint32_t *>(base + w.rt_idx),
                    reinterpret_cast<uint2 *>(base + w.rt_box), reinterpret_cast<uint32_t *>(base + w.rt_key),
                    filter ? reinterpret_cast<uint32_t *>(base + w.rt_mask) : nullptr, filt0, filt1};
    a.ctl = reinterpret_cast<const SortCtl *>(base + w.ctl);
    a.N = N; a.n_tiles = tile_width * tile_height; a.tile_width = tile_width;
    a.multi_cam = C > 1 ? 1u : 0u;
    a.chunk_run = reinterpret_cast<uint32_t *>(base + w.chunk_run);
    a.T_total = bp.T_total; a.P = bp.P; a.M = reinterpret_cast<uint32_t *>(base + w.M);
    a.flatten_ids = flatten_ids; a.cap = (uint32_t)n_isects;
    if (bp.smem > 48 * 1024) {
        GSB_CUDA_TRY(cudaFuncSetAttribute(tile_place_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)bp.smem));
        GSB_CUDA_TRY(cudaFuncSetAttribute(tile_place_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)bp.smem));
    }
    {
        ProfScope ps("isect_emit", s);
        for (uint32_t wnd = 0; wnd < bp.n_win; ++wnd) {
            a.t_lo = wnd * bp.t_win;
            a.t_cnt = min(bp.t_win, bp.T_total - a.t_lo);
            if (filter)
                tile_place_kernel<true><<<bp.P, kBinThreads, bp.smem, s>>>(a);
            else
                tile_place_kernel<false><<<bp.P, kBinThreads, bp.smem, s>>>(a);
            GSB_LAUNCH_CHECK();
        }
    }
    // only the operator API wants the 64-bit keys back (intersect_offset consumes them).  Written here, in order, rather
    // than by the placing lane: scattered 8-byte stores to an array larger than L2 cost more than this pass.
    if (isect_ids) {
        const uint32_t grid = (bp.T_total + kKeyWarps - 1) / kKeyWarps;
        ProfScope psk("isect_keys", s);
        isect_keys_kernel<<<grid, kIsectThreads, 0, s>>>((uint32_t)n_isects, reinterpret_cast<const uint32_t *>(base + w.toff),
                                                        bp.T_total, a.n_tiles, bit_width_u32(tile_width * tile_height),
                                                        flatten_ids, depths, isect_ids);
        GSB_LAUNCH_CHECK();
    }
    return GSB_OK;
}

// EWA entry points used by gsb_fastgs.cu (not part of the C ABI)
size_t isect_plan_ewa_workspace(uint32_t N, uint32_t tile_width, uint32_t tile_height) {
    return plan_ws(N, bin_plan(1, N, tile_width, tile_height), seg_plan(N), true).total;
}
int isect_plan_ewa(uint32_t N, int32_t *counts, const uint2 *boxes, const uint32_t *masks, const float *depths,
                   const float4 *filt0, const float2 *filt1, uint32_t tile_width, uint32_t tile_height, int64_t *n_isects_out,
                   int32_t *tile_offsets_out, void *plan_workspace, size_t plan_workspace_bytes, cudaStream_t s) {
    PlanSource src;
    src.boxes = boxes; src.masks = masks; src.filt0 = filt0; src.filt1 = filt1;
    return plan_impl(1, N, src, depths, tile_width, tile_height, counts, n_isects_out, tile_offsets_out, 1, plan_workspace,
                     plan_workspace_bytes, s);
}
int isect_emit_ewa(uint32_t N, const float4 *filt0, const float2 *filt1, const float *depths, uint32_t tile_width,
                   uint32_t tile_height, uint64_t capacity, const void *plan_workspace, size_t plan_workspace_bytes,
                   int32_t *flatten_ids, cudaStream_t s) {
    return emit_impl(1, N, true, filt0, filt1, depths, tile_width, tile_height, capacity, plan_workspace, plan_workspace_bytes, nullptr,
                     flatten_ids, s);
}
} // namespace gsb

extern "C" int gsb_isect_plan(uint32_t C, uint32_t N, const float *means2d, const int32_t *radii, const float *depths,
                              uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
                              int32_t *tiles_per_gauss, int64_t *n_isects_out, int32_t *tile_offsets_out,
                              int tile_offsets_total, void *plan_workspace, size_t plan_workspace_bytes,
                              gsb_stream_t stream) {
    gsb::PlanSource src;
    src.means2d = means2d; src.radii = radii; src.tile_size = tile_size;
    return gsb::plan_impl(C, N, src, depths, tile_width, tile_height, tiles_per_gauss, n_isects_out, tile_offsets_out,
                          tile_offsets_total, plan_workspace, plan_workspace_bytes, gsb::as_stream(stream));
}

extern "C" int gsb_isect_emit_planned(uint32_t C, uint32_t N, const float *depths, uint32_t tile_width,
                                      uint32_t tile_height, uint64_t n_isects, const void *plan_workspace,
                                      size_t plan_workspace_bytes, int64_t *isect_ids /*nullable*/, int32_t *flatten_ids,
                                      gsb_stream_t stream) {
    return gsb::emit_impl(C, N, false, nullptr, nullptr, depths, tile_width, tile_height, n_isects, plan_workspace, plan_workspace_bytes,
                          isect_ids, flatten_ids, gsb::as_stream(stream));
}

extern "C" int gsb_isect_offsets(uint64_t n_isects, const int64_t *isect_ids_sorted, uint32_t C,
                                 uint32_t tile_width, uint32_t tile_height, int32_t *offsets,
                                 gsb_stream_t stream) {
    const uint32_t n_tiles = tile_width * tile_height;
    const uint64_t total = (uint64_t)C * n_tiles;
    if (total == 0) return GSB_OK;
    if (!offsets) return GSB_E_INVALID;
    cudaStream_t s = gsb::as_stream(stream);
    if (n_isects == 0) { // IntersectTile.cu:268-271
        GSB_CUDA_TRY(cudaMemsetAsync(offsets, 0, total * sizeof(int32_t), s));
        return GSB_OK;
    }
    if (!isect_ids_sorted) return GSB_E_INVALID;
    const uint32_t tile_n_bits = gsb::bit_width_u32(n_tiles);
    const uint32_t grid = (uint32_t)((total + gsb::kIsectThreads - 1) / gsb::kIsectThreads);
    gsb::ProfScope ps("isect_offsets", s);
    gsb::isect_offsets_kernel<<<grid, gsb::kIsectThreads, 0, s>>>(n_isects, isect_ids_sorted, (uint32_t)total,
                                                                  n_tiles, tile_n_bits, offsets);
    GSB_LAUNCH_CHECK();
    return GSB_OK;
}
