// Point cloud -> voxels (SURVEY 8 f2): the step in front of the conv path.
//
// Replaces Point2VoxelKernel / Point2Voxel (spconv/csrc/sparse/pointops.py:120-490).  The reference
// GPU kernels append with atomics, so the voxel ORDER and WHICH points survive the per-voxel cap
// depend on scheduling; here every decision is deterministic and equal to the reference's CPU
// implementation (Point2VoxelCPU::point_to_voxel_static_template, pointops.py:589-695):
//   * a voxel's id is the rank of its FIRST point in input order (atomicMin of the point index per
//     hash slot, then a sort of the minima -- the same first-touch ranking as the conv rulebook);
//   * voxels beyond max_num_voxels are dropped (their points get id -1);
//   * a voxel keeps its first max_num_points_per_voxel points in input order (stable sort of the
//     points by voxel id, position = offset inside the voxel's segment);
//   * empty_mean fills the unused point slots of a voxel with the mean of its kept points.
// Same hash-and-scan building blocks as rulebook.cu (hash.cuh).  Two stages because the voxel count
// sizes the outputs (the reference returns sliced tensors of that length, pointops.py:434-490).
// spx_point2voxel_bounded (MaskedPointToVoxel) does a batch of clouds in one pass with the count kept on the
// device and outputs of a host-known bound; it shares p2v_coord, the insert and the scatter with the stages, and
// groups the points by row with sort_by_key and segment_offsets (segments.cuh).
#include "common.cuh"
#include "hash.cuh"
#include "rank.cuh"
#include "segments.cuh"
#include <cub/cub.cuh>

namespace spx {

struct P2VGeom {
    int ndim, zyx;
    float vsize[SPX_MAX_NDIM], lo[SPX_MAX_NDIM];     // internal (grid) axis order
    int grid[SPX_MAX_NDIM];
};

// grid coordinate of a point on internal axis j: floor((p - lo) / vsize) in fp32, as the reference.
// The cell is range-checked as a float, before any conversion: NaN fails every comparison and inf /
// huge values fail the upper bound, so a point with a non-finite coordinate makes no voxel (a float ->
// int conversion of NaN is undefined and gives 0 on the GPU, which used to put such points in cell 0).
__device__ __forceinline__ bool p2v_coord(const P2VGeom &g, const float *__restrict__ pt, int (&c)[SPX_MAX_NDIM]) {
#pragma unroll
    for (int j = 0; j < SPX_MAX_NDIM; ++j) {
        if (j < g.ndim) {
            const float p = pt[g.zyx ? g.ndim - 1 - j : j];
            const float f = floorf(__fdiv_rn(p - g.lo[j], g.vsize[j]));
            if (!(f >= 0.f && f < 2147483648.f)) return false;
            const int v = (int)f;
            if (v >= g.grid[j]) return false;
            c[j] = v;
        }
    }
    return true;
}

// sample that owns point i: the b in [0, nsamples) with off[b] <= i < off[b+1] (off non-decreasing), -1 when i
// lies before off[0] or at / beyond off[nsamples] (padding)
__device__ __forceinline__ int p2v_sample_of(const int32_t *__restrict__ off, int nsamples, int64_t i) {
    if (i < (int64_t)__ldg(off) || i >= (int64_t)__ldg(off + nsamples)) return -1;
    return last_at_most(off, nsamples, i);
}

// key = b * grid volume + cell (row-major over the internal axes), -1 = no voxel.  sample_off == NULL: one
// sample (b = 0), the single-cloud path.  A point outside every sample is never read.
template <typename Table>
__global__ void p2v_insert_kernel(Table table, P2VGeom g, const float *__restrict__ points, int64_t n, int nf,
                                  const int32_t *__restrict__ sample_off, int nsamples, int64_t *__restrict__ keys) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c[SPX_MAX_NDIM];
    int64_t key = -1;
    const int b = sample_off ? p2v_sample_of(sample_off, nsamples, i) : 0;
    if (b >= 0 && p2v_coord(g, points + i * nf, c)) {
        key = b;
#pragma unroll
        for (int j = 0; j < SPX_MAX_NDIM; ++j) if (j < g.ndim) key = key * g.grid[j] + c[j];
        table.insert_min(key, (int32_t)i);
    }
    keys[i] = key;
}

// occupied slots -> (first point index, slot); one atomic per block
template <typename Table>
__global__ void __launch_bounds__(256)
p2v_collect_kernel(Table table, uint32_t capacity, uint32_t *__restrict__ first_pt, uint32_t *__restrict__ slot_of,
                   int *__restrict__ counter) {
    __shared__ int warp_cnt[8];
    __shared__ int block_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t s = blockIdx.x * 256u + threadIdx.x;
    int64_t key; int32_t val = 0;
    const bool occ = s < capacity && table.occupied(s, key, val);
    const unsigned ball = __ballot_sync(0xffffffffu, occ);
    if (lane == 0) warp_cnt[warp] = __popc(ball);
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < 8; ++w) { const int c = warp_cnt[w]; warp_cnt[w] = tot; tot += c; }
        block_base = tot ? atomicAdd(counter, tot) : 0;
    }
    __syncthreads();
    if (occ) {
        const int pos = block_base + warp_cnt[warp] + __popc(ball & ((1u << lane) - 1u));
        first_pt[pos] = (uint32_t)val;
        slot_of[pos] = s;
    }
}

// rank r (first-touch order): slot value <- r (or -1 when r >= max_voxels), indices[r] <- grid coords
template <typename Table>
__global__ void p2v_assign_kernel(Table table, P2VGeom g, const uint32_t *__restrict__ sorted_slot, int64_t total,
                                  int64_t kept, int32_t *__restrict__ indices) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= total) return;
    const uint32_t s = sorted_slot[r];
    int64_t key; int32_t val;
    table.occupied(s, key, val);
    table.set_value(s, r < kept ? (int32_t)r : -1);
    if (r < kept) {
        int32_t *dst = indices + r * g.ndim;
        for (int j = g.ndim - 1; j >= 0; --j) { dst[j] = (int32_t)(key % g.grid[j]); key /= g.grid[j]; }
    }
}

// per point: voxel id (int64, -1 = outside the range or voxel dropped); sort key = id, invalid last
template <typename Table>
__global__ void p2v_lookup_kernel(Table table, const int64_t *__restrict__ keys, int64_t n, uint32_t invalid_key,
                                  int64_t *__restrict__ pc_voxel_id, uint32_t *__restrict__ sort_key,
                                  uint32_t *__restrict__ sort_val) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int32_t vid = -1;
    const int64_t key = keys[i];
    if (key >= 0) { int32_t v; if (table.find_slot(key, v) >= 0) vid = v; }
    pc_voxel_id[i] = (int64_t)vid;
    sort_key[i] = vid >= 0 ? (uint32_t)vid : invalid_key;
    sort_val[i] = (uint32_t)i;
}

// segment starts of the voxel-sorted point list (ids 0..M-1 are dense: every kept voxel owns at least
// its first point; points without a voxel carry the key M and sort last): start[v] = first position
// with key v, start[M] = first keyless point (or n)
__global__ void p2v_segments_kernel(const uint32_t *__restrict__ sorted_vid, int64_t n, uint32_t M,
                                    int32_t *__restrict__ start) {
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (p > n) return;
    const uint32_t cur = p < n ? sorted_vid[p] : M;
    const uint32_t prev = p > 0 ? sorted_vid[p - 1] : 0xffffffffu;
    if (cur != prev) start[cur] = (int32_t)p;
}

// one thread per (sorted point, feature): voxels[vid][pos][f] = points[i][f] for pos < max_points
__global__ void p2v_scatter_kernel(const float *__restrict__ points, int nf, const uint32_t *__restrict__ sorted_vid,
                                   const uint32_t *__restrict__ sorted_pt, int64_t n, uint32_t num_voxels,
                                   const int32_t *__restrict__ start, int max_points, float *__restrict__ voxels) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t p = idx / nf;
    const int f = (int)(idx - p * nf);
    if (p >= n) return;
    const uint32_t vid = sorted_vid[p];
    if (vid >= num_voxels) return;
    const int pos = (int)(p - start[vid]);
    if (pos >= max_points) return;
    voxels[((int64_t)vid * max_points + pos) * nf + f] = points[(int64_t)sorted_pt[p] * nf + f];
}

// num_per_voxel[v] = min(count, max_points); optional mean fill of the unused slots
__global__ void p2v_finish_kernel(const int32_t *__restrict__ start, int64_t M, int max_points, int nf, int empty_mean,
                                  int32_t *__restrict__ num_per_voxel, float *__restrict__ voxels) {
    const int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (v >= M) return;
    const int cnt = start[v + 1] - start[v];
    const int num = cnt < max_points ? cnt : max_points;
    num_per_voxel[v] = num;
    if (empty_mean && num > 0 && num < max_points) {
        float *vx = voxels + v * (int64_t)max_points * nf;
        for (int f = 0; f < nf; ++f) {
            float acc = 0.f;
            for (int j = 0; j < num; ++j) acc += vx[j * nf + f];
            const float mean = acc / (float)num;
            for (int j = num; j < max_points; ++j) vx[j * nf + f] = mean;
        }
    }
}

// ------------------------------------------------------------------ batched, bounded (MaskedPointToVoxel)
// The voxel count never leaves the device, so nothing may be sized from it: the first-touch ranking is a
// bitmap rank over the point indices (rank.cuh) instead of a sort of the occupied slots, and the outputs
// have a host-known bound.  Sample b owns the points [eff[b], eff[b+1]); its voxels are keyed
// b * grid volume + cell, so the global rank of a voxel's first point is already sample-major.
constexpr int P2V_PLAN_THREADS = 1024;

// inclusive scan (sum, or max of non-negative values) over one block of P2V_PLAN_THREADS; total = block total
template <bool MAX>
__device__ __forceinline__ int p2v_block_scan(int v, int *warp_s, int &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl = MAX ? max(incl, up) : incl + up;
    }
    if (lane == 31) warp_s[warp] = incl;
    __syncthreads();
    int pre = 0, tot = 0;
    for (int w = 0; w < P2V_PLAN_THREADS / 32; ++w) {
        const int s = warp_s[w];
        if (w < warp) pre = MAX ? max(pre, s) : pre + s;
        tot = MAX ? max(tot, s) : tot + s;
    }
    __syncthreads();
    total = tot;
    return MAX ? max(pre, incl) : pre + incl;
}

// eff[b] = max over b' <= b of clamp(off[b'], 0, n), b = 0..nsamples: disjoint, contiguous samples for ANY
// offsets (a decreasing offset gives an empty sample).  off == NULL: one sample of all n points.
__global__ void __launch_bounds__(P2V_PLAN_THREADS)
p2v_offsets_kernel(const int32_t *__restrict__ off, int nsamples, int64_t n, int32_t *__restrict__ eff) {
    __shared__ int warp_s[P2V_PLAN_THREADS / 32];
    int carry = 0;
    for (int b0 = 0; b0 <= nsamples; b0 += P2V_PLAN_THREADS) {
        const int b = b0 + threadIdx.x;
        int v = 0;
        if (b <= nsamples) {
            const int64_t o = off ? (int64_t)__ldg(off + b) : (b == 0 ? 0 : n);
            v = (int)(o < 0 ? 0 : (o > n ? n : o));
        }
        int tot;
        const int incl = max(carry, p2v_block_scan<true>(v, warp_s, tot));
        if (b <= nsamples) eff[b] = incl;
        carry = max(carry, tot);
    }
}

// per point: first[i] = the first point of i's voxel (the table's minimum), -1 = no voxel; the first points are
// marked in the rank bitmap and the last block turns the tile counts into the rank prefix
template <typename Table>
__global__ void __launch_bounds__(256)
p2v_mark_kernel(Table table, const int64_t *__restrict__ keys, int64_t n, int32_t *__restrict__ first,
                uint32_t *__restrict__ bitmap, int *__restrict__ tile_cnt, int64_t tiles, int *__restrict__ done) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) {
        int32_t f = -1;
        const int64_t key = keys[i];
        if (key >= 0) table.find_slot(key, f);
        if (f == (int32_t)i) rank_mark((uint32_t)i, bitmap, tile_cnt);
        first[i] = f;
    }
    int total;
    rank_prefix_last_block<256>(tile_cnt, tiles, done, &total);
}

// one block: per sample, count_b = R(eff[b+1]) - R(eff[b]) voxels (R = first points below a position),
// kept_b = min(count_b, max_voxels), base_b = exclusive scan of kept_b; num_valid = min(sum, bound), status
// bit 0 when the sum exceeds the bound
__global__ void __launch_bounds__(P2V_PLAN_THREADS)
p2v_plan_kernel(const int32_t *__restrict__ eff, int nsamples, const uint32_t *__restrict__ bitmap,
                const int *__restrict__ tile_prefix, int64_t max_voxels, int64_t bound, int32_t *__restrict__ rbase,
                int32_t *__restrict__ kept, int32_t *__restrict__ base, int32_t *__restrict__ num_valid,
                int32_t *__restrict__ status) {
    __shared__ int warp_s[P2V_PLAN_THREADS / 32];
    int carry = 0;
    for (int b0 = 0; b0 < nsamples; b0 += P2V_PLAN_THREADS) {
        const int b = b0 + threadIdx.x;
        int k = 0;
        if (b < nsamples) {
            const int r0 = rank_of((uint32_t)__ldg(eff + b), bitmap, tile_prefix);
            const int r1 = rank_of((uint32_t)__ldg(eff + b + 1), bitmap, tile_prefix);
            k = (int64_t)(r1 - r0) < max_voxels ? r1 - r0 : (int)max_voxels;
            rbase[b] = r0;
            kept[b] = k;
        }
        int tot;
        const int incl = p2v_block_scan<false>(k, warp_s, tot);
        if (b < nsamples) base[b] = carry + incl - k;
        carry += tot;
    }
    if (threadIdx.x == 0) {
        *num_valid = (int64_t)carry < bound ? carry : (int32_t)bound;
        if ((int64_t)carry > bound) atomicOr(status, 1);
    }
}

// per point: output row of its voxel = base_b + (rank of the voxel's first point inside sample b), -1 when the
// voxel is past the sample's cap or the bound; sort key = row (none: bound); the first point of a kept voxel
// writes the voxel's indices row (b, cell)
__global__ void p2v_rows_kernel(P2VGeom g, const int64_t *__restrict__ keys, const int32_t *__restrict__ first,
                                int64_t n, int64_t vol, const uint32_t *__restrict__ bitmap,
                                const int *__restrict__ tile_prefix, const int32_t *__restrict__ rbase,
                                const int32_t *__restrict__ kept, const int32_t *__restrict__ base, int64_t bound,
                                int64_t *__restrict__ pc_voxel_id, uint32_t *__restrict__ sort_key,
                                int32_t *__restrict__ indices) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t f = __ldg(first + i);
    int64_t row = -1;
    if (f >= 0) {
        int64_t key = __ldg(keys + i);
        const int b = (int)(key / vol);
        const int rel = rank_of((uint32_t)f, bitmap, tile_prefix) - __ldg(rbase + b);
        const int64_t r = (int64_t)__ldg(base + b) + rel;
        if (rel < __ldg(kept + b) && r < bound) row = r;
        if (row >= 0 && f == (int32_t)i) {
            int32_t *dst = indices + row * (g.ndim + 1);
            for (int j = g.ndim - 1; j >= 0; --j) { dst[1 + j] = (int32_t)(key % g.grid[j]); key /= g.grid[j]; }
            dst[0] = b;
        }
    }
    pc_voxel_id[i] = row;
    sort_key[i] = row >= 0 ? (uint32_t)row : (uint32_t)bound;
}

// one thread per element of voxels [bound, max_points, nf]: a slot at or beyond the row's point count gets the
// mean of the kept points (empty_mean: the same fp32 sum and division as p2v_finish_kernel) or 0; element
// (v, 0, 0) also writes num_per_voxel[v] and, for a row without points (padding), indices row v = -1
__global__ void p2v_fill_kernel(const int32_t *__restrict__ start, int64_t bound, int max_points, int nf,
                                int empty_mean, int ncols, int32_t *__restrict__ num_per_voxel,
                                int32_t *__restrict__ indices, float *__restrict__ voxels) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t row_elems = (int64_t)max_points * nf;
    if (idx >= bound * row_elems) return;
    const int64_t v = idx / row_elems;
    const int rem = (int)(idx - v * row_elems);
    const int s = rem / nf, f = rem - s * nf;
    const int cnt = __ldg(start + v + 1) - __ldg(start + v);
    const int num = cnt < max_points ? cnt : max_points;
    if (rem == 0) {
        num_per_voxel[v] = num;
        if (cnt == 0) for (int a = 0; a < ncols; ++a) indices[v * ncols + a] = -1;
    }
    if (s < num) return;
    float val = 0.f;
    if (empty_mean && num > 0) {
        const float *vx = voxels + v * row_elems;
        float acc = 0.f;
        for (int j = 0; j < num; ++j) acc += vx[j * nf + f];
        val = acc / (float)num;
    }
    voxels[idx] = val;
}

struct P2VWs {
    void *tbl; int32_t *tvals; uint32_t capacity; bool i64;
    int64_t *keys;
    uint32_t *a0, *a1, *b0, *b1;          // sort buffers (keys / values, in / out), sized max(N, capacity-bound)
    void *sort_tmp; size_t sort_tmp_bytes;
    int32_t *start; int *counter;
};

static bool p2v_i64(const int *grid, int ndim) {
    double v = 1;
    for (int j = 0; j < ndim; ++j) v *= (double)grid[j];
    return v >= 2147483647.0;
}

static int p2v_carve(int64_t n, const int *grid, int ndim, void *workspace, size_t bytes, P2VWs &w) {
    w.i64 = p2v_i64(grid, ndim);
    w.capacity = table_capacity(n, 2);
    WorkspaceCarver ws(workspace, bytes);
    w.tbl = ws.take<char>((size_t)w.capacity * 8);
    w.tvals = w.i64 ? ws.take<int32_t>(w.capacity) : nullptr;
    w.keys = ws.take<int64_t>(n);
    w.a0 = ws.take<uint32_t>(n); w.a1 = ws.take<uint32_t>(n);
    w.b0 = ws.take<uint32_t>(n); w.b1 = ws.take<uint32_t>(n);
    w.sort_tmp_bytes = cub_sort_pairs_temp_bytes(n);
    w.sort_tmp = ws.take<char>(w.sort_tmp_bytes);
    w.start = ws.take<int32_t>(n + 2);
    w.counter = ws.take<int>(64);
    SPX_REQUIRE(ws.ok(), "point2voxel workspace too small: need %zu, have %zu", ws.off, bytes);
    return 0;
}

static int p2v_geom(int ndim, int zyx, const float *vsize, const int *grid, const float *range, P2VGeom &g) {
    SPX_REQUIRE(ndim >= 1 && ndim <= SPX_MAX_NDIM, "point2voxel: ndim must be in [1, %d]", SPX_MAX_NDIM);
    SPX_REQUIRE(vsize && grid && range, "point2voxel: NULL geometry");
    memset(&g, 0, sizeof(g));
    g.ndim = ndim; g.zyx = zyx;
    for (int j = 0; j < ndim; ++j) {
        SPX_REQUIRE(vsize[j] > 0.f && grid[j] > 0, "point2voxel: bad voxel size / grid on axis %d", j);
        g.vsize[j] = vsize[j]; g.lo[j] = range[j]; g.grid[j] = grid[j];
    }
    return 0;
}

struct P2VBoundedWs {
    int32_t *eff, *rbase, *kept, *base;               // [B + 1], [B] x 3
    void *tbl; int32_t *tvals; uint32_t capacity;     // tvals: 64-bit keys only (always carved)
    int64_t *keys; int32_t *first;                    // [N] each
    uint32_t *bitmap; int *tile_cnt; int *done; int64_t tiles; size_t rank_bytes;
    uint32_t *sort_key; int32_t *order;               // [N] each: rows, sorted in place, and the argsort
    void *sort_ws; size_t sort_ws_bytes;
    int32_t *start;                                   // [bound + 1]
    size_t bytes;
};

// the ranks are taken over the positions 0..N (N included: eff[B] may be N), so the bitmap covers N + 1 bits
static void p2v_bounded_carve(int64_t n, int nsamples, int64_t bound, void *workspace, size_t bytes, P2VBoundedWs &w) {
    WorkspaceCarver ws(workspace, bytes);
    w.eff = ws.take<int32_t>((size_t)nsamples + 1);
    w.rbase = ws.take<int32_t>((size_t)nsamples);
    w.kept = ws.take<int32_t>((size_t)nsamples);
    w.base = ws.take<int32_t>((size_t)nsamples);
    w.capacity = table_capacity(n, 2);
    w.tbl = ws.take<char>((size_t)w.capacity * 8);
    w.tvals = ws.take<int32_t>(w.capacity);
    w.keys = ws.take<int64_t>((size_t)n);
    w.first = ws.take<int32_t>((size_t)n);
    w.rank_bytes = rank_scratch_bytes(n + 1, &w.tiles);
    char *rk = ws.take<char>(w.rank_bytes + sizeof(int));
    w.bitmap = (uint32_t *)rk;
    w.tile_cnt = (int *)(w.bitmap + w.tiles * RANK_TILE_WORDS);
    w.done = (int *)(rk + w.rank_bytes);
    w.sort_key = ws.take<uint32_t>((size_t)n);
    w.order = ws.take<int32_t>((size_t)n);
    w.sort_ws_bytes = radix_argsort_workspace_bytes(n);
    w.sort_ws = ws.take<char>(w.sort_ws_bytes);
    w.start = ws.take<int32_t>((size_t)bound + 1);
    w.bytes = ws.off;
}

static bool p2v_bounded_sizes_ok(int64_t n, int nsamples, int64_t bound) {
    return n >= 0 && n < 2147483647ll && nsamples >= 1 && nsamples <= SPX_P2V_MAX_BATCH && bound >= 1 &&
           bound < 2147483647ll;
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_point2voxel_bounded_workspace_size(int64_t num_points, int batch_size, int64_t bound) {
    if (!p2v_bounded_sizes_ok(num_points, batch_size, bound)) return 0;
    P2VBoundedWs w;
    p2v_bounded_carve(num_points, batch_size, bound, nullptr, SIZE_MAX, w);
    return align_up(w.bytes, 256) + 256;
}

extern "C" int spx_point2voxel_bounded(const float *points, int64_t N, int num_features, int ndim, int zyx,
                                       const float *vsize_host, const int *grid_size_host,
                                       const float *coors_range_host, const int32_t *point_offsets, int batch_size,
                                       int64_t max_voxels, int64_t bound, int max_points_per_voxel, int empty_mean,
                                       float *voxels, int32_t *indices, int32_t *num_per_voxel, int64_t *pc_voxel_id,
                                       int32_t *num_valid, int32_t *status, void *workspace, size_t workspace_bytes,
                                       spx_stream_t stream_) {
    SPX_REQUIRE(N >= 0 && N < 2147483647ll, "point2voxel_bounded: %lld points, must be in [0, 2^31 - 2]", (long long)N);
    SPX_REQUIRE(batch_size >= 1 && batch_size <= SPX_P2V_MAX_BATCH, "point2voxel_bounded: batch_size %d not in [1, %d]",
                batch_size, SPX_P2V_MAX_BATCH);
    SPX_REQUIRE(point_offsets != nullptr || batch_size == 1,
                "point2voxel_bounded: point_offsets may be NULL only with batch_size 1");
    SPX_REQUIRE(bound >= 1 && bound < 2147483647ll, "point2voxel_bounded: bound %lld not in [1, 2^31 - 2]",
                (long long)bound);
    SPX_REQUIRE(max_voxels > 0, "point2voxel_bounded: max_voxels must be positive");
    SPX_REQUIRE(max_points_per_voxel > 0, "point2voxel_bounded: max_points_per_voxel must be positive");
    P2VGeom g;
    if (p2v_geom(ndim, zyx, vsize_host, grid_size_host, coors_range_host, g)) return 2;
    SPX_REQUIRE(num_features >= ndim, "point2voxel_bounded: %d features, fewer than the %d coordinates", num_features,
                ndim);
    double keys = (double)batch_size;
    for (int j = 0; j < ndim; ++j) keys *= (double)grid_size_host[j];
    SPX_REQUIRE(keys < 4611686018427387904.0, "point2voxel_bounded: batch_size x grid volume must be below 2^62");
    int64_t vol = 1;
    for (int j = 0; j < ndim; ++j) vol *= grid_size_host[j];
    SPX_REQUIRE(voxels && indices && num_per_voxel && num_valid && status && workspace,
                "point2voxel_bounded: NULL pointer argument");
    SPX_REQUIRE(N == 0 || (points && pc_voxel_id), "point2voxel_bounded: NULL pointer argument");
    const size_t need = spx_point2voxel_bounded_workspace_size(N, batch_size, bound);
    SPX_REQUIRE(workspace_bytes >= need, "point2voxel_bounded: workspace too small: need %zu, have %zu", need,
                workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int ncols = ndim + 1;
    const int64_t row_elems = (int64_t)max_points_per_voxel * num_features;
    if (N == 0) {                           // no points: every row is padding
        SPX_CHECK_CUDA(cudaMemsetAsync(voxels, 0, (size_t)(bound * row_elems) * sizeof(float), stream));
        SPX_CHECK_CUDA(cudaMemsetAsync(indices, 0xff, (size_t)(bound * ncols) * sizeof(int32_t), stream));
        SPX_CHECK_CUDA(cudaMemsetAsync(num_per_voxel, 0, (size_t)bound * sizeof(int32_t), stream));
        SPX_CHECK_CUDA(cudaMemsetAsync(num_valid, 0, sizeof(int32_t), stream));
        return 0;
    }
    P2VBoundedWs w;
    p2v_bounded_carve(N, batch_size, bound, workspace, workspace_bytes, w);
    const bool i64 = keys >= 2147483647.0;
    SPX_CHECK_CUDA(cudaMemsetAsync(w.tbl, 0xFF, (size_t)w.capacity * 8, stream));
    if (i64) SPX_CHECK_CUDA(cudaMemsetAsync(w.tvals, 0x7F, (size_t)w.capacity * 4, stream));
    SPX_CHECK_CUDA(cudaMemsetAsync(w.bitmap, 0, w.rank_bytes + sizeof(int), stream));
    p2v_offsets_kernel<<<1, P2V_PLAN_THREADS, 0, stream>>>(point_offsets, batch_size, N, w.eff);
    SPX_CHECK_LAUNCH("p2v_offsets_kernel");
    const unsigned nblk = (unsigned)div_up64(N, 256);
    if (int rc = visit_table(i64, w.tbl, w.tvals, w.capacity, [&](auto t) {
            p2v_insert_kernel<<<nblk, 256, 0, stream>>>(t, g, points, N, num_features, w.eff, batch_size, w.keys);
            SPX_CHECK_LAUNCH("p2v_insert_kernel");
            p2v_mark_kernel<<<nblk, 256, 0, stream>>>(t, w.keys, N, w.first, w.bitmap, w.tile_cnt, w.tiles, w.done);
            SPX_CHECK_LAUNCH("p2v_mark_kernel");
            return 0;
        })) return rc;
    p2v_plan_kernel<<<1, P2V_PLAN_THREADS, 0, stream>>>(w.eff, batch_size, w.bitmap, w.tile_cnt, max_voxels, bound,
                                                        w.rbase, w.kept, w.base, num_valid, status);
    SPX_CHECK_LAUNCH("p2v_plan_kernel");
    p2v_rows_kernel<<<nblk, 256, 0, stream>>>(g, w.keys, w.first, N, vol, w.bitmap, w.tile_cnt, w.rbase, w.kept,
                                              w.base, bound, pc_voxel_id, w.sort_key, indices);
    SPX_CHECK_LAUNCH("p2v_rows_kernel");
    // stable sort of the points by row (points without a row keyed `bound`, last): position inside a row's
    // segment = rank in input order
    if (int rc = sort_by_key(w.sort_key, N, bound, w.order, w.sort_ws, w.sort_ws_bytes, stream)) return rc;
    if (int rc = segment_offsets(w.sort_key, N, bound, w.start, stream)) return rc;
    p2v_scatter_kernel<<<(unsigned)div_up64(N * num_features, 256), 256, 0, stream>>>(
        points, num_features, w.sort_key, (const uint32_t *)w.order, N, (uint32_t)bound, w.start, max_points_per_voxel,
        voxels);
    SPX_CHECK_LAUNCH("p2v_scatter_kernel");
    p2v_fill_kernel<<<(unsigned)div_up64(bound * row_elems, 256), 256, 0, stream>>>(
        w.start, bound, max_points_per_voxel, num_features, empty_mean, ncols, num_per_voxel, indices, voxels);
    SPX_CHECK_LAUNCH("p2v_fill_kernel");
    return 0;
}

extern "C" size_t spx_point2voxel_workspace_size(int64_t num_points, int ndim) {
    if (num_points < 1) num_points = 1;
    const size_t n = (size_t)num_points;
    size_t total = 0;
    total += align_up((size_t)table_capacity(num_points, 2) * 8, 256) + align_up((size_t)table_capacity(num_points, 2) * 4, 256);
    total += align_up(n * 8, 256) + 4 * align_up(n * 4, 256) + align_up(cub_sort_pairs_temp_bytes(num_points), 256);
    total += align_up((n + 2) * 4, 256) + 256;
    (void)ndim;
    return total + 2048;
}

extern "C" int spx_point2voxel_stage1(const float *points, int64_t N, int num_features, int ndim, int zyx,
                                      const float *vsize_host, const int *grid_size_host,
                                      const float *coors_range_host, int64_t max_voxels, int64_t *num_voxels_host,
                                      int64_t *total_voxels_host, void *workspace, size_t workspace_bytes,
                                      spx_stream_t stream_) {
    SPX_REQUIRE(num_voxels_host != nullptr && total_voxels_host != nullptr, "point2voxel: count pointers are NULL");
    *num_voxels_host = 0;
    *total_voxels_host = 0;
    if (N == 0) return 0;
    SPX_REQUIRE(points && workspace, "point2voxel: NULL pointer argument");
    SPX_REQUIRE(N < 2147483647ll && num_features >= ndim && max_voxels > 0, "point2voxel: bad sizes");
    P2VGeom g;
    if (p2v_geom(ndim, zyx, vsize_host, grid_size_host, coors_range_host, g)) return 2;
    P2VWs w;
    if (p2v_carve(N, grid_size_host, ndim, workspace, workspace_bytes, w)) return 2;
    cudaStream_t stream = (cudaStream_t)stream_;
    SPX_CHECK_CUDA(cudaMemsetAsync(w.tbl, 0xFF, (size_t)w.capacity * 8, stream));
    SPX_CHECK_CUDA(cudaMemsetAsync(w.counter, 0, sizeof(int), stream));
    const unsigned nblk = (unsigned)div_up64(N, 256), cblk = (unsigned)div_up64(w.capacity, 256);
    if (w.i64) SPX_CHECK_CUDA(cudaMemsetAsync(w.tvals, 0x7F, (size_t)w.capacity * 4, stream));
    if (int rc = visit_table(w.i64, w.tbl, w.tvals, w.capacity, [&](auto t) {
            p2v_insert_kernel<<<nblk, 256, 0, stream>>>(t, g, points, N, num_features, nullptr, 1, w.keys);
            SPX_CHECK_LAUNCH("p2v_insert_kernel");
            p2v_collect_kernel<<<cblk, 256, 0, stream>>>(t, w.capacity, w.a0, w.a1, w.counter);
            SPX_CHECK_LAUNCH("p2v_collect_kernel");
            return 0;
        })) return rc;
    int total = 0;
    SPX_CHECK_CUDA(cudaMemcpyAsync(&total, w.counter, sizeof(int), cudaMemcpyDeviceToHost, stream));
    SPX_CHECK_CUDA(cudaStreamSynchronize(stream));
    *total_voxels_host = total;
    *num_voxels_host = total < max_voxels ? total : max_voxels;
    if (total == 0) return 0;
    // rank the voxels by their first point (0..N - 1): (first point, slot) sorted by first point -> b0 / b1
    size_t tmp = w.sort_tmp_bytes;
    SPX_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, tmp, w.a0, w.b0, w.a1, w.b1, total, 0,
                                                   sort_key_bits(N - 1), stream));
    count_launch(3);
    return 0;
}

extern "C" int spx_point2voxel_stage2(const float *points, int64_t N, int num_features, int ndim, int zyx,
                                      const float *vsize_host, const int *grid_size_host,
                                      const float *coors_range_host, int64_t num_voxels, int64_t total_voxels,
                                      int max_points_per_voxel, int empty_mean, float *voxels, int32_t *indices,
                                      int32_t *num_per_voxel, int64_t *pc_voxel_id, void *workspace,
                                      size_t workspace_bytes, spx_stream_t stream_) {
    if (N == 0) return 0;
    SPX_REQUIRE(points && pc_voxel_id && workspace, "point2voxel: NULL pointer argument");
    SPX_REQUIRE(num_voxels >= 0 && num_voxels <= total_voxels && total_voxels <= N, "point2voxel: bad voxel counts");
    SPX_REQUIRE(max_points_per_voxel > 0, "point2voxel: max_points_per_voxel must be positive");
    P2VGeom g;
    if (p2v_geom(ndim, zyx, vsize_host, grid_size_host, coors_range_host, g)) return 2;
    P2VWs w;
    if (p2v_carve(N, grid_size_host, ndim, workspace, workspace_bytes, w)) return 2;
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned nblk = (unsigned)div_up64(N, 256);
    const uint32_t M = (uint32_t)num_voxels;
    SPX_REQUIRE(num_voxels == 0 || (voxels && indices && num_per_voxel), "point2voxel: NULL output");
    if (int rc = visit_table(w.i64, w.tbl, w.tvals, w.capacity, [&](auto t) {
            if (total_voxels) {
                p2v_assign_kernel<<<(unsigned)div_up64(total_voxels, 256), 256, 0, stream>>>(t, g, w.b1, total_voxels, num_voxels, indices);
                SPX_CHECK_LAUNCH("p2v_assign_kernel");
            }
            p2v_lookup_kernel<<<nblk, 256, 0, stream>>>(t, w.keys, N, M, pc_voxel_id, w.a0, w.a1);
            SPX_CHECK_LAUNCH("p2v_lookup_kernel");
            return 0;
        })) return rc;
    if (num_voxels == 0) return 0;
    // stable sort of the points by voxel id: position inside a segment = rank in input order
    size_t tmp = w.sort_tmp_bytes;
    SPX_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, tmp, w.a0, w.b0, w.a1, w.b1, (int)N, 0, sort_key_bits(M),
                                                   stream));
    count_launch(3);
    p2v_segments_kernel<<<(unsigned)div_up64(N + 1, 256), 256, 0, stream>>>(w.b0, N, M, w.start);
    SPX_CHECK_LAUNCH("p2v_segments_kernel");
    p2v_scatter_kernel<<<(unsigned)div_up64(N * num_features, 256), 256, 0, stream>>>(
        points, num_features, w.b0, w.b1, N, M, w.start, max_points_per_voxel, voxels);
    SPX_CHECK_LAUNCH("p2v_scatter_kernel");
    p2v_finish_kernel<<<(unsigned)div_up64(num_voxels, 128), 128, 0, stream>>>(w.start, num_voxels, max_points_per_voxel,
                                                                               num_features, empty_mean, num_per_voxel, voxels);
    SPX_CHECK_LAUNCH("p2v_finish_kernel");
    return 0;
}
