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
#include "common.cuh"
#include "hash.cuh"
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

template <typename Table>
__global__ void p2v_insert_kernel(Table table, P2VGeom g, const float *__restrict__ points, int64_t n, int nf,
                                  int64_t *__restrict__ keys) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c[SPX_MAX_NDIM];
    int64_t key = -1;
    if (p2v_coord(g, points + i * nf, c)) {
        key = 0;
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

struct P2VWs {
    void *tbl; int32_t *tvals; uint32_t capacity; bool i64;
    int64_t *keys;
    uint32_t *a0, *a1, *b0, *b1;          // sort buffers (keys / values, in / out), sized max(N, capacity-bound)
    void *sort_tmp; size_t sort_tmp_bytes;
    int32_t *start; int *counter;
};

static size_t p2v_sort_tmp(int64_t n) {
    // The size query goes through the CUDA runtime: a stale error left by an earlier failed call (e.g. a
    // refused stream capture) would make it return early with bytes = 0, and the workspace computed here
    // would then be smaller than what the same query yields a moment later.  Clear the state first and
    // never return less than a bound that covers CUB's double buffers + histograms.
    cudaGetLastError();
    size_t bytes = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                                    (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)n);
    const size_t floor_bytes = (size_t)(n > 0 ? n : 1) * 16 + (1u << 20);
    if (e != cudaSuccess) { cudaGetLastError(); return floor_bytes; }
    return bytes > floor_bytes ? bytes : floor_bytes;
}

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
    w.sort_tmp_bytes = p2v_sort_tmp(n);
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

}  // namespace spx

using namespace spx;

extern "C" size_t spx_point2voxel_workspace_size(int64_t num_points, int ndim) {
    if (num_points < 1) num_points = 1;
    const size_t n = (size_t)num_points;
    size_t total = 0;
    total += align_up((size_t)table_capacity(num_points, 2) * 8, 256) + align_up((size_t)table_capacity(num_points, 2) * 4, 256);
    total += align_up(n * 8, 256) + 4 * align_up(n * 4, 256) + align_up(p2v_sort_tmp(num_points), 256);
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
    if (!w.i64) {
        Table32 t{(unsigned long long *)w.tbl, w.capacity - 1};
        p2v_insert_kernel<<<nblk, 256, 0, stream>>>(t, g, points, N, num_features, w.keys);
        SPX_CHECK_LAUNCH("p2v_insert_kernel");
        p2v_collect_kernel<<<cblk, 256, 0, stream>>>(t, w.capacity, w.a0, w.a1, w.counter);
    } else {
        SPX_CHECK_CUDA(cudaMemsetAsync(w.tvals, 0x7F, (size_t)w.capacity * 4, stream));
        Table64 t{(long long *)w.tbl, w.tvals, w.capacity - 1};
        p2v_insert_kernel<<<nblk, 256, 0, stream>>>(t, g, points, N, num_features, w.keys);
        SPX_CHECK_LAUNCH("p2v_insert_kernel");
        p2v_collect_kernel<<<cblk, 256, 0, stream>>>(t, w.capacity, w.a0, w.a1, w.counter);
    }
    SPX_CHECK_LAUNCH("p2v_collect_kernel");
    int total = 0;
    SPX_CHECK_CUDA(cudaMemcpyAsync(&total, w.counter, sizeof(int), cudaMemcpyDeviceToHost, stream));
    SPX_CHECK_CUDA(cudaStreamSynchronize(stream));
    *total_voxels_host = total;
    *num_voxels_host = total < max_voxels ? total : max_voxels;
    if (total == 0) return 0;
    // rank the voxels by their first point: (first point, slot) sorted by first point -> b0 / b1
    int end_bit = 1;
    while (end_bit < 32 && ((int64_t)1 << end_bit) < N) ++end_bit;
    size_t tmp = w.sort_tmp_bytes;
    SPX_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, tmp, w.a0, w.b0, w.a1, w.b1, total, 0, end_bit, stream));
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
    if (!w.i64) {
        Table32 t{(unsigned long long *)w.tbl, w.capacity - 1};
        if (total_voxels) {
            p2v_assign_kernel<<<(unsigned)div_up64(total_voxels, 256), 256, 0, stream>>>(t, g, w.b1, total_voxels, num_voxels, indices);
            SPX_CHECK_LAUNCH("p2v_assign_kernel");
        }
        p2v_lookup_kernel<<<nblk, 256, 0, stream>>>(t, w.keys, N, M, pc_voxel_id, w.a0, w.a1);
    } else {
        Table64 t{(long long *)w.tbl, w.tvals, w.capacity - 1};
        if (total_voxels) {
            p2v_assign_kernel<<<(unsigned)div_up64(total_voxels, 256), 256, 0, stream>>>(t, g, w.b1, total_voxels, num_voxels, indices);
            SPX_CHECK_LAUNCH("p2v_assign_kernel");
        }
        p2v_lookup_kernel<<<nblk, 256, 0, stream>>>(t, w.keys, N, M, pc_voxel_id, w.a0, w.a1);
    }
    SPX_CHECK_LAUNCH("p2v_lookup_kernel");
    if (num_voxels == 0) return 0;
    // stable sort of the points by voxel id: position inside a segment = rank in input order
    int end_bit = 1;
    while (end_bit < 32 && ((int64_t)1 << end_bit) <= (int64_t)M) ++end_bit;
    size_t tmp = w.sort_tmp_bytes;
    SPX_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, tmp, w.a0, w.b0, w.a1, w.b1, (int)N, 0, end_bit, stream));
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
