// Per-voxel max / mean / sum of point features (PointVoxelScatter, pytorch/utils.py): the point -> voxel
// reduction of a dynamic VFE, with no host read-back.  ids [P] give every point's output row (pc_voxel_id of
// MaskedPointToVoxel); a point whose id is outside [0, rows) is dropped.
//
//   group   : row32[p] = id or -1 (ps_rows_kernel), then group_rows (segments.cuh) keyed by the rows (dropped
//             points keyed `rows`, i.e. last), so the points of row r are order[offsets[r] .. offsets[r+1]) in
//             ascending point index;
//   reduce  : one thread per 16-byte chunk of an output row (per element when C * e or the pointers do not allow
//             vectors) walks the row's points in that order.  max keeps the winner of max_beats (a NaN beats
//             every number, then the greater value, then the lower point) and copies it bit for bit, with its
//             point in argmax [rows, C]; mean is the fp32 sum divided by the count, rounded once.  sum is the
//             sa_sum_kernel of sparse_add.cu with one operand (sum_segments);
//   backward: one thread per (point, chunk) writes dx once: dy[r] where argmax[r] is the point (max), dy[r] /
//             count[r] (mean), dy[r] (sum: spx_sparse_add_gather with index = row32), 0 for a dropped point.
// The order of every reduction depends only on the row's points, and no float atomics are used, so results are
// bit-reproducible and independent of dropped points, wherever they sit.
#include "rows.cuh"
#include "segments.cuh"

namespace spx {

constexpr int PS_THREADS = 256;
constexpr int PS_INFLIGHT = 4;                   // reduce (max): points loaded per step of a row's walk
constexpr int64_t PS_MAX_ROWS = 2147483647ll;    // P and rows below 2^31 - 1
constexpr int64_t PS_MAX_BLOCKS = 2147483647ll;  // grid.x of the per-element kernels

template <typename I>
__global__ void ps_rows_kernel(const I *__restrict__ ids, int64_t n, int64_t rows, int32_t *__restrict__ row32) {
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int64_t id = (int64_t)__ldg(ids + p);
    row32[p] = id >= 0 && id < rows ? (int32_t)id : -1;
}

template <typename T, int W, bool MEAN>
__global__ void __launch_bounds__(PS_THREADS)
ps_reduce_kernel(const T *__restrict__ x, const int32_t *__restrict__ order, const int32_t *__restrict__ offsets,
                 int64_t rows, int chunks, int channels, T *__restrict__ out, int32_t *__restrict__ argmax) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = idx / chunks;
    const int ch = (int)(idx - r * chunks);
    if (r >= rows) return;
    const int32_t begin = __ldg(offsets + r), end = __ldg(offsets + r + 1);
    float acc[W];
    int arg[W];
#pragma unroll
    for (int j = 0; j < W; ++j) {
        acc[j] = 0.f;
        arg[j] = -1;
    }
    auto fold = [&](const T (&e)[W], int32_t p) {        // the row's points come in ascending index
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const float f = to_float(e[j]);
            if constexpr (MEAN) {
                acc[j] += f;
            } else if (max_beats(f, p, acc[j], arg[j])) {
                acc[j] = f;
                arg[j] = p;
            }
        }
    };
    const T *base = x + ch * W;
    int32_t q = begin;
    // max: INFLIGHT points loaded, then folded in order (one at a time, its conditional update kept the loads
    // serial); the mean's plain loop is pipelined by the compiler and measured faster on long rows
    constexpr int INFLIGHT = MEAN ? 1 : PS_INFLIGHT;
    for (; q + INFLIGHT <= end && INFLIGHT > 1; q += INFLIGHT) {
        int32_t p[INFLIGHT];
        T e[INFLIGHT][W];
#pragma unroll
        for (int u = 0; u < INFLIGHT; ++u) p[u] = __ldg(order + q + u);
#pragma unroll
        for (int u = 0; u < INFLIGHT; ++u) row_load_raw<T, W>(base + (int64_t)p[u] * channels, e[u]);
#pragma unroll
        for (int u = 0; u < INFLIGHT; ++u) fold(e[u], p[u]);
    }
    for (; q < end; ++q) {
        const int32_t p = __ldg(order + q);
        T e[W];
        row_load_raw<T, W>(base + (int64_t)p * channels, e);
        fold(e, p);
    }
    const int64_t o = r * channels + ch * W;
    T res[W];
    if constexpr (MEAN) {
        const float n = (float)(end - begin);
#pragma unroll
        for (int j = 0; j < W; ++j) res[j] = from_float<T>(end > begin ? __fdiv_rn(acc[j], n) : 0.f);
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) {                    // a bit copy of the winner (NaN payloads included)
            res[j] = arg[j] >= 0 ? base[(int64_t)arg[j] * channels + j] : from_float<T>(0.f);
            argmax[o + j] = arg[j];
        }
    }
    row_store_raw<T, W>(out + o, res);
}

template <typename T, int W, bool MEAN>
__global__ void __launch_bounds__(PS_THREADS)
ps_bwd_kernel(const T *__restrict__ dy, const int32_t *__restrict__ row32, int64_t n, int chunks, int channels,
              const int32_t *__restrict__ argmax, const int32_t *__restrict__ count, T *__restrict__ dx) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t p = idx / chunks;
    const int ch = (int)(idx - p * chunks);
    if (p >= n) return;
    const int32_t r = __ldg(row32 + p);
    T e[W];
#pragma unroll
    for (int j = 0; j < W; ++j) e[j] = from_float<T>(0.f);
    if (r >= 0) {
        const int64_t o = (int64_t)r * channels + ch * W;
        if constexpr (MEAN) {
            T g[W];
            row_load_raw<T, W>(dy + o, g);
            const float c = (float)__ldg(count + r);      // >= 1: point p itself counts
#pragma unroll
            for (int j = 0; j < W; ++j) e[j] = from_float<T>(__fdiv_rn(to_float(g[j]), c));
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (__ldg(argmax + o + j) == (int32_t)p) e[j] = dy[o + j];
        }
    }
    row_store_raw<T, W>(dx + p * channels + ch * W, e);
}

// ---------------------------------------------------------------- host side

static int ps_check(const char *who, int mode, int64_t n, int64_t rows, int channels, int dtype) {
    SPX_REQUIRE(mode >= 0 && mode <= 2, "%s: mode must be 0 (max), 1 (mean) or 2 (sum), got %d", who, mode);
    SPX_REQUIRE(n >= 0 && n < PS_MAX_ROWS, "%s: bad point count %lld", who, (long long)n);
    SPX_REQUIRE(rows >= 0 && rows < PS_MAX_ROWS, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(channels >= 1, "%s: channels must be positive, got %d", who, channels);
    SPX_REQUIRE(dtype == SPX_F32 || dtype == SPX_F16 || dtype == SPX_BF16,
                "%s: unsupported dtype %d (float32, float16 and bfloat16 only)", who, dtype);
    const int64_t most = n > rows ? n : rows;
    SPX_REQUIRE(div_up64(most * channels, PS_THREADS) <= PS_MAX_BLOCKS, "%s: %lld rows of %d channels are too many",
                who, (long long)most, channels);
    return 0;
}

template <typename T, int W, bool MEAN>
static int ps_fwd_launch(const void *x, const int32_t *order, const int32_t *offsets, int64_t rows, int channels,
                         void *out, int32_t *argmax, cudaStream_t stream) {
    const int chunks = channels / W;
    ps_reduce_kernel<T, W, MEAN><<<(unsigned)div_up64(rows * chunks, PS_THREADS), PS_THREADS, 0, stream>>>(
        static_cast<const T *>(x), order, offsets, rows, chunks, channels, static_cast<T *>(out), argmax);
    SPX_CHECK_LAUNCH("ps_reduce_kernel");
    return 0;
}

template <typename T>
static int ps_fwd_dispatch(bool mean, const void *x, const int32_t *order, const int32_t *offsets, int64_t rows,
                           int channels, void *out, int32_t *argmax, cudaStream_t stream) {
    constexpr int W = 16 / sizeof(T);
    const RowWidth w = row_width(channels * sizeof(T), x, out);
    const bool vec = w.wide && w.aligned;
    if (mean) return vec ? ps_fwd_launch<T, W, true>(x, order, offsets, rows, channels, out, argmax, stream)
                         : ps_fwd_launch<T, 1, true>(x, order, offsets, rows, channels, out, argmax, stream);
    return vec ? ps_fwd_launch<T, W, false>(x, order, offsets, rows, channels, out, argmax, stream)
               : ps_fwd_launch<T, 1, false>(x, order, offsets, rows, channels, out, argmax, stream);
}

template <typename T, int W, bool MEAN>
static int ps_bwd_launch(const void *dy, const int32_t *row32, int64_t n, int channels, const int32_t *argmax,
                         const int32_t *count, void *dx, cudaStream_t stream) {
    const int chunks = channels / W;
    ps_bwd_kernel<T, W, MEAN><<<(unsigned)div_up64(n * chunks, PS_THREADS), PS_THREADS, 0, stream>>>(
        static_cast<const T *>(dy), row32, n, chunks, channels, argmax, count, static_cast<T *>(dx));
    SPX_CHECK_LAUNCH("ps_bwd_kernel");
    return 0;
}

template <typename T>
static int ps_bwd_dispatch(bool mean, const void *dy, const int32_t *row32, int64_t n, int channels,
                           const int32_t *argmax, const int32_t *count, void *dx, cudaStream_t stream) {
    constexpr int W = 16 / sizeof(T);
    const RowWidth w = row_width(channels * sizeof(T), dy, dx);
    const bool vec = w.wide && w.aligned;
    if (mean) return vec ? ps_bwd_launch<T, W, true>(dy, row32, n, channels, argmax, count, dx, stream)
                         : ps_bwd_launch<T, 1, true>(dy, row32, n, channels, argmax, count, dx, stream);
    return vec ? ps_bwd_launch<T, W, false>(dy, row32, n, channels, argmax, count, dx, stream)
               : ps_bwd_launch<T, 1, false>(dy, row32, n, channels, argmax, count, dx, stream);
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_point_scatter_group_workspace_size(int64_t num_points) {
    return spx_sparse_add_group_workspace_size(num_points);     // the grouping's keys and sort
}

extern "C" int spx_point_scatter_group(const void *ids, int id_bytes, int64_t num_points, int64_t rows, int32_t *row32,
                                       int32_t *order, int32_t *offsets, void *workspace, size_t workspace_bytes,
                                       spx_stream_t stream_) {
    const char *who = "point_scatter_group";
    SPX_REQUIRE(id_bytes == 4 || id_bytes == 8, "%s: ids must be int32 or int64 (4 or 8 bytes), got %d bytes", who,
                id_bytes);
    SPX_REQUIRE(num_points >= 0 && num_points < PS_MAX_ROWS, "%s: bad point count %lld", who, (long long)num_points);
    SPX_REQUIRE(rows >= 0 && rows < PS_MAX_ROWS, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(offsets != nullptr, "%s: NULL pointer argument (offsets)", who);
    SPX_REQUIRE(num_points == 0 || (ids && row32 && order && workspace), "%s: NULL pointer argument (ids, row32, order, "
                "workspace)", who);
    const size_t need = spx_point_scatter_group_workspace_size(num_points);
    SPX_REQUIRE(num_points == 0 || workspace_bytes >= need, "%s: workspace too small: need %zu, have %zu", who, need,
                workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (num_points == 0) return group_rows(nullptr, 0, rows, nullptr, offsets, nullptr, 0, stream, who);
    const unsigned blk = (unsigned)div_up64(num_points, PS_THREADS);
    if (id_bytes == 4)
        ps_rows_kernel<int32_t><<<blk, PS_THREADS, 0, stream>>>(static_cast<const int32_t *>(ids), num_points, rows, row32);
    else
        ps_rows_kernel<int64_t><<<blk, PS_THREADS, 0, stream>>>(static_cast<const int64_t *>(ids), num_points, rows, row32);
    SPX_CHECK_LAUNCH("ps_rows_kernel");
    return group_rows(row32, num_points, rows, order, offsets, workspace, workspace_bytes, stream, who);
}

extern "C" int spx_point_scatter_fwd(int mode, const void *x, int64_t num_points, int channels, int dtype,
                                     const int32_t *order, const int32_t *offsets, int64_t rows, void *out,
                                     int32_t *argmax, spx_stream_t stream_) {
    const char *who = "point_scatter_fwd";
    if (int rc = ps_check(who, mode, num_points, rows, channels, dtype)) return rc;
    SPX_REQUIRE(num_points == 0 || (x && order), "%s: NULL pointer argument (x, order)", who);
    SPX_REQUIRE(rows == 0 || (offsets && out), "%s: NULL pointer argument (offsets, out)", who);
    SPX_REQUIRE(mode != 0 || rows == 0 || argmax, "%s: NULL pointer argument (argmax, needed by max)", who);
    if (rows == 0) return 0;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (mode == 2) return sum_segments(x, num_points, order, offsets, rows, channels, dtype, out, stream);
    return dispatch_dtype(dtype, [&](auto t) {
        return ps_fwd_dispatch<typename decltype(t)::type>(mode == 1, x, order, offsets, rows, channels, out, argmax,
                                                           stream);
    });
}

extern "C" int spx_point_scatter_bwd(int mode, const void *dy, const int32_t *row32, int64_t num_points, int64_t rows,
                                     int channels, int dtype, const int32_t *argmax, const int32_t *count, void *dx,
                                     spx_stream_t stream_) {
    const char *who = "point_scatter_bwd";
    if (int rc = ps_check(who, mode, num_points, rows, channels, dtype)) return rc;
    SPX_REQUIRE(num_points == 0 || (row32 && dx), "%s: NULL pointer argument (row32, dx)", who);
    SPX_REQUIRE(rows == 0 || dy, "%s: NULL pointer argument (dy)", who);
    SPX_REQUIRE(mode != 0 || rows == 0 || argmax, "%s: NULL pointer argument (argmax, needed by max)", who);
    SPX_REQUIRE(mode != 1 || rows == 0 || count, "%s: NULL pointer argument (count, needed by mean)", who);
    if (num_points == 0) return 0;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (mode == 2) {
        spx_sparse_add_operands op;
        memset(&op, 0, sizeof(op));
        op.count = 1;
        op.rows[0] = num_points;
        op.grads[0] = dx;
        return spx_sparse_add_gather(row32, dy, rows, &op, channels, dtype, stream_);
    }
    return dispatch_dtype(dtype, [&](auto t) {
        return ps_bwd_dispatch<typename decltype(t)::type>(mode == 1, dy, row32, num_points, channels, argmax, count, dx,
                                                           stream);
    });
}
