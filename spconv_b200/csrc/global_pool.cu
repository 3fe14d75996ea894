// Per-sample global max / mean pooling over the valid rows of a (possibly padded) feature matrix [rows, C]
// (MaskedGlobalMaxPool / MaskedGlobalAvgPool, pytorch/pool.py).  M = *num_valid (NULL: every row); rows
// [M, rows) are never read, neither features nor coordinates.  Row r counts for sample b when r < M and
// coords[r, 0] == b with 0 <= b < B; other rows are dropped.
//
// Forward:
//   keys     : key[r] = sample of row r, B for padding and dropped rows;
//   group    : sort_by_key (segments.cuh), so the rows of sample b are order[offsets[b] .. offsets[b+1]) in
//              ascending row order whatever the padding;
//   segments : one block finds offsets [B+1] by binary search in the sorted keys (first_at_least), cuts every
//              segment into chunks of GP_CHUNK rows and numbers the chunks (cstart [B+1], an exclusive scan);
//   reduce   : one block per (chunk, channel slice), grid sized for the worst case ceil(rows / GP_CHUNK) + B;
//              blocks past the last chunk exit.  Row lane l folds rows p0 + l, p0 + l + lanes, ... in ascending
//              order, then the lanes merge in a fixed binary tree; the partial goes to workspace [chunk][C];
//   finalize : per (sample, channel) 32 lanes merge the sample's chunks p, p + 32, ... in order, then a fixed
//              tree; writes out, and argmax [B, C] (max) or count [B] (mean) for the backward.
// Max partials are (value, row) pairs ordered by max_beats: a NaN beats every number, then the greater value,
// then, on equality (-0 == +0), the lower row; that is a total order, so the winner is the first row in
// ascending order that attains the maximum (np.argmax).  out is copied from x[argmax] bit for bit.
// Mean partials are fp32 sums; out = sum / count, rounded once.
// Backward: one thread per 16-byte vector of a row writes dy[b] at the argmax rows (max) or dy[b] / count[b]
// (mean), and 0 on padding and dropped rows: every element of din is written once, nothing is scattered.
// The summation order depends only on the sample's valid rows, never on `rows`, M beyond them or the grid,
// and no float atomics are used, so every result is bit-reproducible and independent of padding.
#include "rows.cuh"
#include "segments.cuh"

namespace spx {

constexpr int GP_THREADS = 256;
constexpr int GP_SEG_THREADS = 1024; // the one block of the segments kernel
constexpr int GP_FIN_CH = 8;         // finalize: channels per block
constexpr int GP_FIN_LANES = 32;     // finalize: partial lanes per channel
constexpr int GP_MAX_BATCH = 1 << 20;
constexpr int GP_MAX_CHANNELS = 1 << 16;   // finalize grid.y = C / GP_FIN_CH must stay below 2^16

__global__ void gp_keys_kernel(const int32_t *__restrict__ coords, int64_t rows, int row_ints, int batch_size,
                               const int32_t *__restrict__ num_valid, uint32_t *__restrict__ keys) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= rows) return;
    uint32_t key = (uint32_t)batch_size;
    if (r < valid_rows(num_valid, rows)) {
        const int32_t b = __ldg(coords + r * row_ints);
        if (b >= 0 && b < batch_size) key = (uint32_t)b;
    }
    keys[r] = key;
}

// One block: thread t owns the samples [t * per, (t + 1) * per).  offsets [B+1], cstart [B+1] (first chunk of
// every sample, cstart[B] = number of chunks) and, when count != NULL, count [B].
__global__ void __launch_bounds__(GP_SEG_THREADS)
gp_segments_kernel(const uint32_t *__restrict__ keys, int32_t n, int batch_size, int32_t *__restrict__ offsets,
                   int32_t *__restrict__ cstart, int32_t *__restrict__ count) {
    __shared__ int32_t s_scan[GP_SEG_THREADS];
    const int t = threadIdx.x;
    const int per = (batch_size + GP_SEG_THREADS - 1) / GP_SEG_THREADS;
    const int lo = min(t * per, batch_size), hi = min(lo + per, batch_size);
    int32_t chunks = 0;
    int32_t next = first_at_least(keys, n, (uint32_t)lo);
    for (int b = lo; b < hi; ++b) {
        const int32_t cur = next;
        next = first_at_least(keys, n, (uint32_t)b + 1);
        chunks += (next - cur + GP_CHUNK - 1) / GP_CHUNK;
    }
    s_scan[t] = chunks;
    for (int s = 1; s < GP_SEG_THREADS; s <<= 1) {          // inclusive Hillis-Steele scan of the chunk counts
        __syncthreads();
        const int32_t add = t >= s ? s_scan[t - s] : 0;
        __syncthreads();
        s_scan[t] += add;
    }
    __syncthreads();
    int32_t c = s_scan[t] - chunks;
    next = first_at_least(keys, n, (uint32_t)lo);
    for (int b = lo; b < hi; ++b) {
        const int32_t cur = next;
        next = first_at_least(keys, n, (uint32_t)b + 1);
        offsets[b] = cur;
        cstart[b] = c;
        if (count) count[b] = next - cur;
        c += (next - cur + GP_CHUNK - 1) / GP_CHUNK;
    }
    if (t == GP_SEG_THREADS - 1) {
        offsets[batch_size] = first_at_least(keys, n, (uint32_t)batch_size);
        cstart[batch_size] = s_scan[t];
    }
}

template <typename T, int W, bool MEAN, bool A>
__global__ void __launch_bounds__(GP_THREADS)
gp_reduce_kernel(const T *__restrict__ x, const int32_t *__restrict__ order, const int32_t *__restrict__ offsets,
                 const int32_t *__restrict__ cstart, int batch_size, int channels, int vecs, int tpr,
                 float2 *__restrict__ partials) {
    __shared__ float s_v[GP_THREADS * W];
    __shared__ int s_r[MEAN ? 1 : GP_THREADS * W];
    // sample_chunk (rows.cuh) written out: called, it gives these kernels a different register allocation
    const int32_t k = (int32_t)blockIdx.x;
    if (k >= __ldg(cstart + batch_size)) return;
    const int b = last_at_most(cstart, batch_size, k);
    const int32_t p0 = __ldg(offsets + b) + (k - __ldg(cstart + b)) * GP_CHUNK;
    const int32_t seg_end = __ldg(offsets + b + 1);
    const int32_t end = seg_end < p0 + GP_CHUNK ? seg_end : p0 + GP_CHUNK;
    const int lanes = GP_THREADS / tpr;
    const RowThread t = row_thread(vecs, tpr);
    float acc[W];
    int arg[W];
#pragma unroll
    for (int j = 0; j < W; ++j) {
        acc[j] = MEAN ? 0.f : -INFINITY;
        arg[j] = -1;
    }
    if (t.active) {
        const T *base = x + (int64_t)t.v * W;
        auto fold = [&](const float (&f)[W], int r) {        // rows of a lane come in ascending order
#pragma unroll
            for (int j = 0; j < W; ++j) {
                if constexpr (MEAN) {
                    acc[j] += f[j];
                } else if (max_beats(f[j], r, acc[j], arg[j])) {
                    acc[j] = f[j];
                    arg[j] = r;
                }
            }
        };
        int64_t p = p0 + t.lane;
        for (; p + lanes < end; p += 2 * lanes) {             // two rows in flight (four spill), folded in row order
            int r[2];
            float f[2][W];
#pragma unroll
            for (int u = 0; u < 2; ++u) r[u] = __ldg(order + p + u * lanes);
#pragma unroll
            for (int u = 0; u < 2; ++u) row_load<T, W, A>(base + (int64_t)r[u] * channels, f[u]);
#pragma unroll
            for (int u = 0; u < 2; ++u) fold(f[u], r[u]);
        }
        for (; p < end; p += lanes) {
            const int r = __ldg(order + p);
            float f[W];
            row_load<T, W, A>(base + (int64_t)r * channels, f);
            fold(f, r);
        }
    }
    // fixed tree over the row lanes: at step s, lanes [0, s) fold lanes [s, 2s) into their own slots
    const int slot = threadIdx.x;
#pragma unroll
    for (int j = 0; j < W; ++j) {
        s_v[slot * W + j] = acc[j];
        if constexpr (!MEAN) s_r[slot * W + j] = arg[j];
    }
    for (int s = lanes >> 1; s >= 1; s >>= 1) {
        __syncthreads();
        if (t.lane < s) {
            const int o = slot + s * tpr;
#pragma unroll
            for (int j = 0; j < W; ++j) {
                if constexpr (MEAN) {
                    s_v[slot * W + j] = acc[j] = acc[j] + s_v[o * W + j];
                } else if (max_beats(s_v[o * W + j], s_r[o * W + j], acc[j], arg[j])) {
                    s_v[slot * W + j] = acc[j] = s_v[o * W + j];
                    s_r[slot * W + j] = arg[j] = s_r[o * W + j];
                }
            }
        }
    }
    if (t.lane == 0 && t.active) {
        float2 *dst = partials + (int64_t)k * channels + (int64_t)t.v * W;
#pragma unroll
        for (int j = 0; j < W; ++j) dst[j] = make_float2(acc[j], __int_as_float(arg[j]));
    }
}

// grid (B, ceil(C / GP_FIN_CH)); lane pl of channel cl merges chunks cstart[b] + pl, + 32, ... in order
template <typename T, bool MEAN>
__global__ void __launch_bounds__(GP_FIN_CH * GP_FIN_LANES)
gp_finalize_kernel(const T *__restrict__ x, const float2 *__restrict__ partials, const int32_t *__restrict__ offsets,
                   const int32_t *__restrict__ cstart, int channels, T *__restrict__ out, int32_t *__restrict__ argmax) {
    __shared__ float s_v[GP_FIN_LANES][GP_FIN_CH];
    __shared__ int s_r[GP_FIN_LANES][GP_FIN_CH];
    const int cl = threadIdx.x % GP_FIN_CH, pl = threadIdx.x / GP_FIN_CH;
    const int b = blockIdx.x;
    const int c = blockIdx.y * GP_FIN_CH + cl;
    const bool active = c < channels;
    const int32_t k0 = __ldg(cstart + b), k1 = __ldg(cstart + b + 1);
    float acc = MEAN ? 0.f : -INFINITY;
    int arg = -1;
    if (active)
        for (int32_t k = k0 + pl; k < k1; k += GP_FIN_LANES) {
            const float2 p = partials[(int64_t)k * channels + c];
            if constexpr (MEAN) acc += p.x;
            else if (max_beats(p.x, __float_as_int(p.y), acc, arg)) { acc = p.x; arg = __float_as_int(p.y); }
        }
    s_v[pl][cl] = acc;
    s_r[pl][cl] = arg;
    for (int s = GP_FIN_LANES / 2; s >= 1; s >>= 1) {
        __syncthreads();
        if (pl < s) {
            if constexpr (MEAN) {
                s_v[pl][cl] = acc = acc + s_v[pl + s][cl];
            } else if (max_beats(s_v[pl + s][cl], s_r[pl + s][cl], acc, arg)) {
                s_v[pl][cl] = acc = s_v[pl + s][cl];
                s_r[pl][cl] = arg = s_r[pl + s][cl];
            }
        }
    }
    if (pl != 0 || !active) return;
    const int64_t o = (int64_t)b * channels + c;
    if constexpr (MEAN) {
        const int32_t n = __ldg(offsets + b + 1) - __ldg(offsets + b);
        out[o] = from_float<T>(n > 0 ? __fdiv_rn(acc, (float)n) : 0.f);
    } else {
        out[o] = arg >= 0 ? x[(int64_t)arg * channels + c] : from_float<T>(0.f);
        argmax[o] = arg;
    }
}

template <typename T, int W, bool MEAN>
__global__ void __launch_bounds__(GP_THREADS)
gp_bwd_kernel(const T *__restrict__ dy, const int32_t *__restrict__ coords, int64_t rows, int row_ints,
              int batch_size, int channels, int vecs, const int32_t *__restrict__ num_valid,
              const int32_t *__restrict__ argmax, const int32_t *__restrict__ count, T *__restrict__ din) {
    const int64_t idx = blockIdx.x * (int64_t)GP_THREADS + threadIdx.x;
    const int64_t r = idx / vecs;
    const int v = (int)(idx - r * vecs);
    if (r >= rows) return;
    int b = -1;
    if (r < valid_rows(num_valid, rows)) {
        b = __ldg(coords + r * row_ints);
        if (b >= batch_size) b = -1;
    }
    T e[W];
#pragma unroll
    for (int j = 0; j < W; ++j) e[j] = from_float<T>(0.f);
    if (b >= 0) {
        const int64_t o = (int64_t)b * channels + (int64_t)v * W;
        if constexpr (MEAN) {
            float f[W];
            row_load<T, W>(dy + o, f);
            const float n = (float)__ldg(count + b);           // >= 1: row r itself counts
#pragma unroll
            for (int j = 0; j < W; ++j) e[j] = from_float<T>(__fdiv_rn(f[j], n));
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (__ldg(argmax + o + j) == (int32_t)r) e[j] = dy[o + j];
        }
    }
    row_store_raw<T, W>(din + r * channels + (int64_t)v * W, e);
}

// ---------------------------------------------------------------- host side
static int64_t gp_max_chunks(int64_t rows, int batch_size) {
    return (rows + GP_CHUNK - 1) / GP_CHUNK + batch_size;
}

// keys -> sort_by_key -> segments: order [rows], offsets [B+1], cstart [B+1] and, when count != NULL, count [B]
// (see the top of this file).  keys [rows] and sort_ws (radix_argsort_workspace_bytes(rows)) are scratch.  Shared
// with group_norm.cu.
int group_samples(const int32_t *coords, int64_t rows, int row_ints, int batch_size, const int32_t *num_valid,
                  uint32_t *keys, int32_t *order, void *sort_ws, int32_t *offsets, int32_t *cstart, int32_t *count,
                  cudaStream_t stream) {
    if (rows > 0) {
        gp_keys_kernel<<<(unsigned)div_up64(rows, GP_THREADS), GP_THREADS, 0, stream>>>(
            coords, rows, row_ints, batch_size, num_valid, keys);
        SPX_CHECK_LAUNCH("gp_keys_kernel");
        if (int rc = sort_by_key(keys, rows, batch_size, order, sort_ws, radix_argsort_workspace_bytes(rows), stream))
            return rc;
    }
    gp_segments_kernel<<<1, GP_SEG_THREADS, 0, stream>>>(keys, (int32_t)rows, batch_size, offsets, cstart, count);
    SPX_CHECK_LAUNCH("gp_segments_kernel");
    return 0;
}

static int gp_check(const char *who, int mode, int64_t rows, int row_ints, int batch_size, int channels,
                    int dtype) {
    SPX_REQUIRE(mode == 0 || mode == 1, "%s: mode must be 0 (max) or 1 (mean), got %d", who, mode);
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(row_ints >= 1, "%s: coordinate rows must hold the batch index, got %d ints", who, row_ints);
    SPX_REQUIRE(batch_size >= 1 && batch_size <= GP_MAX_BATCH, "%s: batch_size must be in [1, 2^20], got %d", who,
                batch_size);
    SPX_REQUIRE(channels >= 1 && channels <= GP_MAX_CHANNELS, "%s: channels must be in [1, 65536], got %d", who,
                channels);
    SPX_REQUIRE(dtype == SPX_F32 || dtype == SPX_F16 || dtype == SPX_BF16,
                "%s: unsupported dtype %d (float32, float16 and bfloat16 only)", who, dtype);
    return 0;
}

struct GpFwdArgs {
    int mode;
    const void *x;
    const int32_t *order, *offsets, *cstart;
    int64_t rows;
    int batch_size, channels;
    float2 *partials;
    void *out;
    int32_t *argmax;
};

template <typename T, int W, bool MEAN, bool A> static int gp_fwd_launch(const GpFwdArgs &a, cudaStream_t stream) {
    const int vecs = a.channels / W;
    if (a.rows > 0) {
        const int tpr = row_tpr(vecs);
        const dim3 grid((unsigned)gp_max_chunks(a.rows, a.batch_size), (unsigned)div_up64(vecs, tpr));
        gp_reduce_kernel<T, W, MEAN, A><<<grid, GP_THREADS, 0, stream>>>(
            static_cast<const T *>(a.x), a.order, a.offsets, a.cstart, a.batch_size, a.channels, vecs, tpr,
            a.partials);
        SPX_CHECK_LAUNCH("gp_reduce_kernel");
    }
    const dim3 grid((unsigned)a.batch_size, (unsigned)div_up64(a.channels, GP_FIN_CH));
    gp_finalize_kernel<T, MEAN><<<grid, GP_FIN_CH * GP_FIN_LANES, 0, stream>>>(
        static_cast<const T *>(a.x), a.partials, a.offsets, a.cstart, a.channels, static_cast<T *>(a.out), a.argmax);
    SPX_CHECK_LAUNCH("gp_finalize_kernel");
    return 0;
}

template <typename T> static int gp_fwd_dispatch(const GpFwdArgs &a, cudaStream_t stream) {
    constexpr int W = 16 / sizeof(T);
    const RowWidth w = row_width(a.channels * sizeof(T), a.x);     // a reduction: W whenever wide
    if (!w.wide)
        return a.mode == 1 ? gp_fwd_launch<T, 1, true, false>(a, stream) : gp_fwd_launch<T, 1, false, false>(a, stream);
    if (a.rows == 0 || w.aligned)
        return a.mode == 1 ? gp_fwd_launch<T, W, true, true>(a, stream) : gp_fwd_launch<T, W, false, true>(a, stream);
    return a.mode == 1 ? gp_fwd_launch<T, W, true, false>(a, stream) : gp_fwd_launch<T, W, false, false>(a, stream);
}

struct GpBwdArgs {
    int mode;
    const void *dy;
    const int32_t *coords;
    int64_t rows;
    int row_ints, batch_size, channels;
    const int32_t *num_valid, *argmax, *count;
    void *din;
};

template <typename T, int W, bool MEAN> static int gp_bwd_launch(const GpBwdArgs &a, cudaStream_t stream) {
    const int vecs = a.channels / W;
    gp_bwd_kernel<T, W, MEAN><<<(unsigned)div_up64(a.rows * vecs, GP_THREADS), GP_THREADS, 0, stream>>>(
        static_cast<const T *>(a.dy), a.coords, a.rows, a.row_ints, a.batch_size, a.channels, vecs, a.num_valid,
        a.argmax, a.count, static_cast<T *>(a.din));
    SPX_CHECK_LAUNCH("gp_bwd_kernel");
    return 0;
}

template <typename T> static int gp_bwd_dispatch(const GpBwdArgs &a, cudaStream_t stream) {
    constexpr int W = 16 / sizeof(T);
    const RowWidth w = row_width(a.channels * sizeof(T), a.dy, a.din);
    const bool vec = w.wide && w.aligned;
    if (a.mode == 1) return vec ? gp_bwd_launch<T, W, true>(a, stream) : gp_bwd_launch<T, 1, true>(a, stream);
    return vec ? gp_bwd_launch<T, W, false>(a, stream) : gp_bwd_launch<T, 1, false>(a, stream);
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_global_pool_workspace_size(int64_t rows, int batch_size, int channels) {
    if (rows < 0 || batch_size < 1 || channels < 1) return 0;
    return 2 * align_up((size_t)rows * 4, 256) + radix_argsort_workspace_bytes(rows) +
           2 * align_up((size_t)(batch_size + 1) * 4, 256) +
           align_up((size_t)gp_max_chunks(rows, batch_size) * channels * sizeof(float2), 256) + 1024;
}

extern "C" int spx_global_pool_fwd(int mode, const void *features, const int32_t *coords, int64_t rows, int row_ints,
                                   int batch_size, int channels, int dtype, const int32_t *num_valid, void *out,
                                   int32_t *argmax, int32_t *count, void *workspace, size_t workspace_bytes,
                                   spx_stream_t stream_) {
    const char *who = "global_pool_fwd";
    if (int rc = gp_check(who, mode, rows, row_ints, batch_size, channels, dtype)) return rc;
    SPX_REQUIRE(out && workspace, "%s: NULL pointer argument (out, workspace)", who);
    SPX_REQUIRE(rows == 0 || (features && coords), "%s: NULL pointer argument (features, coords)", who);
    SPX_REQUIRE(mode == 1 || argmax, "%s: NULL pointer argument (argmax, needed by max pooling)", who);
    SPX_REQUIRE(mode == 0 || count, "%s: NULL pointer argument (count, needed by mean pooling)", who);
    const size_t need = spx_global_pool_workspace_size(rows, batch_size, channels);
    SPX_REQUIRE(workspace_bytes >= need, "%s: workspace too small: need %zu, have %zu", who, need, workspace_bytes);
    WorkspaceCarver ws(workspace, workspace_bytes);
    uint32_t *keys = ws.take<uint32_t>((size_t)rows);
    int32_t *order = ws.take<int32_t>((size_t)rows);
    void *sort_ws = ws.take<char>(radix_argsort_workspace_bytes(rows));
    int32_t *offsets = ws.take<int32_t>((size_t)batch_size + 1);
    int32_t *cstart = ws.take<int32_t>((size_t)batch_size + 1);
    float2 *partials = ws.take<float2>((size_t)gp_max_chunks(rows, batch_size) * channels);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (int rc = group_samples(coords, rows, row_ints, batch_size, num_valid, keys, order, sort_ws, offsets, cstart,
                               mode == 1 ? count : nullptr, stream))
        return rc;
    GpFwdArgs a{mode, features, order, offsets, cstart, rows, batch_size, channels, partials, out, argmax};
    return dispatch_dtype(dtype, [&](auto t) { return gp_fwd_dispatch<typename decltype(t)::type>(a, stream); });
}

extern "C" int spx_global_pool_bwd(int mode, const void *dy, const int32_t *coords, int64_t rows, int row_ints,
                                   int batch_size, int channels, int dtype, const int32_t *num_valid,
                                   const int32_t *argmax, const int32_t *count, void *din, spx_stream_t stream_) {
    const char *who = "global_pool_bwd";
    if (int rc = gp_check(who, mode, rows, row_ints, batch_size, channels, dtype)) return rc;
    SPX_REQUIRE(dy, "%s: NULL pointer argument (dy)", who);
    SPX_REQUIRE(rows == 0 || (coords && din), "%s: NULL pointer argument (coords, din)", who);
    SPX_REQUIRE(mode == 1 || argmax, "%s: NULL pointer argument (argmax, needed by max pooling)", who);
    SPX_REQUIRE(mode == 0 || count, "%s: NULL pointer argument (count, needed by mean pooling)", who);
    if (rows == 0) return 0;
    GpBwdArgs a{mode, dy, coords, rows, row_ints, batch_size, channels, num_valid, argmax, count, din};
    cudaStream_t stream = (cudaStream_t)stream_;
    return dispatch_dtype(dtype, [&](auto t) { return gp_bwd_dispatch<typename decltype(t)::type>(a, stream); });
}
