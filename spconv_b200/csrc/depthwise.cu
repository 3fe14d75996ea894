// Depthwise sparse convolution (groups = in_channels = out_channels = C) on the rulebook tables.
//
// The filter is KRSC with one input channel per group: W [C, kv] (= [C, *ksize, 1]), read as given.  A table
// T [kv, rows] (row stride `stride`, -1 = no pair) is walked in ascending kernel offset k; every sum is fp32 from
// +0 and rounded once to the output dtype.  No float atomics anywhere:
//   fwd    y[o, c]  = act(sum_k W[c, k] * x[T[k][o], c] + b[c])
//   dgrad  dx[i, c] = sum_k W[c, k] * dy[T[k'][i], c],  k' = k, or kv - 1 - k with reverse_offsets (SubM walks its
//                     forward table: T_fwd[kv - 1 - k][i] == T_bwd[k][i]), so both give the same order
//   wgrad  dW[c, k] = sum over o with T[k][o] >= 0 of dy[o, c] * x[T[k][o], c]
//
// fwd / dgrad: one thread per (row, vector of V channels).  A block holds DW_THREADS / tpr rows of one slice of
// tpr vectors; per tile of DW_KT offsets it stages the slice's filter taps (as fp32, transposed to [k][c]) and the
// table entries of its rows in shared memory -- the table rows are read as whole 128-byte lines rather than one
// small segment per warp -- then each thread gathers its row for those offsets, DW_U table entries at a time with
// their loads in flight together (entries < 0 are skipped), summed in ascending offset order.
// wgrad: one block per (chunk of DW_CHUNK rows, channel slice, tile of DW_KW offsets).  Row lane l folds rows
// r0 + l, r0 + l + lanes, ... in ascending order, the lanes merge in a fixed binary tree, and the chunk's partial
// goes to workspace [chunks][C][kv]; the finalize kernel sums the partials in ascending chunk order.  The result
// depends on the row indices alone: a chunk of padding rows (no pair, or dy = 0) adds +0.
#include "rows.cuh"

namespace spx {

constexpr int DW_THREADS = 256;
constexpr int DW_KT = 16;        // fwd / dgrad: offsets per shared-memory tile
constexpr int DW_U = 4;          // fwd / dgrad: gathers in flight per thread
constexpr int DW_CHUNK = 512;    // wgrad: rows per partial
constexpr int DW_FIN = 16;       // finalize: partial loads in flight per thread

// ---------------------------------------------------------------- fwd / dgrad: gather over the offsets
template <typename T, int V, bool REV>
__device__ __forceinline__ void dw_gather(const T *__restrict__ src, const T *__restrict__ weight, const T *__restrict__ bias,
                                          T *__restrict__ dst, const int32_t *__restrict__ table, int64_t stride, int kv,
                                          int64_t rows, int channels, int vecs, int tpr, int act, float alpha) {
    __shared__ float s_w[DW_KT][32 * V];
    __shared__ int32_t s_t[DW_KT][DW_THREADS];
    const int rpb = DW_THREADS / tpr;                    // rows per block
    const int slice_ch = tpr * V;
    const int ch_base = blockIdx.y * slice_ch;
    const int64_t r0 = (int64_t)blockIdx.x * rpb;
    const RowThread t = row_thread(vecs, tpr);
    const int c0 = t.v * V;                              // first channel of the thread
    const int64_t row = r0 + t.lane;
    const bool live = t.active && row < rows;
    float acc[V];
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] = 0.f;
    for (int k0 = 0; k0 < kv; k0 += DW_KT) {
        const int kt = kv - k0 < DW_KT ? kv - k0 : DW_KT;
        __syncthreads();                                 // the previous tile is no longer read
        for (int e = threadIdx.x; e < DW_KT * slice_ch; e += DW_THREADS) {
            const int kk = e % DW_KT, cl = e / DW_KT;    // consecutive threads: consecutive taps of one channel
            const int c = ch_base + cl;
            s_w[kk][cl] = (kk < kt && c < channels) ? to_float(__ldg(weight + (int64_t)c * kv + k0 + kk)) : 0.f;
        }
        for (int e = threadIdx.x; e < DW_KT * rpb; e += DW_THREADS) {
            const int kk = e / rpb, rl = e % rpb;        // consecutive threads: consecutive rows of one offset
            const int k = k0 + kk;
            const int64_t r = r0 + rl;
            s_t[kk][rl] = (kk < kt && r < rows) ? __ldg(table + (int64_t)(REV ? kv - 1 - k : k) * stride + r) : -1;
        }
        __syncthreads();
        if (!live) continue;
        const int cl0 = c0 - ch_base;
        for (int kk = 0; kk < kt; kk += DW_U) {
            int32_t idx[DW_U];
            float f[DW_U][V];
#pragma unroll
            for (int u = 0; u < DW_U; ++u) {
                idx[u] = kk + u < kt ? s_t[kk + u][t.lane] : -1;
                if (idx[u] >= 0) {
                    row_load<T, V>(src + (int64_t)idx[u] * channels + c0, f[u]);
                } else {
#pragma unroll
                    for (int j = 0; j < V; ++j) f[u][j] = 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < DW_U; ++u) {
                if (idx[u] < 0) continue;
#pragma unroll
                for (int j = 0; j < V; ++j) acc[j] = fmaf(s_w[kk + u][cl0 + j], f[u][j], acc[j]);
            }
        }
    }
    if (!live) return;
    if (bias != nullptr || act != SPX_ACT_NONE) {
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const float b = bias != nullptr ? to_float(__ldg(bias + c0 + j)) : 0.f;
            acc[j] = apply_act(acc[j] + b, act, alpha);
        }
    }
    row_store<T, V>(dst + row * channels + c0, acc);
}

template <typename T, int V>
__global__ void __launch_bounds__(DW_THREADS)
depthwise_fwd_kernel(const T *__restrict__ x, const T *__restrict__ weight, const T *__restrict__ bias, T *__restrict__ y,
                     const int32_t *__restrict__ table, int64_t stride, int kv, int64_t rows, int channels, int vecs,
                     int tpr, int act, float alpha) {
    dw_gather<T, V, false>(x, weight, bias, y, table, stride, kv, rows, channels, vecs, tpr, act, alpha);
}

template <typename T, int V, bool REV>
__global__ void __launch_bounds__(DW_THREADS)
depthwise_dgrad_kernel(const T *__restrict__ dy, const T *__restrict__ weight, T *__restrict__ dx,
                       const int32_t *__restrict__ table, int64_t stride, int kv, int64_t rows, int channels, int vecs,
                       int tpr) {
    dw_gather<T, V, REV>(dy, weight, nullptr, dx, table, stride, kv, rows, channels, vecs, tpr, SPX_ACT_NONE, 0.f);
}

// ---------------------------------------------------------------- wgrad: per-chunk partials, then finalize
template <int V> struct DwKw { static constexpr int value = V == 1 ? 16 : 32 / V; };   // offsets per wgrad block

template <typename T, int V, bool A>
__global__ void __launch_bounds__(DW_THREADS)
depthwise_wgrad_partial_kernel(const T *__restrict__ x, const T *__restrict__ dy, const int32_t *__restrict__ table,
                               int64_t stride, int kv, int64_t rows, int channels, int vecs, int tpr,
                               float *__restrict__ partials) {
    constexpr int KW = DwKw<V>::value;
    __shared__ float s_red[KW * V][DW_THREADS];
    const int lanes = DW_THREADS / tpr;
    const RowThread t = row_thread(vecs, tpr);
    const int c0 = t.v * V;
    const int64_t r0 = (int64_t)blockIdx.x * DW_CHUNK;
    const int k0 = blockIdx.z * KW;
    const int64_t end = rows < r0 + DW_CHUNK ? rows : r0 + DW_CHUNK;
    float acc[KW][V];
#pragma unroll
    for (int kw = 0; kw < KW; ++kw)
#pragma unroll
        for (int j = 0; j < V; ++j) acc[kw][j] = 0.f;
    if (t.active) {
        for (int64_t r = r0 + t.lane; r < end; r += lanes) {      // rows in ascending order
            int32_t idx[KW];
#pragma unroll
            for (int kw = 0; kw < KW; ++kw) idx[kw] = k0 + kw < kv ? __ldg(table + (int64_t)(k0 + kw) * stride + r) : -1;
            bool any = false;
#pragma unroll
            for (int kw = 0; kw < KW; ++kw) any |= idx[kw] >= 0;
            if (!any) continue;
            float g[V];
            row_load<T, V, A>(dy + r * channels + c0, g);
#pragma unroll
            for (int kw = 0; kw < KW; ++kw) {
                if (idx[kw] < 0) continue;
                float f[V];
                row_load<T, V, A>(x + (int64_t)idx[kw] * channels + c0, f);
#pragma unroll
                for (int j = 0; j < V; ++j) acc[kw][j] = fmaf(g[j], f[j], acc[kw][j]);
            }
        }
    }
    // fixed tree over the row lanes: at step s, lanes [0, s) add lanes [s, 2s) into their own slots
#pragma unroll
    for (int kw = 0; kw < KW; ++kw)
#pragma unroll
        for (int j = 0; j < V; ++j) s_red[kw * V + j][threadIdx.x] = acc[kw][j];
    for (int s = lanes >> 1; s >= 1; s >>= 1) {
        __syncthreads();
        if (t.lane < s) {
            const int o = threadIdx.x + s * tpr;
#pragma unroll
            for (int kw = 0; kw < KW; ++kw)
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    acc[kw][j] += s_red[kw * V + j][o];
                    s_red[kw * V + j][threadIdx.x] = acc[kw][j];
                }
        }
    }
    if (t.lane != 0 || !t.active) return;
    float *dst = partials + (int64_t)blockIdx.x * channels * kv;
#pragma unroll
    for (int j = 0; j < V; ++j) {
        const int c = c0 + j;
#pragma unroll
        for (int kw = 0; kw < KW; ++kw)
            if (k0 + kw < kv) dst[(int64_t)c * kv + k0 + kw] = acc[kw][j];
    }
}

// dW[c, k] = partials[0][c][k] + partials[1][c][k] + ... in ascending chunk order, rounded once; 0 without chunks
template <typename T>
__global__ void __launch_bounds__(DW_THREADS)
depthwise_wgrad_finalize_kernel(const float *__restrict__ partials, int64_t chunks, int64_t elems, T *__restrict__ dweight) {
    const int64_t e = blockIdx.x * (int64_t)DW_THREADS + threadIdx.x;
    if (e >= elems) return;
    float s = 0.f;
    int64_t q = 0;
    for (; q + DW_FIN <= chunks; q += DW_FIN) {
        float p[DW_FIN];
#pragma unroll
        for (int u = 0; u < DW_FIN; ++u) p[u] = __ldg(partials + (q + u) * elems + e);
#pragma unroll
        for (int u = 0; u < DW_FIN; ++u) s += p[u];
    }
    for (; q < chunks; ++q) s += __ldg(partials + q * elems + e);
    dweight[e] = from_float<T>(s);
}

// ---------------------------------------------------------------- launchers
template <typename T, int V>
static int launch_gather(bool fwd, bool rev, const void *src, const void *weight, const void *bias, void *dst,
                         const int32_t *table, int64_t stride, int kv, int64_t rows, int channels, int act, float alpha,
                         cudaStream_t stream) {
    const int vecs = channels / V, tpr = row_tpr(vecs);
    const dim3 grid((unsigned)div_up64(rows, DW_THREADS / tpr), (unsigned)div_up64(vecs, tpr));
    if (fwd) {
        depthwise_fwd_kernel<T, V><<<grid, DW_THREADS, 0, stream>>>((const T *)src, (const T *)weight, (const T *)bias,
                                                                    (T *)dst, table, stride, kv, rows, channels, vecs, tpr,
                                                                    act, alpha);
        SPX_CHECK_LAUNCH("depthwise_fwd_kernel");
    } else if (rev) {
        depthwise_dgrad_kernel<T, V, true><<<grid, DW_THREADS, 0, stream>>>((const T *)src, (const T *)weight, (T *)dst,
                                                                            table, stride, kv, rows, channels, vecs, tpr);
        SPX_CHECK_LAUNCH("depthwise_dgrad_kernel");
    } else {
        depthwise_dgrad_kernel<T, V, false><<<grid, DW_THREADS, 0, stream>>>((const T *)src, (const T *)weight, (T *)dst,
                                                                             table, stride, kv, rows, channels, vecs, tpr);
        SPX_CHECK_LAUNCH("depthwise_dgrad_kernel");
    }
    return 0;
}

template <typename T>
static int dispatch_gather(bool vec, bool fwd, bool rev, const void *src, const void *weight, const void *bias, void *dst,
                           const int32_t *table, int64_t stride, int kv, int64_t rows, int channels, int act,
                           float alpha, cudaStream_t stream) {
    if (vec)
        return launch_gather<T, 16 / sizeof(T)>(fwd, rev, src, weight, bias, dst, table, stride, kv, rows, channels, act,
                                                alpha, stream);
    return launch_gather<T, 1>(fwd, rev, src, weight, bias, dst, table, stride, kv, rows, channels, act, alpha, stream);
}

static int64_t dw_chunks(int64_t rows) { return (rows + DW_CHUNK - 1) / DW_CHUNK; }

template <typename T, int V, bool A>
static int launch_wgrad(const void *x, const void *dy, void *dweight, const int32_t *table, int64_t stride, int kv,
                        int64_t rows, int channels, float *partials, cudaStream_t stream) {
    const int64_t chunks = dw_chunks(rows);
    if (chunks > 0) {
        const int vecs = channels / V, tpr = row_tpr(vecs);
        const dim3 grid((unsigned)chunks, (unsigned)div_up64(vecs, tpr), (unsigned)div_up64(kv, DwKw<V>::value));
        depthwise_wgrad_partial_kernel<T, V, A><<<grid, DW_THREADS, 0, stream>>>((const T *)x, (const T *)dy, table, stride,
                                                                              kv, rows, channels, vecs, tpr, partials);
        SPX_CHECK_LAUNCH("depthwise_wgrad_partial_kernel");
    }
    const int64_t elems = (int64_t)channels * kv;
    depthwise_wgrad_finalize_kernel<T><<<(unsigned)div_up64(elems, DW_THREADS), DW_THREADS, 0, stream>>>(
        partials, chunks, elems, (T *)dweight);
    SPX_CHECK_LAUNCH("depthwise_wgrad_finalize_kernel");
    return 0;
}

// The partial sums' order follows the vector width: a misaligned x or dy keeps the width of the aligned call and
// only loads element by element, so the weight gradient does not depend on where the operands start.
template <typename T>
static int dispatch_wgrad(RowWidth w, const void *x, const void *dy, void *dweight, const int32_t *table,
                          int64_t stride, int kv, int64_t rows, int channels, float *partials, cudaStream_t stream) {
    constexpr int W = 16 / sizeof(T);
    if (!w.wide) return launch_wgrad<T, 1, false>(x, dy, dweight, table, stride, kv, rows, channels, partials, stream);
    if (w.aligned) return launch_wgrad<T, W, true>(x, dy, dweight, table, stride, kv, rows, channels, partials, stream);
    return launch_wgrad<T, W, false>(x, dy, dweight, table, stride, kv, rows, channels, partials, stream);
}

}  // namespace spx

using namespace spx;

static int check_depthwise(const char *who, int64_t stride, int kv, int64_t rows, int channels, int dtype) {
    SPX_REQUIRE(kv >= 1 && kv <= 4096, "%s: kernel volume must be in [1, 4096], got %d", who, kv);
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(channels >= 1 && channels <= (1 << 20), "%s: bad channel count %d", who, channels);
    SPX_REQUIRE(dtype == SPX_F32 || dtype == SPX_F16 || dtype == SPX_BF16, "%s: unsupported dtype %d", who, dtype);
    SPX_REQUIRE(stride >= rows, "%s: table stride %lld is below the row count %lld", who, (long long)stride,
                (long long)rows);
    return 0;
}

extern "C" int spx_depthwise_fwd(const void *features, const void *weight, const void *bias, void *out,
                                 const int32_t *table, int64_t table_stride, int kv, int64_t n_out, int channels,
                                 int dtype, int act, float act_alpha, spx_stream_t stream_) {
    if (check_depthwise("depthwise_fwd", table_stride, kv, n_out, channels, dtype)) return 2;
    SPX_REQUIRE(act == SPX_ACT_NONE || act == SPX_ACT_RELU || act == SPX_ACT_SIGMOID || act == SPX_ACT_LEAKY_RELU,
                "depthwise_fwd: bad activation %d", act);
    if (n_out == 0) return 0;
    SPX_REQUIRE(weight && out && table, "depthwise_fwd: NULL pointer argument");
    const RowWidth w = row_width((int64_t)channels * dtype_bytes(dtype), features, out);
    cudaStream_t stream = (cudaStream_t)stream_;
    return dispatch_dtype(dtype, [&](auto t) {
        return dispatch_gather<typename decltype(t)::type>(w.wide && w.aligned, true, false, features, weight, bias, out,
                                                           table, table_stride, kv, n_out, channels, act, act_alpha,
                                                           stream);
    });
}

extern "C" int spx_depthwise_dgrad(const void *out_bp, const void *weight, void *din, const int32_t *table,
                                   int64_t table_stride, int kv, int64_t n_in, int channels, int dtype,
                                   int reverse_offsets, spx_stream_t stream_) {
    if (check_depthwise("depthwise_dgrad", table_stride, kv, n_in, channels, dtype)) return 2;
    if (n_in == 0) return 0;
    SPX_REQUIRE(weight && din && table, "depthwise_dgrad: NULL pointer argument");
    const RowWidth w = row_width((int64_t)channels * dtype_bytes(dtype), out_bp, din);
    const bool rev = reverse_offsets != 0;
    cudaStream_t stream = (cudaStream_t)stream_;
    return dispatch_dtype(dtype, [&](auto t) {
        return dispatch_gather<typename decltype(t)::type>(w.wide && w.aligned, false, rev, out_bp, weight, nullptr, din,
                                                           table, table_stride, kv, n_in, channels, SPX_ACT_NONE, 0.f,
                                                           stream);
    });
}

extern "C" size_t spx_depthwise_wgrad_workspace_size(int64_t n_out, int kv, int channels) {
    if (n_out <= 0 || kv <= 0 || channels <= 0) return 0;
    return align_up((size_t)dw_chunks(n_out) * (size_t)kv * (size_t)channels * sizeof(float), 256);
}

extern "C" int spx_depthwise_wgrad(const void *features, const void *out_bp, void *dweight, const int32_t *table,
                                   int64_t table_stride, int kv, int64_t n_out, int channels, int dtype,
                                   void *workspace, size_t workspace_bytes, spx_stream_t stream_) {
    if (check_depthwise("depthwise_wgrad", table_stride, kv, n_out, channels, dtype)) return 2;
    SPX_REQUIRE(dweight != nullptr, "depthwise_wgrad: dweight is NULL");
    SPX_REQUIRE(n_out == 0 || (out_bp && table), "depthwise_wgrad: NULL pointer argument");
    const size_t need = spx_depthwise_wgrad_workspace_size(n_out, kv, channels);
    SPX_REQUIRE(workspace_bytes >= need && (need == 0 || workspace != nullptr),
                "depthwise_wgrad: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    const RowWidth w = row_width((int64_t)channels * dtype_bytes(dtype), features, out_bp);
    float *partials = (float *)workspace;
    cudaStream_t stream = (cudaStream_t)stream_;
    return dispatch_dtype(dtype, [&](auto t) {
        return dispatch_wgrad<typename decltype(t)::type>(w, features, out_bp, dweight, table, table_stride, kv, n_out,
                                                          channels, partials, stream);
    });
}
