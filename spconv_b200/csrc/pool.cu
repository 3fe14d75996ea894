// Sparse max / average pooling on the rulebook tables (SURVEY 8 f1).
//
// Replaces IndiceMaxPool (spconv/csrc/sparse/maxpool.py:41-341, host drivers :343-588):
//   forward_implicit_gemm_kernel / backward_implicit_gemm_kernel          (max, dense pair tables)
//   forward_avgpool_implicit_gemm_kernel / backward_avgpool_...           (mean + neighbour count)
//   forward_kernel / backward_kernel                                      (ConvAlgo.Native, compact pairs)
// Pure HBM-bound gather work: one thread owns one 16-byte channel chunk of one output row and walks
// the kv table entries of that row; the row indices are warp-broadcast loads, the feature rows are
// read and written as 16-byte vectors, so the entry points refuse a feature pointer that is not
// 16-byte aligned.  The Native variants run on the same kernels after the compact pairs have been
// scattered into a dense table (spx_pairs_to_table) -- no atomics on features, results independent
// of the pair order.
#include "common.cuh"

namespace spx {

template <typename T> struct Vec16 { static constexpr int N = 16 / sizeof(T); };

template <typename T> __device__ __forceinline__ void load_vec(const T *p, float (&f)[16 / sizeof(T)]) {
    const uint4 v = *reinterpret_cast<const uint4 *>(p);
    const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
    for (int j = 0; j < (int)(16 / sizeof(T)); ++j) f[j] = to_float(e[j]);
}
template <typename T> __device__ __forceinline__ T cast_out(float v) { return from_float<T>(v); }
template <> __device__ __forceinline__ int8_t cast_out<int8_t>(float v) { return (int8_t)(int)v; }

template <typename T> __device__ __forceinline__ void store_vec(T *p, const float (&f)[16 / sizeof(T)]) {
    uint4 v;
    T *e = reinterpret_cast<T *>(&v);
#pragma unroll
    for (int j = 0; j < (int)(16 / sizeof(T)); ++j) e[j] = cast_out<T>(f[j]);
    *reinterpret_cast<uint4 *>(p) = v;
}

template <typename T> __device__ __forceinline__ float lowest_of();
template <> __device__ __forceinline__ float lowest_of<float>() { return -3.402823466e+38f; }
template <> __device__ __forceinline__ float lowest_of<__half>() { return -65504.f; }
template <> __device__ __forceinline__ float lowest_of<__nv_bfloat16>() { return -3.3895313892515355e+38f; }
template <> __device__ __forceinline__ float lowest_of<int8_t>() { return -128.f; }

// Max: a candidate replaces the running max only when it is greater, as in the reference -- NaN never
// wins, and of two equal values (-0 and +0) the first stays.
// MODE 0: max, accumulator starts at lowest()   (maxpool.py:76-117)
// MODE 1: max, accumulator starts at 0          (Native: the output buffer is zero-initialised and
//                                                only raised, spconv/pytorch/ops.py:1910 + maxpool.py:63-66)
// MODE 2: mean over the valid entries, count written to count_out   (maxpool.py:211-259)
template <typename T, int MODE>
__global__ void pool_fwd_kernel(const T *__restrict__ x, T *__restrict__ out, const int32_t *__restrict__ table,
                                int64_t stride, int kv, int64_t rows, int chunks, int channels,
                                int32_t *__restrict__ count_out) {
    constexpr int N = Vec16<T>::N;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t o = idx / chunks;
    const int ch = (int)(idx - o * chunks);
    if (o >= rows) return;
    float acc[N];
#pragma unroll
    for (int j = 0; j < N; ++j) acc[j] = MODE == 0 ? lowest_of<T>() : 0.f;
    int count = 0;
    for (int k = 0; k < kv; ++k) {
        const int32_t i = __ldg(table + (int64_t)k * stride + o);
        if (i < 0) continue;
        ++count;
        float f[N];
        load_vec(x + (int64_t)i * channels + ch * N, f);
#pragma unroll
        for (int j = 0; j < N; ++j) acc[j] = MODE == 2 ? acc[j] + f[j] : (f[j] > acc[j] ? f[j] : acc[j]);
    }
    if (MODE == 2) {
        // a division, as the reference (maxpool.py:255): acc * (1 / count) differs from it in the last
        // bit for about a third of the sums at count 3
#pragma unroll
        for (int j = 0; j < N; ++j) acc[j] = count > 0 ? acc[j] / (float)count : 0.f;
        if (count_out && ch == 0) count_out[o] = count;
    }
    store_vec(out + o * channels + ch * N, acc);
}

// max: din[i] = sum over the outputs o that i feeds of (x[i] == y[o]) ? dy[o] : 0   (maxpool.py:159-208)
// avg: din[i] = sum_o dy[o] * count[o]   -- the reference multiplies by the count (maxpool.py:262-300);
//      reproduced as is so that gradients match the reference bit for bit in fp32
template <typename T, bool AVG>
__global__ void pool_bwd_kernel(const T *__restrict__ x, const T *__restrict__ y, const T *__restrict__ dy,
                                T *__restrict__ din, const int32_t *__restrict__ table_bwd, int64_t stride, int kv,
                                int64_t rows, int chunks, int channels, const int32_t *__restrict__ count) {
    constexpr int N = Vec16<T>::N;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t i = idx / chunks;
    const int ch = (int)(idx - i * chunks);
    if (i >= rows) return;
    float xin[N], acc[N];
#pragma unroll
    for (int j = 0; j < N; ++j) { acc[j] = 0.f; xin[j] = 0.f; }
    if (!AVG) load_vec(x + i * channels + ch * N, xin);
    for (int k = 0; k < kv; ++k) {
        const int32_t o = __ldg(table_bwd + (int64_t)k * stride + i);
        if (o < 0) continue;
        float g[N];
        load_vec(dy + (int64_t)o * channels + ch * N, g);
        if (AVG) {
            const float c = (float)__ldg(count + o);
#pragma unroll
            for (int j = 0; j < N; ++j) acc[j] += g[j] * c;
        } else {
            float yo[N];
            load_vec(y + (int64_t)o * channels + ch * N, yo);
#pragma unroll
            for (int j = 0; j < N; ++j) acc[j] += xin[j] == yo[j] ? g[j] : 0.f;
        }
    }
    store_vec(din + i * channels + ch * N, acc);
}

// rows of each sample, in input order: out[b * N + count[b]++] = i  (maxpool.py:303-341 uses an
// atomic append; here ranks come from a stable block scan so the order is deterministic = CPU order,
// maxpool.py:599-620)
__global__ void global_pool_count_kernel(const int32_t *__restrict__ coords, int64_t n, int row_ints, int batch,
                                         int32_t *__restrict__ counts) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = coords[i * row_ints];
    if (b >= 0 && b < batch) atomicAdd(&counts[b], 1);
}
__global__ void global_pool_rank_kernel(const int32_t *__restrict__ coords, int64_t n, int row_ints, int batch,
                                        int32_t *__restrict__ out) {
    // one block per sample: ordered compaction of the rows whose batch index is blockIdx.x
    __shared__ int warp_tot[32];
    __shared__ int carry;
    const int b = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += blockDim.x) {
        const int64_t i = base + threadIdx.x;
        const bool mine = i < n && coords[i * row_ints] == b;
        const unsigned ball = __ballot_sync(0xffffffffu, mine);
        if (lane == 0) warp_tot[warp] = __popc(ball);
        __syncthreads();
        int before = carry;
        for (int w2 = 0; w2 < warp; ++w2) before += warp_tot[w2];
        if (mine) out[(int64_t)b * n + before + __popc(ball & ((1u << lane) - 1u))] = (int32_t)i;
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int w2 = 0; w2 < nwarp; ++w2) t += warp_tot[w2]; carry += t; }
        __syncthreads();
    }
}

template <typename T>
static int launch_fwd(int mode, const void *x, void *out, const int32_t *table, int64_t stride, int kv, int64_t rows,
                      int channels, int32_t *count_out, cudaStream_t stream) {
    const int chunks = channels / Vec16<T>::N;
    const int64_t total = rows * chunks;
    const unsigned nblk = (unsigned)div_up64(total, 256);
    if (mode == 0)
        pool_fwd_kernel<T, 0><<<nblk, 256, 0, stream>>>((const T *)x, (T *)out, table, stride, kv, rows, chunks, channels, nullptr);
    else if (mode == 1)
        pool_fwd_kernel<T, 1><<<nblk, 256, 0, stream>>>((const T *)x, (T *)out, table, stride, kv, rows, chunks, channels, nullptr);
    else
        pool_fwd_kernel<T, 2><<<nblk, 256, 0, stream>>>((const T *)x, (T *)out, table, stride, kv, rows, chunks, channels, count_out);
    SPX_CHECK_LAUNCH("pool_fwd_kernel");
    return 0;
}

template <typename T>
static int launch_bwd(bool avg, const void *x, const void *y, const void *dy, void *din, const int32_t *table,
                      int64_t stride, int kv, int64_t rows, int channels, const int32_t *count, cudaStream_t stream) {
    const int chunks = channels / Vec16<T>::N;
    const unsigned nblk = (unsigned)div_up64(rows * chunks, 256);
    if (avg)
        pool_bwd_kernel<T, true><<<nblk, 256, 0, stream>>>((const T *)x, (const T *)y, (const T *)dy, (T *)din, table, stride, kv, rows, chunks, channels, count);
    else
        pool_bwd_kernel<T, false><<<nblk, 256, 0, stream>>>((const T *)x, (const T *)y, (const T *)dy, (T *)din, table, stride, kv, rows, chunks, channels, count);
    SPX_CHECK_LAUNCH("pool_bwd_kernel");
    return 0;
}

}  // namespace spx

using namespace spx;

static int check_pool(const char *who, int kv, int channels, int dtype, int64_t rows, bool allow_i8) {
    SPX_REQUIRE(kv >= 1 && kv <= 4096, "%s: bad kernel volume %d", who, kv);
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "%s: bad row count", who);
    const int e = dtype_bytes(dtype);
    SPX_REQUIRE(e != 0 && (allow_i8 || dtype != SPX_I8), "%s: unsupported dtype %d", who, dtype);
    SPX_REQUIRE(channels > 0 && (channels * e) % 16 == 0,
                "%s: channels * element size must be a multiple of 16 bytes (got %d x %d)", who, channels, e);
    return 0;
}

extern "C" int spx_indice_pool_fwd(int mode, const void *features, void *out, const int32_t *pair_fwd,
                                   int64_t pair_stride, int kv, int64_t n_out, int channels, int dtype,
                                   int32_t *count_out, spx_stream_t stream_) {
    SPX_REQUIRE(mode >= 0 && mode <= 2, "indice_pool_fwd: mode must be 0 (max), 1 (max, zero floor) or 2 (mean)");
    if (check_pool("indice_pool_fwd", kv, channels, dtype, n_out, mode != 2)) return 2;
    if (n_out == 0) return 0;
    SPX_REQUIRE(features && out && pair_fwd, "indice_pool_fwd: NULL pointer argument");
    SPX_REQUIRE_ALIGNED16(features, "indice_pool_fwd");
    SPX_REQUIRE_ALIGNED16(out, "indice_pool_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    switch (dtype) {
        case SPX_F32: return launch_fwd<float>(mode, features, out, pair_fwd, pair_stride, kv, n_out, channels, count_out, stream);
        case SPX_F16: return launch_fwd<__half>(mode, features, out, pair_fwd, pair_stride, kv, n_out, channels, count_out, stream);
        case SPX_BF16: return launch_fwd<__nv_bfloat16>(mode, features, out, pair_fwd, pair_stride, kv, n_out, channels, count_out, stream);
        case SPX_I8: return launch_fwd<int8_t>(mode, features, out, pair_fwd, pair_stride, kv, n_out, channels, count_out, stream);
    }
    return 2;
}

extern "C" int spx_indice_pool_bwd(int mode, const void *features, const void *out_features, const void *out_bp,
                                   void *din, const int32_t *pair_bwd, int64_t pair_stride, int kv, int64_t n_in,
                                   int channels, int dtype, const int32_t *count_out, spx_stream_t stream_) {
    SPX_REQUIRE(mode >= 0 && mode <= 2, "indice_pool_bwd: bad mode %d", mode);
    if (check_pool("indice_pool_bwd", kv, channels, dtype, n_in, false)) return 2;
    if (n_in == 0) return 0;
    const bool avg = mode == 2;
    SPX_REQUIRE(out_bp && din && pair_bwd, "indice_pool_bwd: NULL pointer argument");
    SPX_REQUIRE(avg ? count_out != nullptr : (features && out_features), "indice_pool_bwd: missing %s",
                avg ? "count_out" : "features / out_features");
    SPX_REQUIRE_ALIGNED16(features, "indice_pool_bwd");
    SPX_REQUIRE_ALIGNED16(out_features, "indice_pool_bwd");
    SPX_REQUIRE_ALIGNED16(out_bp, "indice_pool_bwd");
    SPX_REQUIRE_ALIGNED16(din, "indice_pool_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    switch (dtype) {
        case SPX_F32: return launch_bwd<float>(avg, features, out_features, out_bp, din, pair_bwd, pair_stride, kv, n_in, channels, count_out, stream);
        case SPX_F16: return launch_bwd<__half>(avg, features, out_features, out_bp, din, pair_bwd, pair_stride, kv, n_in, channels, count_out, stream);
        case SPX_BF16: return launch_bwd<__nv_bfloat16>(avg, features, out_features, out_bp, din, pair_bwd, pair_stride, kv, n_in, channels, count_out, stream);
    }
    return 2;
}

extern "C" int spx_global_pool_rearrange(const int32_t *coords, int64_t n, int row_ints, int batch_size,
                                         int32_t *out_indices, int32_t *counts, spx_stream_t stream_) {
    SPX_REQUIRE(batch_size > 0 && row_ints >= 1 && n >= 0, "global_pool_rearrange: bad arguments");
    SPX_REQUIRE(out_indices && counts, "global_pool_rearrange: NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    SPX_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * batch_size, stream));
    if (n == 0) return 0;
    SPX_REQUIRE(coords != nullptr, "global_pool_rearrange: coords is NULL");
    global_pool_count_kernel<<<(unsigned)div_up64(n, 256), 256, 0, stream>>>(coords, n, row_ints, batch_size, counts);
    SPX_CHECK_LAUNCH("global_pool_count_kernel");
    global_pool_rank_kernel<<<batch_size, 256, 0, stream>>>(coords, n, row_ints, batch_size, out_indices);
    SPX_CHECK_LAUNCH("global_pool_rank_kernel");
    return 0;
}
