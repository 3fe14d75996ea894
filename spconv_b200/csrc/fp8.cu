// FP8 (e4m3) quantisation of feature rows (include/spconv_b200.h, spx_fp8_quantize).
//
// Dynamic mode is two launches: fp8_amax_kernel folds |x| of the valid rows into one partial maximum per block,
// and fp8_cast_kernel, in every block, folds those partials into the scale before it casts.  A maximum does not
// depend on the order it is taken in, so the scale is bit-reproducible without float atomics.  With a given scale
// only the cast runs.  The rows are cut into W-element vectors as in rows.cuh; W never changes a result.
#include "gemm.cuh"
#include "rows.cuh"

using namespace spx;

namespace {

constexpr int Q_THREADS = 256;
constexpr int Q_MAX_BLOCKS = 1024;      // partial maxima in the workspace
constexpr float E4M3_MAX = 448.f;

int quant_blocks(int64_t vecs) {
    const int64_t b = div_up64(vecs, (int64_t)Q_THREADS * 4);
    return (int)(b < 1 ? 1 : (b > Q_MAX_BLOCKS ? Q_MAX_BLOCKS : b));
}

// maximum of v over the block, returned to every thread
__device__ __forceinline__ float block_max(float v) {
    __shared__ float s_warp[Q_THREADS / 32];
    __shared__ float s_total;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = s_warp[0];
        for (int w = 1; w < Q_THREADS / 32; ++w) m = fmaxf(m, s_warp[w]);
        s_total = m;
    }
    __syncthreads();
    return s_total;
}

// partial[blockIdx.x] = max |x| over the finite elements of rows [0, M) this block visits (0 when none)
template <typename T, int W>
__global__ void __launch_bounds__(Q_THREADS) fp8_amax_kernel(const T *x, int64_t rows, int channels,
                                                             const int32_t *num_valid, float *partial) {
    const int64_t vecs = valid_rows(num_valid, rows) * channels / W;
    float m = 0.f;
    for (int64_t v = (int64_t)blockIdx.x * Q_THREADS + threadIdx.x; v < vecs; v += (int64_t)gridDim.x * Q_THREADS) {
        float f[W];
        row_load<T, W>(x + v * W, f);
#pragma unroll
        for (int j = 0; j < W; ++j)
            if (isfinite(f[j])) m = fmaxf(m, fabsf(f[j]));
    }
    m = block_max(m);
    if (threadIdx.x == 0) partial[blockIdx.x] = m;
}

template <int W> struct Bytes;
template <> struct Bytes<1> { using type = uint8_t; };
template <> struct Bytes<4> { using type = uint32_t; };
template <> struct Bytes<8> { using type = uint2; };

// y = satfinite_rne(x / scale) on rows [0, M), 0 on rows [M, rows).  scale: *scale_in, or amax / 448 of the
// nparts partial maxima (1 when the amax is 0); block 0 writes it to scale_out.
template <typename T, int W>
__global__ void __launch_bounds__(Q_THREADS) fp8_cast_kernel(const T *x, int64_t rows, int channels,
                                                             const int32_t *num_valid, const float *scale_in,
                                                             const float *partial, int nparts, uint8_t *y,
                                                             float *scale_out) {
    float scale;
    if (scale_in) {
        scale = __ldg(scale_in);
    } else {
        float m = 0.f;
        for (int i = threadIdx.x; i < nparts; i += Q_THREADS) m = fmaxf(m, partial[i]);
        m = block_max(m);
        scale = m > 0.f ? __fdiv_rn(m, E4M3_MAX) : 1.f;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && scale_out) *scale_out = scale;
    const int64_t valid = valid_rows(num_valid, rows) * channels / W;
    const int64_t vecs = rows * channels / W;
    for (int64_t v = (int64_t)blockIdx.x * Q_THREADS + threadIdx.x; v < vecs; v += (int64_t)gridDim.x * Q_THREADS) {
        union { typename Bytes<W>::type word; uint8_t b[W]; } q;
        if (v < valid) {
            float f[W];
            row_load<T, W>(x + v * W, f);
#pragma unroll
            for (int j = 0; j < W; ++j) q.b[j] = float_to_e4m3(__fdiv_rn(f[j], scale));
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j) q.b[j] = 0;
        }
        *reinterpret_cast<typename Bytes<W>::type *>(y + v * W) = q.word;
    }
}

template <typename T, int W>
int launch_quantize(const T *x, int64_t rows, int channels, const int32_t *num_valid, const float *scale_in,
                    uint8_t *y, float *scale_out, float *partial, cudaStream_t stream) {
    const int blocks = quant_blocks(rows * channels / W);
    if (!scale_in) {
        fp8_amax_kernel<T, W><<<blocks, Q_THREADS, 0, stream>>>(x, rows, channels, num_valid, partial);
        SPX_CHECK_LAUNCH("fp8_amax_kernel");
    }
    fp8_cast_kernel<T, W><<<blocks, Q_THREADS, 0, stream>>>(x, rows, channels, num_valid, scale_in, partial, blocks,
                                                            y, scale_out);
    SPX_CHECK_LAUNCH("fp8_cast_kernel");
    return 0;
}

}  // namespace

extern "C" size_t spx_fp8_quantize_workspace_size(int64_t rows, int channels) {
    (void)rows; (void)channels;
    return (size_t)Q_MAX_BLOCKS * sizeof(float);
}

extern "C" int spx_fp8_quantize(const spx_fp8_quant *q, void *workspace, size_t workspace_bytes,
                                spx_stream_t stream) {
    const char *who = "fp8_quantize";
    SPX_REQUIRE(q != nullptr, "%s: argument block is NULL", who);
    const void *x = q->x;
    void *out = q->out;
    const int dtype = q->dtype, channels = q->channels;
    const int64_t rows = q->rows;
    const int32_t *num_valid = q->num_valid;
    const float *scale_in = q->scale_in;
    float *scale_out = q->scale_out;
    SPX_REQUIRE(dtype == SPX_F32 || dtype == SPX_F16 || dtype == SPX_BF16, "%s: dtype %d not supported", who, dtype);
    SPX_REQUIRE(rows >= 0 && channels >= 1, "%s: bad shape [%lld, %d]", who, (long long)rows, channels);
    SPX_REQUIRE(rows * channels == 0 || (x && out), "%s: NULL tensor", who);
    SPX_REQUIRE(scale_in || scale_out, "%s: dynamic quantisation needs scale_out", who);
    SPX_REQUIRE(scale_in || (workspace && workspace_bytes >= spx_fp8_quantize_workspace_size(rows, channels)),
                "%s: workspace too small (%zu < %zu)", who, workspace_bytes,
                spx_fp8_quantize_workspace_size(rows, channels));
    cudaStream_t st = (cudaStream_t)stream;
    const RowWidth rw = row_width((int64_t)channels * dtype_bytes(dtype), x, out);
    return dispatch_dtype(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int VW = 16 / (int)sizeof(T);
        if (rw.wide && rw.aligned)
            return launch_quantize<T, VW>((const T *)x, rows, channels, num_valid, scale_in, (uint8_t *)out, scale_out,
                                          (float *)workspace, st);
        return launch_quantize<T, 1>((const T *)x, rows, channels, num_valid, scale_in, (uint8_t *)out, scale_out,
                                     (float *)workspace, st);
    });
}
