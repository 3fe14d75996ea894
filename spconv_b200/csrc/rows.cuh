// Shared pieces of the row-wise kernels over a feature matrix [rows, C]: BatchNorm, GroupNorm, the global pools,
// depthwise convolution, sparse_add and the point scatter.
//
// A row of C elements of T is cut into vectors of W elements.  A launcher picks W once per call (row_width):
//   element-wise kernels : W = 16 / sizeof(T) when the row is wide and every operand is 16-byte aligned, else
//                          W = 1.  W does not change what they compute.
//   reductions           : W = 16 / sizeof(T) whenever the row is wide; a misaligned operand keeps that W and only
//                          moves element by element (A = false).  W decides which rows and channels each thread
//                          folds, and so the order of the sums: the results must not depend on where the operands
//                          start.
// A block of a row kernel holds `tpr` threads per row (row_tpr) and `lanes` = threads / tpr rows in flight;
// blockIdx.y selects a slice of tpr vectors.
#pragma once
#include "common.cuh"
#include "segments.cuh"

namespace spx {

// ---------------------------------------------------------------- host: dispatch and block layout
template <typename T> struct Type { using type = T; };

// f(Type<T>{}) with the element type of dtype: float32, float16 or (any other value) bfloat16.  The caller has
// checked dtype.
template <typename F> static inline int dispatch_dtype(int dtype, F &&f) {
    switch (dtype) {
        case SPX_F32: return f(Type<float>{});
        case SPX_F16: return f(Type<__half>{});
        default: return f(Type<__nv_bfloat16>{});
    }
}

struct RowWidth {
    bool wide;       // the row splits into 16-byte vectors
    bool aligned;    // every given operand starts on a 16-byte boundary (NULL passes)
};
template <typename... P> static inline RowWidth row_width(int64_t row_bytes, const P *...operands) {
    return {row_bytes % 16 == 0, (true && ... && aligned16(operands))};
}

// threads per row: a power of two >= the row's vectors, at most 32
static inline int row_tpr(int vecs) {
    int tpr = 1;
    while (tpr < vecs && tpr < 32) tpr <<= 1;
    return tpr;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------- device: row access
// W elements at p, converted to float.  A: one 16-byte access when W * sizeof(T) == 16; otherwise W element
// accesses.  Both give the same values.
template <typename T, int W, bool A = true> __device__ __forceinline__ void row_load(const T *p, float (&f)[W]) {
    if constexpr (A && W * sizeof(T) == 16) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
        const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = to_float(e[j]);
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = to_float(__ldg(p + j));
    }
}
template <typename T, int W, bool A = true> __device__ __forceinline__ void row_store(T *p, const float (&f)[W]) {
    if constexpr (A && W * sizeof(T) == 16) {
        uint4 v;
        T *e = reinterpret_cast<T *>(&v);
#pragma unroll
        for (int j = 0; j < W; ++j) e[j] = from_float<T>(f[j]);
        *reinterpret_cast<uint4 *>(p) = v;
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) p[j] = from_float<T>(f[j]);
    }
}

// the same, bit for bit, for the kernels that copy elements: one 16-byte vector (W * sizeof(T) == 16) or W == 1
template <typename T, int W> __device__ __forceinline__ void row_load_raw(const T *p, T (&e)[W]) {
    if constexpr (W * sizeof(T) == 16) {
        *reinterpret_cast<uint4 *>(e) = __ldg(reinterpret_cast<const uint4 *>(p));
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) e[j] = __ldg(p + j);
    }
}
template <typename T, int W> __device__ __forceinline__ void row_store_raw(T *p, const T (&e)[W]) {
    if constexpr (W * sizeof(T) == 16) {
        *reinterpret_cast<uint4 *>(p) = *reinterpret_cast<const uint4 *>(e);
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) p[j] = e[j];
    }
}

// ---------------------------------------------------------------- device: block layout and valid rows
struct RowThread {
    int lane;        // row lane of the thread
    int v;           // vector of the row
    bool active;     // v < vecs
};
__device__ __forceinline__ RowThread row_thread(int vecs, int tpr) {
    RowThread t;
    t.lane = threadIdx.x / tpr;
    t.v = blockIdx.y * tpr + (threadIdx.x % tpr);
    t.active = t.v < vecs;
    return t;
}

// M = *num_valid clamped to [0, rows]; NULL: every row
__device__ __forceinline__ int64_t valid_rows(const int32_t *num_valid, int64_t rows) {
    if (num_valid == nullptr) return rows;
    const int64_t m = __ldg(num_valid);
    return m < 0 ? 0 : (m > rows ? rows : m);
}

// ---- per-sample chunks (global_pool.cu's group_samples): the rows of sample b are the sorted positions
// [offsets[b], offsets[b+1]), cut into chunks of GP_CHUNK numbered from cstart[b]; cstart[B] chunks in all
constexpr int GP_CHUNK = 512;        // rows per partial

// The chunk of block blockIdx.x: its sample and sorted positions [p0, end).  False past the last chunk.
__device__ __forceinline__ bool sample_chunk(const int32_t *offsets, const int32_t *cstart, int batch_size, int &b,
                                             int32_t &p0, int32_t &end) {
    const int32_t k = (int32_t)blockIdx.x;
    if (k >= __ldg(cstart + batch_size)) return false;
    b = last_at_most(cstart, batch_size, k);          // empty samples own no chunk
    p0 = __ldg(offsets + b) + (k - __ldg(cstart + b)) * GP_CHUNK;
    const int32_t seg_end = __ldg(offsets + b + 1);
    end = seg_end < p0 + GP_CHUNK ? seg_end : p0 + GP_CHUNK;
    return true;
}

// ---------------------------------------------------------------- device: merges and lane trees
// The max rule of the global pool and the point scatter: does (v, r) beat (bv, br)?  r < 0 marks an empty side.
// A NaN beats every number, then the greater value, then, on equality (-0 == +0), the lower row: a total order
// whose winner is the first row in ascending order that attains the maximum (np.argmax).
__device__ __forceinline__ bool max_beats(float v, int r, float bv, int br) {
    if (r < 0) return false;
    if (br < 0) return true;
    const bool n = isnan(v), bn = isnan(bv);
    if (n != bn) return n;
    if (!n && v != bv) return v > bv;
    return r < br;
}

// Chan et al.: fold (nb, mb, qb) into (na, ma, qa).  An empty side changes nothing, bit for bit.
__device__ __forceinline__ void chan_merge(float &na, float &ma, float &qa, float nb, float mb, float qb) {
    if (nb == 0.f) return;
    if (na == 0.f) { na = nb; ma = mb; qa = qb; return; }
    const float n = na + nb, d = mb - ma, f = __fdiv_rn(nb, n);
    ma = fmaf(d, f, ma);
    qa = qa + qb + d * d * na * f;
    na = n;
}

// Fixed tree over the row lanes of a block (lane = threadIdx.x / tpr, as in row_thread): at step s, lanes [0, s) fold
// lanes [s, 2s) into their own slots, so lane 0 ends with the block's total.  Shared memory: s_mean, s_q
// [threads * W], s_n [threads].
// Welford (count n, mean[], M2 q[]) merged by Chan's rule:
template <int W>
__device__ __forceinline__ void welford_lane_tree(float *s_mean, float *s_q, float *s_n, int lanes, int tpr, float &n,
                                                  float (&mean)[W], float (&q)[W]) {
    const int slot = threadIdx.x, lane = threadIdx.x / tpr;
#pragma unroll
    for (int j = 0; j < W; ++j) { s_mean[slot * W + j] = mean[j]; s_q[slot * W + j] = q[j]; }
    s_n[slot] = n;
    for (int s = lanes >> 1; s >= 1; s >>= 1) {
        __syncthreads();
        if (lane < s) {
            const int o = slot + s * tpr;
            const float nb = s_n[o];
#pragma unroll
            for (int j = 0; j < W; ++j) {
                float na = n;
                chan_merge(na, mean[j], q[j], nb, s_mean[o * W + j], s_q[o * W + j]);
                s_mean[slot * W + j] = mean[j];
                s_q[slot * W + j] = q[j];
            }
            s_n[slot] = n = n + nb;
        }
    }
}

// ... and two sums a[], b[] (shared memory s_a, s_b [threads * W]):
template <int W>
__device__ __forceinline__ void pair_sum_lane_tree(float *s_a, float *s_b, int lanes, int tpr, float (&a)[W],
                                                   float (&b)[W]) {
    const int slot = threadIdx.x, lane = threadIdx.x / tpr;
#pragma unroll
    for (int j = 0; j < W; ++j) { s_a[slot * W + j] = a[j]; s_b[slot * W + j] = b[j]; }
    for (int s = lanes >> 1; s >= 1; s >>= 1) {
        __syncthreads();
        if (lane < s) {
            const int o = slot + s * tpr;
#pragma unroll
            for (int j = 0; j < W; ++j) {
                s_a[slot * W + j] = a[j] = a[j] + s_a[o * W + j];
                s_b[slot * W + j] = b[j] = b[j] + s_b[o * W + j];
            }
        }
    }
}
#endif  // __CUDACC__

}  // namespace spx
