// Sum of sparse tensors whose coordinates differ (reference: spconv/pytorch/functional.py:441-544,
// sparse_add / sparse_add_hash_based).
//
// The union of the coordinates is not computed here.  It is the regular-conv rulebook of a 1x..x1,
// stride-1, padding-0 convolution over the operands' coordinates concatenated in visit order
// (spx_conv_rulebook_stage1/2): out_inds are the distinct in-range coordinates in first-touch order and
// pair_bwd[0] maps every visited row to its output row (-1 = out of range).  This file adds:
//   group  : a stable radix argsort of those output rows (dropped rows keyed M, i.e. last) and the segment
//            offsets, so the rows of output o are order[offsets[o] .. offsets[o+1]), ascending in visit order;
//            the first of them is the row that created o;
//   fwd    : output-stationary sum of every segment in fp32, in visit order, rounded once; each output
//            element is written by exactly one thread (no atomics, bit-reproducible);
//   gather : rows[g] = index[g] >= 0 ? src[index[g]] : 0 into per-operand row blocks -- the backward pass
//            (index = pair_bwd[0]) and the head-row gather of RemoveDuplicate.
// Feature rows are moved as 16-byte vectors when every row and base pointer allows it, else per element.
#include "common.cuh"

namespace spx {
size_t radix_argsort_workspace_bytes(int64_t n);
int radix_argsort_pair(uint32_t *mask0, int32_t *argsort0, int64_t n0, uint32_t *mask1, int32_t *argsort1, int64_t n1,
                       int key_bits, void *ws0, size_t ws0_bytes, void *ws1, size_t ws1_bytes, cudaStream_t stream);

constexpr int SA_THREADS = 256;
constexpr int SA_MAX = SPX_SPARSE_ADD_MAX_OPERANDS;

// the operand table as a kernel parameter: base pointers plus the first visited row of every operand
struct SaOperands {
    int count;
    const void *features[SA_MAX];
    void *grads[SA_MAX];
    int64_t start[SA_MAX + 1];
};

// operand that holds visited row g: the last t with start[t] <= g (empty operands are skipped that way)
__device__ __forceinline__ int operand_of(const SaOperands &ops, int64_t g) {
    int lo = 0, hi = ops.count - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (ops.start[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void sa_keys_kernel(const int32_t *__restrict__ dst, int64_t n, uint32_t m, uint32_t *__restrict__ keys) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t o = __ldg(dst + i);
    keys[i] = o < 0 ? m : (uint32_t)o;
}

// keys sorted ascending: offsets[o] = first position whose key is >= o, for o = 0..m
__global__ void sa_offsets_kernel(const uint32_t *__restrict__ keys, int64_t n, uint32_t m, int32_t *__restrict__ offsets) {
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int64_t k = keys[p];
    const int64_t prev = p == 0 ? -1 : (int64_t)keys[p - 1];
    for (int64_t o = prev + 1; o <= k; ++o) offsets[o] = (int32_t)p;
    if (p == n - 1)
        for (int64_t o = k + 1; o <= (int64_t)m; ++o) offsets[o] = (int32_t)n;
}

// W elements of T per thread: W * sizeof(T) == 16 (vector path) or W == 1
template <typename T, int W> __device__ __forceinline__ void load_row(const T *p, float (&f)[W]) {
    if constexpr (W * sizeof(T) == 16) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
        const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = to_float(e[j]);
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = to_float(p[j]);
    }
}
template <typename T, int W> __device__ __forceinline__ void store_row(T *p, const float (&f)[W]) {
    if constexpr (W * sizeof(T) == 16) {
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

// one thread = W channels of one output row; the rows of the segment are added in visit order
template <typename T, int W>
__global__ void __launch_bounds__(SA_THREADS)
sa_sum_kernel(const __grid_constant__ SaOperands ops, const int32_t *__restrict__ order, const int32_t *__restrict__ offsets,
              int64_t M, int chunks, int channels, T *__restrict__ out) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t o = idx / chunks;
    const int ch = (int)(idx - o * chunks);
    if (o >= M) return;
    float acc[W];
#pragma unroll
    for (int j = 0; j < W; ++j) acc[j] = 0.f;
    const int32_t end = __ldg(offsets + o + 1);
    for (int32_t p = __ldg(offsets + o); p < end; ++p) {
        const int64_t g = __ldg(order + p);
        const int t = operand_of(ops, g);
        float f[W];
        load_row<T, W>(static_cast<const T *>(ops.features[t]) + (g - ops.start[t]) * channels + ch * W, f);
#pragma unroll
        for (int j = 0; j < W; ++j) acc[j] += f[j];
    }
    store_row<T, W>(out + o * channels + ch * W, acc);
}

// rows are copied bit for bit: U is a 16-byte vector or an integer of the element's size
template <typename U>
__global__ void __launch_bounds__(SA_THREADS)
sa_gather_kernel(const __grid_constant__ SaOperands ops, const int32_t *__restrict__ index, int64_t rows, int chunks,
                 const U *__restrict__ src) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t g = idx / chunks;
    const int ch = (int)(idx - g * chunks);
    if (g >= rows) return;
    const int t = operand_of(ops, g);
    U *dst = static_cast<U *>(ops.grads[t]);
    if (dst == nullptr) return;
    const int32_t s = __ldg(index + g);
    U v{};
    if (s >= 0) v = __ldg(src + (int64_t)s * chunks + ch);
    dst[(g - ops.start[t]) * chunks + ch] = v;
}

static int make_operands(const spx_sparse_add_operands *in, bool fwd, int64_t &total, SaOperands &ops, const char *who) {
    SPX_REQUIRE(in != nullptr, "%s: operands is NULL", who);
    SPX_REQUIRE(in->count >= 1 && in->count <= SA_MAX, "%s: %d operands, must be in [1, %d]", who, in->count, SA_MAX);
    memset(&ops, 0, sizeof(ops));
    ops.count = in->count;
    total = 0;
    for (int t = 0; t < in->count; ++t) {
        SPX_REQUIRE(in->rows[t] >= 0, "%s: operand %d has a negative row count", who, t);
        SPX_REQUIRE(in->rows[t] == 0 || (fwd ? in->features[t] != nullptr : true),
                    "%s: features of operand %d are NULL", who, t);
        ops.features[t] = in->features[t];
        ops.grads[t] = in->grads[t];
        ops.start[t] = total;
        total += in->rows[t];
        SPX_REQUIRE(total < 2147483647ll, "%s: the operands hold %lld rows, at most 2^31 - 2 are supported", who,
                    (long long)total);
    }
    ops.start[in->count] = total;
    return 0;
}

static int check_features(int channels, int dtype, const char *who) {
    SPX_REQUIRE(channels >= 1, "%s: channels must be positive, got %d", who, channels);
    SPX_REQUIRE(dtype == SPX_F32 || dtype == SPX_F16 || dtype == SPX_BF16,
                "%s: unsupported dtype %d (float32, float16 and bfloat16 only)", who, dtype);
    return 0;
}

static bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }

template <typename T, int W>
static int launch_sum(const SaOperands &ops, const int32_t *order, const int32_t *offsets, int64_t M, int channels, void *out,
                      cudaStream_t stream) {
    const int chunks = channels / W;
    sa_sum_kernel<T, W><<<(unsigned)div_up64(M * chunks, SA_THREADS), SA_THREADS, 0, stream>>>(
        ops, order, offsets, M, chunks, channels, static_cast<T *>(out));
    SPX_CHECK_LAUNCH("sa_sum_kernel");
    return 0;
}

template <typename T>
static int dispatch_sum(const SaOperands &ops, const int32_t *order, const int32_t *offsets, int64_t M, int channels,
                        void *out, cudaStream_t stream) {
    constexpr int W = 16 / sizeof(T);
    bool vec = (channels * (int)sizeof(T)) % 16 == 0 && aligned16(out);
    for (int t = 0; t < ops.count; ++t) vec = vec && aligned16(ops.features[t]);
    if (vec) return launch_sum<T, W>(ops, order, offsets, M, channels, out, stream);
    return launch_sum<T, 1>(ops, order, offsets, M, channels, out, stream);
}

template <typename U>
static int launch_gather(const SaOperands &ops, const int32_t *index, int64_t rows, int64_t row_bytes, const void *src,
                         cudaStream_t stream) {
    const int chunks = (int)(row_bytes / (int64_t)sizeof(U));
    sa_gather_kernel<U><<<(unsigned)div_up64(rows * chunks, SA_THREADS), SA_THREADS, 0, stream>>>(
        ops, index, rows, chunks, static_cast<const U *>(src));
    SPX_CHECK_LAUNCH("sa_gather_kernel");
    return 0;
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_sparse_add_group_workspace_size(int64_t rows) {
    if (rows < 0) return 0;
    return align_up((size_t)rows * 4, 256) + radix_argsort_workspace_bytes(rows) + 1024;
}

extern "C" int spx_sparse_add_group(const int32_t *dst, int64_t rows, int64_t M, int32_t *order, int32_t *offsets,
                                    void *workspace, size_t workspace_bytes, spx_stream_t stream_) {
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "sparse_add_group: bad row count %lld", (long long)rows);
    SPX_REQUIRE(M >= 0 && M <= rows, "sparse_add_group: output count %lld not in [0, %lld]", (long long)M, (long long)rows);
    SPX_REQUIRE(offsets != nullptr, "sparse_add_group: offsets is NULL");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (rows == 0) {
        SPX_CHECK_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int32_t), stream));
        return 0;
    }
    SPX_REQUIRE(dst && order && workspace, "sparse_add_group: NULL pointer argument");
    SPX_REQUIRE(workspace_bytes >= spx_sparse_add_group_workspace_size(rows),
                "sparse_add_group: workspace too small: need %zu, have %zu", spx_sparse_add_group_workspace_size(rows),
                workspace_bytes);
    WorkspaceCarver ws(workspace, workspace_bytes);
    uint32_t *keys = ws.take<uint32_t>((size_t)rows);
    void *sort_ws = ws.take<char>(radix_argsort_workspace_bytes(rows));
    const unsigned blk = (unsigned)div_up64(rows, SA_THREADS);
    sa_keys_kernel<<<blk, SA_THREADS, 0, stream>>>(dst, rows, (uint32_t)M, keys);
    SPX_CHECK_LAUNCH("sa_keys_kernel");
    int key_bits = 1;                                  // enough bits for the keys 0..M
    while (key_bits < 32 && (M >> key_bits) != 0) ++key_bits;
    if (int rc = radix_argsort_pair(keys, order, rows, nullptr, nullptr, 0, key_bits, sort_ws,
                                    radix_argsort_workspace_bytes(rows), nullptr, 0, stream))
        return rc;
    sa_offsets_kernel<<<blk, SA_THREADS, 0, stream>>>(keys, rows, (uint32_t)M, offsets);
    SPX_CHECK_LAUNCH("sa_offsets_kernel");
    return 0;
}

extern "C" int spx_sparse_add_fwd(const spx_sparse_add_operands *operands, const int32_t *order, const int32_t *offsets,
                                  int64_t M, int channels, int dtype, void *out, spx_stream_t stream_) {
    SaOperands ops;
    int64_t total = 0;
    if (int rc = make_operands(operands, true, total, ops, "sparse_add_fwd")) return rc;
    if (int rc = check_features(channels, dtype, "sparse_add_fwd")) return rc;
    SPX_REQUIRE(M >= 0 && M <= total, "sparse_add_fwd: output count %lld not in [0, %lld]", (long long)M, (long long)total);
    if (M == 0) return 0;
    SPX_REQUIRE(order && offsets && out, "sparse_add_fwd: NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    switch (dtype) {
        case SPX_F32: return dispatch_sum<float>(ops, order, offsets, M, channels, out, stream);
        case SPX_F16: return dispatch_sum<__half>(ops, order, offsets, M, channels, out, stream);
        case SPX_BF16: return dispatch_sum<__nv_bfloat16>(ops, order, offsets, M, channels, out, stream);
    }
    return 2;
}

extern "C" int spx_sparse_add_gather(const int32_t *index, const void *src, int64_t src_rows,
                                     const spx_sparse_add_operands *operands, int channels, int dtype,
                                     spx_stream_t stream_) {
    SaOperands ops;
    int64_t total = 0;
    if (int rc = make_operands(operands, false, total, ops, "sparse_add_gather")) return rc;
    if (int rc = check_features(channels, dtype, "sparse_add_gather")) return rc;
    SPX_REQUIRE(src_rows >= 0, "sparse_add_gather: bad source row count");
    if (total == 0) return 0;
    bool any = false;
    for (int t = 0; t < ops.count; ++t) any = any || (operands->rows[t] > 0 && ops.grads[t] != nullptr);
    if (!any) return 0;
    SPX_REQUIRE(index != nullptr, "sparse_add_gather: index is NULL");
    SPX_REQUIRE(src != nullptr || src_rows == 0, "sparse_add_gather: src is NULL");
    cudaStream_t stream = (cudaStream_t)stream_;
    const int64_t row_bytes = (int64_t)channels * dtype_bytes(dtype);
    bool vec = row_bytes % 16 == 0 && aligned16(src);
    for (int t = 0; t < ops.count; ++t) vec = vec && aligned16(ops.grads[t]);
    if (vec) return launch_gather<uint4>(ops, index, total, row_bytes, src, stream);
    if (dtype_bytes(dtype) == 4) return launch_gather<uint32_t>(ops, index, total, row_bytes, src, stream);
    return launch_gather<uint16_t>(ops, index, total, row_bytes, src, stream);
}
