// Sum of sparse tensors whose coordinates differ (reference: spconv/pytorch/functional.py:441-544,
// sparse_add / sparse_add_hash_based).
//
// The union of the coordinates is not computed here.  It is the regular-conv rulebook of a 1x..x1,
// stride-1, padding-0 convolution over the operands' coordinates concatenated in visit order
// (spx_conv_rulebook_stage1/2): out_inds are the distinct in-range coordinates in first-touch order and
// pair_bwd[0] maps every visited row to its output row (-1 = out of range).  This file adds:
//   group  : group_rows, the grouping of segments.cuh keyed by those output rows (dropped rows keyed M, i.e.
//            last), so the rows of output o are order[offsets[o] .. offsets[o+1]), ascending in visit order;
//            the first of them is the row that created o;
//   fwd    : output-stationary sum of every segment in fp32, in visit order, rounded once; each output
//            element is written by exactly one thread (no atomics, bit-reproducible);
//   gather : rows[g] = index[g] >= 0 ? src[index[g]] : 0 into per-operand row blocks -- the backward pass
//            (index = pair_bwd[0]) and the head-row gather of RemoveDuplicate.
// Feature rows are moved as 16-byte vectors when every row and base pointer allows it, else per element.
#include "rows.cuh"
#include "segments.cuh"

namespace spx {
int validate_sparse_add_union(const spx_conv_geometry *g, int64_t N, int64_t bound);

constexpr int SA_THREADS = 256;
constexpr int SA_MAX = SPX_SPARSE_ADD_MAX_OPERANDS;

// the operand table as a kernel parameter: base pointers plus the first visited row of every operand
struct SaOperands {
    int count;
    const void *features[SA_MAX];
    void *grads[SA_MAX];
    int64_t start[SA_MAX + 1];
};

// operand that holds visited row g: the last t with start[t] <= g (empty operands are skipped that way).  Not
// last_at_most: ops lives in the kernel parameters, which __ldg cannot read.
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
        row_load<T, W>(static_cast<const T *>(ops.features[t]) + (g - ops.start[t]) * channels + ch * W, f);
#pragma unroll
        for (int j = 0; j < W; ++j) acc[j] += f[j];
    }
    row_store<T, W>(out + o * channels + ch * W, acc);
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
    RowWidth w = row_width(channels * sizeof(T), out);
    for (int t = 0; t < ops.count; ++t) w.aligned = w.aligned && aligned16(ops.features[t]);
    if (w.wide && w.aligned) return launch_sum<T, W>(ops, order, offsets, M, channels, out, stream);
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

// ------------------------------------------------------------------ padded operands (masked_sparse_add)
// Operand t's valid rows are [0, valid_t), valid_t = *num_valid[t] clamped to [0, rows_t] (NULL: every row).
// The visit order is the one sparse_add takes for the unpadded operands: the largest valid count first (ties:
// the earliest operand), then the others in argument order.  The counts live on the device, so every block of
// the pack kernel decides the order itself from the <= 64 counts (no extra launch, no read-back).
struct SaPlan {
    int count;
    const int32_t *num_valid[SA_MAX];
    int64_t start[SA_MAX + 1];                 // argument order
};

// row g of the argument-order concatenation -> position pos(g) of the packed array: the valid rows of the
// operands in visit order (exactly the concatenation sparse_add ranks), then every padding row in argument
// order with coordinates -1 (dropped by the union).  packed[pos] = coordinates, src[pos] = g.
__global__ void __launch_bounds__(SA_THREADS)
sa_pack_kernel(const __grid_constant__ SaPlan plan, const int32_t *__restrict__ indices, int ncols,
               int32_t *__restrict__ packed, int32_t *__restrict__ src) {
    __shared__ int64_t valid[SA_MAX], vstart[SA_MAX], pstart[SA_MAX];
    const int t = threadIdx.x;
    if (t < plan.count) {
        const int64_t rows = plan.start[t + 1] - plan.start[t];
        int64_t v = rows;
        if (plan.num_valid[t] != nullptr) {
            v = *plan.num_valid[t];
            v = v < 0 ? 0 : (v > rows ? rows : v);
        }
        valid[t] = v;
    }
    __syncthreads();
    if (t == 0) {
        int largest = 0;
        for (int i = 1; i < plan.count; ++i)
            if (valid[i] > valid[largest]) largest = i;
        int64_t v = valid[largest];
        vstart[largest] = 0;
        for (int i = 0; i < plan.count; ++i)
            if (i != largest) { vstart[i] = v; v += valid[i]; }
        for (int i = 0; i < plan.count; ++i) {                 // the tail starts at V = sum of the valid counts
            pstart[i] = v;
            v += plan.start[i + 1] - plan.start[i] - valid[i];
        }
    }
    __syncthreads();
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + t;
    if (g >= plan.start[plan.count]) return;
    int lo = 0, hi = plan.count - 1;                           // the last operand with start <= g (operand_of)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (plan.start[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    const int64_t r = g - plan.start[lo];
    const bool ok = r < valid[lo];
    const int64_t pos = ok ? vstart[lo] + r : pstart[lo] + (r - valid[lo]);
    for (int a = 0; a < ncols; ++a) packed[pos * ncols + a] = ok ? __ldg(indices + g * ncols + a) : -1;
    src[pos] = (int32_t)g;
}

// back to argument order: order_arg[p] = src[order[p]] (the segments keep their ascending visit order),
// dst_arg[src[p]] = dst[p]
__global__ void sa_remap_kernel(const int32_t *__restrict__ src, const int32_t *__restrict__ order,
                                const int32_t *__restrict__ dst, int64_t n, int32_t *__restrict__ order_arg,
                                int32_t *__restrict__ dst_arg) {
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    order_arg[p] = __ldg(src + __ldg(order + p));
    dst_arg[__ldg(src + p)] = __ldg(dst + p);
}

// heads[o] = the row that created output o (o < M), else -1; inverse[heads[o]] = o.  inverse is -1 beforehand.
__global__ void sa_heads_kernel(const int32_t *__restrict__ order, const int32_t *__restrict__ offsets,
                                const int32_t *__restrict__ num_out, int64_t bound, int32_t *__restrict__ heads,
                                int32_t *__restrict__ inverse) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= bound) return;
    const int32_t h = o < (int64_t)*num_out ? __ldg(order + __ldg(offsets + o)) : -1;
    heads[o] = h;
    if (h >= 0) inverse[h] = (int32_t)o;
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_sparse_add_group_workspace_size(int64_t rows) {
    if (rows < 0) return 0;
    return align_up((size_t)rows * 4, 256) + radix_argsort_workspace_bytes(rows) + 1024;
}

namespace spx {
// The grouping of spx_sparse_add_group and spx_point_scatter_group: order [rows] and offsets [M + 1] of dst [rows].
// M may exceed rows here; with rows == 0 all M + 1 offsets are 0.  0 <= rows < 2^31 - 1, 0 <= M < 2^31 - 1.
int group_rows(const int32_t *dst, int64_t rows, int64_t M, int32_t *order, int32_t *offsets, void *workspace,
               size_t workspace_bytes, cudaStream_t stream, const char *who) {
    SPX_REQUIRE(offsets != nullptr, "%s: offsets is NULL", who);
    if (rows == 0) {
        SPX_CHECK_CUDA(cudaMemsetAsync(offsets, 0, (size_t)(M + 1) * sizeof(int32_t), stream));
        return 0;
    }
    SPX_REQUIRE(dst && order && workspace, "%s: NULL pointer argument", who);
    SPX_REQUIRE(workspace_bytes >= spx_sparse_add_group_workspace_size(rows),
                "%s: workspace too small: need %zu, have %zu", who, spx_sparse_add_group_workspace_size(rows),
                workspace_bytes);
    WorkspaceCarver ws(workspace, workspace_bytes);
    uint32_t *keys = ws.take<uint32_t>((size_t)rows);
    void *sort_ws = ws.take<char>(radix_argsort_workspace_bytes(rows));
    const unsigned blk = (unsigned)div_up64(rows, SA_THREADS);
    sa_keys_kernel<<<blk, SA_THREADS, 0, stream>>>(dst, rows, (uint32_t)M, keys);
    SPX_CHECK_LAUNCH("sa_keys_kernel");
    if (int rc = sort_by_key(keys, rows, M, order, sort_ws, radix_argsort_workspace_bytes(rows), stream)) return rc;
    return segment_offsets(keys, rows, M, offsets, stream);
}

static int sum_dtype(const SaOperands &ops, const int32_t *order, const int32_t *offsets, int64_t M, int channels,
                     int dtype, void *out, cudaStream_t stream) {
    return dispatch_dtype(dtype, [&](auto t) {
        return dispatch_sum<typename decltype(t)::type>(ops, order, offsets, M, channels, out, stream);
    });
}

// The sum of spx_point_scatter_fwd: one operand x [rows, channels] and M segments, M may exceed rows.  The caller
// has checked every argument.
int sum_segments(const void *x, int64_t rows, const int32_t *order, const int32_t *offsets, int64_t M, int channels,
                 int dtype, void *out, cudaStream_t stream) {
    SaOperands ops;
    memset(&ops, 0, sizeof(ops));
    ops.count = 1;
    ops.features[0] = x;
    ops.start[1] = rows;
    return sum_dtype(ops, order, offsets, M, channels, dtype, out, stream);
}
}  // namespace spx

extern "C" int spx_sparse_add_group(const int32_t *dst, int64_t rows, int64_t M, int32_t *order, int32_t *offsets,
                                    void *workspace, size_t workspace_bytes, spx_stream_t stream_) {
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "sparse_add_group: bad row count %lld", (long long)rows);
    SPX_REQUIRE(M >= 0 && M <= rows, "sparse_add_group: output count %lld not in [0, %lld]", (long long)M, (long long)rows);
    return group_rows(dst, rows, M, order, offsets, workspace, workspace_bytes, (cudaStream_t)stream_,
                      "sparse_add_group");
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
    return sum_dtype(ops, order, offsets, M, channels, dtype, out, (cudaStream_t)stream_);
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
    RowWidth w = row_width(row_bytes, src);
    for (int t = 0; t < ops.count; ++t) w.aligned = w.aligned && aligned16(ops.grads[t]);
    if (w.wide && w.aligned) return launch_gather<uint4>(ops, index, total, row_bytes, src, stream);
    if (dtype_bytes(dtype) == 4) return launch_gather<uint32_t>(ops, index, total, row_bytes, src, stream);
    return launch_gather<uint16_t>(ops, index, total, row_bytes, src, stream);
}

// ------------------------------------------------------------------ padded operands (masked_sparse_add)
namespace {
struct PlanWs {
    int32_t *packed, *src, *dst, *order;
    void *union_ws, *group_ws;
    size_t union_bytes, group_bytes, bytes;
};

void carve_plan_ws(const spx_conv_geometry *g, int64_t rows, int64_t bound, void *workspace, size_t bytes, PlanWs &w) {
    WorkspaceCarver ws(workspace, bytes);
    w.packed = ws.take<int32_t>((size_t)rows * (g->ndim + 1));
    w.src = ws.take<int32_t>((size_t)rows);
    w.dst = ws.take<int32_t>((size_t)rows);
    w.order = ws.take<int32_t>((size_t)rows);
    w.union_bytes = spx_sparse_add_union_workspace_size(g, rows, bound);
    w.union_ws = ws.take<char>(w.union_bytes);
    w.group_bytes = spx_sparse_add_group_workspace_size(rows);
    w.group_ws = ws.take<char>(w.group_bytes);
    w.bytes = ws.off;
}
}  // namespace

extern "C" size_t spx_masked_sparse_add_workspace_size(const spx_conv_geometry *g, int64_t rows, int64_t bound) {
    if (!g || g->ndim < 1 || g->ndim > SPX_MAX_NDIM || rows < 0 || bound < 0 || bound > rows) return 0;
    if (rows == 0) return 256;
    if (spx_sparse_add_union_workspace_size(g, rows, bound) == 0) return 0;
    PlanWs w;
    carve_plan_ws(g, rows, bound, nullptr, SIZE_MAX, w);
    return align_up(w.bytes, 256) + 256;
}

extern "C" int spx_masked_sparse_add_plan(const spx_conv_geometry *g, const spx_sparse_add_operands *operands,
                                          const int32_t *const *num_valid, const int32_t *indices, int64_t bound,
                                          int32_t *out_inds, int32_t *dst, int32_t *order, int32_t *offsets,
                                          int32_t *num_out, int32_t *status, void *workspace, size_t workspace_bytes,
                                          spx_stream_t stream_) {
    SaOperands ops;
    int64_t rows = 0;
    if (int rc = make_operands(operands, false, rows, ops, "masked_sparse_add_plan")) return rc;
    SPX_REQUIRE(g != nullptr && g->ndim >= 1 && g->ndim <= SPX_MAX_NDIM, "masked_sparse_add_plan: bad geometry");
    SPX_REQUIRE(bound >= (rows > 0 ? 1 : 0) && bound <= rows && bound < (1ll << 30),
                "masked_sparse_add_plan: bound must be in [1, rows] and below 2^30, got %lld for %lld rows",
                (long long)bound, (long long)rows);
    SPX_REQUIRE(offsets && num_out && status, "masked_sparse_add_plan: NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (rows == 0) {                       // nothing to visit: M = 0, offsets [1] = {0}
        SPX_CHECK_CUDA(cudaMemsetAsync(num_out, 0, sizeof(int32_t), stream));
        SPX_CHECK_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int32_t), stream));
        return 0;
    }
    if (validate_sparse_add_union(g, rows, bound)) return 2;
    SPX_REQUIRE(indices && out_inds && dst && order && workspace, "masked_sparse_add_plan: NULL pointer argument");
    const size_t need = spx_masked_sparse_add_workspace_size(g, rows, bound);
    SPX_REQUIRE(workspace_bytes >= need, "masked_sparse_add_plan: workspace too small: need %zu, have %zu", need,
                workspace_bytes);
    PlanWs w;
    carve_plan_ws(g, rows, bound, workspace, workspace_bytes, w);
    SaPlan plan;
    memset(&plan, 0, sizeof(plan));
    plan.count = ops.count;
    for (int t = 0; t < ops.count; ++t) plan.num_valid[t] = num_valid ? num_valid[t] : nullptr;
    memcpy(plan.start, ops.start, sizeof(plan.start));
    const unsigned blk = (unsigned)div_up64(rows, SA_THREADS);
    const int ncols = g->ndim + 1;
    sa_pack_kernel<<<blk, SA_THREADS, 0, stream>>>(plan, indices, ncols, w.packed, w.src);
    SPX_CHECK_LAUNCH("sa_pack_kernel");
    if (int rc = spx_sparse_add_union(g, w.packed, rows, bound, out_inds, w.dst, num_out, status, w.union_ws,
                                      w.union_bytes, stream_)) return rc;
    if (int rc = spx_sparse_add_group(w.dst, rows, bound, w.order, offsets, w.group_ws, w.group_bytes, stream_)) return rc;
    sa_remap_kernel<<<blk, SA_THREADS, 0, stream>>>(w.src, w.order, w.dst, rows, order, dst);
    SPX_CHECK_LAUNCH("sa_remap_kernel");
    return 0;
}

extern "C" int spx_masked_sparse_add_heads(const int32_t *order, const int32_t *offsets, const int32_t *num_out,
                                           int64_t bound, int64_t rows, int32_t *heads, int32_t *inverse,
                                           spx_stream_t stream_) {
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "masked_sparse_add_heads: bad row count %lld", (long long)rows);
    SPX_REQUIRE(bound >= 0 && bound <= rows, "masked_sparse_add_heads: bound %lld not in [0, %lld]", (long long)bound,
                (long long)rows);
    if (rows == 0) return 0;
    SPX_REQUIRE(order && offsets && num_out && inverse && (heads || bound == 0),
                "masked_sparse_add_heads: NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    SPX_CHECK_CUDA(cudaMemsetAsync(inverse, 0xff, (size_t)rows * sizeof(int32_t), stream));
    if (bound == 0) return 0;
    sa_heads_kernel<<<(unsigned)div_up64(bound, SA_THREADS), SA_THREADS, 0, stream>>>(order, offsets, num_out, bound,
                                                                                       heads, inverse);
    SPX_CHECK_LAUNCH("sa_heads_kernel");
    return 0;
}
