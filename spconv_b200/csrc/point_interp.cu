// Voxel -> point interpolation (VoxelPointInterpolator, pytorch/utils.py): the devoxelisation of point-voxel
// networks (SPVCNN's voxel_to_point), trilinear or nearest, from a sparse tensor at any stride, with no host
// read-back.  pos [P, ndim] are fp32 positions in the tensor's index space (voxel v's feature sits at v).
//
//   plan    : clear the table, insert the usable rows (r < num_valid, batch and coordinates in range; the lowest
//             row wins a duplicated coordinate, insert_min), then one thread per point computes its K = 2^ndim
//             corners (1 for nearest) and their weights and finds them with the K probes in flight
//             (find_many): index [P, K] (-1 = no such row) and weight [P, K] fp32.  Then group_rows
//             (segments.cuh) over the P * K entries keyed by index (-1 keyed `rows`, i.e. last): the entries of
//             row r are order[offsets[r] .. offsets[r+1]) in ascending entry e = p * K + j;
//   forward : one thread per (point, 16-byte vector) loads its K corner rows together and adds w_j * x[idx_j] in
//             ascending j in fp32 (no FMA), rounded once;
//   backward: one thread per (row, vector) walks the row's entries in ascending e and adds w_e * dy[e / K] in fp32,
//             rounded once; every element of dx is written once (0 for a row without entries).
// Every sum has an order fixed by the coordinates and the points alone, and no float atomics are used, so results
// are bit-reproducible and independent of padding rows and dropped points.
#include "hash.cuh"
#include "rows.cuh"
#include "segments.cuh"

namespace spx {

constexpr int PI_THREADS = 256;
constexpr int PI_INFLIGHT = 4;                   // backward: entries loaded per step of a row's walk
constexpr int64_t PI_MAX = 2147483647ll;         // rows, P and P * K below 2^31 - 1

struct PiGeom {
    int ndim, batch;
    int dims[SPX_MAX_NDIM];
};

template <typename Table>
__global__ void pi_insert_kernel(Table table, PiGeom g, const int32_t *__restrict__ indices, int64_t rows,
                                 const int32_t *__restrict__ num_valid) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= rows || i >= valid_rows(num_valid, rows)) return;
    const int32_t *row = indices + i * (g.ndim + 1);
    int c[SPX_MAX_NDIM + 1];
    c[0] = __ldg(row);
    bool ok = c[0] >= 0 && c[0] < g.batch;
#pragma unroll
    for (int a = 0; a < SPX_MAX_NDIM; ++a) {
        if (a < g.ndim) {
            c[a + 1] = __ldg(row + a + 1);
            ok = ok && c[a + 1] >= 0 && c[a + 1] < g.dims[a];
        }
    }
    if (ok) table.insert_min(linear_key(c, g.dims, g.ndim), (int32_t)i);
}

// One thread per point.  The range check runs on the float, before any conversion: NaN fails both comparisons,
// +-inf and huge values fail one, so only a point with a possible corner reaches floorf's int conversion.  The
// upper bound is compared in double, exact for every int shape.
template <typename Table, int NDIM, bool NEAREST>
__global__ void __launch_bounds__(PI_THREADS)
pi_probe_kernel(Table table, PiGeom g, const float *__restrict__ pos, const int32_t *__restrict__ batch_ids, int64_t n,
                int normalize, int32_t *__restrict__ index, float *__restrict__ weight) {
    constexpr int K = NEAREST ? 1 : 1 << NDIM;
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int b = __ldg(batch_ids + p);
    bool keep = b >= 0 && b < g.batch;
    int base[NDIM];
    float f[NDIM];
#pragma unroll
    for (int a = 0; a < NDIM; ++a) {
        const float q = __ldg(pos + p * NDIM + a);
        keep = keep && q >= -1.f && (double)q < (double)g.dims[a];
        const float fl = floorf(q);
        base[a] = keep ? (int)fl : 0;
        f[a] = keep ? __fsub_rn(q, fl) : 0.f;           // exact: q and floor(q) share their leading bits
    }
    int64_t key[K];
    bool live[K];
    float w[K];
#pragma unroll
    for (int j = 0; j < K; ++j) {
        int c[SPX_MAX_NDIM + 1] = {b, 0, 0, 0, 0};
        bool ok = keep;
        float wj = 1.f;
#pragma unroll
        for (int a = 0; a < NDIM; ++a) {
            const int bit = NEAREST ? (f[a] >= 0.5f ? 1 : 0) : (j >> a) & 1;
            c[a + 1] = base[a] + bit;
            ok = ok && c[a + 1] >= 0 && c[a + 1] < g.dims[a];
            if constexpr (!NEAREST) {
                const float fa = bit ? f[a] : __fsub_rn(1.f, f[a]);
                wj = a == 0 ? fa : __fmul_rn(wj, fa);
            }
        }
        live[j] = ok;
        key[j] = ok ? linear_key(c, g.dims, NDIM) : 0;
        w[j] = wj;
    }
    int32_t v[K];
    find_many<K>(table, key, live, v);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (v[j] >= 0) s = __fadd_rn(s, w[j]);
    const float d = __fadd_rn(s, 1e-8f);
#pragma unroll
    for (int j = 0; j < K; ++j) {
        index[p * K + j] = v[j];
        weight[p * K + j] = v[j] < 0 ? 0.f : (normalize ? __fdiv_rn(w[j], d) : w[j]);
    }
}

template <typename T, int W, int K>
__global__ void __launch_bounds__(PI_THREADS)
pi_fwd_kernel(const T *__restrict__ x, const int32_t *__restrict__ index, const float *__restrict__ weight, int64_t n,
              int chunks, int channels, T *__restrict__ y) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t p = idx / chunks;
    const int ch = (int)(idx - p * chunks);
    if (p >= n) return;
    int32_t r[K];
    float w[K];
#pragma unroll
    for (int j = 0; j < K; ++j) {
        r[j] = __ldg(index + p * K + j);
        w[j] = __ldg(weight + p * K + j);
    }
    float e[K][W];                                       // the K rows loaded together, then folded in order
#pragma unroll
    for (int j = 0; j < K; ++j) {
        if (r[j] >= 0) row_load<T, W>(x + (int64_t)r[j] * channels + ch * W, e[j]);
    }
    float acc[W];
#pragma unroll
    for (int c = 0; c < W; ++c) acc[c] = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        if (r[j] >= 0) {
#pragma unroll
            for (int c = 0; c < W; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(w[j], e[j][c]));
        }
    }
    row_store<T, W>(y + p * channels + ch * W, acc);
}

template <typename T, int W>
__global__ void __launch_bounds__(PI_THREADS)
pi_bwd_kernel(const T *__restrict__ dy, const float *__restrict__ weight, const int32_t *__restrict__ order,
              const int32_t *__restrict__ offsets, int64_t rows, int kshift, int chunks, int channels,
              T *__restrict__ dx) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = idx / chunks;
    const int ch = (int)(idx - r * chunks);
    if (r >= rows) return;
    const int32_t end = __ldg(offsets + r + 1);
    float acc[W];
#pragma unroll
    for (int c = 0; c < W; ++c) acc[c] = 0.f;
    const T *base = dy + ch * W;
    int32_t q = __ldg(offsets + r);
    for (; q + PI_INFLIGHT <= end; q += PI_INFLIGHT) {
        int32_t e[PI_INFLIGHT];
        float w[PI_INFLIGHT], g[PI_INFLIGHT][W];
#pragma unroll
        for (int u = 0; u < PI_INFLIGHT; ++u) e[u] = __ldg(order + q + u);
#pragma unroll
        for (int u = 0; u < PI_INFLIGHT; ++u) {
            w[u] = __ldg(weight + e[u]);
            row_load<T, W>(base + (int64_t)(e[u] >> kshift) * channels, g[u]);
        }
#pragma unroll
        for (int u = 0; u < PI_INFLIGHT; ++u)
#pragma unroll
            for (int c = 0; c < W; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(w[u], g[u][c]));
    }
    for (; q < end; ++q) {
        const int32_t e = __ldg(order + q);
        const float w = __ldg(weight + e);
        float g[W];
        row_load<T, W>(base + (int64_t)(e >> kshift) * channels, g);
#pragma unroll
        for (int c = 0; c < W; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(w, g[c]));
    }
    row_store<T, W>(dx + r * channels + ch * W, acc);
}

// ---------------------------------------------------------------- host side

static int pi_corners(int ndim, int mode) { return mode == 1 ? 1 : 1 << ndim; }

static int pi_kshift(int corners) {
    int s = 0;
    while ((1 << s) < corners) ++s;
    return s;
}

// 64-bit keys once batch * volume reaches 2^31 - 1, the rule of the SubM rulebook
static bool pi_i64(const PiGeom &g) {
    double v = (double)g.batch;
    for (int a = 0; a < g.ndim; ++a) v *= (double)g.dims[a];
    return v >= 2147483647.0;
}

struct PiLayout {
    uint32_t capacity;
    bool i64;
    void *tbl;
    int32_t *tvals;
    void *group_ws;
    size_t group_bytes, bytes;
};

static void pi_carve(const PiGeom &g, int64_t rows, int64_t entries, void *workspace, size_t bytes, PiLayout &L) {
    L.i64 = pi_i64(g);
    L.capacity = table_capacity(rows);
    WorkspaceCarver ws(workspace, bytes);
    L.tbl = ws.take<unsigned long long>(L.capacity);
    L.tvals = L.i64 ? ws.take<int32_t>(L.capacity) : nullptr;
    L.group_bytes = spx_sparse_add_group_workspace_size(entries);
    L.group_ws = ws.take<char>(L.group_bytes);
    L.bytes = ws.off;
}

static int pi_geom(const char *who, int ndim, const int *shape_host, int batch_size, PiGeom &g) {
    SPX_REQUIRE(ndim >= 1 && ndim <= SPX_MAX_NDIM, "%s: ndim must be in [1, %d], got %d", who, SPX_MAX_NDIM, ndim);
    SPX_REQUIRE(shape_host != nullptr, "%s: NULL pointer argument (spatial_shape)", who);
    SPX_REQUIRE(batch_size >= 1, "%s: batch_size must be positive, got %d", who, batch_size);
    memset(&g, 0, sizeof(g));
    g.ndim = ndim;
    g.batch = batch_size;
    for (int a = 0; a < ndim; ++a) {
        SPX_REQUIRE(shape_host[a] >= 1, "%s: spatial_shape[%d] must be positive, got %d", who, a, shape_host[a]);
        g.dims[a] = shape_host[a];
    }
    return 0;
}

static int pi_sizes(const char *who, int mode, int ndim, int64_t rows, int64_t n) {
    SPX_REQUIRE(mode == 0 || mode == 1, "%s: mode must be 0 (trilinear) or 1 (nearest), got %d", who, mode);
    SPX_REQUIRE(rows >= 0 && rows < PI_MAX, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(n >= 0 && n < PI_MAX, "%s: bad point count %lld", who, (long long)n);
    SPX_REQUIRE(n * pi_corners(ndim, mode) < PI_MAX, "%s: %lld points of %d corners are too many", who, (long long)n,
                pi_corners(ndim, mode));
    return 0;
}

static int pi_features(const char *who, int64_t rows, int64_t n, int corners, int channels, int dtype) {
    SPX_REQUIRE(corners == 1 || corners == 2 || corners == 4 || corners == 8 || corners == 16,
                "%s: corners must be 1, 2, 4, 8 or 16, got %d", who, corners);
    SPX_REQUIRE(rows >= 0 && rows < PI_MAX, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(n >= 0 && n * corners < PI_MAX, "%s: bad point count %lld", who, (long long)n);
    SPX_REQUIRE(channels >= 1, "%s: channels must be positive, got %d", who, channels);
    SPX_REQUIRE(dtype == SPX_F32 || dtype == SPX_F16 || dtype == SPX_BF16,
                "%s: unsupported dtype %d (float32, float16 and bfloat16 only)", who, dtype);
    const int64_t most = n > rows ? n : rows;
    SPX_REQUIRE(div_up64(most * channels, PI_THREADS) <= PI_MAX, "%s: %lld rows of %d channels are too many", who,
                (long long)most, channels);
    return 0;
}

template <typename Table, int NDIM>
static int pi_probe_launch(const Table &t, const PiGeom &g, const float *pos, const int32_t *batch_ids, int64_t n,
                           int mode, int normalize, int32_t *index, float *weight, cudaStream_t stream) {
    const unsigned blk = (unsigned)div_up64(n, PI_THREADS);
    if (mode == 1) pi_probe_kernel<Table, NDIM, true><<<blk, PI_THREADS, 0, stream>>>(t, g, pos, batch_ids, n, normalize,
                                                                                       index, weight);
    else pi_probe_kernel<Table, NDIM, false><<<blk, PI_THREADS, 0, stream>>>(t, g, pos, batch_ids, n, normalize, index,
                                                                              weight);
    SPX_CHECK_LAUNCH("pi_probe_kernel");
    return 0;
}

template <typename T, int W, int K>
static int pi_fwd_launch(const void *x, const int32_t *index, const float *weight, int64_t n, int channels, void *y,
                         cudaStream_t stream) {
    const int chunks = channels / W;
    pi_fwd_kernel<T, W, K><<<(unsigned)div_up64(n * chunks, PI_THREADS), PI_THREADS, 0, stream>>>(
        static_cast<const T *>(x), index, weight, n, chunks, channels, static_cast<T *>(y));
    SPX_CHECK_LAUNCH("pi_fwd_kernel");
    return 0;
}

template <typename T, int W>
static int pi_fwd_corners(int corners, const void *x, const int32_t *index, const float *weight, int64_t n,
                          int channels, void *y, cudaStream_t stream) {
    switch (corners) {
        case 1: return pi_fwd_launch<T, W, 1>(x, index, weight, n, channels, y, stream);
        case 2: return pi_fwd_launch<T, W, 2>(x, index, weight, n, channels, y, stream);
        case 4: return pi_fwd_launch<T, W, 4>(x, index, weight, n, channels, y, stream);
        case 8: return pi_fwd_launch<T, W, 8>(x, index, weight, n, channels, y, stream);
        default: return pi_fwd_launch<T, W, 16>(x, index, weight, n, channels, y, stream);
    }
}

template <typename T, int W>
static int pi_bwd_launch(const void *dy, const float *weight, const int32_t *order, const int32_t *offsets,
                         int64_t rows, int corners, int channels, void *dx, cudaStream_t stream) {
    const int chunks = channels / W;
    pi_bwd_kernel<T, W><<<(unsigned)div_up64(rows * chunks, PI_THREADS), PI_THREADS, 0, stream>>>(
        static_cast<const T *>(dy), weight, order, offsets, rows, pi_kshift(corners), chunks, channels,
        static_cast<T *>(dx));
    SPX_CHECK_LAUNCH("pi_bwd_kernel");
    return 0;
}

}  // namespace spx

using namespace spx;

static size_t pi_plan_workspace_size(int ndim, const int *spatial_shape_host, int batch_size, int64_t rows,
                                     int64_t num_points, int mode) {
    if (ndim < 1 || ndim > SPX_MAX_NDIM || !spatial_shape_host || batch_size < 1 || rows < 0 || rows >= PI_MAX ||
        num_points < 0 || (mode != 0 && mode != 1))
        return 0;
    const int64_t entries = num_points * pi_corners(ndim, mode);
    if (entries >= PI_MAX) return 0;
    PiGeom g;
    memset(&g, 0, sizeof(g));
    g.ndim = ndim;
    g.batch = batch_size;
    for (int a = 0; a < ndim; ++a) g.dims[a] = spatial_shape_host[a] > 0 ? spatial_shape_host[a] : 1;
    PiLayout L;
    pi_carve(g, rows, entries, nullptr, SIZE_MAX, L);
    return align_up(L.bytes, 256) + 256;
}

static int pi_plan(int ndim, const int *spatial_shape_host, int batch_size, const int32_t *indices, int64_t rows,
                   const int32_t *num_valid, const float *pos, const int32_t *batch_ids, int64_t num_points, int mode,
                   int normalize, int32_t *index, float *weight, int32_t *order, int32_t *offsets, void *workspace,
                   size_t workspace_bytes, cudaStream_t stream) {
    const char *who = "point_interp_plan";
    PiGeom g;
    if (int rc = pi_geom(who, ndim, spatial_shape_host, batch_size, g)) return rc;
    if (int rc = pi_sizes(who, mode, ndim, rows, num_points)) return rc;
    SPX_REQUIRE(normalize == 0 || normalize == 1, "%s: normalize must be 0 or 1, got %d", who, normalize);
    SPX_REQUIRE(offsets && workspace, "%s: NULL pointer argument (offsets, workspace)", who);
    SPX_REQUIRE(rows == 0 || indices, "%s: NULL pointer argument (indices)", who);
    SPX_REQUIRE(num_points == 0 || (pos && batch_ids && index && weight && order),
                "%s: NULL pointer argument (pos, batch_ids, index, weight, order)", who);
    const size_t need = pi_plan_workspace_size(ndim, spatial_shape_host, batch_size, rows, num_points, mode);
    SPX_REQUIRE(workspace_bytes >= need, "%s: workspace too small: need %zu, have %zu", who, need, workspace_bytes);
    const int64_t entries = num_points * pi_corners(ndim, mode);
    PiLayout L;
    pi_carve(g, rows, entries, workspace, workspace_bytes, L);
    if (num_points > 0) {
        SPX_CHECK_CUDA(cudaMemsetAsync(L.tbl, 0xFF, (size_t)L.capacity * 8, stream));
        if (L.i64) SPX_CHECK_CUDA(cudaMemsetAsync(L.tvals, 0x7F, (size_t)L.capacity * 4, stream));
        if (int rc = visit_table(L.i64, L.tbl, L.tvals, L.capacity, [&](auto t) {
                if (rows > 0) {
                    pi_insert_kernel<<<(unsigned)div_up64(rows, PI_THREADS), PI_THREADS, 0, stream>>>(t, g, indices,
                                                                                                      rows, num_valid);
                    SPX_CHECK_LAUNCH("pi_insert_kernel");
                }
                using Table = decltype(t);
                switch (ndim) {
                    case 1: return pi_probe_launch<Table, 1>(t, g, pos, batch_ids, num_points, mode, normalize, index,
                                                             weight, stream);
                    case 2: return pi_probe_launch<Table, 2>(t, g, pos, batch_ids, num_points, mode, normalize, index,
                                                             weight, stream);
                    case 3: return pi_probe_launch<Table, 3>(t, g, pos, batch_ids, num_points, mode, normalize, index,
                                                             weight, stream);
                    default: return pi_probe_launch<Table, 4>(t, g, pos, batch_ids, num_points, mode, normalize,
                                                              index, weight, stream);
                }
            })) return rc;
    }
    return group_rows(index, entries, rows, order, offsets, L.group_ws, L.group_bytes, stream, who);
}

static int pi_fwd(const void *x, int64_t rows, int channels, int dtype, const int32_t *index, const float *weight,
                  int64_t num_points, int corners, void *y, cudaStream_t stream) {
    const char *who = "point_interp_fwd";
    if (int rc = pi_features(who, rows, num_points, corners, channels, dtype)) return rc;
    SPX_REQUIRE(num_points == 0 || (index && weight && y), "%s: NULL pointer argument (index, weight, y)", who);
    SPX_REQUIRE(rows == 0 || x, "%s: NULL pointer argument (x)", who);
    if (num_points == 0) return 0;
    return dispatch_dtype(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int W = 16 / sizeof(T);
        const RowWidth w = row_width(channels * sizeof(T), x, y);
        if (w.wide && w.aligned) return pi_fwd_corners<T, W>(corners, x, index, weight, num_points, channels, y, stream);
        return pi_fwd_corners<T, 1>(corners, x, index, weight, num_points, channels, y, stream);
    });
}

static int pi_bwd(const void *dy, int64_t num_points, int corners, int channels, int dtype, const float *weight,
                  const int32_t *order, const int32_t *offsets, int64_t rows, void *dx, cudaStream_t stream) {
    const char *who = "point_interp_bwd";
    if (int rc = pi_features(who, rows, num_points, corners, channels, dtype)) return rc;
    SPX_REQUIRE(rows == 0 || (offsets && dx), "%s: NULL pointer argument (offsets, dx)", who);
    SPX_REQUIRE(num_points == 0 || (dy && weight && order), "%s: NULL pointer argument (dy, weight, order)", who);
    if (rows == 0) return 0;
    return dispatch_dtype(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int W = 16 / sizeof(T);
        const RowWidth w = row_width(channels * sizeof(T), dy, dx);
        if (w.wide && w.aligned)
            return pi_bwd_launch<T, W>(dy, weight, order, offsets, rows, corners, channels, dx, stream);
        return pi_bwd_launch<T, 1>(dy, weight, order, offsets, rows, corners, channels, dx, stream);
    });
}

extern "C" size_t spx_point_interp_plan_workspace_size(const spx_point_interp *a) {
    if (a == nullptr) return 0;
    return pi_plan_workspace_size(a->ndim, a->spatial_shape, a->batch_size, a->rows, a->num_points, a->mode);
}

extern "C" int spx_point_interp_plan(const spx_point_interp *a, void *workspace, size_t workspace_bytes,
                                     spx_stream_t stream) {
    SPX_REQUIRE(a != nullptr, "point_interp_plan: the argument block is NULL");
    return pi_plan(a->ndim, a->spatial_shape, a->batch_size, a->indices, a->rows, a->num_valid, a->pos, a->batch_ids,
                   a->num_points, a->mode, a->normalize, a->index, a->weight, a->order, a->offsets, workspace,
                   workspace_bytes, (cudaStream_t)stream);
}

extern "C" int spx_point_interp_fwd(const spx_point_interp *a, spx_stream_t stream) {
    SPX_REQUIRE(a != nullptr, "point_interp_fwd: the argument block is NULL");
    SPX_REQUIRE(a->ndim >= 1 && a->ndim <= SPX_MAX_NDIM, "point_interp_fwd: ndim must be in [1, %d], got %d",
                SPX_MAX_NDIM, a->ndim);
    SPX_REQUIRE(a->mode == 0 || a->mode == 1, "point_interp_fwd: mode must be 0 (trilinear) or 1 (nearest), got %d",
                a->mode);
    return pi_fwd(a->x, a->rows, a->channels, a->dtype, a->index, a->weight, a->num_points, pi_corners(a->ndim, a->mode),
                  a->y, (cudaStream_t)stream);
}

extern "C" int spx_point_interp_bwd(const spx_point_interp *a, spx_stream_t stream) {
    SPX_REQUIRE(a != nullptr, "point_interp_bwd: the argument block is NULL");
    SPX_REQUIRE(a->ndim >= 1 && a->ndim <= SPX_MAX_NDIM, "point_interp_bwd: ndim must be in [1, %d], got %d",
                SPX_MAX_NDIM, a->ndim);
    SPX_REQUIRE(a->mode == 0 || a->mode == 1, "point_interp_bwd: mode must be 0 (trilinear) or 1 (nearest), got %d",
                a->mode);
    return pi_bwd(a->dy, a->num_points, pi_corners(a->ndim, a->mode), a->channels, a->dtype, a->weight, a->order,
                  a->offsets, a->rows, a->dx, (cudaStream_t)stream);
}
