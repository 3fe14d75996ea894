// Rulebook (indice-pair) generation for SubM and regular/transposed sparse convolution.
//
// Replaces the reference's hash + atomic-append kernels (spconv/csrc/sparse/indices.py:292-939)
// and their host drivers (spconv/csrc/sparse/all.py:1660-2218).  Design differences, on purpose:
//   * one packed 64-bit slot {key:32 | value:32} per hash entry so a probe is ONE 8-byte load
//     (the reference probes split key/value arrays: "performance bound", indices.py:791);
//   * the dense tables pair_fwd / pair_bwd are written exactly once, coalesced, -1 included
//     (no torch.full(-1) pre-pass + scattered writes);
//   * every ordering decision is deterministic and equal to the reference *CPU* rulebook
//     (indices.py:1640-1778): outputs of a regular conv are ranked by first touch in
//     offset-major order (atomicMin of k*N+i, then a radix sort of the minima), compact
//     "Native" pairs come from a stable per-offset scan instead of atomicAggInc.
#include "common.cuh"
#include "gemm.cuh"
#include "hash.cuh"
#include "rank.cuh"
#include "rows.cuh"
#include "segments.cuh"
#include <cub/cub.cuh>

namespace spx {
int validate_sparse_add_union(const spx_conv_geometry *g, int64_t N, int64_t bound);
}

namespace spx {

// ------------------------------------------------------------------ geometry
struct Geom {
    int ndim, batch, kv;
    int in_dims[SPX_MAX_NDIM], out_dims[SPX_MAX_NDIM], ksize[SPX_MAX_NDIM];
    int stride[SPX_MAX_NDIM], padding[SPX_MAX_NDIM], dilation[SPX_MAX_NDIM];
    int transposed;
};

static Geom make_geom(const spx_conv_geometry *g, bool subm) {
    Geom r;
    memset(&r, 0, sizeof(r));
    r.ndim = g->ndim;
    r.batch = g->batch_size;
    r.kv = 1;
    r.transposed = g->transposed;
    for (int a = 0; a < g->ndim; ++a) {
        r.in_dims[a] = g->in_dims[a];
        r.ksize[a] = g->ksize[a];
        r.dilation[a] = g->dilation[a];
        r.kv *= g->ksize[a];
        if (subm) {  // indices.py:1648-1657: stride 1, pad = (k/2)*dil, out dims = in dims
            r.out_dims[a] = g->in_dims[a];
            r.stride[a] = 1;
            r.padding[a] = (g->ksize[a] / 2) * g->dilation[a];
        } else {
            r.out_dims[a] = g->out_dims[a];
            r.stride[a] = g->stride[a];
            r.padding[a] = g->padding[a];
        }
    }
    return r;
}

static bool needs_i64(const Geom &g, const int *dims) {
    // same rule as the reference: int64 keys once batch * prod(dims) reaches 2^31
    // (spconv/pytorch/ops.py:188-190, ConvProblem::check_npq_not_overflow)
    double v = (double)g.batch;
    for (int a = 0; a < g.ndim; ++a) v *= (double)dims[a];
    return v >= 2147483647.0;
}

// ------------------------------------------------------------------ coordinate helpers
__device__ __forceinline__ void load_coord(const int32_t *indices, int64_t i, int ndim, int (&c)[SPX_MAX_NDIM + 1]) {
    if (ndim == 3) {
        int4 v = __ldg(reinterpret_cast<const int4 *>(indices) + i);
        c[0] = v.x; c[1] = v.y; c[2] = v.z; c[3] = v.w;
    } else {
        const int32_t *p = indices + i * (ndim + 1);
#pragma unroll
        for (int a = 0; a <= SPX_MAX_NDIM; ++a) if (a <= ndim) c[a] = __ldg(p + a);
    }
}

__device__ __forceinline__ void offset_taps(int k, const int *ksize, int ndim, int (&r)[SPX_MAX_NDIM]) {
#pragma unroll
    for (int a = SPX_MAX_NDIM - 1; a >= 0; --a) if (a < ndim) { r[a] = k % ksize[a]; k /= ksize[a]; }
}

// ------------------------------------------------------------------ SubM
template <typename Table>
__global__ void subm_insert_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= N) return;
    int c[SPX_MAX_NDIM + 1];
    load_coord(indices, i, g.ndim, c);
    table.insert_min(linear_key(c, g.in_dims, g.ndim), (int32_t)i);
}

// one thread per voxel, all kv offsets: pair_fwd[k][o] = index of the voxel at
// coord(o) - pad + r_k * dil (query_nhw, indices.py:222-236), coalesced writes, no atomics.
template <typename Table>
__global__ void subm_probe_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N,
                                  int32_t *__restrict__ pair_fwd, int32_t *__restrict__ pair_bwd,
                                  uint32_t *__restrict__ mask, int words) {
    int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= N) return;
    int c[SPX_MAX_NDIM + 1];
    load_coord(indices, o, g.ndim, c);
    const int kv = g.kv;
    uint32_t mword = 0;
    int r[SPX_MAX_NDIM] = {0, 0, 0, 0};
    for (int k = 0; k < kv; ++k) {
        int32_t found = -1;
        if (k == kv / 2) {
            found = (int32_t)o;   // centre: identity (indices.py:1671-1676)
        } else {
            int q[SPX_MAX_NDIM + 1];
            q[0] = c[0];
            bool valid = c[0] >= 0 && c[0] < g.batch;
#pragma unroll
            for (int a = 0; a < SPX_MAX_NDIM; ++a) {
                if (a < g.ndim) {
                    q[a + 1] = c[a + 1] - g.padding[a] + r[a] * g.dilation[a];
                    valid = valid && q[a + 1] >= 0 && q[a + 1] < g.in_dims[a];
                }
            }
            if (valid) {
                int32_t v;
                if (table.find_slot(linear_key(q, g.in_dims, g.ndim), v) >= 0) found = v;
            }
        }
        pair_fwd[(int64_t)k * N + o] = found;
        if (pair_bwd) pair_bwd[(int64_t)(kv - 1 - k) * N + o] = found;
        if (found >= 0) mword |= 1u << (k & 31);
        if (mask && ((k & 31) == 31 || k == kv - 1)) {
            mask[o * words + (k >> 5)] = mword;
            mword = 0;
        }
        // advance taps row-major, last axis fastest (ConvOutLocIter::operator++, indices.py:117-127)
#pragma unroll
        for (int a = SPX_MAX_NDIM - 1; a >= 0; --a) {
            if (a < g.ndim) {
                if (++r[a] < g.ksize[a]) break;
                r[a] = 0;
            }
        }
    }
}

// 3-D, 3x3x3 (any dilation), 32-bit keys -- the shape of every SubMConv3d in SECOND-style nets.
// (The generic kernel above exposes one L2 round trip per offset and spends ~150 instructions per
// probe on generic n-d index arithmetic.)
// A warp probes ONE kernel offset for K3_VOX = 128 consecutive voxels (four per lane), a block
// (27 warps) covers all offsets of those voxels.  The kernel is a chain of dependent L2 round
// trips (coordinates -> slot -> collision chain -> stores); per-offset state is one key / slot per
// voxel, so every thread keeps four independent probes in flight at full occupancy, and chains
// advance in rounds (one extra round trip per round for the whole warp, not per probe).  The
// warp's hit ballots are the columns of mask bits of its offset; thread v assembles voxel v's mask
// word from the 27 ballots.  Rows of the table are staged in shared memory for the row-major copy.
constexpr int K3_VOX = 128;                    // voxels per block; block = 27 warps
constexpr int K3_PER_LANE = K3_VOX / 32;
__global__ void __launch_bounds__(27 * 32, 2)
subm_probe_k3_kernel(Table32 table, Geom g, const int32_t *__restrict__ indices, int64_t N,
                     int32_t *__restrict__ pair_fwd, int32_t *__restrict__ pair_bwd,
                     uint32_t *__restrict__ mask, int32_t *__restrict__ row_table) {
    __shared__ uint32_t hit_col[27][K3_PER_LANE];
    __shared__ int32_t row_stage[K3_VOX][27];     // odd row stride: conflict-free both ways
    const int lane = threadIdx.x & 31;
    const int k = threadIdx.x >> 5;               // warp-uniform kernel offset, k = (rz*3 + ry)*3 + rx
    const int rz = k / 9, ry = (k / 3) % 3, rx = k % 3;
    const int64_t vbase = blockIdx.x * (int64_t)K3_VOX;
    const int D0 = g.in_dims[0], D1 = g.in_dims[1], D2 = g.in_dims[2];
    // q_a = c_a + (r_a - 1) * dil_a   (pad = dil for ksize 3), r_a in {0,1,2}
    const int oz = (rz - 1) * g.dilation[0], oy = (ry - 1) * g.dilation[1], ox = (rx - 1) * g.dilation[2];
    int4 c[K3_PER_LANE];
#pragma unroll
    for (int j = 0; j < K3_PER_LANE; ++j) {
        const int64_t o = vbase + j * 32 + lane;
        c[j] = o < N ? __ldg(reinterpret_cast<const int4 *>(indices) + o) : make_int4(-1, 0, 0, 0);
    }
    uint32_t key[K3_PER_LANE], h[K3_PER_LANE];
    unsigned long long cur[K3_PER_LANE];
    uint32_t pending = 0;
#pragma unroll
    for (int j = 0; j < K3_PER_LANE; ++j) {
        const int qz = c[j].y + oz, qy = c[j].z + oy, qx = c[j].w + ox;
        const bool valid = k != 13 && c[j].x >= 0 && c[j].x < g.batch && qz >= 0 && qz < D0 && qy >= 0 && qy < D1 &&
                           qx >= 0 && qx < D2;
        key[j] = (uint32_t)(((c[j].x * D0 + qz) * D1 + qy) * D2 + qx);
        h[j] = mix32(key[j]) & table.cap_mask;
        cur[j] = valid ? __ldg(&table.slots[h[j]]) : Table32::EMPTY;
    }
#pragma unroll
    for (int j = 0; j < K3_PER_LANE; ++j)
        if (cur[j] != Table32::EMPTY && (uint32_t)(cur[j] >> 32) != key[j]) pending |= 1u << j;
    while (pending) {                             // collision chains (short at load factor <= 0.25)
#pragma unroll
        for (int j = 0; j < K3_PER_LANE; ++j)
            if (pending & (1u << j)) { h[j] = (h[j] + 1) & table.cap_mask; cur[j] = __ldg(&table.slots[h[j]]); }
#pragma unroll
        for (int j = 0; j < K3_PER_LANE; ++j)
            if ((pending & (1u << j)) && (cur[j] == Table32::EMPTY || (uint32_t)(cur[j] >> 32) == key[j]))
                pending &= ~(1u << j);
    }
#pragma unroll
    for (int j = 0; j < K3_PER_LANE; ++j) {
        const int64_t o = vbase + j * 32 + lane;
        int32_t found = cur[j] != Table32::EMPTY ? (int32_t)(uint32_t)cur[j] : -1;
        if (k == 13 && o < N) found = (int32_t)o;     // centre: identity
        if (o < N) {
            pair_fwd[(int64_t)k * N + o] = found;
            if (pair_bwd) pair_bwd[(int64_t)(26 - k) * N + o] = found;
        }
        const uint32_t hits = __ballot_sync(0xffffffffu, found >= 0);
        if (lane == 0) hit_col[k][j] = hits;
        row_stage[j * 32 + lane][k] = found;
    }
    __syncthreads();
    if (mask && threadIdx.x < K3_VOX && vbase + threadIdx.x < N) {
        const int v = threadIdx.x;
        uint32_t m = 0;
#pragma unroll
        for (int kk = 0; kk < 27; ++kk) m |= ((hit_col[kk][v >> 5] >> (v & 31)) & 1u) << kk;
        mask[vbase + v] = m;
    }
    if (row_table) {
        // row-major copy [N][32] (one 128-byte line per voxel, -1 padded) for build_tile_table_rows_kernel:
        // the permuted re-read then costs 4 sectors per row instead of one per (row, offset)
        for (int e = threadIdx.x; e < K3_VOX * 32; e += 27 * 32) {
            const int v = e >> 5, kk = e & 31;
            if (vbase + v < N) row_table[(vbase + v) * 32 + kk] = kk < 27 ? row_stage[v][kk] : -1;
        }
    }
}

// ------------------------------------------------------------------ regular / transposed conv
__device__ __forceinline__ bool conv_out_coord(const Geom &g, const int (&c)[SPX_MAX_NDIM + 1],
                                               const int (&r)[SPX_MAX_NDIM], int (&o)[SPX_MAX_NDIM + 1]) {
    bool valid = c[0] >= 0 && c[0] < g.batch;
    o[0] = c[0];
#pragma unroll
    for (int a = 0; a < SPX_MAX_NDIM; ++a) {
        if (a < g.ndim) {
            if (g.transposed) {   // query_nhw_out, indices.py:253-269
                o[a + 1] = c[a + 1] * g.stride[a] - g.padding[a] + r[a] * g.dilation[a];
                valid = valid && o[a + 1] >= 0 && o[a + 1] < g.out_dims[a];
            } else {              // query_npq, indices.py:141-203
                int h = c[a + 1] + g.padding[a] - r[a] * g.dilation[a];
                o[a + 1] = h / g.stride[a];
                valid = valid && o[a + 1] >= 0 && o[a + 1] < g.out_dims[a] && (h % g.stride[a] == 0);
            }
        }
    }
    return valid;
}

// 3-D, non-transposed fast path of query_npq (indices.py:141-203): the taps of the block's offset
// are decoded once per block, the stride division is a shift for strides 1 and 2, everything else
// is three fused range tests.  (The generic helpers spend ~150 instructions per (input, offset)
// on run-time-ndim loops and two integer divisions per axis.)
struct Taps3 { int r0, r1, r2; };
__device__ __forceinline__ Taps3 block_taps3(const Geom &g, int k) {
    Taps3 t;
    t.r2 = k % g.ksize[2]; k /= g.ksize[2];
    t.r1 = k % g.ksize[1]; k /= g.ksize[1];
    t.r0 = k;
    return t;
}
__device__ __forceinline__ bool axis_out(int c, int pad, int r, int dil, int stride, int odim, int &o) {
    const int h = c + pad - r * dil;
    if (h < 0) return false;
    if (stride == 1) o = h;
    else if (stride == 2) { if (h & 1) return false; o = h >> 1; }
    else { o = h / stride; if (o * stride != h) return false; }
    return o < odim;
}
// The inverse relations, for a rulebook onto given output coordinates (spx_cross_rulebook_all): the input
// coordinate c that output o reads through tap r, valid iff it lies in [0, idim).  Regular conv (the c with
// axis_out(c, r) = o): c = o * stride - pad + r * dil.  Transposed: c = (o + pad - r * dil) / stride, exact.
// validate_cross keeps every intermediate inside int.
__device__ __forceinline__ bool axis_in(int o, int pad, int r, int dil, int stride, int idim, int &c) {
    c = o * stride - pad + r * dil;
    return c >= 0 && c < idim;
}
__device__ __forceinline__ bool axis_in_transposed(int o, int pad, int r, int dil, int stride, int idim, int &c) {
    const int h = o + pad - r * dil;
    if (h < 0) return false;
    if (stride == 1) c = h;
    else if (stride == 2) { if (h & 1) return false; c = h >> 1; }
    else { c = h / stride; if (c * stride != h) return false; }
    return c < idim;
}
__device__ __forceinline__ bool conv3_out_key(const Geom &g, const int4 c, const Taps3 &t, int64_t &key) {
    int o0, o1, o2;
    if (c.x < 0 || c.x >= g.batch) return false;
    if (!axis_out(c.y, g.padding[0], t.r0, g.dilation[0], g.stride[0], g.out_dims[0], o0)) return false;
    if (!axis_out(c.z, g.padding[1], t.r1, g.dilation[1], g.stride[1], g.out_dims[1], o1)) return false;
    if (!axis_out(c.w, g.padding[2], t.r2, g.dilation[2], g.stride[2], g.out_dims[2], o2)) return false;
    key = (((int64_t)c.x * g.out_dims[0] + o0) * g.out_dims[1] + o1) * g.out_dims[2] + o2;
    return true;
}

// 3-D, 3x3x3, non-transposed: one thread per INPUT voxel walks the 27 offsets.  The per-axis output
// coordinates of the three taps are computed once (9 divisions-by-stride instead of 81), and with a
// stride > 1 most (axis, tap) pairs fail the divisibility test, so only the surviving combinations
// (3.4 of 27 on average at stride 2) reach the hash table.  The grid-(N, kv) kernels re-read the
// coordinates 27 times and spend a thread per rejected combination.
struct Axis3 { int o[3]; };
__device__ __forceinline__ Axis3 axis_taps3(int c, int pad, int dil, int stride, int odim) {
    Axis3 a;
#pragma unroll
    for (int r = 0; r < 3; ++r) { int o; a.o[r] = axis_out(c, pad, r, dil, stride, odim, o) ? o : -1; }
    return a;
}

// pair_bwd[k][i] = output of (input i, offset k) or -1 (every element written, coalesced over i);
// pair_fwd[k][o] = i scattered; mask_bwd[i] (optional) = bits of the offsets that hit an output
template <typename Table>
__global__ void conv_pairs_k3_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N, int64_t M,
                                     int32_t *__restrict__ pair_fwd, int32_t *__restrict__ pair_bwd,
                                     uint32_t *__restrict__ mask_bwd, uint32_t *__restrict__ mask_fwd_or) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
    const bool bok = c.x >= 0 && c.x < g.batch;
    const Axis3 az = axis_taps3(c.y, g.padding[0], g.dilation[0], g.stride[0], g.out_dims[0]);
    const Axis3 ay = axis_taps3(c.z, g.padding[1], g.dilation[1], g.stride[1], g.out_dims[1]);
    const Axis3 ax = axis_taps3(c.w, g.padding[2], g.dilation[2], g.stride[2], g.out_dims[2]);
    uint32_t mword = 0;
#pragma unroll
    for (int r0 = 0; r0 < 3; ++r0) {
#pragma unroll
        for (int r1 = 0; r1 < 3; ++r1) {
#pragma unroll
            for (int r2 = 0; r2 < 3; ++r2) {
                const int k = (r0 * 3 + r1) * 3 + r2;
                int32_t out = -1;
                if (bok && az.o[r0] >= 0 && ay.o[r1] >= 0 && ax.o[r2] >= 0) {
                    const int64_t key = (((int64_t)c.x * g.out_dims[0] + az.o[r0]) * g.out_dims[1] + ay.o[r1]) *
                                            g.out_dims[2] + ax.o[r2];
                    int32_t v;
                    if (table.find_slot(key, v) >= 0) out = v;
                }
                pair_bwd[(int64_t)k * N + i] = out;
                if (out >= 0) {
                    pair_fwd[(int64_t)k * M + out] = (int32_t)i;
                    mword |= 1u << k;
                    if (mask_fwd_or) atomicOr(&mask_fwd_or[out], 1u << k);   // zeroed by conv_assign_rank_kernel
                }
            }
        }
    }
    if (mask_bwd) mask_bwd[i] = mword;
}


// ---- append-on-create variants (default path): the thread whose CAS creates a table entry records
// the slot, so the distinct outputs are known without scanning the (mostly empty) table afterwards.
// Created slots are staged in shared memory and a block reserves its range of the global list with
// ONE atomic.  `state`: [0] number of created entries, [1] overflow flag (a probe chain exceeded
// CONV_MAX_PROBES: the optimistically sized table was too small, the host re-runs with the full size).
constexpr int CONV_MAX_PROBES = 96;
constexpr int APPEND_THREADS = 128;

template <typename Table>
__global__ void __launch_bounds__(APPEND_THREADS)
conv_insert_k3_append_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N,
                             uint32_t *__restrict__ slot_list, int *__restrict__ state) {
    __shared__ uint32_t stage[APPEND_THREADS * 27];
    __shared__ int cnt_s, base_s;
    if (threadIdx.x == 0) cnt_s = 0;
    __syncthreads();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < N) {
        const int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
        if (c.x >= 0 && c.x < g.batch) {
            const Axis3 az = axis_taps3(c.y, g.padding[0], g.dilation[0], g.stride[0], g.out_dims[0]);
            const Axis3 ay = axis_taps3(c.z, g.padding[1], g.dilation[1], g.stride[1], g.out_dims[1]);
            const Axis3 ax = axis_taps3(c.w, g.padding[2], g.dilation[2], g.stride[2], g.out_dims[2]);
#pragma unroll
            for (int r0 = 0; r0 < 3; ++r0) {
                if (az.o[r0] < 0) continue;
                const int64_t kz = (int64_t)c.x * g.out_dims[0] + az.o[r0];
#pragma unroll
                for (int r1 = 0; r1 < 3; ++r1) {
                    if (ay.o[r1] < 0) continue;
                    const int64_t kzy = kz * g.out_dims[1] + ay.o[r1];
#pragma unroll
                    for (int r2 = 0; r2 < 3; ++r2) {
                        if (ax.o[r2] < 0) continue;
                        const int k = (r0 * 3 + r1) * 3 + r2;
                        bool created;
                        const int64_t slot = table.insert_min_slot(kzy * g.out_dims[2] + ax.o[r2],
                                                                   (int32_t)((int64_t)k * N + i), created, CONV_MAX_PROBES);
                        if (slot < 0) state[1] = 1;
                        else if (created) stage[atomicAdd(&cnt_s, 1)] = (uint32_t)slot;
                    }
                }
            }
        }
    }
    __syncthreads();
    const int cnt = cnt_s;
    if (threadIdx.x == 0) base_s = cnt ? atomicAdd(state, cnt) : 0;
    __syncthreads();
    for (int j = threadIdx.x; j < cnt; j += APPEND_THREADS) slot_list[base_s + j] = stage[j];
}

// grid (ceil(N/T), kv): one (input, offset) per thread -> at most one creation per thread
template <typename Table, bool FAST3>
__global__ void __launch_bounds__(APPEND_THREADS)
conv_insert_append_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N,
                          uint32_t *__restrict__ slot_list, int *__restrict__ state) {
    __shared__ int warp_cnt[APPEND_THREADS / 32];
    __shared__ int base_s;
    __shared__ Taps3 taps;
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int k = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (FAST3 && threadIdx.x == 0) taps = block_taps3(g, k);
    __syncthreads();
    bool created = false;
    int64_t slot = 0;
    if (i < N) {
        int64_t key = 0;
        bool valid;
        if constexpr (FAST3) {
            const int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
            valid = conv3_out_key(g, c, taps, key);
        } else {
            int c[SPX_MAX_NDIM + 1], o[SPX_MAX_NDIM + 1], r[SPX_MAX_NDIM];
            load_coord(indices, i, g.ndim, c);
            offset_taps(k, g.ksize, g.ndim, r);
            valid = conv_out_coord(g, c, r, o);
            if (valid) key = linear_key(o, g.out_dims, g.ndim);
        }
        if (valid) {
            slot = table.insert_min_slot(key, (int32_t)((int64_t)k * N + i), created, CONV_MAX_PROBES);
            if (slot < 0) { state[1] = 1; created = false; }
        }
    }
    const unsigned ball = __ballot_sync(0xffffffffu, created);
    if (lane == 0) warp_cnt[warp] = __popc(ball);
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < APPEND_THREADS / 32; ++w) { const int c = warp_cnt[w]; warp_cnt[w] = tot; tot += c; }
        base_s = tot ? atomicAdd(state, tot) : 0;
    }
    __syncthreads();
    if (created) slot_list[base_s + warp_cnt[warp] + __popc(ball & ((1u << lane) - 1u))] = (uint32_t)slot;
}

// ---- ranking the outputs by first touch WITHOUT a sort.  Every output's final payload p = k*N + i
// (the smallest (offset, input) pair that produces it) is distinct, so the rank of an output is the
// number of outputs with a smaller payload: the bitmap / tile-prefix / popcount ranking of rank.cuh
// over [0, kv*N).  conv_mark_kernel marks and its last block builds the tile prefix;
// conv_assign_rank_kernel ranks.  Replaces a radix sort of the payloads (1 + 2 x 3 launches at 22 key bits).

// one launch clears everything stage 1 needs: hash table (0xFF), 64-bit-key value array (0x7F), ranking scratch and counters (0)
__global__ void conv_clear_kernel(uint4 *__restrict__ table, int64_t table_vec, uint4 *__restrict__ tvals, int64_t tvals_vec,
                                  uint4 *__restrict__ zero, int64_t zero_vec) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const uint4 ff = make_uint4(~0u, ~0u, ~0u, ~0u), sf = make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu),
                zz = make_uint4(0u, 0u, 0u, 0u);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < table_vec; i += stride) table[i] = ff;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < tvals_vec; i += stride) tvals[i] = sf;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < zero_vec; i += stride) zero[i] = zz;
}

constexpr int MARK_THREADS = 256;
// mark every output's final payload; the LAST block to finish turns the tile counts into an exclusive prefix
template <typename Table>
__global__ void __launch_bounds__(MARK_THREADS)
conv_mark_kernel(Table table, const uint32_t *__restrict__ slot_list, int64_t M, uint32_t *__restrict__ bitmap,
                 int *__restrict__ tile_cnt, int64_t tiles, int *__restrict__ done) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j < M)      // final payload: all inserts finished in an earlier kernel
        rank_mark((uint32_t)table.value_at(slot_list[j]), bitmap, tile_cnt);
    int total;
    rank_prefix_last_block<MARK_THREADS>(tile_cnt, tiles, done, &total);
}

// created slot j -> rank r of its payload: write r into the slot, decode the key into out_inds[r]
template <typename Table>
__global__ void conv_assign_rank_kernel(Table table, Geom g, const uint32_t *__restrict__ slot_list, int64_t M,
                                        const uint32_t *__restrict__ bitmap, const int *__restrict__ tile_prefix,
                                        int32_t *__restrict__ out_inds, uint32_t *__restrict__ mask_zero,
                                        int32_t *__restrict__ pair_fill, int kv) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= M) return;
    if (pair_fill)                                  // column j of the forward table: -1 until the pairs kernel fills it
        for (int k = 0; k < kv; ++k) pair_fill[(int64_t)k * M + j] = -1;
    const uint32_t s = slot_list[j];
    int64_t key; int32_t val;
    table.occupied(s, key, val);
    const int r = rank_of((uint32_t)val, bitmap, tile_prefix);
    table.set_value(s, r);
    if (mask_zero) mask_zero[r] = 0u;              // the pairs kernel ORs the forward masks into it
    int32_t *dst = out_inds + (int64_t)r * (g.ndim + 1);
    for (int a = g.ndim - 1; a >= 0; --a) {
        dst[a + 1] = (int32_t)(key % g.out_dims[a]);
        key /= g.out_dims[a];
    }
    dst[0] = (int32_t)key;
}

// grid (ceil(N/T), kv): pair_bwd[k][i] = o (every element written), pair_fwd[k][o] = i
template <typename Table, bool FAST3>
__global__ void conv_pairs_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N, int64_t M,
                                  int32_t *__restrict__ pair_fwd, int32_t *__restrict__ pair_bwd) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int k = blockIdx.y;
    int32_t out = -1;
    if constexpr (FAST3) {
        __shared__ Taps3 taps;
        if (threadIdx.x == 0) taps = block_taps3(g, k);
        __syncthreads();
        if (i >= N) return;
        const int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
        int64_t key;
        int32_t v;
        if (conv3_out_key(g, c, taps, key) && table.find_slot(key, v) >= 0) out = v;
    } else {
        if (i >= N) return;
        int c[SPX_MAX_NDIM + 1], o[SPX_MAX_NDIM + 1], r[SPX_MAX_NDIM];
        load_coord(indices, i, g.ndim, c);
        offset_taps(k, g.ksize, g.ndim, r);
        if (conv_out_coord(g, c, r, o)) {
            int32_t v;
            if (table.find_slot(linear_key(o, g.out_dims, g.ndim), v) >= 0) out = v;
        }
    }
    pair_bwd[(int64_t)k * N + i] = out;
    if (out >= 0) pair_fwd[(int64_t)k * M + out] = (int32_t)i;
}

// mask[row] = bits of the non-negative entries of table[:, row]
__global__ void table_mask_kernel(const int32_t *__restrict__ table, int64_t rows, int kv, int words,
                                  uint32_t *__restrict__ mask) {
    int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= rows) return;
    uint32_t m = 0;
    for (int k = 0; k < kv; ++k) {
        if (table[(int64_t)k * rows + r] >= 0) m |= 1u << (k & 31);
        if ((k & 31) == 31 || k == kv - 1) { mask[r * words + (k >> 5)] = m; m = 0; }
    }
}

// ------------------------------------------------------------------ bounded regular conv (no host read-back)
// The caller gives an upper limit `bound` on the outputs; the table holds at most 4 x bound slots, so the
// distinct outputs are found by scanning it instead of keeping a list of created slots, and the count
// never leaves the device.  Every output is ranked (same bitmap ranking, so rows below the count equal
// the unbounded rulebook bit for bit); outputs ranked >= bound get the value -1, which the pairs kernels
// above already treat as "no output": the deterministic truncation.  `state`: [0] number of outputs
// (written by the marking kernel), [1] probe-chain overflow, [2] completion counter of the marking kernel.
template <typename Table>
__global__ void conv_insert_k3_bounded_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N,
                              int *__restrict__ state) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
    if (c.x < 0 || c.x >= g.batch) return;
    const Axis3 az = axis_taps3(c.y, g.padding[0], g.dilation[0], g.stride[0], g.out_dims[0]);
    const Axis3 ay = axis_taps3(c.z, g.padding[1], g.dilation[1], g.stride[1], g.out_dims[1]);
    const Axis3 ax = axis_taps3(c.w, g.padding[2], g.dilation[2], g.stride[2], g.out_dims[2]);
#pragma unroll
    for (int r0 = 0; r0 < 3; ++r0) {
        if (az.o[r0] < 0) continue;
        const int64_t kz = (int64_t)c.x * g.out_dims[0] + az.o[r0];
#pragma unroll
        for (int r1 = 0; r1 < 3; ++r1) {
            if (ay.o[r1] < 0) continue;
            const int64_t kzy = kz * g.out_dims[1] + ay.o[r1];
#pragma unroll
            for (int r2 = 0; r2 < 3; ++r2) {
                if (ax.o[r2] < 0) continue;
                const int k = (r0 * 3 + r1) * 3 + r2;
                bool created;
                if (table.insert_min_slot(kzy * g.out_dims[2] + ax.o[r2], (int32_t)((int64_t)k * N + i), created,
                                          CONV_MAX_PROBES) < 0)
                    state[1] = 1;
            }
        }
    }
}

// grid (ceil(N/T), kv): one (input, offset) per thread
template <typename Table, bool FAST3>
__global__ void __launch_bounds__(APPEND_THREADS)
conv_insert_bounded_kernel(Table table, Geom g, const int32_t *__restrict__ indices, int64_t N, int *__restrict__ state) {
    __shared__ Taps3 taps;
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int k = blockIdx.y;
    if (FAST3 && threadIdx.x == 0) taps = block_taps3(g, k);
    __syncthreads();
    if (i >= N) return;
    int64_t key = 0;
    bool valid;
    if constexpr (FAST3) {
        const int4 c = __ldg(reinterpret_cast<const int4 *>(indices) + i);
        valid = conv3_out_key(g, c, taps, key);
    } else {
        int c[SPX_MAX_NDIM + 1], o[SPX_MAX_NDIM + 1], r[SPX_MAX_NDIM];
        load_coord(indices, i, g.ndim, c);
        offset_taps(k, g.ksize, g.ndim, r);
        valid = conv_out_coord(g, c, r, o);
        if (valid) key = linear_key(o, g.out_dims, g.ndim);
    }
    bool created;
    if (valid && table.insert_min_slot(key, (int32_t)((int64_t)k * N + i), created, CONV_MAX_PROBES) < 0) state[1] = 1;
}

// one thread per table slot: mark the final payload of every output; the last block builds the tile
// prefix and leaves the number of outputs in state[0]
template <typename Table>
__global__ void __launch_bounds__(MARK_THREADS)
conv_mark_table_kernel(Table table, int64_t capacity, uint32_t *__restrict__ bitmap, int *__restrict__ tile_cnt,
                       int64_t tiles, int *__restrict__ state) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t key; int32_t val;
    if (s < capacity && table.occupied((uint32_t)s, key, val)) rank_mark((uint32_t)val, bitmap, tile_cnt);
    int total;
    if (rank_prefix_last_block<MARK_THREADS>(tile_cnt, tiles, state + 2, &total) && threadIdx.x == 0) state[0] = total;
}

// one thread per table slot and per output row (grid covers max(capacity, bound)):
//   slot s:  payload -> rank r; r < bound: the slot's value becomes r and out_inds[r] its coordinate,
//            else the value becomes -1 (dropped).  After a probe-chain overflow every slot is emptied
//            instead, so the pairs kernel finds nothing and cannot walk a full table for ever.
//   row j:   column j of pair_fwd = -1 (the pairs kernel fills it), mask 0 where the pairs kernel ORs into
//            it, and for j >= M (padding) out_inds[j] = -1.
// Thread 0 publishes num_out and ORs the status bits.
template <typename Table>
__global__ void conv_assign_table_kernel(Table table, Geom g, int64_t capacity, int64_t bound,
                                         const uint32_t *__restrict__ bitmap, const int *__restrict__ tile_prefix,
                                         const int *__restrict__ state, int32_t *__restrict__ out_inds,
                                         uint32_t *__restrict__ mask_zero, int32_t *__restrict__ pair_fill, int kv,
                                         int32_t *__restrict__ num_out, int32_t *__restrict__ status) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const bool overflow = state[1] != 0;
    const int64_t total = overflow ? 0 : state[0];
    const int64_t M = total < bound ? total : bound;
    if (j == 0) {
        *num_out = (int32_t)M;
        const int bits = (total > bound ? 1 : 0) | (overflow ? 2 : 0);
        if (bits) atomicOr(status, bits);
    }
    if (j < bound) {
        for (int k = 0; k < kv; ++k) pair_fill[(int64_t)k * bound + j] = -1;
        if (mask_zero) mask_zero[j] = 0u;
        if (j >= M) {
            int32_t *dst = out_inds + j * (g.ndim + 1);
            for (int a = 0; a <= g.ndim; ++a) dst[a] = -1;
        }
    }
    if (j >= capacity) return;
    const uint32_t s = (uint32_t)j;
    if (overflow) { table.clear_slot(s); return; }
    int64_t key; int32_t val;
    if (!table.occupied(s, key, val)) return;
    const int r = rank_of((uint32_t)val, bitmap, tile_prefix);
    if (r >= bound) { table.set_value(s, -1); return; }
    table.set_value(s, r);
    int32_t *dst = out_inds + (int64_t)r * (g.ndim + 1);
    for (int a = g.ndim - 1; a >= 0; --a) {
        dst[a + 1] = (int32_t)(key % g.out_dims[a]);
        key /= g.out_dims[a];
    }
    dst[0] = (int32_t)key;
}

// zero rows [*count, rows) of a row-major matrix; V = uint4 (16-byte stores) or uint16_t
template <typename V>
__global__ void zero_rows_from_count_kernel(V *__restrict__ p, int64_t rows, int64_t row_vec,
                                            const int32_t *__restrict__ count) {
    int64_t m = *count;
    m = m < 0 ? 0 : (m > rows ? rows : m);
    const int64_t n = (rows - m) * row_vec, stride = (int64_t)gridDim.x * blockDim.x;
    V *q = p + m * row_vec;
    V z;
    memset(&z, 0, sizeof(V));
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) q[i] = z;
}

// ------------------------------------------------------------------ Native compact pairs (stable scan)
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 4;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// rows: regular conv -> kv rows (row k of pair_bwd); SubM -> kv/2 rows
__global__ void native_count_kernel(const int32_t *__restrict__ pair_bwd, int64_t N, int *__restrict__ block_counts,
                                    int nblk) {
    int row = blockIdx.y;
    int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        int64_t i = base + j * SCAN_THREADS + threadIdx.x;
        if (i < N && pair_bwd[(int64_t)row * N + i] >= 0) ++cnt;
    }
    typedef cub::BlockReduce<int, SCAN_THREADS> BR;
    __shared__ typename BR::TempStorage tmp;
    int total = BR(tmp).Sum(cnt);
    if (threadIdx.x == 0) block_counts[row * nblk + blockIdx.x] = total;
}

// one block per row: exclusive scan of the block counts, total -> num[row]
__global__ void native_scan_kernel(int *__restrict__ block_counts, int nblk, int32_t *__restrict__ num) {
    int row = blockIdx.x;
    typedef cub::BlockScan<int, SCAN_THREADS> BS;
    __shared__ typename BS::TempStorage tmp;
    __shared__ int carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int b0 = 0; b0 < nblk; b0 += SCAN_THREADS) {
        int b = b0 + threadIdx.x;
        int v = b < nblk ? block_counts[row * nblk + b] : 0;
        int excl, agg;
        BS(tmp).ExclusiveSum(v, excl, agg);
        int carry = carry_s;
        if (b < nblk) block_counts[row * nblk + b] = carry + excl;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + agg;
        __syncthreads();
    }
    if (threadIdx.x == 0) num[row] = carry_s;
}

__global__ void native_write_kernel(const int32_t *__restrict__ pair_bwd, int64_t N, int kv, int is_subm,
                                    const int *__restrict__ block_offsets, int nblk, int32_t *__restrict__ pairs) {
    int row = blockIdx.y;
    int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
    // blocked arrangement keeps ascending-i order inside the tile
    int32_t vals[SCAN_ITEMS];
    int flags[SCAN_ITEMS];
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        int64_t i = base + (int64_t)threadIdx.x * SCAN_ITEMS + j;
        vals[j] = i < N ? pair_bwd[(int64_t)row * N + i] : -1;
        flags[j] = vals[j] >= 0;
        cnt += flags[j];
    }
    typedef cub::BlockScan<int, SCAN_THREADS> BS;
    __shared__ typename BS::TempStorage tmp;
    int excl;
    BS(tmp).ExclusiveSum(cnt, excl);
    int pos = block_offsets[row * nblk + blockIdx.x] + excl;
    int32_t *pin = pairs, *pout = pairs + (int64_t)kv * N;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        if (flags[j]) {
            int32_t i = (int32_t)(base + (int64_t)threadIdx.x * SCAN_ITEMS + j);
            int32_t o = vals[j];
            pin[(int64_t)row * N + pos] = i;
            pout[(int64_t)row * N + pos] = o;
            if (is_subm) {   // mirrored entry, indices.py:1696-1699
                pin[(int64_t)(kv - 1 - row) * N + pos] = o;
                pout[(int64_t)(kv - 1 - row) * N + pos] = i;
            }
            ++pos;
        }
    }
}

__global__ void subm_centre_kernel(int32_t *__restrict__ pairs, int64_t N, int kv) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= N) return;
    pairs[(int64_t)(kv / 2) * N + i] = (int32_t)i;
    pairs[(int64_t)kv * N + (int64_t)(kv / 2) * N + i] = (int32_t)i;
}

// compact pairs -> dense tables (ConvAlgo.Native operator path)
__global__ void pairs_to_table_kernel(const int32_t *__restrict__ pairs, const int32_t *__restrict__ num, int kv,
                                      int64_t pair_stride, int64_t n_in, int64_t n_out, int is_subm, int inverse,
                                      int32_t *__restrict__ table_fwd, int32_t *__restrict__ table_bwd,
                                      uint32_t *__restrict__ mask_fwd, uint32_t *__restrict__ mask_bwd, int words) {
    int k = blockIdx.y;
    int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t cnt;
    if (is_subm) {   // mirror rule, spconv/pytorch/ops.py:962-968
        if (k == kv / 2) cnt = n_in;
        else cnt = k < kv / 2 ? num[k] : num[kv - 1 - k];
    } else {
        cnt = num[k];
    }
    if (j >= cnt) return;
    int32_t a = pairs[(int64_t)k * pair_stride + j];
    int32_t b = pairs[(int64_t)kv * pair_stride + (int64_t)k * pair_stride + j];
    int32_t i = inverse ? b : a, o = inverse ? a : b;
    if (i < 0 || o < 0 || i >= n_in || o >= n_out) return;
    if (table_fwd) table_fwd[(int64_t)k * n_out + o] = i;
    if (table_bwd) table_bwd[(int64_t)k * n_in + i] = o;
    if (mask_fwd) atomicOr(&mask_fwd[o * words + (k >> 5)], 1u << (k & 31));
    if (mask_bwd) atomicOr(&mask_bwd[i * words + (k >> 5)], 1u << (k & 31));
}

// ------------------------------------------------------------------ rulebook onto given output coordinates
// spx_cross_rulebook_all: the source rows x and the target rows t are both given.  A source row is usable when it is
// below its num_valid, its batch is in [0, batch) and every coordinate is inside in_dims; a target row is active under
// the same conditions against out_dims and when no lower active row has its coordinate.  Each set has its own hash
// table, filled by insert_min, so the lowest row wins a duplicated coordinate on either side.
constexpr int CROSS_THREADS = 128;
constexpr int CROSS_CHUNK = 8;                  // taps whose probe chains advance together (find_many)

template <int NDIM>
__device__ __forceinline__ bool load_usable(const int32_t *__restrict__ indices, int64_t row, const int *dims, int batch,
                                            int (&c)[SPX_MAX_NDIM + 1]) {
    load_coord(indices, row, NDIM, c);
    bool ok = c[0] >= 0 && c[0] < batch;
#pragma unroll
    for (int a = 0; a < NDIM; ++a) ok = ok && c[a + 1] >= 0 && c[a + 1] < dims[a];
    return ok;
}

// threads [0, n) insert the usable source rows into src_table (keys over in_dims), threads [n, n + m) the usable
// target rows into dst_table (keys over out_dims)
template <typename Table, int NDIM>
__global__ void __launch_bounds__(CROSS_THREADS)
cross_insert_kernel(Table src_table, Table dst_table, Geom g, const int32_t *__restrict__ src, int64_t n,
                    const int32_t *__restrict__ src_valid, const int32_t *__restrict__ dst, int64_t m,
                    const int32_t *__restrict__ dst_valid) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const bool is_src = j < n;
    const int64_t row = is_src ? j : j - n;
    if (row >= (is_src ? n : m) || row >= valid_rows(is_src ? src_valid : dst_valid, is_src ? n : m)) return;
    int dims[SPX_MAX_NDIM] = {0, 0, 0, 0};
#pragma unroll
    for (int a = 0; a < NDIM; ++a) dims[a] = is_src ? g.in_dims[a] : g.out_dims[a];
    int c[SPX_MAX_NDIM + 1] = {0, 0, 0, 0, 0};
    if (!load_usable<NDIM>(is_src ? src : dst, row, dims, g.batch, c)) return;
    if (is_src) src_table.insert_min(linear_key(c, dims, NDIM), (int32_t)row);
    else dst_table.insert_min(linear_key(c, dims, NDIM), (int32_t)row);
}

// one thread per target row o: pair_fwd[k][o] and mask_fwd[o] written in full (-1 / 0 for an inactive row), and
// for every hit i the scatter pair_bwd[k][i] = o plus bit k of mask_bwd[i] (pair_bwd / mask_bwd cleared before).
// A (source row, tap) pair maps to at most one coordinate and the active targets are distinct, so every pair_bwd
// element has at most one writer.  The taps are probed CROSS_CHUNK at a time with their chains in flight together.
template <typename Table, int NDIM, bool TRANSPOSED>
__global__ void __launch_bounds__(CROSS_THREADS)
cross_probe_kernel(Table src_table, Table dst_table, Geom g, const int32_t *__restrict__ dst, int64_t m,
                   const int32_t *__restrict__ dst_valid, int64_t n, int32_t *__restrict__ pair_fwd,
                   int32_t *__restrict__ pair_bwd, uint32_t *__restrict__ mask_fwd, uint32_t *__restrict__ mask_bwd,
                   int words) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= m) return;
    int c[SPX_MAX_NDIM + 1] = {0, 0, 0, 0, 0};
    bool active = o < valid_rows(dst_valid, m) && load_usable<NDIM>(dst, o, g.out_dims, g.batch, c);
    if (active) {
        int32_t v = -1;
        active = dst_table.find_slot(linear_key(c, g.out_dims, NDIM), v) >= 0 && v == (int32_t)o;
    }
    const int kv = g.kv;
    int r[NDIM];
#pragma unroll
    for (int a = 0; a < NDIM; ++a) r[a] = 0;
    uint32_t mword = 0;
    for (int k0 = 0; k0 < kv; k0 += CROSS_CHUNK) {
        int64_t key[CROSS_CHUNK];
        bool live[CROSS_CHUNK];
        int32_t v[CROSS_CHUNK];
#pragma unroll
        for (int j = 0; j < CROSS_CHUNK; ++j) {
            int q[SPX_MAX_NDIM + 1] = {c[0], 0, 0, 0, 0};
            bool ok = active && k0 + j < kv;
#pragma unroll
            for (int a = 0; a < NDIM; ++a) {
                int ca = 0;
                const bool in = TRANSPOSED
                    ? axis_in_transposed(c[a + 1], g.padding[a], r[a], g.dilation[a], g.stride[a], g.in_dims[a], ca)
                    : axis_in(c[a + 1], g.padding[a], r[a], g.dilation[a], g.stride[a], g.in_dims[a], ca);
                ok = ok && in;
                q[a + 1] = ca;
            }
            live[j] = ok;
            key[j] = ok ? linear_key(q, g.in_dims, NDIM) : 0;
#pragma unroll
            for (int a = NDIM - 1; a >= 0; --a) {          // next tap, last axis fastest
                if (++r[a] < g.ksize[a]) break;
                r[a] = 0;
            }
        }
        find_many<CROSS_CHUNK>(src_table, key, live, v);
#pragma unroll
        for (int j = 0; j < CROSS_CHUNK; ++j) {
            const int k = k0 + j;
            if (k >= kv) break;
            pair_fwd[(int64_t)k * m + o] = v[j];
            if (v[j] >= 0) {
                mword |= 1u << (k & 31);
                pair_bwd[(int64_t)k * n + v[j]] = (int32_t)o;
                atomicOr(&mask_bwd[(int64_t)v[j] * words + (k >> 5)], 1u << (k & 31));
            }
            if ((k & 31) == 31 || k == kv - 1) {
                mask_fwd[o * words + (k >> 5)] = mword;
                mword = 0;
            }
        }
    }
}

// ------------------------------------------------------------------ argsort helpers
__global__ void iota_kernel(int32_t *__restrict__ p, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) p[i] = (int32_t)i;
}
__global__ void gather_word_kernel(const uint32_t *__restrict__ mask, const int32_t *__restrict__ perm, int64_t n,
                                   int words, int w, uint32_t *__restrict__ out) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = mask[(int64_t)perm[i] * words + w];
}
__global__ void gather_rows_kernel(const uint32_t *__restrict__ src, const int32_t *__restrict__ perm, int64_t n,
                                   int words, uint32_t *__restrict__ dst) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int w = 0; w < words; ++w) dst[i * words + w] = src[(int64_t)perm[i] * words + w];
}

// ------------------------------------------------------------------ tile-blocked gather table
// one block per 128-row tile; see include/spconv_b200.h (spx_build_tile_table)
constexpr int TT_SPLIT = 4;                     // threads per tile row: offsets k = q, q + 4, ...
// (blockIdx.y picks one of up to two jobs: a regular conv builds its forward and backward tables in one launch)
struct TtJob {
    const int32_t *pair; int64_t pair_stride;
    const int32_t *argsort; const uint32_t *mask;
    int64_t rows;
    int32_t *table; uint32_t *tile_mask;
};
struct TtJobs { TtJob j[2]; };

__global__ void __launch_bounds__(128 * TT_SPLIT)
build_tile_table_kernel(const TtJobs jobs, int kv, int words) {
    const TtJob &J = jobs.j[blockIdx.y];
    const int64_t t = blockIdx.x;
    if (t * 128 >= J.rows) return;
    const int32_t *__restrict__ pair = J.pair;
    const int64_t pair_stride = J.pair_stride;
    const int32_t *__restrict__ argsort = J.argsort;
    const uint32_t *__restrict__ mask = J.mask;
    const int64_t rows = J.rows;
    int32_t *__restrict__ table = J.table;
    uint32_t *__restrict__ tile_mask = J.tile_mask;
    const int r = threadIdx.x & 127;
    const int q = threadIdx.x >> 7;             // warp-uniform
    const int64_t j = t * 128 + r;
    int32_t src = -1;
    if (j < rows) src = argsort ? __ldg(argsort + j) : (int32_t)j;
    int32_t *blk = table + t * (int64_t)(kv + 1) * 128;
    // 3N x 4 threads with <= 8 independent scattered 4-byte loads each: the kernel is a pure
    // L2-latency problem, so it is sized for memory-level parallelism, not for work per thread
    const int32_t *col = pair + (src >= 0 ? src : 0);
    // An offset whose bit is clear in the row's mask stores -1.  A mask split clears the offsets of the
    // other split while pair still holds them, and the GEMM kernels gather every entry >= 0 of a stage
    // they run (an all-zero tile still runs one stage at offset 0).  Without a split a bit is clear
    // exactly where the pair is -1.
    uint32_t rm0 = ~0u, rm1 = ~0u, rm2 = ~0u, rm3 = ~0u;
    if (mask && j < rows) {
        const uint32_t *mr = mask + j * words;
        rm0 = __ldg(mr);
        if (words > 1) rm1 = __ldg(mr + 1);
        if (words > 2) rm2 = __ldg(mr + 2);
        if (words > 3) rm3 = __ldg(mr + 3);
    }
#pragma unroll 8
    for (int k = q; k < kv; k += TT_SPLIT) {
        const uint32_t w = k < 32 ? rm0 : k < 64 ? rm1 : k < 96 ? rm2 : rm3;
        blk[k * 128 + r] = src >= 0 && ((w >> (k & 31)) & 1u) ? __ldg(col + (int64_t)k * pair_stride) : -1;
    }
    if (q == 0) blk[kv * 128 + r] = src;
    __shared__ uint32_t red[4][4];
    if (q == 0) {
        for (int w = 0; w < words; ++w) {
            uint32_t m = 0;
            if (j < rows) {
                if (mask) m = __ldg(mask + j * words + w);
                else { int hi = kv - 32 * w; m = hi >= 32 ? 0xffffffffu : ((1u << hi) - 1u); }
            }
            m = __reduce_or_sync(0xffffffffu, m);
            if ((r & 31) == 0) red[w][r >> 5] = m;
        }
    }
    __syncthreads();
    if (threadIdx.x < words) tile_mask[t * words + threadIdx.x] = red[threadIdx.x][0] | red[threadIdx.x][1] |
                                                                  red[threadIdx.x][2] | red[threadIdx.x][3];
}

// same table from the row-major copy [rows][32] written by subm_probe_k3_kernel (kv <= 32):
// 4 threads per row, two 16-byte loads each, stores coalesced over the rows of the tile
__global__ void __launch_bounds__(128 * TT_SPLIT)
build_tile_table_rows_kernel(const int32_t *__restrict__ row_table, int kv, const int32_t *__restrict__ argsort,
                             const uint32_t *__restrict__ mask, int64_t rows, int32_t *__restrict__ table,
                             uint32_t *__restrict__ tile_mask) {
    const int64_t t = blockIdx.x;
    const int r = threadIdx.x & 127;
    const int q = threadIdx.x >> 7;
    const int64_t j = t * 128 + r;
    int32_t src = -1;
    if (j < rows) src = argsort ? __ldg(argsort + j) : (int32_t)j;
    int32_t *blk = table + t * (int64_t)(kv + 1) * 128;
    int4 v0 = make_int4(-1, -1, -1, -1), v1 = v0;
    if (src >= 0) {
        const int4 *rp = reinterpret_cast<const int4 *>(row_table + (int64_t)src * 32 + q * 8);
        v0 = __ldg(rp); v1 = __ldg(rp + 1);
    }
    const int32_t vals[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int k = q * 8 + i;
        if (k < kv) blk[k * 128 + r] = vals[i];
    }
    if (q == 0) blk[kv * 128 + r] = src;
    __shared__ uint32_t red[4];
    if (q == 0) {
        uint32_t m = 0;
        if (j < rows) m = mask ? __ldg(mask + j) : (kv >= 32 ? 0xffffffffu : ((1u << kv) - 1u));
        m = __reduce_or_sync(0xffffffffu, m);
        if ((r & 31) == 0) red[r >> 5] = m;
    }
    __syncthreads();
    if (threadIdx.x == 0) tile_mask[t] = red[0] | red[1] | red[2] | red[3];
}

// Schedule records for the dynamically scheduled kernels: tiles in order of decreasing stage count
// (= popcount of the tile mask), ties in ascending tile order (stable => deterministic).  Handing
// tiles out heaviest-first through an atomic ticket is LPT list scheduling: on the 100 k-voxel
// cloud the static round-robin assignment leaves the slowest CTA 1.6x over the mean, LPT 1.07x.
// One block; chunks of 1024 tiles are ranked with warp match_any + per-warp bucket counts.
constexpr int TO_THREADS = 1024;
constexpr int TO_BUCKETS = 130;                 // stage counts 0..128 (+1 spare)
struct ToJob { const uint32_t *tile_mask; int tiles; int32_t *rec; int32_t *state; };
struct ToJobs { ToJob j[2]; };
__global__ void __launch_bounds__(TO_THREADS)
tile_order_kernel(const ToJobs jobs, int words) {
    const ToJob &J = jobs.j[blockIdx.x];
    const uint32_t *__restrict__ tile_mask = J.tile_mask;
    const int tiles = J.tiles;
    int32_t *__restrict__ rec = J.rec;
    int32_t *__restrict__ state = J.state;
    __shared__ int bucket_base[TO_BUCKETS];
    __shared__ int wcnt[TO_THREADS / 32][TO_BUCKETS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < TT_STATE_INTS) state[tid] = 0;
    for (int i = tid; i < TO_BUCKETS; i += TO_THREADS) bucket_base[i] = 0;
    __syncthreads();
    auto load_mask = [&](int t, uint32_t (&m)[4]) {
        uint32_t any = 0;
#pragma unroll
        for (int w = 0; w < 4; ++w) { m[w] = w < words ? __ldg(tile_mask + (int64_t)t * words + w) : 0u; any |= m[w]; }
        if (!any) m[0] = 1u;                     // an empty tile still runs one (all-zero) stage
        return __popc(m[0]) + __popc(m[1]) + __popc(m[2]) + __popc(m[3]);
    };
    // bucket sizes
    for (int t = tid; t < tiles; t += TO_THREADS) {
        uint32_t m[4];
        atomicAdd(&bucket_base[load_mask(t, m)], 1);
    }
    __syncthreads();
    if (warp == 0) {                              // exclusive scan, heaviest bucket first (one warp, shuffles)
        int carry = 0;
        for (int base = TO_BUCKETS - 1; base >= 0; base -= 32) {
            const int c = base - lane;
            const int n = c >= 0 ? bucket_base[c] : 0;
            int incl = n;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int up = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += up;
            }
            if (c >= 0) bucket_base[c] = carry + incl - n;
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    __syncthreads();
    for (int t0 = 0; t0 < tiles; t0 += TO_THREADS) {
        for (int i = tid; i < (TO_THREADS / 32) * TO_BUCKETS; i += TO_THREADS) (&wcnt[0][0])[i] = 0;
        __syncthreads();
        const int t = t0 + tid;
        const bool ok = t < tiles;
        uint32_t m[4] = {0, 0, 0, 0};
        const int c = ok ? load_mask(t, m) : TO_BUCKETS - 1;
        const unsigned peers = __match_any_sync(0xffffffffu, ok ? c : -1);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (ok && rank == 0) wcnt[warp][c] = __popc(peers);
        __syncthreads();
        const int live_warps = min(TO_THREADS / 32, (tiles - t0 + 31) / 32);     // warps that hold tiles
        for (int b = tid; b < TO_BUCKETS; b += TO_THREADS) {
            int run = bucket_base[b];
            for (int w = 0; w < live_warps; ++w) { const int n = wcnt[w][b]; wcnt[w][b] = run; run += n; }
            bucket_base[b] = run;
        }
        __syncthreads();
        if (ok) {
            int32_t *r = rec + (int64_t)(wcnt[warp][c] + rank) * TT_REC_INTS;
            *reinterpret_cast<int4 *>(r) = make_int4(t, (int)m[0], (int)m[1], (int)m[2]);
            *reinterpret_cast<int4 *>(r + 4) = make_int4((int)m[3], 0, 0, 0);
        }
        __syncthreads();
    }
}

}  // namespace spx

using namespace spx;

// ====================================================================== C ABI
static int validate_geom(const spx_conv_geometry *g) {
    SPX_REQUIRE(g != nullptr, "geometry is NULL");
    SPX_REQUIRE(g->ndim >= 1 && g->ndim <= SPX_MAX_NDIM, "ndim must be in [1, %d], got %d", SPX_MAX_NDIM, g->ndim);
    SPX_REQUIRE(g->batch_size > 0, "batch_size must be positive");
    for (int a = 0; a < g->ndim; ++a) {
        SPX_REQUIRE(g->ksize[a] > 0 && g->dilation[a] > 0 && g->in_dims[a] > 0, "bad ksize/dilation/dims on axis %d", a);
    }
    return 0;
}

// a regular (not SubM) conv also reads the strides and the output dims
static int validate_strides(const spx_conv_geometry *g) {
    for (int a = 0; a < g->ndim; ++a)
        SPX_REQUIRE(g->stride[a] > 0 && g->out_dims[a] > 0, "bad stride/out_dims on axis %d", a);
    return 0;
}

static int64_t kernel_volume(const spx_conv_geometry *g) {
    int64_t kv = 1;
    for (int a = 0; a < g->ndim; ++a) kv *= g->ksize[a];
    return kv;
}

struct RbLayout {   // workspace layout shared by the rulebook entry points
    size_t table_bytes, table_vals_bytes;
    uint32_t capacity;
    bool i64;
};

// `items` is exact for SubM (factor 4); for a regular conv it is the UPPER BOUND on outputs
// (typically ~7x the real count), so factor 2 already means a load factor well below 0.1
static RbLayout rb_layout(const Geom &g, int64_t items, const int *dims, int factor = 4) {
    RbLayout L;
    L.i64 = needs_i64(g, dims);
    L.capacity = table_capacity(items, factor);
    L.table_bytes = (size_t)L.capacity * 8;
    L.table_vals_bytes = L.i64 ? (size_t)L.capacity * 4 : 0;
    return L;
}

extern "C" int64_t spx_conv_max_out(const spx_conv_geometry *g, int64_t num_in) {
    // all.py:1559-1580, with the transposed case bounded by kv*N (ops.py:569-570)
    int64_t res = num_in, kv = 1;
    for (int i = 0; i < g->ndim; ++i) {
        kv *= g->ksize[i];
        if (g->ksize[i] > g->stride[i]) res *= (g->ksize[i] + g->stride[i] - 1) / g->stride[i];
    }
    if (g->transposed) res = kv * num_in;
    if (res > kv * num_in) res = kv * num_in;
    return res;
}

static bool subm_k3_path(const Geom &gg) {
    return !needs_i64(gg, gg.in_dims) && gg.ndim == 3 && gg.ksize[0] == 3 && gg.ksize[1] == 3 && gg.ksize[2] == 3;
}

// row_table: NULL, or (subm_k3_path only) [N][32] that the probe kernel fills with the rows of pair_fwd
static int subm_rulebook(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int32_t *pair_fwd,
                         int32_t *pair_bwd, uint32_t *mask, int32_t *row_table, void *workspace,
                         size_t workspace_bytes, spx_stream_t stream_) {
    if (validate_geom(g)) return 2;
    for (int a = 0; a < g->ndim; ++a)
        SPX_REQUIRE(g->ksize[a] % 2 == 1, "subm only support odd ksize");
    SPX_REQUIRE(N >= 0 && N < 2147483647ll, "bad N");
    if (N == 0) return 0;
    SPX_REQUIRE(indices && pair_fwd && workspace, "NULL pointer argument");
    SPX_REQUIRE_ALIGNED16(indices, "subm_rulebook");
    cudaStream_t stream = (cudaStream_t)stream_;
    Geom gg = make_geom(g, true);
    SPX_REQUIRE((int64_t)gg.kv * N < 2147483647ll * 4, "kv*N too large");
    RbLayout L = rb_layout(gg, N, gg.in_dims);
    WorkspaceCarver ws(workspace, workspace_bytes);
    void *tbl = ws.take<char>(L.table_bytes);
    int32_t *tvals = L.i64 ? ws.take<int32_t>(L.capacity) : nullptr;
    SPX_REQUIRE(ws.ok(), "rulebook workspace too small: need %zu, have %zu", ws.off, workspace_bytes);
    int words = (gg.kv + 31) / 32;
    const int T = 128;
    unsigned nblk = (unsigned)div_up64(N, T);
    SPX_CHECK_CUDA(cudaMemsetAsync(tbl, 0xFF, L.table_bytes, stream));
    if (L.i64) SPX_CHECK_CUDA(cudaMemsetAsync(tvals, 0x7F, (size_t)L.capacity * 4, stream));
    return visit_table(L.i64, tbl, tvals, L.capacity, [&](auto t) {
        subm_insert_kernel<<<nblk, T, 0, stream>>>(t, gg, indices, N);
        SPX_CHECK_LAUNCH("subm_insert_kernel");
        if constexpr (std::is_same_v<decltype(t), Table32>) {   // subm_k3_path implies 32-bit keys
            if (subm_k3_path(gg)) {
                subm_probe_k3_kernel<<<(unsigned)div_up64(N, K3_VOX), 27 * 32, 0, stream>>>(t, gg, indices, N, pair_fwd,
                                                                                            pair_bwd, mask, row_table);
                SPX_CHECK_LAUNCH("subm_probe_kernel");
                return 0;
            }
        }
        subm_probe_kernel<<<nblk, T, 0, stream>>>(t, gg, indices, N, pair_fwd, pair_bwd, mask, words);
        SPX_CHECK_LAUNCH("subm_probe_kernel");
        return 0;
    });
}

extern "C" int spx_subm_rulebook(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int32_t *pair_fwd,
                                 int32_t *pair_bwd, uint32_t *mask, void *workspace, size_t workspace_bytes,
                                 spx_stream_t stream) {
    return subm_rulebook(g, indices, N, pair_fwd, pair_bwd, mask, nullptr, workspace, workspace_bytes, stream);
}


namespace {
struct ConvWs {
    void *tbl; int32_t *tvals;
    uint32_t *slot;                             // table slots of the created outputs
    uint32_t *rank_bitmap; int *rank_tiles;     // first-touch ranking: bitmap over kv*N + tile counts
    size_t rank_bytes; int64_t rank_ntiles;
    int *counter;
    size_t bytes;                               // end of the carved layout
    RbLayout L;
};

// which table capacity stage 1 ended up with (the optimistic size, or the full one after an overflow);
// stage 2 is called right after stage 1 on the same thread with the same workspace
struct ConvStage1Record { const void *ws; uint32_t capacity; };
thread_local ConvStage1Record g_stage1 = {nullptr, 0};

// Optimistic table size: the bound on the outputs (spx_conv_max_out, e.g. 8 N for 3^3 stride 2) is what
// isolated points would produce; LiDAR-like clouds yield ~0.5 N.  A table for a quarter of the bound
// (load <= 0.5 if M <= bound / 4) is cleared and probed 4x cheaper; a probe chain longer than
// CONV_MAX_PROBES flags an overflow and stage 1 re-runs with the full size.
uint32_t optimistic_capacity(int64_t max_out, uint32_t full_capacity) {
    uint32_t cap = table_capacity((max_out + 3) / 4, 2);
    return cap < full_capacity ? cap : full_capacity;
}
// The one definition of the regular-conv workspace layout: spx_rulebook_workspace_size carves it
// dry (workspace NULL, bytes SIZE_MAX) and reads w.bytes.  rank_bitmap .. counter + 64 must stay
// contiguous: conv_clear_kernel zeroes that range in one pass.
int carve_conv_ws(const spx_conv_geometry *g, const Geom &gg, int64_t N, void *workspace, size_t bytes, ConvWs &w) {
    int64_t max_out = spx_conv_max_out(g, N);
    w.L = rb_layout(gg, max_out, gg.out_dims, 2);
    WorkspaceCarver ws(workspace, bytes);
    w.tbl = ws.take<char>(w.L.table_bytes);
    w.tvals = w.L.i64 ? ws.take<int32_t>(w.L.capacity) : nullptr;
    w.slot = ws.take<uint32_t>(max_out);
    w.rank_bytes = rank_scratch_bytes((int64_t)gg.kv * N, &w.rank_ntiles);
    w.rank_bitmap = (uint32_t *)ws.take<char>(w.rank_bytes);
    w.rank_tiles = (int *)(w.rank_bitmap + w.rank_ntiles * RANK_TILE_WORDS);
    w.counter = ws.take<int>(64);
    w.bytes = ws.off;
    SPX_REQUIRE(ws.ok(), "rulebook workspace too small: need %zu, have %zu", ws.off, bytes);
    return 0;
}

// which of the insert and pairs kernels a regular conv runs
struct ConvKind {
    bool fast3;   // 3-D, not transposed: each block's offset precomputed once (block_taps3)
    bool k3;      // and 3x3x3: one thread per input point walks all 27 offsets
    explicit ConvKind(const Geom &gg)
        : fast3(gg.ndim == 3 && !gg.transposed),
          k3(fast3 && gg.ksize[0] == 3 && gg.ksize[1] == 3 && gg.ksize[2] == 3) {}
    // 3x3x3 (one mask word): the pairs kernel ORs the forward masks too (zeroed by the assign kernel)
    uint32_t *mask_fwd_or(uint32_t *mask_fwd) const { return k3 ? mask_fwd : nullptr; }
};

// reset the hash table of `capacity` slots and zero the ranking scratch and counters [rank_bitmap, end),
// which the carvers keep contiguous
int clear_conv_scratch(const RbLayout &L, uint32_t capacity, void *tbl, int32_t *tvals, uint32_t *rank_bitmap,
                       const int *end, cudaStream_t stream) {
    const int64_t zero_vec = (int64_t)(((const char *)end - (const char *)rank_bitmap) / 16);
    conv_clear_kernel<<<sm_count() * 4, 256, 0, stream>>>((uint4 *)tbl, (int64_t)capacity / 2,
                                                          L.i64 ? (uint4 *)tvals : nullptr,
                                                          L.i64 ? (int64_t)capacity / 4 : 0,
                                                          (uint4 *)rank_bitmap, zero_vec);
    SPX_CHECK_LAUNCH("conv_clear_kernel");
    return 0;
}

// After the outputs are assigned: the pair tables (pair_fwd has `rows` rows, M or the bound), then the masks that
// the pairs kernel did not write.  A NULL mask is not wanted.
template <typename Table>
int conv_pairs_and_masks(Table t, const Geom &gg, ConvKind kind, const int32_t *indices, int64_t N, int64_t rows,
                         int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd, uint32_t *mask_bwd,
                         cudaStream_t stream) {
    const int T = 128, words = (gg.kv + 31) / 32;
    uint32_t *mask_fwd_or = kind.mask_fwd_or(mask_fwd);
    if (N > 0) {
        const dim3 grid((unsigned)div_up64(N, T), gg.kv);
        if (kind.k3) conv_pairs_k3_kernel<<<(unsigned)div_up64(N, T), T, 0, stream>>>(t, gg, indices, N, rows, pair_fwd, pair_bwd, mask_bwd, mask_fwd_or);
        else if (kind.fast3) conv_pairs_kernel<Table, true><<<grid, T, 0, stream>>>(t, gg, indices, N, rows, pair_fwd, pair_bwd);
        else conv_pairs_kernel<Table, false><<<grid, T, 0, stream>>>(t, gg, indices, N, rows, pair_fwd, pair_bwd);
        SPX_CHECK_LAUNCH("conv_pairs_kernel");
    }
    if (mask_fwd && !mask_fwd_or) {
        table_mask_kernel<<<(unsigned)div_up64(rows, 256), 256, 0, stream>>>(pair_fwd, rows, gg.kv, words, mask_fwd);
        SPX_CHECK_LAUNCH("table_mask_kernel");
    }
    if (mask_bwd && !kind.k3 && N > 0) {        // the 3x3x3 pairs kernel has already written it
        table_mask_kernel<<<(unsigned)div_up64(N, 256), 256, 0, stream>>>(pair_bwd, N, gg.kv, words, mask_bwd);
        SPX_CHECK_LAUNCH("table_mask_kernel");
    }
    return 0;
}
}  // namespace

extern "C" size_t spx_rulebook_workspace_size(const spx_conv_geometry *g, int64_t num_in, int64_t max_out, int is_subm) {
    if (!g || g->ndim < 1 || g->ndim > SPX_MAX_NDIM) return 0;
    Geom gg = make_geom(g, is_subm != 0);
    size_t total = 256;
    if (is_subm) {
        RbLayout L = rb_layout(gg, num_in, gg.in_dims);
        total += align_up(L.table_bytes, 256) + align_up(L.table_vals_bytes, 256);
    } else {
        (void)max_out;                           // the bound is recomputed by both stages
        ConvWs w;
        carve_conv_ws(g, gg, num_in, nullptr, SIZE_MAX, w);
        total += align_up(w.bytes, 256);
    }
    return total + 1024;
}

extern "C" int spx_conv_rulebook_stage1(const spx_conv_geometry *g, const int32_t *indices, int64_t N,
                                        int64_t *num_out_host, void *workspace, size_t workspace_bytes,
                                        spx_stream_t stream_) {
    if (validate_geom(g)) return 2;
    SPX_REQUIRE(num_out_host != nullptr, "num_out_host is NULL");
    *num_out_host = 0;
    if (N == 0) return 0;
    SPX_REQUIRE(indices && workspace, "NULL pointer argument");
    SPX_REQUIRE_ALIGNED16(indices, "conv_rulebook_stage1");
    if (validate_strides(g)) return 2;
    cudaStream_t stream = (cudaStream_t)stream_;
    Geom gg = make_geom(g, false);
    SPX_REQUIRE((int64_t)gg.kv * N < 2000000000ll, "kv*N must stay below 2e9 (kv=%d, N=%lld)", gg.kv, (long long)N);
    ConvWs w;
    if (carve_conv_ws(g, gg, N, workspace, workspace_bytes, w)) return 2;
    const dim3 grid((unsigned)div_up64(N, 128), gg.kv);
    const ConvKind kind(gg);
    g_stage1 = {workspace, w.L.capacity};
    // optimistic table, append-on-create, outputs ranked by first touch without a sort
    const int64_t max_out = spx_conv_max_out(g, N);
    int host_state[2] = {0, 0};
    uint32_t capacity = optimistic_capacity(max_out, w.L.capacity);
    for (int attempt = 0; attempt < 2; ++attempt) {
        if (int rc = clear_conv_scratch(w.L, capacity, w.tbl, w.tvals, w.rank_bitmap, w.counter + 64, stream)) return rc;
        if (int rc = visit_table(w.L.i64, w.tbl, w.tvals, capacity, [&](auto t) {
                using Table = decltype(t);
                if (kind.k3) conv_insert_k3_append_kernel<<<(unsigned)div_up64(N, APPEND_THREADS), APPEND_THREADS, 0, stream>>>(t, gg, indices, N, w.slot, w.counter);
                else if (kind.fast3) conv_insert_append_kernel<Table, true><<<grid, APPEND_THREADS, 0, stream>>>(t, gg, indices, N, w.slot, w.counter);
                else conv_insert_append_kernel<Table, false><<<grid, APPEND_THREADS, 0, stream>>>(t, gg, indices, N, w.slot, w.counter);
                SPX_CHECK_LAUNCH("conv_insert_append_kernel");
                return 0;
            })) return rc;
        SPX_CHECK_CUDA(cudaMemcpyAsync(host_state, w.counter, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        SPX_CHECK_CUDA(cudaStreamSynchronize(stream));
        if (!host_state[1]) break;
        SPX_REQUIRE(capacity < w.L.capacity, "conv rulebook: hash table overflow at full capacity (%u slots)", capacity);
        capacity = w.L.capacity;                     // rare: far more outputs than the optimistic guess
    }
    g_stage1.capacity = capacity;
    const int m_host = host_state[0];
    *num_out_host = m_host;
    if (m_host == 0) return 0;
    const unsigned mblk = (unsigned)div_up64(m_host, MARK_THREADS);
    return visit_table(w.L.i64, w.tbl, w.tvals, capacity, [&](auto t) {
        conv_mark_kernel<<<mblk, MARK_THREADS, 0, stream>>>(t, w.slot, m_host, w.rank_bitmap, w.rank_tiles, w.rank_ntiles, w.counter + 2);
        SPX_CHECK_LAUNCH("conv_mark_kernel");
        return 0;
    });
}

extern "C" int spx_conv_rulebook_stage2(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int64_t M,
                                        int32_t *out_inds, int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd,
                                        uint32_t *mask_bwd, void *workspace, size_t workspace_bytes,
                                        spx_stream_t stream_) {
    if (validate_geom(g)) return 2;
    if (N == 0 || M == 0) return 0;
    SPX_REQUIRE(indices && out_inds && pair_fwd && pair_bwd && workspace, "NULL pointer argument");
    SPX_REQUIRE_ALIGNED16(indices, "conv_rulebook_stage2");
    cudaStream_t stream = (cudaStream_t)stream_;
    Geom gg = make_geom(g, false);
    ConvWs w;
    if (carve_conv_ws(g, gg, N, workspace, workspace_bytes, w)) return 2;
    const ConvKind kind(gg);
    SPX_REQUIRE(g_stage1.ws == workspace && g_stage1.capacity != 0,
                "conv_rulebook_stage2 must follow conv_rulebook_stage1 on the same thread with the same workspace");
    return visit_table(w.L.i64, w.tbl, w.tvals, g_stage1.capacity, [&](auto t) {
        conv_assign_rank_kernel<<<(unsigned)div_up64(M, 256), 256, 0, stream>>>(t, gg, w.slot, M, w.rank_bitmap, w.rank_tiles, out_inds, kind.mask_fwd_or(mask_fwd), pair_fwd, gg.kv);
        SPX_CHECK_LAUNCH("conv_assign_rank_kernel");
        return conv_pairs_and_masks(t, gg, kind, indices, N, M, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
    });
}

extern "C" size_t spx_native_pairs_workspace_size(int64_t N, int kv) {
    int64_t nblk = div_up64(N > 0 ? N : 1, SCAN_TILE);
    return (size_t)kv * nblk * sizeof(int) + 1024;
}

extern "C" int spx_native_pairs(const int32_t *pair_bwd, int64_t N, int kv, int is_subm, int32_t *pairs,
                                int32_t *indice_pair_num, void *workspace, size_t workspace_bytes,
                                spx_stream_t stream_) {
    SPX_REQUIRE(kv > 0 && N >= 0, "bad kv / N");
    SPX_REQUIRE(pairs && indice_pair_num, "NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    SPX_CHECK_CUDA(cudaMemsetAsync(indice_pair_num, 0, sizeof(int32_t) * kv, stream));
    if (N == 0) return 0;
    SPX_REQUIRE(pair_bwd && workspace, "NULL pointer argument");
    SPX_CHECK_CUDA(cudaMemsetAsync(pairs, 0xFF, (size_t)2 * kv * N * 4, stream));
    int rows = is_subm ? kv / 2 : kv;
    int nblk = (int)div_up64(N, SCAN_TILE);
    WorkspaceCarver ws(workspace, workspace_bytes);
    int *counts = ws.take<int>((size_t)kv * nblk);
    SPX_REQUIRE(ws.ok(), "native-pairs workspace too small: need %zu, have %zu", ws.off, workspace_bytes);
    if (rows > 0) {
        dim3 grid(nblk, rows);
        native_count_kernel<<<grid, SCAN_THREADS, 0, stream>>>(pair_bwd, N, counts, nblk);
        SPX_CHECK_LAUNCH("native_count_kernel");
        native_scan_kernel<<<rows, SCAN_THREADS, 0, stream>>>(counts, nblk, indice_pair_num);
        SPX_CHECK_LAUNCH("native_scan_kernel");
        native_write_kernel<<<grid, SCAN_THREADS, 0, stream>>>(pair_bwd, N, kv, is_subm, counts, nblk, pairs);
        SPX_CHECK_LAUNCH("native_write_kernel");
    }
    if (is_subm) {
        subm_centre_kernel<<<(unsigned)div_up64(N, 256), 256, 0, stream>>>(pairs, N, kv);
        SPX_CHECK_LAUNCH("subm_centre_kernel");
    }
    return 0;
}

extern "C" int spx_pairs_to_table(const int32_t *pairs, const int32_t *indice_pair_num, int kv, int64_t pair_stride,
                                  int64_t n_in, int64_t n_out, int is_subm, int inverse, int32_t *table_fwd,
                                  int32_t *table_bwd, uint32_t *mask_fwd, uint32_t *mask_bwd, spx_stream_t stream_) {
    SPX_REQUIRE(pairs && indice_pair_num && kv > 0, "NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    int words = (kv + 31) / 32;
    if (table_fwd && n_out > 0) SPX_CHECK_CUDA(cudaMemsetAsync(table_fwd, 0xFF, (size_t)kv * n_out * 4, stream));
    if (table_bwd && n_in > 0) SPX_CHECK_CUDA(cudaMemsetAsync(table_bwd, 0xFF, (size_t)kv * n_in * 4, stream));
    if (mask_fwd && n_out > 0) SPX_CHECK_CUDA(cudaMemsetAsync(mask_fwd, 0, (size_t)n_out * words * 4, stream));
    if (mask_bwd && n_in > 0) SPX_CHECK_CUDA(cudaMemsetAsync(mask_bwd, 0, (size_t)n_in * words * 4, stream));
    int64_t span = pair_stride;
    if (span <= 0) return 0;
    dim3 grid((unsigned)div_up64(span, 256), kv);
    pairs_to_table_kernel<<<grid, 256, 0, stream>>>(pairs, indice_pair_num, kv, pair_stride, n_in, n_out, is_subm,
                                                    inverse, table_fwd, table_bwd, mask_fwd, mask_bwd, words);
    SPX_CHECK_LAUNCH("pairs_to_table_kernel");
    return 0;
}


extern "C" size_t spx_mask_argsort_workspace_size(int64_t N, int words) {
    if (N <= 0) return 256;
    if (words == 1) return radix_argsort_workspace_bytes(N);
    size_t n = (size_t)N;
    return 4 * align_up(n * 4, 256) + align_up(n * 4 * (size_t)words, 256) + align_up(cub_sort_pairs_temp_bytes(N), 256) + 1024;
}

extern "C" int spx_mask_argsort(uint32_t *mask, int32_t *argsort, int64_t N, int words, int kv, int do_sort,
                                void *workspace, size_t workspace_bytes, spx_stream_t stream_) {
    SPX_REQUIRE(words >= 1 && words <= 4, "mask words must be in [1,4], got %d", words);
    if (N == 0) return 0;
    SPX_REQUIRE(mask && argsort, "NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    unsigned nblk = (unsigned)div_up64(N, 256);
    if (!do_sort) {
        iota_kernel<<<nblk, 256, 0, stream>>>(argsort, N);
        SPX_CHECK_LAUNCH("iota_kernel");
        return 0;
    }
    SPX_REQUIRE(workspace != nullptr, "workspace is NULL");
    if (words == 1)   // hand-written 9-bit-digit stable radix argsort (sort.cu)
        return radix_argsort_pair(mask, argsort, N, nullptr, nullptr, 0, kv > 0 && kv < 32 ? kv : 32, workspace,
                                  workspace_bytes, nullptr, 0, stream);
    WorkspaceCarver ws(workspace, workspace_bytes);
    uint32_t *keys_in = ws.take<uint32_t>(N);
    uint32_t *keys_out = ws.take<uint32_t>(N);
    int32_t *perm_a = ws.take<int32_t>(N);
    int32_t *perm_b = ws.take<int32_t>(N);
    uint32_t *rows_tmp = ws.take<uint32_t>((size_t)N * words);
    size_t tmp_bytes = cub_sort_pairs_temp_bytes(N);
    void *tmp = ws.take<char>(tmp_bytes);
    SPX_REQUIRE(ws.ok(), "argsort workspace too small: need %zu, have %zu", ws.off, workspace_bytes);
    iota_kernel<<<nblk, 256, 0, stream>>>(perm_a, N);
    SPX_CHECK_LAUNCH("iota_kernel");
    // LSD over words: least significant word (last) first; stable sorts compose
    int32_t *cur = perm_a, *nxt = perm_b;
    for (int w = words - 1; w >= 0; --w) {
        gather_word_kernel<<<nblk, 256, 0, stream>>>(mask, cur, N, words, w, keys_in);
        SPX_CHECK_LAUNCH("gather_word_kernel");
        SPX_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, (const uint32_t *)keys_in, keys_out,
                                                       (const int32_t *)cur, nxt, (int)N, 0, 32, stream));
        count_launch(3);
        int32_t *t = cur; cur = nxt; nxt = t;
    }
    SPX_CHECK_CUDA(cudaMemcpyAsync(argsort, cur, (size_t)N * 4, cudaMemcpyDeviceToDevice, stream));
    gather_rows_kernel<<<nblk, 256, 0, stream>>>(mask, argsort, N, words, rows_tmp);
    SPX_CHECK_LAUNCH("gather_rows_kernel");
    SPX_CHECK_CUDA(cudaMemcpyAsync(mask, rows_tmp, (size_t)N * words * 4, cudaMemcpyDeviceToDevice, stream));
    return 0;
}

extern "C" size_t spx_tile_table_elems(int64_t rows, int kv) {
    return (size_t)tt_total_elems(div_up64(rows > 0 ? rows : 1, 128), kv);
}

// row_table: NULL, or the [rows][32] copy of `pair` (kv <= 32) written by subm_rulebook; then `pair` is not read
static int build_tile_table(const int32_t *pair, int64_t pair_stride, int kv, const int32_t *argsort,
                            const uint32_t *mask, int64_t rows, const int32_t *row_table, int32_t *table,
                            uint32_t *tile_mask, spx_stream_t stream_) {
    SPX_REQUIRE(kv >= 1 && kv <= 128, "build_tile_table: kernel volume %d not in [1,128]", kv);
    if (rows == 0) return 0;
    SPX_REQUIRE((pair || row_table) && table && tile_mask, "build_tile_table: NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    int words = (kv + 31) / 32;
    if (row_table) {
        SPX_REQUIRE(kv <= 32, "build_tile_table: row_table holds at most 32 offsets per row, kv = %d", kv);
        SPX_REQUIRE(aligned16(row_table), "build_tile_table: row_table must be 16-byte aligned");
        build_tile_table_rows_kernel<<<(unsigned)div_up64(rows, 128), 128 * TT_SPLIT, 0, stream>>>(
            row_table, kv, argsort, mask, rows, table, tile_mask);
        SPX_CHECK_LAUNCH("build_tile_table_rows_kernel");
    } else {
        TtJobs jobs;
        memset(&jobs, 0, sizeof(jobs));
        jobs.j[0] = TtJob{pair, pair_stride, argsort, mask, rows, table, tile_mask};
        build_tile_table_kernel<<<dim3((unsigned)div_up64(rows, 128), 1), 128 * TT_SPLIT, 0, stream>>>(jobs, kv, words);
        SPX_CHECK_LAUNCH("build_tile_table_kernel");
    }
    const int64_t tiles = div_up64(rows, 128);
    SPX_REQUIRE(tiles < 2147483647ll, "build_tile_table: too many tiles");
    SPX_REQUIRE(aligned16(table), "build_tile_table: table must be 16-byte aligned");
    int32_t *rec = table + tt_blocks_elems(tiles, kv);
    ToJobs oj;
    memset(&oj, 0, sizeof(oj));
    oj.j[0] = ToJob{tile_mask, (int)tiles, rec, rec + tiles * TT_REC_INTS};
    tile_order_kernel<<<1, TO_THREADS, 0, stream>>>(oj, words);
    SPX_CHECK_LAUNCH("tile_order_kernel");
    return 0;
}

extern "C" int spx_build_tile_table(const int32_t *pair, int64_t pair_stride, int kv, const int32_t *argsort,
                                    const uint32_t *mask, int64_t rows, int32_t *table, uint32_t *tile_mask,
                                    spx_stream_t stream) {
    return build_tile_table(pair, pair_stride, kv, argsort, mask, rows, nullptr, table, tile_mask, stream);
}

// forward + backward tile tables of a regular conv in one launch each (gather kernel, schedule records)
static int build_tile_tables_pair(int kv, const int32_t *pair0, const int32_t *argsort0, const uint32_t *mask0, int64_t rows0,
                                  int32_t *table0, uint32_t *tmask0, const int32_t *pair1, const int32_t *argsort1,
                                  const uint32_t *mask1, int64_t rows1, int32_t *table1, uint32_t *tmask1,
                                  cudaStream_t stream) {
    SPX_REQUIRE(kv >= 1 && kv <= 128, "build_tile_table: kernel volume %d not in [1,128]", kv);
    const int words = (kv + 31) / 32;
    const int64_t tiles0 = div_up64(rows0, 128), tiles1 = div_up64(rows1, 128);
    SPX_REQUIRE(tiles0 < 2147483647ll && tiles1 < 2147483647ll, "build_tile_table: too many tiles");
    SPX_REQUIRE(aligned16(table0) && aligned16(table1), "build_tile_table: table must be 16-byte aligned");
    TtJobs jobs;
    memset(&jobs, 0, sizeof(jobs));
    jobs.j[0] = TtJob{pair0, rows0, argsort0, mask0, rows0, table0, tmask0};
    jobs.j[1] = TtJob{pair1, rows1, argsort1, mask1, rows1, table1, tmask1};
    const int64_t tmax = tiles0 > tiles1 ? tiles0 : tiles1;
    build_tile_table_kernel<<<dim3((unsigned)tmax, 2), 128 * TT_SPLIT, 0, stream>>>(jobs, kv, words);
    SPX_CHECK_LAUNCH("build_tile_table_kernel");
    int32_t *rec0 = table0 + tt_blocks_elems(tiles0, kv), *rec1 = table1 + tt_blocks_elems(tiles1, kv);
    ToJobs oj;
    memset(&oj, 0, sizeof(oj));
    oj.j[0] = ToJob{tmask0, (int)tiles0, rec0, rec0 + tiles0 * TT_REC_INTS};
    oj.j[1] = ToJob{tmask1, (int)tiles1, rec1, rec1 + tiles1 * TT_REC_INTS};
    tile_order_kernel<<<2, TO_THREADS, 0, stream>>>(oj, words);
    SPX_CHECK_LAUNCH("tile_order_kernel");
    return 0;
}

// ====================================================================== fused host entry points
// One C-ABI call per rulebook (the eager Python path was paying ~10 us of interpreter + ctypes +
// allocator time for every separate call, workspace query and scratch tensor).  Pure orchestration of
// the kernels behind the separate entry points; scratch regions are carved from ONE caller-provided
// workspace.

// the row-major copy of pair_fwd that subm_probe_k3_kernel writes for the tile-table build
static size_t subm_row_table_bytes(const spx_conv_geometry *g, int64_t N) {
    return subm_k3_path(make_geom(g, true)) ? align_up((size_t)N * 32 * sizeof(int32_t), 256) : 0;
}

extern "C" size_t spx_subm_rulebook_all_workspace_size(const spx_conv_geometry *g, int64_t N) {
    if (!g || g->ndim < 1 || g->ndim > SPX_MAX_NDIM) return 0;
    const int kv = (int)kernel_volume(g);
    const size_t a = spx_rulebook_workspace_size(g, N, 0, 1);
    const size_t b = spx_mask_argsort_workspace_size(N, (kv + 31) / 32);
    return align_up(a > b ? a : b, 256) + subm_row_table_bytes(g, N) + 256;
}

extern "C" int spx_subm_rulebook_all(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int32_t *pair_fwd,
                                     int32_t *pair_bwd, uint32_t *mask, int32_t *argsort, int do_sort,
                                     int32_t *tile_table, uint32_t *tile_mask, void *workspace, size_t workspace_bytes,
                                     spx_stream_t stream) {
    if (validate_geom(g)) return 2;
    if (N == 0) return 0;
    SPX_REQUIRE(mask && argsort && tile_table && tile_mask && workspace, "subm_rulebook_all: NULL pointer argument");
    SPX_REQUIRE(workspace_bytes >= spx_subm_rulebook_all_workspace_size(g, N), "subm_rulebook_all: workspace too small");
    const int kv = (int)kernel_volume(g);
    const int words = (kv + 31) / 32;
    const size_t rb = spx_rulebook_workspace_size(g, N, 0, 1), as = spx_mask_argsort_workspace_size(N, words);
    const size_t shared = align_up(rb > as ? rb : as, 256);          // rulebook and sort scratch are used one after the other
    int32_t *row_table = subm_row_table_bytes(g, N) ? (int32_t *)((char *)workspace + shared) : nullptr;
    if (int rc = subm_rulebook(g, indices, N, pair_fwd, pair_bwd, mask, row_table, workspace, rb, stream)) return rc;
    if (int rc = spx_mask_argsort(mask, argsort, N, words, kv, do_sort, workspace, as, stream)) return rc;
    return build_tile_table(pair_fwd, N, kv, argsort, mask, N, row_table, tile_table, tile_mask, stream);
}

// both mask argsorts + both tile tables of a regular conv whose pair tables and masks are in place
// (M rows forward, N rows backward; the backward direction is skipped for inference)
static int conv_sort_and_tiles(int kv, int64_t N, int64_t M, int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd,
                               uint32_t *mask_bwd, int32_t *argsort_fwd, int32_t *argsort_bwd, int do_sort,
                               int32_t *table_fwd, uint32_t *tmask_fwd, int32_t *table_bwd, uint32_t *tmask_bwd,
                               void *sort_ws, size_t sort_bytes, spx_stream_t stream) {
    const int words = (kv + 31) / 32;
    const bool train = argsort_bwd != nullptr;
    if (words == 1 && do_sort && train) {
        // both mask sorts, then both tile tables, two jobs per launch
        const size_t half = (sort_bytes / 2) & ~(size_t)255;
        const int key_bits = kv < 32 ? kv : 32;
        if (int rc = radix_argsort_pair(mask_fwd, argsort_fwd, M, mask_bwd, argsort_bwd, N, key_bits, sort_ws, half,
                                        (char *)sort_ws + half, half, (cudaStream_t)stream)) return rc;
        return build_tile_tables_pair(kv, pair_fwd, argsort_fwd, mask_fwd, M, table_fwd, tmask_fwd, pair_bwd, argsort_bwd,
                                      mask_bwd, N, table_bwd, tmask_bwd, (cudaStream_t)stream);
    }
    if (int rc = spx_mask_argsort(mask_fwd, argsort_fwd, M, words, kv, do_sort, sort_ws, sort_bytes, stream)) return rc;
    if (int rc = spx_build_tile_table(pair_fwd, M, kv, argsort_fwd, mask_fwd, M, table_fwd, tmask_fwd, stream)) return rc;
    if (!train) return 0;
    if (int rc = spx_mask_argsort(mask_bwd, argsort_bwd, N, words, kv, do_sort, sort_ws, sort_bytes, stream)) return rc;
    return spx_build_tile_table(pair_bwd, N, kv, argsort_bwd, mask_bwd, N, table_bwd, tmask_bwd, stream);
}

extern "C" size_t spx_conv_rulebook_all_workspace_size(const spx_conv_geometry *g, int64_t N) {
    if (!g || g->ndim < 1 || g->ndim > SPX_MAX_NDIM) return 0;
    const int kv = (int)kernel_volume(g);
    const int64_t max_rows = spx_conv_max_out(g, N) > N ? spx_conv_max_out(g, N) : N;
    return align_up(spx_rulebook_workspace_size(g, N, 0, 0), 256) +
           2 * align_up(spx_mask_argsort_workspace_size(max_rows, (kv + 31) / 32), 256) + 256;   // two sorts side by side
}

// stage 2 + both mask argsorts + both tile tables (the backward ones are skipped for inference)
extern "C" int spx_conv_rulebook_stage2_all(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int64_t M,
                                            int32_t *out_inds, int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd,
                                            uint32_t *mask_bwd, int32_t *argsort_fwd, int32_t *argsort_bwd, int do_sort,
                                            int32_t *table_fwd, uint32_t *tmask_fwd, int32_t *table_bwd,
                                            uint32_t *tmask_bwd, void *workspace, size_t workspace_bytes,
                                            spx_stream_t stream) {
    if (validate_geom(g)) return 2;
    if (N == 0 || M == 0) return 0;
    SPX_REQUIRE(mask_fwd && mask_bwd && argsort_fwd && table_fwd && tmask_fwd && workspace,
                "conv_rulebook_stage2_all: NULL pointer argument");
    const bool train = argsort_bwd != nullptr;
    SPX_REQUIRE((table_bwd != nullptr) == train && (tmask_bwd != nullptr) == train,
                "conv_rulebook_stage2_all: argsort_bwd, table_bwd and tmask_bwd must all be given (training) or all be "
                "NULL (inference)");
    SPX_REQUIRE(workspace_bytes >= spx_conv_rulebook_all_workspace_size(g, N), "conv_rulebook_stage2_all: workspace too small");
    const int kv = (int)kernel_volume(g);
    const size_t rb = spx_rulebook_workspace_size(g, N, 0, 0);
    void *sort_ws = (char *)workspace + align_up(rb, 256);
    const size_t sort_bytes = workspace_bytes - align_up(rb, 256);
    if (int rc = spx_conv_rulebook_stage2(g, indices, N, M, out_inds, pair_fwd, pair_bwd, mask_fwd, mask_bwd, workspace, rb, stream)) return rc;
    return conv_sort_and_tiles(kv, N, M, pair_fwd, pair_bwd, mask_fwd, mask_bwd, argsort_fwd, argsort_bwd, do_sort,
                               table_fwd, tmask_fwd, table_bwd, tmask_bwd, sort_ws, sort_bytes, stream);
}

// ====================================================================== bounded regular-conv rulebook
namespace {
struct BoundedWs {
    void *tbl; int32_t *tvals;
    uint32_t *rank_bitmap; int *rank_tiles; int64_t rank_ntiles;
    int *state;
    void *sort_ws; size_t sort_bytes;
    int32_t *pair_scratch;
    size_t bytes;
    RbLayout L;
};

// rank_bitmap .. state + 64 stay contiguous: conv_clear_kernel zeroes that range in one pass.
// The table is sized from the bound alone (load <= 0.5 with `bound` outputs): there is no second attempt.
// `sorts`: the conv rulebook's two mask-sort scratch areas; without them (the sparse_add union) a
// pair_fwd [bound] that the kernels write and nobody reads takes their place.
void carve_bounded_ws(const Geom &gg, int64_t N, int64_t bound, bool sorts, void *workspace, size_t bytes, BoundedWs &w) {
    w.L = rb_layout(gg, bound, gg.out_dims, 2);
    WorkspaceCarver ws(workspace, bytes);
    w.tbl = ws.take<char>(w.L.table_bytes);
    w.tvals = w.L.i64 ? ws.take<int32_t>(w.L.capacity) : nullptr;
    const size_t rank_bytes = rank_scratch_bytes((int64_t)gg.kv * N, &w.rank_ntiles);
    w.rank_bitmap = (uint32_t *)ws.take<char>(rank_bytes);
    w.rank_tiles = (int *)(w.rank_bitmap + w.rank_ntiles * RANK_TILE_WORDS);
    w.state = ws.take<int>(64);
    const int64_t max_rows = bound > N ? bound : N;
    w.sort_bytes = sorts ? 2 * align_up(spx_mask_argsort_workspace_size(max_rows, (gg.kv + 31) / 32), 256) : 0;
    w.sort_ws = sorts ? ws.take<char>(w.sort_bytes) : nullptr;     // two sorts side by side
    w.pair_scratch = sorts ? nullptr : ws.take<int32_t>((size_t)bound);
    w.bytes = ws.off;
}

// clear the table, the ranking scratch and the state, then insert, rank, assign and pair on the table
int run_bounded(const Geom &gg, const BoundedWs &w, const int32_t *indices, int64_t N, int64_t bound, int32_t *out_inds,
                int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd, uint32_t *mask_bwd, int32_t *num_out,
                int32_t *status, cudaStream_t stream) {
    if (int rc = clear_conv_scratch(w.L, w.L.capacity, w.tbl, w.tvals, w.rank_bitmap, w.state + 64, stream)) return rc;
    const ConvKind kind(gg);
    const int64_t capacity = w.L.capacity;
    return visit_table(w.L.i64, w.tbl, w.tvals, w.L.capacity, [&](auto t) {
        using Table = decltype(t);
        if (N > 0) {
            const dim3 grid((unsigned)div_up64(N, 128), gg.kv);
            if (kind.k3) conv_insert_k3_bounded_kernel<<<(unsigned)div_up64(N, APPEND_THREADS), APPEND_THREADS, 0, stream>>>(t, gg, indices, N, w.state);
            else if (kind.fast3) conv_insert_bounded_kernel<Table, true><<<grid, APPEND_THREADS, 0, stream>>>(t, gg, indices, N, w.state);
            else conv_insert_bounded_kernel<Table, false><<<grid, APPEND_THREADS, 0, stream>>>(t, gg, indices, N, w.state);
            SPX_CHECK_LAUNCH("conv_insert_bounded_kernel");
        }
        conv_mark_table_kernel<<<(unsigned)div_up64(capacity, MARK_THREADS), MARK_THREADS, 0, stream>>>(
            t, capacity, w.rank_bitmap, w.rank_tiles, w.rank_ntiles, w.state);
        SPX_CHECK_LAUNCH("conv_mark_table_kernel");
        const int64_t span = capacity > bound ? capacity : bound;
        conv_assign_table_kernel<<<(unsigned)div_up64(span, 256), 256, 0, stream>>>(
            t, gg, capacity, bound, w.rank_bitmap, w.rank_tiles, w.state, out_inds, kind.mask_fwd_or(mask_fwd), pair_fwd,
            gg.kv, num_out, status);
        SPX_CHECK_LAUNCH("conv_assign_table_kernel");
        return conv_pairs_and_masks(t, gg, kind, indices, N, bound, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
    });
}

int validate_bounded(const spx_conv_geometry *g, int64_t N, int64_t bound) {
    if (validate_geom(g) || validate_strides(g)) return 2;
    SPX_REQUIRE(bound > 0 && bound < (1ll << 30), "bound must be in [1, 2^30), got %lld", (long long)bound);
    SPX_REQUIRE(N >= 0, "bad N");
    const int64_t kv = kernel_volume(g);
    SPX_REQUIRE(kv <= 128, "conv_rulebook_bounded: kernel volume %lld not in [1,128]", (long long)kv);
    SPX_REQUIRE(kv * N < 2000000000ll, "kv*N must stay below 2e9 (kv=%lld, N=%lld)", (long long)kv, (long long)N);
    return 0;
}
}  // namespace

extern "C" size_t spx_conv_rulebook_bounded_workspace_size(const spx_conv_geometry *g, int64_t N, int64_t bound) {
    if (!g || g->ndim < 1 || g->ndim > SPX_MAX_NDIM || N < 0 || bound <= 0 || bound >= (1ll << 30)) return 0;
    BoundedWs w;
    carve_bounded_ws(make_geom(g, false), N, bound, true, nullptr, SIZE_MAX, w);
    return align_up(w.bytes, 256) + 256;
}

extern "C" int spx_conv_rulebook_bounded_all(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int64_t bound,
                                             int32_t *out_inds, int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd,
                                             uint32_t *mask_bwd, int32_t *argsort_fwd, int32_t *argsort_bwd, int do_sort,
                                             int32_t *table_fwd, uint32_t *tmask_fwd, int32_t *table_bwd,
                                             uint32_t *tmask_bwd, int32_t *num_out, int32_t *status, void *workspace,
                                             size_t workspace_bytes, spx_stream_t stream_) {
    if (validate_bounded(g, N, bound)) return 2;
    SPX_REQUIRE(out_inds && pair_fwd && mask_fwd && argsort_fwd && table_fwd && tmask_fwd && num_out && status && workspace,
                "conv_rulebook_bounded_all: NULL pointer argument");
    SPX_REQUIRE(N == 0 || (indices && pair_bwd && mask_bwd), "conv_rulebook_bounded_all: NULL pointer argument");
    SPX_REQUIRE_ALIGNED16(indices, "conv_rulebook_bounded_all");
    const bool train = argsort_bwd != nullptr;
    SPX_REQUIRE((table_bwd != nullptr) == train && (tmask_bwd != nullptr) == train,
                "conv_rulebook_bounded_all: argsort_bwd, table_bwd and tmask_bwd must all be given (training) or all be "
                "NULL (inference)");
    const size_t need = spx_conv_rulebook_bounded_workspace_size(g, N, bound);
    SPX_REQUIRE(workspace_bytes >= need, "conv_rulebook_bounded_all: workspace too small: need %zu, have %zu", need,
                workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    const Geom gg = make_geom(g, false);
    BoundedWs w;
    carve_bounded_ws(gg, N, bound, true, workspace, workspace_bytes, w);
    if (int rc = run_bounded(gg, w, indices, N, bound, out_inds, pair_fwd, pair_bwd, mask_fwd, mask_bwd, num_out, status,
                             stream)) return rc;
    return conv_sort_and_tiles(gg.kv, N, bound, pair_fwd, pair_bwd, mask_fwd, mask_bwd, argsort_fwd, argsort_bwd, do_sort,
                               table_fwd, tmask_fwd, table_bwd, tmask_bwd, w.sort_ws, w.sort_bytes, stream_);
}

// ---- the union of sparse_add: the bounded rulebook of a 1x..x1, stride-1, padding-0 convolution, without its masks,
// mask sorts and tile tables (the union reads out_inds, dst = pair_bwd[0] and the count only)
int spx::validate_sparse_add_union(const spx_conv_geometry *g, int64_t N, int64_t bound) {
    if (validate_geom(g)) return 2;
    for (int a = 0; a < g->ndim; ++a)
        SPX_REQUIRE(g->ksize[a] == 1 && g->stride[a] == 1 && g->padding[a] == 0 && g->dilation[a] == 1 &&
                    g->out_dims[a] == g->in_dims[a] && !g->transposed,
                    "sparse_add_union: the geometry must be 1x..x1, stride 1, padding 0, out_dims = in_dims (axis %d)", a);
    SPX_REQUIRE(N > 0 && N < 2147483647ll, "sparse_add_union: bad row count %lld", (long long)N);
    SPX_REQUIRE(bound > 0 && bound <= N && bound < (1ll << 30), "sparse_add_union: bound must be in [1, min(rows, 2^30)), "
                "got %lld for %lld rows", (long long)bound, (long long)N);
    return 0;
}

extern "C" size_t spx_sparse_add_union_workspace_size(const spx_conv_geometry *g, int64_t N, int64_t bound) {
    if (!g || g->ndim < 1 || g->ndim > SPX_MAX_NDIM || N <= 0 || bound <= 0 || bound > N || bound >= (1ll << 30)) return 0;
    BoundedWs w;
    carve_bounded_ws(make_geom(g, false), N, bound, false, nullptr, SIZE_MAX, w);
    return align_up(w.bytes, 256) + 256;
}

extern "C" int spx_sparse_add_union(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int64_t bound,
                                    int32_t *out_inds, int32_t *dst, int32_t *num_out, int32_t *status, void *workspace,
                                    size_t workspace_bytes, spx_stream_t stream) {
    if (validate_sparse_add_union(g, N, bound)) return 2;
    SPX_REQUIRE(indices && out_inds && dst && num_out && status && workspace, "sparse_add_union: NULL pointer argument");
    SPX_REQUIRE_ALIGNED16(indices, "sparse_add_union");
    const size_t need = spx_sparse_add_union_workspace_size(g, N, bound);
    SPX_REQUIRE(workspace_bytes >= need, "sparse_add_union: workspace too small: need %zu, have %zu", need, workspace_bytes);
    const Geom gg = make_geom(g, false);
    BoundedWs w;
    carve_bounded_ws(gg, N, bound, false, workspace, workspace_bytes, w);
    return run_bounded(gg, w, indices, N, bound, out_inds, w.pair_scratch, dst, nullptr, nullptr, num_out, status,
                       (cudaStream_t)stream);
}

extern "C" int spx_zero_rows_from_count(void *ptr, int64_t rows, int64_t row_bytes, const int32_t *count,
                                        spx_stream_t stream_) {
    SPX_REQUIRE(rows >= 0 && row_bytes > 0 && row_bytes % 2 == 0, "zero_rows_from_count: bad rows / row_bytes");
    if (rows == 0) return 0;
    SPX_REQUIRE(ptr && count, "zero_rows_from_count: NULL pointer argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    const unsigned blocks = (unsigned)sm_count() * 4;
    if (row_bytes % 16 == 0 && aligned16(ptr))
        zero_rows_from_count_kernel<<<blocks, 256, 0, stream>>>((uint4 *)ptr, rows, row_bytes / 16, count);
    else
        zero_rows_from_count_kernel<<<blocks, 256, 0, stream>>>((uint16_t *)ptr, rows, row_bytes / 2, count);
    SPX_CHECK_LAUNCH("zero_rows_from_count_kernel");
    return 0;
}

// ====================================================================== rulebook onto given output coordinates
namespace {
// Both tables use 64-bit keys when either grid needs them.  The capacities are powers of two >= 1024, so the two key
// arrays are contiguous, and so are the two value arrays.  The mask sorts run after the probe, so their scratch shares
// the workspace with the hash tables.
struct CrossWs {
    void *src_tbl, *dst_tbl;
    int32_t *src_vals, *dst_vals;
    uint32_t src_cap, dst_cap;
    bool i64;
    size_t table_bytes, sort_bytes;
};

void carve_cross_ws(const Geom &gg, int64_t N, int64_t M, void *workspace, size_t bytes, CrossWs &w) {
    w.i64 = needs_i64(gg, gg.in_dims) || needs_i64(gg, gg.out_dims);
    w.src_cap = table_capacity(N);
    w.dst_cap = table_capacity(M);
    WorkspaceCarver ws(workspace, bytes);
    w.src_tbl = ws.take<unsigned long long>(w.src_cap);
    w.dst_tbl = ws.take<unsigned long long>(w.dst_cap);
    w.src_vals = w.i64 ? ws.take<int32_t>(w.src_cap) : nullptr;
    w.dst_vals = w.i64 ? ws.take<int32_t>(w.dst_cap) : nullptr;
    w.table_bytes = ws.off;
    w.sort_bytes = 2 * align_up(spx_mask_argsort_workspace_size(N > M ? N : M, (gg.kv + 31) / 32), 256);
}

int validate_cross(const spx_conv_geometry *g, int64_t N, int64_t M) {
    if (validate_geom(g) || validate_strides(g)) return 2;
    const int64_t kv = kernel_volume(g);
    SPX_REQUIRE(kv <= 128, "cross_rulebook_all: kernel volume %lld not in [1,128]", (long long)kv);
    for (int a = 0; a < g->ndim; ++a) {
        const int64_t dims = g->in_dims[a] > g->out_dims[a] ? g->in_dims[a] : g->out_dims[a];
        SPX_REQUIRE(g->padding[a] >= 0 && dims * g->stride[a] + g->padding[a] +
                                              (int64_t)(g->ksize[a] - 1) * g->dilation[a] < 2147483647ll,
                    "cross_rulebook_all: padding must be >= 0 and the coordinates of axis %d must stay below 2^31 "
                    "- 1", a);
    }
    SPX_REQUIRE(N >= 0 && N < 2147483647ll && M >= 0 && M < 2147483647ll,
                "cross_rulebook_all: bad row counts (%lld source, %lld target)", (long long)N, (long long)M);
    return 0;
}

template <typename Table, int NDIM>
int cross_launch(const Table &src_table, const Table &dst_table, const Geom &gg, const int32_t *indices, int64_t N,
                 const int32_t *num_valid, const int32_t *out_indices, int64_t M, const int32_t *out_num_valid,
                 int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd, uint32_t *mask_bwd, cudaStream_t stream) {
    cross_insert_kernel<Table, NDIM><<<(unsigned)div_up64(N + M, CROSS_THREADS), CROSS_THREADS, 0, stream>>>(
        src_table, dst_table, gg, indices, N, num_valid, out_indices, M, out_num_valid);
    SPX_CHECK_LAUNCH("cross_insert_kernel");
    const unsigned blk = (unsigned)div_up64(M, CROSS_THREADS);
    const int words = (gg.kv + 31) / 32;
    if (gg.transposed)
        cross_probe_kernel<Table, NDIM, true><<<blk, CROSS_THREADS, 0, stream>>>(
            src_table, dst_table, gg, out_indices, M, out_num_valid, N, pair_fwd, pair_bwd, mask_fwd, mask_bwd, words);
    else
        cross_probe_kernel<Table, NDIM, false><<<blk, CROSS_THREADS, 0, stream>>>(
            src_table, dst_table, gg, out_indices, M, out_num_valid, N, pair_fwd, pair_bwd, mask_fwd, mask_bwd, words);
    SPX_CHECK_LAUNCH("cross_probe_kernel");
    return 0;
}

template <typename Table>
int cross_tables(const Table &src_table, const Table &dst_table, const Geom &gg, const int32_t *indices, int64_t N,
                 const int32_t *num_valid, const int32_t *out_indices, int64_t M, const int32_t *out_num_valid,
                 int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask_fwd, uint32_t *mask_bwd, cudaStream_t stream) {
    switch (gg.ndim) {
        case 1: return cross_launch<Table, 1>(src_table, dst_table, gg, indices, N, num_valid, out_indices, M,
                                              out_num_valid, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
        case 2: return cross_launch<Table, 2>(src_table, dst_table, gg, indices, N, num_valid, out_indices, M,
                                              out_num_valid, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
        case 3: return cross_launch<Table, 3>(src_table, dst_table, gg, indices, N, num_valid, out_indices, M,
                                              out_num_valid, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
        default: return cross_launch<Table, 4>(src_table, dst_table, gg, indices, N, num_valid, out_indices, M,
                                               out_num_valid, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
    }
}
}  // namespace

extern "C" size_t spx_cross_rulebook_all_workspace_size(const spx_conv_geometry *g, int64_t N, int64_t M) {
    if (!g || g->ndim < 1 || g->ndim > SPX_MAX_NDIM || N < 0 || M < 0) return 0;
    CrossWs w;
    carve_cross_ws(make_geom(g, false), N, M, nullptr, SIZE_MAX, w);
    return align_up(w.table_bytes > w.sort_bytes ? w.table_bytes : w.sort_bytes, 256) + 256;
}

extern "C" int spx_cross_rulebook_all(const spx_conv_geometry *g, const int32_t *src_indices, int64_t N,
                                      const int32_t *num_valid, const int32_t *out_indices, int64_t M,
                                      const int32_t *out_num_valid, int32_t *pair_fwd, int32_t *pair_bwd,
                                      uint32_t *mask_fwd, uint32_t *mask_bwd, int32_t *argsort_fwd,
                                      int32_t *argsort_bwd, int do_sort, int32_t *table_fwd, uint32_t *tmask_fwd,
                                      int32_t *table_bwd, uint32_t *tmask_bwd, void *workspace,
                                      size_t workspace_bytes, spx_stream_t stream_) {
    if (validate_cross(g, N, M)) return 2;
    SPX_REQUIRE(workspace, "cross_rulebook_all: NULL pointer argument (workspace)");
    SPX_REQUIRE(M == 0 || (out_indices && pair_fwd && mask_fwd && argsort_fwd && table_fwd && tmask_fwd),
                "cross_rulebook_all: NULL pointer argument (out_indices, pair_fwd, mask_fwd, argsort_fwd, table_fwd, "
                "tmask_fwd)");
    SPX_REQUIRE(N == 0 || (src_indices && pair_bwd && mask_bwd),
                "cross_rulebook_all: NULL pointer argument (src_indices, pair_bwd, mask_bwd)");
    const bool train = argsort_bwd != nullptr;
    SPX_REQUIRE(N == 0 || ((table_bwd != nullptr) == train && (tmask_bwd != nullptr) == train),
                "cross_rulebook_all: argsort_bwd, table_bwd and tmask_bwd must all be given (training) or all be "
                "NULL (inference)");
    if (N > 0) SPX_REQUIRE_ALIGNED16(src_indices, "cross_rulebook_all");
    if (M > 0) SPX_REQUIRE_ALIGNED16(out_indices, "cross_rulebook_all");
    const size_t need = spx_cross_rulebook_all_workspace_size(g, N, M);
    SPX_REQUIRE(workspace_bytes >= need, "cross_rulebook_all: workspace too small: need %zu, have %zu", need,
                workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    const Geom gg = make_geom(g, false);
    const int kv = gg.kv, words = (kv + 31) / 32;
    CrossWs w;
    carve_cross_ws(gg, N, M, workspace, workspace_bytes, w);
    if (N > 0) {                                  // the probe scatters into the backward direction
        SPX_CHECK_CUDA(cudaMemsetAsync(pair_bwd, 0xFF, (size_t)kv * N * 4, stream));
        SPX_CHECK_CUDA(cudaMemsetAsync(mask_bwd, 0, (size_t)N * words * 4, stream));
    }
    if (M > 0) {
        const size_t slots = (size_t)w.src_cap + w.dst_cap;      // each pair of arrays is contiguous
        SPX_CHECK_CUDA(cudaMemsetAsync(w.src_tbl, 0xFF, slots * 8, stream));
        if (w.i64) SPX_CHECK_CUDA(cudaMemsetAsync(w.src_vals, 0x7F, slots * 4, stream));
        int rc;
        if (w.i64)
            rc = cross_tables(Table64{(long long *)w.src_tbl, w.src_vals, w.src_cap - 1},
                              Table64{(long long *)w.dst_tbl, w.dst_vals, w.dst_cap - 1}, gg, src_indices, N, num_valid,
                              out_indices, M, out_num_valid, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
        else
            rc = cross_tables(Table32{(unsigned long long *)w.src_tbl, w.src_cap - 1},
                              Table32{(unsigned long long *)w.dst_tbl, w.dst_cap - 1}, gg, src_indices, N, num_valid,
                              out_indices, M, out_num_valid, pair_fwd, pair_bwd, mask_fwd, mask_bwd, stream);
        if (rc) return rc;
    }
    if (M > 0 && N > 0)
        return conv_sort_and_tiles(kv, N, M, pair_fwd, pair_bwd, mask_fwd, mask_bwd, argsort_fwd, argsort_bwd, do_sort,
                                   table_fwd, tmask_fwd, table_bwd, tmask_bwd, workspace, w.sort_bytes, stream_);
    // one side empty: the other side's sort and tile table alone
    if (M > 0) {
        if (int rc = spx_mask_argsort(mask_fwd, argsort_fwd, M, words, kv, do_sort, workspace, w.sort_bytes, stream_))
            return rc;
        return spx_build_tile_table(pair_fwd, M, kv, argsort_fwd, mask_fwd, M, table_fwd, tmask_fwd, stream_);
    }
    if (N > 0 && train) {
        if (int rc = spx_mask_argsort(mask_bwd, argsort_bwd, N, words, kv, do_sort, workspace, w.sort_bytes, stream_))
            return rc;
        return spx_build_tile_table(pair_bwd, N, kv, argsort_bwd, mask_bwd, N, table_bwd, tmask_bwd, stream_);
    }
    return 0;
}
