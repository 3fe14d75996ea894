// wgmma weight gradient:  dW[:, k, :] = sum_o dout[o, :]^T x[pair_fwd[k][o], :].
//
// GEMM view per 128-voxel tile:  D_g[128 x c_out] += A_g[128 x 128 voxels] * B[c_out x 128 voxels]^T
//   * the contraction runs over VOXELS; for 16-bit types both operands are MN-major wgmma
//     operands built from the very same "rows of channels" shared-memory image the forward pass
//     uses (a gathered row of C channels is one K-slice of an MN-major tile).  tf32 wgmma reads
//     K-major operands only, so the fp32 producers transpose while they gather (register loads,
//     4-byte shared stores) instead of copying rows with cp.async;
//   * A_g stacks as many kernel offsets as fit M = 128 (two offsets for C_in = 64 fp16),
//     B is the dout tile, loaded once per voxel tile and shared by all offsets;
//   * the fp32 accumulators of G groups stay resident in the registers of two consumer
//     warpgroups (64 rows each) for ALL tiles a CTA visits (G * c_out = 256 columns); the groups
//     that do not fit are handled by further "pass" CTA columns (gridDim.y), so the filter
//     gradient is never spilled;
//   * each CTA finally stores its accumulators to an fp32 partial buffer and a small second
//     kernel sums the partials in a fixed order (deterministic; the reference's split-K does the
//     same with fp32 workspaces, spconv/csrc/sparse/convops.py:1236-1243, :2421-2436).
// Roles: warps 0-7 consumers (wgmma + final store), 8-9 gather producers (16-byte cp.async, 64
// tile rows per warp), 10 tile feeder (index-block ring + per-tile group sets), 11 idle.  Tiles
// are assigned STATICALLY so the summation order of dW -- and with it the result -- is
// reproducible bit for bit, but not round-robin: the schedule records list the tiles by
// decreasing offset count, and CTA c takes records c, 2C-1-c, 2C+c, 4C-1-c, ... (a snake over
// rows of C = chunks records).  Every CTA then holds one tile of every cost rank, which is LPT
// list scheduling without a run-time counter.
#include "gemm.cuh"
#include "peer.cuh"
#include "wgmma.cuh"
#include <stdlib.h>

namespace spx {

constexpr int WG_TILE = 128;
constexpr int WG_CONS_WARPS = 8;        // two consumer warpgroups, M rows 0-63 / 64-127 of every group
constexpr int WG_PROD_WARPS = 2;        // 64 tile rows per producer warp
constexpr int WG_PROD_THREADS = WG_PROD_WARPS * 32;
constexpr int WG_SCHED_WARP = WG_CONS_WARPS + WG_PROD_WARPS;
constexpr int WG_THREADS = 3 * 128;     // warps 0-7 consumers | 8-9 producers | 10 tile feeder | 11 idle
constexpr int WG_ACC_COLS = 256;        // accumulator columns per consumer row: G groups x c_out (128 registers)
constexpr int WG_MAX_STAGES = 6;
constexpr int WG_SMEM_BUDGET = 200 * 1024;    // operand stages are sized inside this ...
constexpr int WG_SMEM_MAX = 224 * 1024;       // ... what is left up to here buys deeper index prefetch
constexpr int WG_MAX_IDX = 4;                 // index-block ring depth (prefetch distance = depth - 1 tiles)
constexpr int WG_MAX_B = 3;                   // dout tile buffers

struct WgParams {
    const uint8_t *x; int xb, span_x, lg_span_x, apo, apg, atom_elems;
    const uint8_t *d; int db, span_d, lg_span_d, lg_cpr_d;
    int n, ab_bf16;
    int groups_total, groups_per_pass;
    int stages, a_stage_bytes, b_buf_bytes, b_bufs, idx_bytes, idx_bufs;
    int64_t rows;
    const int32_t *tile_table;   // [tiles][kv+1][128]
    const uint32_t *tile_mask;   // [tiles][words]
    const int32_t *sched_rec;    // [tiles][TT_REC_INTS] {tile, mask[4]}: tiles by decreasing offset count (gemm.cuh)
    int kv, words, c_in;
    float *partial; int64_t partial_stride;
    int ldx, ldd;                // grouped instances: bytes between gathered x rows / dout rows (full rows)
};

// Atoms are stacked in natural offset order: atom a holds channels (a % apo) of offset a / apo, and a
// group (one M = 128 accumulator) covers atoms [g apg, (g + 1) apg) -- offsets k, k + 1 for 64
// 16-bit channels; atoms past kv apo in the last group are padding.  Pairing k with its point
// mirror kv-1-k was tried: on tilted surface patches the two are rarely active together (the
// dz = +-1 groups of config 2 had both halves active in 1-23 of their 48-270 active tiles), and 37 %
// of its warpgroup-atom wgmma multiplied zero fill; natural pairs cut the stages from 5543 to 4761
// (tools/wgrad_schedule_model.py).

// bit gl: the atoms of local group gl that warpgroup 0 reads (M rows 0-63) hold an offset active in
// the tile; bit 16 + gl: the same for warpgroup 1 (rows 64-127).  gmask = [16][2 halves][4 words].
__device__ __forceinline__ uint32_t active_halves(const uint32_t (&tm)[4], const uint32_t *gmask, int ng, int words) {
    uint32_t act = 0;
    if (words == 1) {                                   // kv <= 32: the common 3x3x3 case
        for (int gl = 0; gl < ng; ++gl) {
            act |= (tm[0] & gmask[gl * 8]) ? 1u << gl : 0u;
            act |= (tm[0] & gmask[gl * 8 + 4]) ? 0x10000u << gl : 0u;
        }
        return act;
    }
    for (int gl = 0; gl < ng; ++gl)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t *m = gmask + gl * 8 + h * 4;
            if ((tm[0] & m[0]) | (tm[1] & m[1]) | (tm[2] & m[2]) | (tm[3] & m[3])) act |= 1u << (16 * h + gl);
        }
    return act;
}

// mask bits of offsets k_lo..k_hi.  The offsets of half a group are an aligned run of 1, 2 or 4
// offsets (apg / apo is a power of two), so they never straddle a mask word.
__device__ __forceinline__ uint32_t offset_run_bits(int k_lo, int k_hi) {
    return (2u << (k_hi & 31)) - (1u << (k_lo & 31));
}

// record visited by CTA `chunk` at step i (snake order over the cost-sorted schedule records)
__device__ __forceinline__ int64_t wg_rec_index(int64_t i, int chunk, int chunks) {
    return i * chunks + ((i & 1) ? (chunks - 1 - chunk) : chunk);
}
__device__ __forceinline__ void wg_load_rec(const int32_t *__restrict__ rec, int64_t r, int64_t &tile, uint32_t (&m)[4]) {
    const int4 a = __ldg(reinterpret_cast<const int4 *>(rec + r * TT_REC_INTS));
    const int b = __ldg(rec + r * TT_REC_INTS + 4);
    tile = a.x; m[0] = (uint32_t)a.y; m[1] = (uint32_t)a.z; m[2] = (uint32_t)a.w; m[3] = (uint32_t)b;
}

__device__ __forceinline__ uint32_t pick_word(const uint32_t (&m)[4], int w) {
    return w == 0 ? m[0] : (w == 1 ? m[1] : (w == 2 ? m[2] : m[3]));     // selects, no local-memory indexing
}

// tf32: element (row, voxel) of a K-major operand with `rows` rows and 128 voxels, cut into
// four 32-voxel (128-byte) SWIZZLE_128B sub-tiles
__device__ __forceinline__ uint32_t kmajor_tf32_off(uint32_t row, uint32_t voxel, uint32_t rows) {
    return (voxel >> 5) * rows * 128u + swizzle_offset(row * 128u + ((voxel & 31u) << 2), 128u);
}
__device__ __forceinline__ void st_shared_f32x4_t(uint32_t base, uint32_t row0, uint32_t voxel, uint32_t rows, float4 v) {
    const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int t = 0; t < 4; ++t)
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + kmajor_tf32_off(row0 + t, voxel, rows)), "f"(f[t]) : "memory");
}

// CPA = 16-byte chunks per x-atom row (span_x / 16), CPD = 16-byte chunks per dout row (db / 16)
template <int CPA, int CPD, bool TF32 = false>
__global__ void __launch_bounds__(WG_THREADS, 1)
tc_wgrad_kernel(const WgParams p) {
    constexpr bool GROUPED = false;
#include "tc_wgrad_body.cuh"
}

template <int CPA, int CPD>
__global__ void __launch_bounds__(WG_THREADS, 1)
tc_grouped_wgrad_kernel(const WgParams p) {
    constexpr bool TF32 = false, GROUPED = true;
#include "tc_wgrad_body.cuh"
}

// 4 outputs per thread (float4 partial reads), the chunk range split over the 8 warps of a block,
// partial sums combined through shared memory in warp order (fixed order => deterministic)
constexpr int RED_WARPS = 8;
template <typename T>
__global__ void __launch_bounds__(RED_WARPS * 32)
wgrad_reduce_kernel(const float *__restrict__ partial, int64_t stride, int chunks, int64_t total,
                    T *__restrict__ dw) {
    __shared__ float4 acc_s[RED_WARPS][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = ((int64_t)blockIdx.x * 32 + lane) * 4;      // total % 4 == 0 (channels % 16 == 0)
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < total) {
        const int per = (chunks + RED_WARPS - 1) / RED_WARPS;
        const int c0 = warp * per, c1 = min(chunks, c0 + per);
#pragma unroll 4
        for (int c = c0; c < c1; ++c) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(partial + (int64_t)c * stride + i));
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
    }
    acc_s[warp][lane] = s;
    __syncthreads();
    if (warp == 0 && i < total) {
        float4 t = acc_s[0][lane];
#pragma unroll
        for (int w = 1; w < RED_WARPS; ++w) {
            const float4 v = acc_s[w][lane];
            t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
        }
        dw[i] = from_float<T>(t.x); dw[i + 1] = from_float<T>(t.y);
        dw[i + 2] = from_float<T>(t.z); dw[i + 3] = from_float<T>(t.w);
    }
}

// ------------------------------------------------------------------ host side
static bool wg_span_ok(int bytes) { return bytes == 32 || bytes == 64 || (bytes >= 128 && bytes % 128 == 0); }

struct WgPlan { WgParams p; int passes, chunks; size_t smem; };

static bool make_plan(const WgradArgs &a, WgPlan &pl) {
    if (a.dtype != SPX_F16 && a.dtype != SPX_BF16 && a.dtype != SPX_F32) return false;
    if (!a.tile_table || !a.tile_mask) return false;                 // built by spx_build_tile_table
    if (!aligned16(a.x) || !aligned16(a.dout)) return false;         // 16-byte cp.async / float4 row gathers
    const bool tf32 = a.dtype == SPX_F32;       // fp32 reaches here only in TF32 mode (api_gemm.cu)
    const int e = tf32 ? 4 : 2;
    if (a.c_in % 16 || a.c_out % 16 || a.c_in > 256 || a.c_out > 256) return false;
    // tf32: whole 128-byte atoms of 32 channels on both operands, dout rows of at most 256 bytes (at
    // c_out = 128 two 64 KB x stages and two dout tiles exceed WG_SMEM_MAX);
    // spx_debug_configure bit 4096 sends it back to the FMA kernel (A/B)
    if (tf32 && (a.c_in % 32 || a.c_out % 32 || a.c_out > 64 || runtime_cfg().tf32_wgrad_fma)) return false;
    if (!wg_span_ok(a.c_in * e) || !wg_span_ok(a.c_out * e)) return false;
    WgParams &p = pl.p;
    memset(&p, 0, sizeof(p));
    p.xb = a.c_in * e; p.span_x = p.xb < 128 ? p.xb : 128;
    p.lg_span_x = p.span_x == 128 ? 7 : (p.span_x == 64 ? 6 : 5);
    p.apo = p.xb / p.span_x;
    // the producers split an atom index into (offset slot, chunk) with a shift and a mask: 384- to
    // 896-byte rows (192 16-bit channels, 96 / 160 / 192 / 224 fp32 channels) run on the FMA kernel
    if (p.apo & (p.apo - 1)) return false;
    p.atom_elems = p.span_x / e;
    p.apg = 128 / p.atom_elems;
    p.db = a.c_out * e; p.span_d = p.db < 128 ? p.db : 128;
    p.lg_span_d = p.span_d == 128 ? 7 : (p.span_d == 64 ? 6 : 5);
    if (p.db & (p.db - 1)) return false;
    p.lg_cpr_d = 0;
    while ((1 << p.lg_cpr_d) < (p.db >> 4)) ++p.lg_cpr_d;
    p.n = a.c_out;
    p.ab_bf16 = a.dtype == SPX_BF16;
    const int atoms_total = a.kv * p.apo;
    p.groups_total = (atoms_total + p.apg - 1) / p.apg;
    p.groups_per_pass = WG_ACC_COLS / a.c_out;          // = G of the kernel instance
    if (p.groups_per_pass > 16) p.groups_per_pass = 16;
    pl.passes = (p.groups_total + p.groups_per_pass - 1) / p.groups_per_pass;
    p.a_stage_bytes = p.apg * WG_TILE * p.span_x;
    p.b_buf_bytes = WG_TILE * p.db;
    p.idx_bytes = (int)align_up((size_t)(a.kv + 1) * 512, 1024);
    // tf32 stages are twice as large (64 KB per group of four 32-channel atoms): two of them only fit without the
    // head-room the 16-bit plans keep for a deeper index ring
    int avail = (tf32 ? WG_SMEM_MAX - 2048 : WG_SMEM_BUDGET) - 2 * p.b_buf_bytes - 2 * p.idx_bytes;
    if (avail < 2 * p.a_stage_bytes) return false;
    p.stages = avail / p.a_stage_bytes;
    if (p.stages > WG_MAX_STAGES) p.stages = WG_MAX_STAGES;
    // A third dout buffer where it fits: the producers issue the dout tile of tile t+1 right after the
    // first x stage of tile t, and with two buffers that waits until the consumers have retired the
    // last group of tile t-1 -- a gather latency on every tile.  Stage count and index ring come first.
    p.b_bufs = 2;
    size_t fixed = 2 * (size_t)p.b_buf_bytes + (size_t)p.stages * p.a_stage_bytes + 1024 + 1024;
    if (fixed + p.b_buf_bytes + 2 * (size_t)p.idx_bytes <= (size_t)WG_SMEM_MAX) { p.b_bufs = 3; fixed += p.b_buf_bytes; }
    p.idx_bufs = 2;
    while (p.idx_bufs < WG_MAX_IDX && fixed + (size_t)(p.idx_bufs + 1) * p.idx_bytes <= (size_t)WG_SMEM_MAX) ++p.idx_bufs;
    pl.smem = fixed + (size_t)p.idx_bufs * p.idx_bytes;
    int64_t tiles = div_up64(a.n_out, WG_TILE);
    int chunks = sm_count() / pl.passes;
    if (chunks < 1) chunks = 1;
    if (chunks > tiles) chunks = (int)tiles;
    if (chunks < 1) chunks = 1;
    pl.chunks = chunks;
    p.rows = a.n_out; p.tile_table = a.tile_table; p.tile_mask = a.tile_mask;
    p.sched_rec = a.tile_table + tt_blocks_elems(tiles, a.kv);
    p.kv = a.kv; p.words = (a.kv + 31) / 32; p.c_in = a.c_in;
    p.x = (const uint8_t *)a.x; p.d = (const uint8_t *)a.dout;
    p.partial_stride = (int64_t)a.kv * a.c_in * a.c_out;
    return true;
}

bool tc_wgrad_supported(const WgradArgs &a) {
    WgPlan pl;
    return make_plan(a, pl);
}

size_t tc_wgrad_workspace_size(const WgradArgs &a) {
    WgPlan pl;
    if (!make_plan(a, pl)) return 256;
    // chunk count depends on the SM count only through an upper bound; size for the bound
    return (size_t)pl.chunks * pl.p.partial_stride * sizeof(float) + 256;
}

// ldx != 0: one group of a grouped conv (16-bit only): x rows ldx and dout rows ldd elements apart; the reduction
// writes the group's contiguous dW block a.dw.  A grouped call is never given peers (api_gemm.cu pushes the whole dW).
int tc_wgrad(const WgradArgs &a, cudaStream_t stream, int64_t ldx, int64_t ldd) {
    WgPlan pl;
    SPX_REQUIRE(make_plan(a, pl), "tc_wgrad: unsupported shape");
    SPX_REQUIRE(!ldx || (a.dtype != SPX_F32 && !a.peers), "tc_wgrad: grouped calls are 16-bit and local");
    pl.p.ldx = (int)ldx * 2; pl.p.ldd = (int)ldd * 2;
    pl.p.partial = (float *)a.workspace;
    SPX_REQUIRE((size_t)pl.chunks * pl.p.partial_stride * sizeof(float) <= a.workspace_bytes,
                "tc_wgrad: workspace too small");
    SPX_REQUIRE(aligned16(a.workspace), "tc_wgrad: workspace must be 16-byte aligned");
    dim3 grid(pl.chunks, pl.passes);
    const int cpa = pl.p.span_x >> 4, cpd = pl.p.db >> 4;
    using KernelFn = void (*)(const WgParams);
    KernelFn fn = nullptr;
    if (a.dtype == SPX_F32) {
        if (cpa == 8 && cpd == 8) fn = tc_wgrad_kernel<8, 8, true>;
        if (cpa == 8 && cpd == 16) fn = tc_wgrad_kernel<8, 16, true>;
    } else {
#define WG_PICK(A, D) if (cpa == A && cpd == D) fn = ldx ? tc_grouped_wgrad_kernel<A, D> : tc_wgrad_kernel<A, D>;
#define WG_PICK_ROW(A) WG_PICK(A, 2) WG_PICK(A, 4) WG_PICK(A, 8) WG_PICK(A, 16) WG_PICK(A, 32)
        WG_PICK_ROW(2) WG_PICK_ROW(4) WG_PICK_ROW(8)
#undef WG_PICK_ROW
#undef WG_PICK
    }
    SPX_REQUIRE(fn != nullptr, "tc_wgrad: no kernel instance for this channel layout");
    if (!func_configured((const void *)fn, current_device()))      // per-device attribute
        SPX_CHECK_CUDA(cudaFuncSetAttribute((const void *)fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            WG_SMEM_MAX));
    fn<<<grid, WG_THREADS, pl.smem, stream>>>(pl.p);
    SPX_CHECK_LAUNCH(ldx ? "tc_grouped_wgrad_kernel" : "tc_wgrad_kernel");
    const int64_t total = pl.p.partial_stride;
    if (a.peers)        // data-parallel: the reduction of the partials IS the send side of the exchange (peer.cu); the
                        // caller finishes it (peer_finish writes dW) after the work it wants to overlap
        return peer_push(pl.p.partial, total, pl.chunks, nullptr, total, a.dtype, a.peers, stream);
    unsigned nblk = (unsigned)div_up64(total, 128);
    if (a.dtype == SPX_F32)
        wgrad_reduce_kernel<float><<<nblk, RED_WARPS * 32, 0, stream>>>(pl.p.partial, total, pl.chunks, total, (float *)a.dw);
    else if (a.dtype == SPX_F16)
        wgrad_reduce_kernel<__half><<<nblk, RED_WARPS * 32, 0, stream>>>(pl.p.partial, total, pl.chunks, total, (__half *)a.dw);
    else
        wgrad_reduce_kernel<__nv_bfloat16><<<nblk, RED_WARPS * 32, 0, stream>>>(pl.p.partial, total, pl.chunks, total, (__nv_bfloat16 *)a.dw);
    SPX_CHECK_LAUNCH("wgrad_reduce_kernel");
    return 0;
}

}  // namespace spx
