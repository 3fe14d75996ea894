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
    constexpr int E = TF32 ? 4 : 2;
    constexpr int N = CPD * 16 / E;                              // wgmma N = c_out
    constexpr int G = WG_ACC_COLS / N < 16 ? WG_ACC_COLS / N : 16;   // resident groups per CTA
    constexpr int KSTEPS = WG_TILE * E / 32;                     // 32-byte k-steps over the 128 voxels
    constexpr int LG_CPA = CPA == 2 ? 1 : (CPA == 4 ? 2 : 3);
    constexpr int RPI = 32 / CPA;
    constexpr int LG_CPD = CPD == 2 ? 1 : (CPD == 4 ? 2 : (CPD == 8 ? 3 : (CPD == 16 ? 4 : 5)));
    constexpr int RPI_D = 32 / CPD;                              // dout rows covered by one warp-wide cp.async
    constexpr int DB = CPD * 16;
    constexpr int SPAN_D = DB < 128 ? DB : 128;
    constexpr int LG_SPAN_D = SPAN_D == 128 ? 7 : (SPAN_D == 64 ? 6 : 5);
    constexpr int SPAN_X = CPA * 16;
    constexpr int LG_SPAN_X = LG_CPA + 4;
    constexpr int ROWS_PW = WG_TILE / WG_PROD_WARPS;           // tile rows per producer warp
    constexpr int ITERS = ROWS_PW / RPI > 0 ? ROWS_PW / RPI : 1;   // copies per thread per atom
    constexpr int ITERS_D = ROWS_PW / RPI_D;                       // copies per thread per dout tile
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
    uint8_t *smem = smem_raw + pad;
    const uint32_t smem_base = raw_addr + pad;
    // layout: [b_bufs x B buffer][stages x A stage][idx_bufs x index block][barriers]
    const uint32_t b_base = smem_base;
    const uint32_t a_base = smem_base + (uint32_t)p.b_bufs * p.b_buf_bytes;
    const uint32_t idx_off = (uint32_t)p.b_bufs * p.b_buf_bytes + (uint32_t)p.stages * p.a_stage_bytes;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + idx_off + (uint32_t)p.idx_bufs * p.idx_bytes);
    uint64_t *full_a = bars;                          // [stages]
    uint64_t *empty_a = bars + WG_MAX_STAGES;         // [stages]
    uint64_t *full_b = bars + 2 * WG_MAX_STAGES;                // [WG_MAX_B]
    uint64_t *empty_b = bars + 2 * WG_MAX_STAGES + WG_MAX_B;     // [WG_MAX_B]
    uint64_t *idx_full = bars + 2 * WG_MAX_STAGES + 2 * WG_MAX_B;                // [WG_MAX_IDX]
    uint64_t *idx_empty = bars + 2 * WG_MAX_STAGES + 2 * WG_MAX_B + WG_MAX_IDX;  // [WG_MAX_IDX]
    uint32_t *gmask = reinterpret_cast<uint32_t *>(bars + 2 * WG_MAX_STAGES + 2 * WG_MAX_B + 2 * WG_MAX_IDX);  // [16][2][4] offsets of each warpgroup's half of each group of this pass
    uint32_t *slot_info = gmask + 16 * 8;             // [WG_MAX_IDX][8]: {active halves, tile mask[4]} per ring slot

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t num_tiles = (p.rows + WG_TILE - 1) / WG_TILE;
    const int chunk = blockIdx.x, chunks = gridDim.x;

    // Groups are dealt to the passes round-robin (pass y owns groups y, y + passes, ...).  Balancing the
    // passes by their active-tile counts (LPT, computed in every CTA's prologue) cut the busiest CTA of
    // config 2 from 54 to 41 stages, but not the training step: the input-gradient kernel runs beside
    // this one and fills the SMs that lighter passes leave early, so the step pays for total SM time,
    // which the prologue only adds to (DESIGN.md section 7).
    const int g_first = blockIdx.y, g_step = gridDim.y;
    const int ng = g_first < p.groups_total ? (p.groups_total - g_first + g_step - 1) / g_step : 0;
    if (threadIdx.x < 32) {
        // local group gl = thread / 2, warpgroup half h = thread % 2: atoms [g apg + h apg / 2, ...)
        const int gl = (int)threadIdx.x >> 1, h = (int)threadIdx.x & 1;
        const int g = g_first + gl * g_step, hp = p.apg >> 1;
        const int k_lo = (g * p.apg + h * hp) / p.apo;
        const int k_hi = min((g * p.apg + (h + 1) * hp - 1) / p.apo, p.kv - 1);
        const uint32_t bits = gl < ng && k_lo <= k_hi ? offset_run_bits(k_lo, k_hi) : 0u;
#pragma unroll
        for (int w = 0; w < 4; ++w) gmask[threadIdx.x * 4 + w] = w == (k_lo >> 5) ? bits : 0u;
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full_a[s], WG_PROD_THREADS); mbar_init(&empty_a[s], WG_CONS_WARPS); }
        for (int b = 0; b < p.b_bufs; ++b) { mbar_init(&full_b[b], WG_PROD_THREADS); mbar_init(&empty_b[b], WG_CONS_WARPS); }
        for (int b = 0; b < p.idx_bufs; ++b) { mbar_init(&idx_full[b], 1); mbar_init(&idx_empty[b], WG_PROD_WARPS); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp >= WG_CONS_WARPS && warp < WG_SCHED_WARP) {
        // ================================================= producers
        const int pw = warp - WG_CONS_WARPS;
        int stage = 0; uint32_t phase = 0;
        int bbuf = 0; uint32_t bphase = 0;               // next B buffer to fill, its phase
        // per-lane constants of the atom gather: chunk chb of rows r0 + itc*RPI of this warp's rows
        const int r0 = lane >> LG_CPA;
        const uint32_t chb = (uint32_t)(lane & (CPA - 1)) << 4;
        const uint8_t *x_lane = p.x + chb;
        uint32_t dst_off[ITERS];
#pragma unroll
        for (int itc = 0; itc < ITERS; ++itc)
            dst_off[itc] = swizzle_offset(((uint32_t)(pw * ROWS_PW + r0 + itc * RPI) << LG_SPAN_X) + chb, SPAN_X);
        const int lg_apo = p.apo == 1 ? 0 : (p.apo == 2 ? 1 : (p.apo == 4 ? 2 : 3));   // apo: 1, 2, 4 or 8 (make_plan)
        // per-lane constants of the dout gather: chunk chd of rows rd0 + itc*RPI_D of this warp's rows
        const int rd0 = lane >> LG_CPD;
        const uint32_t chd = (uint32_t)(lane & (CPD - 1)) << 4;
        const uint8_t *d_lane = p.d + chd;
        // index-block ring (filled by the feeder warp): slot / use count advance with the tiles
        const int nring = p.idx_bufs;
        // dout tile (B operand) of the tile whose index block is idx_s; source rows = block row kv
        auto issue_b = [&](const int32_t *idx_s) {
            const int bb = bbuf;
            mbar_wait_silent(&empty_b[bb], bphase ^ 1u);
            const uint32_t dstb = b_base + (uint32_t)bb * p.b_buf_bytes;
            const int32_t *rows_s = idx_s + p.kv * 128 + pw * ROWS_PW + rd0;
            if constexpr (TF32) {
                // batches of 8 rows keep the float4 loads in flight without spilling; the row indices
                // are read per batch, as a whole-tile register array would be indexed dynamically
#pragma unroll 1
                for (int i0 = 0; i0 < ITERS_D; i0 += 8) {
                    float4 v[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int32_t r = i0 + i < ITERS_D ? rows_s[(i0 + i) * RPI_D] : -1;
                        v[i] = r >= 0 ? __ldg(reinterpret_cast<const float4 *>(d_lane + (int64_t)r * DB)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (i0 + i < ITERS_D)
                            st_shared_f32x4_t(dstb, chd >> 2, (uint32_t)(pw * ROWS_PW + rd0 + (i0 + i) * RPI_D), (uint32_t)N, v[i]);
                }
                fence_proxy_async_smem();
                mbar_arrive(&full_b[bb]);
            } else {
                int32_t rsrc[ITERS_D];                    // all index loads first, then the copies
#pragma unroll
                for (int itc = 0; itc < ITERS_D; ++itc) rsrc[itc] = rows_s[itc * RPI_D];
#pragma unroll
                for (int itc = 0; itc < ITERS_D; ++itc) {
                    const uint32_t row_in_tile = (uint32_t)(pw * ROWS_PW + rd0 + itc * RPI_D);
                    const uint32_t off = (chd >> LG_SPAN_D) * (uint32_t)(WG_TILE * SPAN_D) +
                                         swizzle_offset((row_in_tile << LG_SPAN_D) + (chd & (uint32_t)(SPAN_D - 1)), SPAN_D);
                    cp_async_16(dstb + off, d_lane + (int64_t)max(rsrc[itc], 0) * DB, rsrc[itc] >= 0 ? 16u : 0u);
                }
                cp_async_mbar_arrive_noinc(&full_b[bb]);
            }
            if (++bbuf == p.b_bufs) { bbuf = 0; bphase ^= 1u; }
        };
        auto idx_block = [&](int b) {
            return reinterpret_cast<const int32_t *>(smem + idx_off + (size_t)b * p.idx_bytes);
        };
        // Software pipeline over tiles: the feeder warp keeps the ring of index blocks (and each
        // tile's group set) filled nring-1 tiles ahead; right after the first x stage of tile t
        // the dout tile of t+1 is issued -- nothing but the first x stage sits on the boundary.
        auto read_slot = [&](int slot, uint32_t use, uint32_t (&m)[4]) -> uint32_t {
            mbar_wait_silent(&idx_full[slot], use & 1u);
            const volatile uint32_t *r = slot_info + slot * 8;
            m[0] = r[1]; m[1] = r[2]; m[2] = r[3]; m[3] = r[4];
            return r[0];
        };
        int cur_slot = 0; uint32_t cur_use = 0;          // ring position of the tile being gathered
        uint32_t tm[4] = {0, 0, 0, 0}, tm1[4] = {0, 0, 0, 0};
        uint32_t act = 0;
        if (wg_rec_index(0, chunk, chunks) < num_tiles) {
            act = read_slot(0, 0u, tm);
            if (act) issue_b(idx_block(0));
        }
        for (int64_t step = 0; wg_rec_index(step, chunk, chunks) < num_tiles; ++step) {
            const bool has_next = wg_rec_index(step + 1, chunk, chunks) < num_tiles;
            int nxt_slot = cur_slot + 1; uint32_t nxt_use = cur_use;
            if (nxt_slot == nring) { nxt_slot = 0; ++nxt_use; }
            uint32_t act_next = 0;
            bool next_ready = !has_next;
            auto prepare_next = [&]() {
                act_next = read_slot(nxt_slot, nxt_use, tm1);
                if (act_next) issue_b(idx_block(nxt_slot));
                next_ready = true;
            };
            const int32_t *idx_s = idx_block(cur_slot);
            // ---- gathered x atoms, one stage per active group.  A warpgroup's half without an active
            // offset is not copied at all: its consumer warpgroup skips the stage's wgmma.
            for (uint32_t rem = (act | act >> 16) & 0xFFFFu; rem; rem &= rem - 1) {
                const int gl = __ffs(rem) - 1;
                const int g = g_first + gl * g_step;
                mbar_wait_silent(&empty_a[stage], phase ^ 1u);
                const uint32_t a_stage = a_base + (uint32_t)stage * p.a_stage_bytes;
                for (int s = 0; s < p.apg; ++s) {
                    if (!((act >> (gl + (s >= (p.apg >> 1) ? 16 : 0))) & 1u)) continue;
                    const int a = g * p.apg + s;
                    const int k = a >> lg_apo;
                    const int cb = a & (p.apo - 1);
                    const bool active = k < p.kv && ((pick_word(tm, k >> 5) >> (k & 31)) & 1u);
                    const int32_t *idx_k = idx_s + (active ? k : 0) * 128 + pw * ROWS_PW + r0;
                    const uint8_t *x_atom = x_lane + cb * SPAN_X;
                    int32_t ridx[ITERS];                      // all index loads first, then the copies
#pragma unroll
                    for (int itc = 0; itc < ITERS; ++itc) ridx[itc] = active ? idx_k[itc * RPI] : -1;
                    if constexpr (TF32) {
                        // M row = s * 32 + channel inside the atom, K = voxel of the tile
#pragma unroll
                        for (int itc = 0; itc < ITERS; ++itc) {
                            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (ridx[itc] >= 0) v = __ldg(reinterpret_cast<const float4 *>(x_atom + (int64_t)ridx[itc] * p.xb));
                            st_shared_f32x4_t(a_stage, (uint32_t)(s * 32) + (chb >> 2),
                                              (uint32_t)(pw * ROWS_PW + r0 + itc * RPI), (uint32_t)WG_TILE, v);
                        }
                    } else {
                        const uint32_t atom_base = a_stage + (uint32_t)s * (uint32_t)(WG_TILE * SPAN_X);
#pragma unroll
                        for (int itc = 0; itc < ITERS; ++itc)
                            cp_async_16(atom_base + dst_off[itc], x_atom + (int64_t)max(ridx[itc], 0) * p.xb,
                                        ridx[itc] >= 0 ? 16u : 0u);
                    }
                }
                if constexpr (TF32) {
                    fence_proxy_async_smem();
                    mbar_arrive(&full_a[stage]);
                } else {
                    cp_async_mbar_arrive_noinc(&full_a[stage]);
                }
                if (++stage == p.stages) { stage = 0; phase ^= 1u; }
                if (!next_ready) prepare_next();
            }
            if (!next_ready) prepare_next();
            __syncwarp();
            if (lane == 0) mbar_arrive(&idx_empty[cur_slot]);
#pragma unroll
            for (int w = 0; w < 4; ++w) tm[w] = tm1[w];
            act = act_next;
            cur_slot = nxt_slot; cur_use = nxt_use;
        }
    } else if (warp == WG_SCHED_WARP) {
        // ================================================= tile feeder
        // Per tile of this CTA (static snake order, so the summation order of dW is fixed): compute
        // the active group halves of this pass from the tile mask, publish them with the mask through
        // the ring slot, and bulk-copy the tile's index block -- only when the pass has work for
        // the tile.  Schedule records are fetched 32 at a time, one per lane.
        const uint32_t blk_bytes = (uint32_t)(p.kv + 1) * 512u;
        const int nring = p.idx_bufs;
        int slot = 0; uint32_t use = 0;
        uint32_t mw[4] = {0, 0, 0, 0};
        int64_t mtile = 0;
        for (int64_t i = 0; wg_rec_index(i, chunk, chunks) < num_tiles; ++i) {
            if ((i & 31) == 0) {                         // the next 32 schedule records, one per lane
                const int64_t r = wg_rec_index(i + lane, chunk, chunks);
                if (r < num_tiles) wg_load_rec(p.sched_rec, r, mtile, mw);
            }
            uint32_t tm[4];
#pragma unroll
            for (int w = 0; w < 4; ++w) tm[w] = __shfl_sync(0xffffffffu, mw[w], (int)(i & 31));
            const int64_t tile = __shfl_sync(0xffffffffu, mtile, (int)(i & 31));
            const uint32_t act = active_halves(tm, gmask, ng, p.words);
            mbar_wait_silent(&idx_empty[slot], (use & 1u) ^ 1u);
            if (lane == 0) {
                uint32_t *r = slot_info + slot * 8;
                r[0] = act; r[1] = tm[0]; r[2] = tm[1]; r[3] = tm[2]; r[4] = tm[3];
                if (act) {
                    mbar_arrive_expect_tx(&idx_full[slot], blk_bytes);
                    bulk_copy_g2s(smem_base + idx_off + (uint32_t)slot * p.idx_bytes,
                                  p.tile_table + tile * (int64_t)(p.kv + 1) * 128, blk_bytes, &idx_full[slot]);
                } else {
                    mbar_arrive(&idx_full[slot]);
                }
            }
            __syncwarp();
            if (++slot == nring) { slot = 0; ++use; }
        }
    } else if (warp < WG_CONS_WARPS) {
        // ================================================= consumers: warpgroup wg owns M rows 64 wg .. 64 wg + 63 of every group
        const int wg = warp >> 2;
        int stage = 0; uint32_t phase = 0;
        int bbuf = 0; uint32_t bphase = 0;               // next B buffer to read, its phase
        uint32_t tm[4] = {0, 0, 0, 0};
        int64_t tile_unused = 0;
        if (wg_rec_index(0, chunk, chunks) < num_tiles)
            wg_load_rec(p.sched_rec, wg_rec_index(0, chunk, chunks), tile_unused, tm);
        // 16-bit: both operands MN-major, LBO = distance between swizzle-wide atoms along M / N, SBO = 8 voxel
        // rows.  tf32: K-major 128-byte rows, SBO = one 8-row swizzle atom, k-steps walk 32-voxel sub-tiles.
        const uint64_t a_hi = TF32 ? gmma_desc_hi(16u, 1024u, 128u)
                                   : gmma_desc_hi((uint32_t)(WG_TILE * SPAN_X), 8u * SPAN_X, SPAN_X);
        const uint64_t b_hi = TF32 ? gmma_desc_hi(16u, 1024u, 128u)
                                   : gmma_desc_hi((uint32_t)(WG_TILE * SPAN_D), 8u * SPAN_D, SPAN_D);
        // this warpgroup's first M row: 64 rows of 128 bytes (tf32) / 64 channels = 64 / atom_elems atoms (16-bit)
        const uint32_t a_wg = TF32 ? (uint32_t)wg * 64u * 128u : (uint32_t)wg * 64u * WG_TILE * E;
        float acc[G][N / 2];
#pragma unroll
        for (int gl = 0; gl < G; ++gl)
#pragma unroll
            for (int i = 0; i < N / 2; ++i) acc[gl][i] = 0.f;
        // One wgmma group stays in flight: it reads A stage `held` and, when it was the last group of its
        // tile, dout buffer `held_b`; both are released once it has retired (wait_group 1 after the next
        // group is issued).  A stage this warpgroup has no active atoms in is not multiplied (its rows
        // are zero): the group in flight is retired and both stages are released at once, so the
        // producers never wait on a stage held across stages this warpgroup skips.
        int held = -1, held_b = -1;
        for (int64_t step = 0; wg_rec_index(step, chunk, chunks) < num_tiles; ++step) {
            const int64_t next = wg_rec_index(step + 1, chunk, chunks);
            uint32_t tm_next[4] = {0, 0, 0, 0};
            if (next < num_tiles) wg_load_rec(p.sched_rec, next, tile_unused, tm_next);
            const uint32_t halves = active_halves(tm, gmask, ng, p.words);
            const uint32_t act = (halves | halves >> 16) & 0xFFFFu;
            const uint32_t mine = (halves >> (16 * wg)) & 0xFFFFu;
            if (act) {
                const int bb = bbuf;
                mbar_wait_silent(&full_b[bb], bphase);
                const uint32_t b16 = (b_base + (uint32_t)bb * p.b_buf_bytes) >> 4;
#pragma unroll
                for (int gl = 0; gl < G; ++gl) {
                    if (!((act >> gl) & 1u)) continue;
                    mbar_wait_silent(&full_a[stage], phase);
                    if (!((mine >> gl) & 1u)) {
                        wgmma_wait<0>();
                        __syncwarp();
                        if (lane == 0) {
                            if (held >= 0) mbar_arrive(&empty_a[held]);
                            if (held_b >= 0) mbar_arrive(&empty_b[held_b]);
                            mbar_arrive(&empty_a[stage]);
                        }
                        held = -1; held_b = -1;
                        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
                        continue;
                    }
                    fence_proxy_async_smem();     // generic-proxy writes (cp.async / st.shared) -> wgmma operand reads
                    const uint32_t a16 = (a_base + (uint32_t)stage * p.a_stage_bytes + a_wg) >> 4;
                    fence_regs(acc[gl]);
                    wgmma_fence();
#pragma unroll
                    for (int j = 0; j < KSTEPS; ++j) {
                        if constexpr (TF32) {
                            // k-step j = 8 voxels: sub-tile j / 4, 32-byte column j % 4
                            const uint32_t ao = (uint32_t)(j >> 2) * (WG_TILE * 128u / 16u) + (uint32_t)(j & 3) * 2u;
                            const uint32_t bo = (uint32_t)(j >> 2) * (N * 128u / 16u) + (uint32_t)(j & 3) * 2u;
                            Wgmma<N>::tf32(acc[gl], a_hi | (uint64_t)((a16 + ao) & 0x3FFFu),
                                           b_hi | (uint64_t)((b16 + bo) & 0x3FFFu), 1u);
                        } else {
                            // k-step j = 16 voxel rows of both MN-major operands
                            const uint64_t a_desc = a_hi | (uint64_t)((a16 + (uint32_t)j * SPAN_X) & 0x3FFFu);
                            const uint64_t b_desc = b_hi | (uint64_t)((b16 + (uint32_t)j * SPAN_D) & 0x3FFFu);
                            if (p.ab_bf16) Wgmma<N>::template bf16<1, 1>(acc[gl], a_desc, b_desc, 1u);
                            else Wgmma<N>::template f16<1, 1>(acc[gl], a_desc, b_desc, 1u);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<1>();
                    fence_regs(acc[gl]);
                    __syncwarp();
                    if (lane == 0) {
                        if (held >= 0) mbar_arrive(&empty_a[held]);
                        if (held_b >= 0) mbar_arrive(&empty_b[held_b]);
                    }
                    held = stage; held_b = -1;
                    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
                }
                if (held >= 0) {
                    held_b = bb;                  // released with the tile's last group
                } else {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_b[bb]);
                }
                if (++bbuf == p.b_bufs) { bbuf = 0; bphase ^= 1u; }
            }
#pragma unroll
            for (int w = 0; w < 4; ++w) tm[w] = tm_next[w];
        }
        wgmma_wait<0>();
#pragma unroll
        for (int gl = 0; gl < G; ++gl) fence_regs(acc[gl]);
        // ================================================= accumulators -> fp32 partials
        // register i of thread t holds M row 64 wg + 16 (warp % 4) + t / 4 + 8 ((i / 2) % 2),
        // column 8 (i / 4) + 2 (t % 4) + i % 2
        float *part = p.partial + (int64_t)chunk * p.partial_stride;
#pragma unroll
        for (int gl = 0; gl < G; ++gl) {
            if (gl >= ng) break;
            const int g = g_first + gl * g_step;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int L = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;   // M index inside the group
                const int s = L / p.atom_elems;
                const int ce = L - s * p.atom_elems;
                const int a = g * p.apg + s;
                const int k = a / p.apo;
                const int c = (a - k * p.apo) * p.atom_elems + ce;
                if (k >= p.kv) continue;
                float *dst = part + (int64_t)k * p.c_in + c;
#pragma unroll
                for (int nb8 = 0; nb8 < N / 8; ++nb8)
#pragma unroll
                    for (int j = 0; j < 2; ++j)
                        dst[(int64_t)(nb8 * 8 + 2 * (lane & 3) + j) * p.kv * p.c_in] = acc[gl][nb8 * 4 + 2 * h + j];
            }
        }
    }

    __syncthreads();
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

int tc_wgrad(const WgradArgs &a, cudaStream_t stream) {
    WgPlan pl;
    SPX_REQUIRE(make_plan(a, pl), "tc_wgrad: unsupported shape");
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
#define WG_PICK(A, D) if (cpa == A && cpd == D) fn = tc_wgrad_kernel<A, D>;
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
    SPX_CHECK_LAUNCH("tc_wgrad_kernel");
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
