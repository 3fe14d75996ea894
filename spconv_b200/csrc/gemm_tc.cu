// wgmma / TMA masked implicit GEMM: forward and input-gradient (and the int8 and fp8 inference forwards).
//
// Persistent CTAs (one per SM) work on 128-row output tiles (rows in mask_argsort order).  Tiles
// are handed out DYNAMICALLY: a scheduler warp draws tickets from an atomic counter and takes
// tiles from the schedule records behind the tile table (heaviest first = LPT list scheduling,
// see gemm.cuh / rulebook.cu); the tile's gather indices arrive as ONE bulk async copy
// (cp.async.bulk) of its block of the tile table (spx_build_tile_table), one tile ahead.  For
// each kernel offset whose bit is set in the tile's OR-mask:
//   * 2 producer warps gather the 128 input rows into a swizzled K-major shared-memory tile with
//     16-byte cp.async (zero-fill for "-1 = no neighbour"); all per-lane addressing is hoisted
//     out of the pipeline (compile-time chunk count CPR), the row indices of the next offset are
//     read before the wait for the next free stage;
//   * the TMA warp loads that offset's KRSC weight slice W[:, k, :] (a strided 2-D box);
//   * two consumer warpgroups (rows 0-63 and 64-127) issue wgmma.mma_async (M = 64 each,
//     N = out channels, K = 32 bytes per instruction) accumulating the whole offset sum in
//     registers (one group stays in flight: a stage is released once the next stage's group is
//     issued), and store their rows (bias / activation / int8 requantisation) once the tile's
//     last offset is in; the producers meanwhile fill the stages of the next tile.  The
//     destination rows come from the argsort row of the tile's index block, read at the tile's
//     start; bias and scales from shared memory, loaded once per CTA.
// 384 threads leave 168 registers per thread: room for the accumulator fragment (128 fp32 per
// consumer thread at N = 256) and for the hoisted per-lane gather addressing of the producers.
//
// Reference being replaced: ConvMain::implicit_gemm2 as called from
// spconv/csrc/sparse/convops.py:2196-2235 (fwd) and :2394-2419 (dgrad); the kernel itself lives
// in the un-vendored cumm package (Ampere mma.sync at best, spconv/core.py:502-830).
//
// The input-gradient pass is the same kernel: A = gathered dout rows, contraction over the
// out channels, and the SAME 16-bit weight box is consumed as an MN-major B operand (wgmma
// transpose-B), so no transposed copy of the filter is ever made.  tf32 wgmma only reads K-major
// operands: for the fp32 input gradient the TMA warp writes the weight slice transposed into
// the stage with ordinary loads and stores instead.
#include "gemm.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <atomic>
#include <mutex>
#include <stdlib.h>

namespace spx {

constexpr int TC_TILE_M = 128;
constexpr int TC_CONS_WARPS = 8;         // two consumer warpgroups, 64 tile rows each
constexpr int TC_PROD_WARPS = 2;         // 64 tile rows per producer warp
constexpr int TC_PROD_THREADS = TC_PROD_WARPS * 32;
constexpr int TC_TMA_WARP = TC_CONS_WARPS + TC_PROD_WARPS;
constexpr int TC_SCHED_WARP = TC_TMA_WARP + 1;
constexpr int TC_THREADS = 3 * 128;      // warps 0-7 consumers | 8-9 gather producers | 10 weight TMA | 11 tile scheduler + index copies
constexpr int TC_INFO_DEPTH = 4;         // tile-info ring (scheduler -> every role)
constexpr int TC_INFO_READERS = TC_PROD_WARPS + TC_CONS_WARPS + 1;   // producer warps, consumer warps, TMA warp
constexpr int TC_MAX_STAGES = 8;
constexpr int TC_SMEM_BUDGET = 200 * 1024;   // operand stages + index blocks per CTA (227 KB is the sm_90 limit)

struct TcParams {
    // gathered operand A
    const uint8_t *x;
    int xb;                 // bytes per gathered row (contraction length in bytes) = CPR * 16
    // weight operand B (TMA box = [b_rows x span_b bytes] per sub-tile)
    int span_b, b_subtiles, b_sub_bytes, b_bytes, b_mn_major, b_kstep16_mn;
    int b_transposed;       // 1: fp32 input gradient, the TMA warp writes W[:, k, :]^T as a K-major operand
    const float *w;         // the filter (b_transposed only)
    int c_in, c_out;
    int w_inner_elems;      // c_in (elements between consecutive offsets along the TMA inner dim)
    int span_b_elems;       // span_b / elem bytes
    int n;                  // wgmma N (output channels of this pass)
    int ab_bf16;            // 16-bit kernels: operands are bf16 (else fp16)
    int stages, a_stage_bytes, stage_bytes, idx_bytes;
    // rows
    int64_t rows;
    const int32_t *tile_table;   // [tiles][kv+1][128]
    const int32_t *sched_rec;    // [tiles][TT_REC_INTS] schedule records, heaviest tile first (gemm.cuh)
    int *sched_state;            // [0] ticket counter, [1] finished CTAs; zero between launches
    const int32_t *argsort;      // order the tile table was built with (NULL = identity); the epilogue reads its
                                 // destination rows from row kv of each index block, which holds this order
    int kv, words, reverse;
    // epilogue
    void *y;
    int out_dtype;          // spx_dtype of y
    int epi_mode;           // 0: float bias+act, 1: int8 quantised inference, 2: fp8 inference
    const void *bias;       // dtype of y (mode 0)
    int act; float alpha;
    const float *scale, *bias_f32;
    const int8_t *output_add;
    float output_add_scale;
    // fp8 epilogue (KIND_E4M3): scale = w_scale, bias_f32 = bias, output_add = the residual in out_dtype
    const float *in_scale, *add_scale, *out_scale;
    int ldy;                // elements between output (and residual) rows: c_out, of which this pass writes N
    int ldx;                // grouped instances: bytes between gathered rows (the full row, of which a group reads xb)
};

// iterate set bits of a <=128-bit tile mask in ascending order (register-only: no indexed array)
struct BitIter {
    uint32_t m0, m1, m2, m3;
    __device__ __forceinline__ BitIter(const uint32_t (&t)[4]) : m0(t[0]), m1(t[1]), m2(t[2]), m3(t[3]) {}
    __device__ __forceinline__ int next() {
        if (m0) { int b = __ffs(m0) - 1; m0 &= m0 - 1; return b; }
        if (m1) { int b = __ffs(m1) - 1; m1 &= m1 - 1; return 32 + b; }
        if (m2) { int b = __ffs(m2) - 1; m2 &= m2 - 1; return 64 + b; }
        if (m3) { int b = __ffs(m3) - 1; m3 &= m3 - 1; return 96 + b; }
        return -1;
    }
};

// ------------------------------------------------------------------ epilogue
// two adjacent accumulator columns -> OUT type.  OUT is an spx_dtype code.
template <int OUT>
__device__ __forceinline__ void store2(uint8_t *dst, float a, float b) {
    if constexpr (OUT == SPX_F32) {
        *reinterpret_cast<float2 *>(dst) = make_float2(a, b);
    } else if constexpr (OUT == SPX_F16) {
        *reinterpret_cast<__half2 *>(dst) = __floats2half2_rn(a, b);
    } else if constexpr (OUT == SPX_BF16) {
        *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(a, b);
    } else {   // int8: clip(rint(.)) -- numpy round-half-even
        const int qa = (int)fminf(fmaxf(rintf(a), -128.f), 127.f), qb = (int)fminf(fmaxf(rintf(b), -128.f), 127.f);
        *reinterpret_cast<uint16_t *>(dst) = (uint16_t)((uint32_t)(uint8_t)(int8_t)qa | ((uint32_t)(uint8_t)(int8_t)qb << 8));
    }
}

template <int OUT> struct OutElem { static constexpr int bytes = OUT == SPX_F32 ? 4 : (OUT == SPX_I8 ? 1 : 2); };

template <int OUT>
__device__ __forceinline__ float load_bias(const void *bias, int j) {
    if constexpr (OUT == SPX_F32) return ((const float *)bias)[j];
    else if constexpr (OUT == SPX_F16) return __half2float(((const __half *)bias)[j]);
    else return __bfloat162float(((const __nv_bfloat16 *)bias)[j]);
}

// Store one warpgroup's accumulator fragment: register i of thread t holds row
// (t / 4) % 8 + 16 * warp + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (t % 4) + i % 2.
// ec: the CTA's epilogue constants in shared memory, ec[j] = bias (float mode) or scale (int8 mode),
// ec[N + j] = the int8 bias.  A float-mode call without bias and activation (the input gradient, and
// every conv layer followed by a norm) runs the PLAIN instance: convert and store, no per-element
// branches between the stores.  STRIDED (grouped instances): output rows are p.ldy elements apart, not N.
template <int OUT, bool INT8_MODE, int N, typename Acc, bool PLAIN = false, bool STRIDED = false>
__device__ __forceinline__ void epilogue_frag(const TcParams &p, const float *ec, const Acc (&acc)[N / 2], int64_t dst_lo,
                                              int64_t dst_hi, int lane) {
    if constexpr (!INT8_MODE && !PLAIN) {
        if (p.bias == nullptr && p.act == SPX_ACT_NONE) {
            epilogue_frag<OUT, false, N, Acc, true, STRIDED>(p, ec, acc, dst_lo, dst_hi, lane);
            return;
        }
    }
    constexpr int EB = OutElem<OUT>::bytes;
    const bool has_bias = !PLAIN && (INT8_MODE ? (p.bias_f32 != nullptr) : (p.bias != nullptr));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t dst = h ? dst_hi : dst_lo;
        if (dst < 0) continue;
        uint8_t *row_ptr = (uint8_t *)p.y + dst * (int64_t)(STRIDED ? p.ldy : N) * EB;
#pragma unroll
        for (int nb = 0; nb < N / 8; ++nb) {
            const int col = nb * 8 + 2 * (lane & 3);
            float f[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const Acc v = acc[nb * 4 + 2 * h + j];
                if constexpr (!INT8_MODE) {
                    f[j] = (float)v;
                    if (has_bias) f[j] += ec[col + j];
                } else {
                    // int8 inference: y = acc * scale[k] + bias[k] (+ add * add_scale)   test/test_all_algo.py:272-287
                    f[j] = (float)(int32_t)v * ec[col + j];
                    if (has_bias) f[j] += ec[N + col + j];
                    if (p.output_add) f[j] += (float)p.output_add[dst * (int64_t)N + col + j] * p.output_add_scale;
                }
                if (!PLAIN && p.act != SPX_ACT_NONE) f[j] = apply_act(f[j], p.act, p.alpha);
            }
            store2<OUT>(row_ptr + col * EB, f[0], f[1]);
        }
    }
}

// The fp8 epilogue (gemm.cuh fp8_epilogue) of one warpgroup fragment, same layout as epilogue_frag.  ec[j] = s_j,
// ec[N + j] = bias.  add_s / out_s: the residual and output scales, read once per tile.  Rows are p.ldy apart.
template <int OUT, int N>
__device__ __forceinline__ void epilogue_fp8(const TcParams &p, const float *ec, const float (&acc)[N / 2],
                                             int64_t dst_lo, int64_t dst_hi, int lane, float add_s, float out_s) {
    constexpr int EB = OUT == SPX_F32 ? 4 : (OUT == SPX_E4M3 ? 1 : 2);
    const float *bias = p.bias_f32 ? ec + N : nullptr;
    const void *add = (const void *)p.output_add;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t dst = h ? dst_hi : dst_lo;
        if (dst < 0) continue;
        uint8_t *row_ptr = (uint8_t *)p.y + dst * (int64_t)p.ldy * EB;
#pragma unroll
        for (int nb = 0; nb < N / 8; ++nb) {
            const int col = nb * 8 + 2 * (lane & 3);
            float f[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const float a = add ? load_out_elem<OUT>(add, dst * (int64_t)p.ldy + col + j) : 0.f;
                f[j] = fp8_epilogue(acc[nb * 4 + 2 * h + j], ec[col + j], bias, col + j, add != nullptr, a, add_s,
                                    p.act, p.alpha);
            }
            if constexpr (OUT == SPX_E4M3)
                *reinterpret_cast<uint16_t *>(row_ptr + col) = float2_to_e4m3x2(__fdiv_rn(f[0], out_s), __fdiv_rn(f[1], out_s));
            else
                store2<OUT>(row_ptr + col * EB, f[0], f[1]);
        }
    }
}

// one K step of 32 bytes: D[64 x N] += A[64 x 32 B] * B[N x 32 B]^T
template <int KIND, int N, typename Acc>
__device__ __forceinline__ void mma_step(Acc (&acc)[N / 2], uint64_t a, uint64_t b, int b_mn, int bf16) {
    if constexpr (KIND == KIND_F16) {
        if (bf16) {
            if (b_mn) Wgmma<N>::template bf16<0, 1>(acc, a, b, 1u);
            else Wgmma<N>::template bf16<0, 0>(acc, a, b, 1u);
        } else {
            if (b_mn) Wgmma<N>::template f16<0, 1>(acc, a, b, 1u);
            else Wgmma<N>::template f16<0, 0>(acc, a, b, 1u);
        }
    } else if constexpr (KIND == KIND_TF32) {
        Wgmma<N>::tf32(acc, a, b, 1u);
    } else if constexpr (KIND == KIND_I8) {
        Wgmma<N>::s8(acc, a, b, 1u);
    } else {
        Wgmma<N>::e4m3(acc, a, b, 1u);
    }
}

// The kernel body; tc_gather_gemm_kernel (16-bit, tf32, int8), tc_gather_gemm_fp8_kernel (e4m3) and
// tc_grouped_gemm_kernel (16-bit, one group of a grouped conv) launch it.  GROUPED: gathered rows are p.ldx bytes
// apart and output rows p.ldy elements; everything else is the dense instance.
template <int KIND, int CPR, int N, bool GROUPED = false>
__device__ __forceinline__ void tc_gather_gemm_body(const CUtensorMap &tmap_w, const TcParams &p) {
    using Acc = typename std::conditional<KIND == KIND_I8, int32_t, float>::type;
    constexpr int LG_CPR = CPR == 2 ? 1 : CPR == 4 ? 2 : CPR == 8 ? 3 : CPR == 16 ? 4 : 5;
    constexpr int RPI = 32 / CPR;            // rows covered by one warp-wide cp.async instruction
    constexpr int XB = CPR * 16;             // bytes per gathered row
    constexpr int SPAN_A = XB < 128 ? XB : 128;
    constexpr int LG_SPAN_A = SPAN_A == 128 ? 7 : (SPAN_A == 64 ? 6 : 5);
    constexpr int A_SUB_BYTES = TC_TILE_M * SPAN_A;
    constexpr int A_SUBTILES = XB / SPAN_A;
    constexpr int Q_A = SPAN_A / 32;         // k-steps (32 B) per A sub-tile
    constexpr int ROWS_PW = TC_TILE_M / TC_PROD_WARPS;          // tile rows per producer warp
    constexpr int ITERS = ROWS_PW / RPI > 0 ? ROWS_PW / RPI : 1;  // cp.async per thread per stage
    static_assert(ROWS_PW * CPR >= 32, "a producer warp must cover at least one full cp.async instruction");

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // dynamic smem base is only guaranteed 16-byte aligned: align manually to 1024
    const uint32_t raw_addr = smem_u32(smem_raw);
    const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
    uint8_t *smem = smem_raw + pad;
    const uint32_t smem_base = raw_addr + pad;

    const uint32_t idx_off = (uint32_t)p.stages * p.stage_bytes;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + idx_off + 2u * p.idx_bytes);
    uint64_t *full = bars;                                // [stages]  producers + TMA -> consumers
    uint64_t *empty = bars + TC_MAX_STAGES;               // [stages]  consumers -> producers + TMA
    uint64_t *idx_full = bars + 2 * TC_MAX_STAGES;        // [2] bulk copy -> producers
    uint64_t *idx_empty = bars + 2 * TC_MAX_STAGES + 2;   // [2] producers -> bulk copy
    uint64_t *info_full = bars + 2 * TC_MAX_STAGES + 4;                    // [TC_INFO_DEPTH] scheduler -> roles
    uint64_t *info_empty = bars + 2 * TC_MAX_STAGES + 4 + TC_INFO_DEPTH;   // [TC_INFO_DEPTH] roles -> scheduler
    int32_t *info = reinterpret_cast<int32_t *>(bars + 2 * TC_MAX_STAGES + 4 + 2 * TC_INFO_DEPTH);   // [TC_INFO_DEPTH][8]: {tile, mask[4]}
    float *ec = reinterpret_cast<float *>(smem + idx_off + 2u * p.idx_bytes + 1024u);   // [2][N] epilogue constants

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t num_tiles = (p.rows + TC_TILE_M - 1) / TC_TILE_M;

    // Tiles are handed out dynamically: the scheduler warp draws a ticket, looks the tile and its
    // offset set up in the schedule records (heaviest first => LPT list scheduling) and publishes
    // them through the info ring; every other role consumes ring entries in order.  Entry n uses
    // ring slot n % TC_INFO_DEPTH and index buffer n % 2; tile < 0 ends the stream.
    auto read_info = [&](int n, uint32_t (&tm)[4]) -> int {
        const int e = n & (TC_INFO_DEPTH - 1);
        mbar_wait_silent(&info_full[e], (uint32_t)((n / TC_INFO_DEPTH) & 1));
        const volatile int32_t *r = info + e * 8;
        const int tile = r[0];
        tm[0] = (uint32_t)r[1]; tm[1] = (uint32_t)r[2]; tm[2] = (uint32_t)r[3]; tm[3] = (uint32_t)r[4];
        __syncwarp();
        if (lane == 0) mbar_arrive(&info_empty[e]);
        return tile;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(&full[s], TC_PROD_THREADS + 1);    // cp.async arrivals + 1 arrival of the weight loader
            mbar_init(&empty[s], TC_CONS_WARPS);         // one release per consumer warp
        }
        for (int a = 0; a < 2; ++a) {
            mbar_init(&idx_full[a], 1);      // expect_tx arrival of the bulk copy
            mbar_init(&idx_empty[a], TC_PROD_WARPS + TC_CONS_WARPS);   // one release per producer / consumer warp
        }
        for (int e = 0; e < TC_INFO_DEPTH; ++e) {
            mbar_init(&info_full[e], 1);
            mbar_init(&info_empty[e], TC_INFO_READERS);  // one release per reading warp
        }
        mbar_fence_init();
        tma_prefetch_desc(&tmap_w);
    }
    // epilogue constants, read once per CTA instead of once per element and tile
    for (int j = threadIdx.x; j < N; j += TC_THREADS) {
        if constexpr (KIND == KIND_I8) {
            ec[j] = __ldg(p.scale + j);
            if (p.bias_f32) ec[N + j] = __ldg(p.bias_f32 + j);
        } else if constexpr (KIND == KIND_E4M3) {
            ec[j] = __fmul_rn(__ldg(p.in_scale), __ldg(p.scale + j));     // s_j = in_scale * w_scale[j]
            if (p.bias_f32) ec[N + j] = __ldg(p.bias_f32 + j);
        } else if (p.bias) {
            if constexpr (KIND == KIND_TF32) ec[j] = load_bias<SPX_F32>(p.bias, j);
            else ec[j] = p.out_dtype == SPX_F16 ? load_bias<SPX_F16>(p.bias, j) : load_bias<SPX_BF16>(p.bias, j);
        }
    }
    __syncthreads();

    if (warp >= TC_CONS_WARPS && warp < TC_TMA_WARP) {
        // ================================================= gather producers
        const int pw = warp - TC_CONS_WARPS;
        // per-lane constants: chunk ch of rows r0 + itc*RPI (itc = 0..CPR-1) of this warp's 32 rows
        const int r0 = lane >> LG_CPR;
        const uint32_t byte_in_row = (uint32_t)(lane & (CPR - 1)) << 4;
        const uint8_t *x_lane = p.x + byte_in_row;
        uint32_t dst_off[ITERS];
#pragma unroll
        for (int itc = 0; itc < ITERS; ++itc) {
            const uint32_t row_in_tile = (uint32_t)(pw * ROWS_PW + r0 + itc * RPI);
            const uint32_t sub = byte_in_row >> LG_SPAN_A;
            const uint32_t within = byte_in_row & (uint32_t)(SPAN_A - 1);
            dst_off[itc] = sub * (uint32_t)A_SUB_BYTES + swizzle_offset((row_in_tile << LG_SPAN_A) + within, SPAN_A);
        }
        int stage = 0; uint32_t phase = 0;
        for (int n = 0;; ++n) {
            uint32_t tm[4];
            if (read_info(n, tm) < 0) break;
            const int buf = n & 1;
            mbar_wait_silent(&idx_full[buf], (uint32_t)((n >> 1) & 1));
            const int32_t *idx_lane = reinterpret_cast<const int32_t *>(smem + idx_off + (size_t)buf * p.idx_bytes) +
                                      pw * ROWS_PW + r0;
            BitIter it(tm);
            // the index loads of offset k+1 are issued before the wait on the next free stage
            int k = it.next();
            int32_t ridx[ITERS];
            if (k >= 0) {
#pragma unroll
                for (int itc = 0; itc < ITERS; ++itc) ridx[itc] = idx_lane[k * 128 + itc * RPI];
            }
            while (k >= 0) {
                mbar_wait_silent(&empty[stage], phase ^ 1u);
                const uint32_t a_stage = smem_base + (uint32_t)stage * p.stage_bytes;
#pragma unroll
                for (int itc = 0; itc < ITERS; ++itc)
                    cp_async_16(a_stage + dst_off[itc], x_lane + (int64_t)max(ridx[itc], 0) * (GROUPED ? p.ldx : XB),
                                ridx[itc] >= 0 ? 16u : 0u);
                cp_async_mbar_arrive_noinc(&full[stage]);
                k = it.next();
                if (k >= 0) {
#pragma unroll
                    for (int itc = 0; itc < ITERS; ++itc) ridx[itc] = idx_lane[k * 128 + itc * RPI];
                }
                if (++stage == p.stages) { stage = 0; phase ^= 1u; }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&idx_empty[buf]);
        }
    } else if (warp == TC_TMA_WARP) {
        // ================================================= weight loader: one weight box per (tile, offset) stage
        // all 32 lanes walk the loops together (the CTA-wide barrier at the end must be reached
        // convergently); lane 0 issues the copies
        int stage = 0; uint32_t phase = 0;
        for (int n = 0;; ++n) {
            uint32_t tm[4];
            if (read_info(n, tm) < 0) break;
            BitIter it(tm);
            for (int k = it.next(); k >= 0; k = it.next()) {
                mbar_wait_silent(&empty[stage], phase ^ 1u);
                const int kw = p.reverse ? p.kv - 1 - k : k;
                const uint32_t b_stage = smem_base + (uint32_t)stage * p.stage_bytes + p.a_stage_bytes;
                if (p.b_transposed) {
                    // W[o][kw][i] -> row i, byte 4*o of a K-major [c_in x c_out] fp32 operand
                    const int i4s = p.c_in >> 2;
                    const float *wk = p.w + (int64_t)kw * p.c_in;
                    for (int q = lane; q < p.c_out * i4s; q += 32) {
                        const int o = q / i4s, i4 = (q - o * i4s) * 4;
                        const float4 v = __ldg(reinterpret_cast<const float4 *>(wk + (int64_t)o * p.kv * p.c_in + i4));
                        const uint32_t kb = (uint32_t)o * 4u;
                        const uint32_t sub = kb / (uint32_t)p.span_b, within = kb % (uint32_t)p.span_b;
                        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            const uint32_t off = sub * (uint32_t)p.b_sub_bytes +
                                                 swizzle_offset((uint32_t)(i4 + t) * (uint32_t)p.span_b + within, (uint32_t)p.span_b);
                            asm volatile("st.shared.f32 [%0], %1;" ::"r"(b_stage + off), "f"(vv[t]) : "memory");
                        }
                    }
                    fence_proxy_async_smem();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&full[stage]);
                } else if (lane == 0) {
                    mbar_arrive_expect_tx(&full[stage], (uint32_t)p.b_bytes);
                    for (int sb = 0; sb < p.b_subtiles; ++sb)
                        tma_load_2d(b_stage + sb * p.b_sub_bytes, &tmap_w, &full[stage],
                                    kw * p.w_inner_elems + sb * p.span_b_elems, 0);
                }
                __syncwarp();
                if (++stage == p.stages) { stage = 0; phase ^= 1u; }
            }
        }
    } else if (warp == TC_SCHED_WARP) {
        // ================================================= tile scheduler + gather-index blocks
        // A free index buffer is the permission to look ONE tile ahead: the ticket for entry n is
        // drawn only when the buffer of entry n-2 has been released, so a CTA never hoards tiles
        // and the tail of the kernel is at most one (light) tile long.
        const uint32_t blk_bytes = (uint32_t)(p.kv + 1) * 512u;
        for (int n = 0;; ++n) {
            const int b = n & 1, e = n & (TC_INFO_DEPTH - 1);
            mbar_wait_silent(&idx_empty[b], (uint32_t)(((n >> 1) & 1) ^ 1));
            mbar_wait_silent(&info_empty[e], (uint32_t)(((n / TC_INFO_DEPTH) & 1) ^ 1));
            int tile = -1;
            if (lane == 0) {
                const int ticket = atomicAdd(p.sched_state, 1);
                int4 r0 = make_int4(-1, 1, 0, 0), r1 = make_int4(0, 0, 0, 0);
                if ((int64_t)ticket < num_tiles) {
                    const int4 *rp = reinterpret_cast<const int4 *>(p.sched_rec + (int64_t)ticket * TT_REC_INTS);
                    r0 = __ldg(rp); r1 = __ldg(rp + 1);
                }
                tile = r0.x;
                int32_t *dst = info + e * 8;
                dst[0] = r0.x; dst[1] = r0.y; dst[2] = r0.z; dst[3] = r0.w; dst[4] = r1.x;
                if (tile >= 0) {
                    mbar_arrive_expect_tx(&idx_full[b], blk_bytes);
                    bulk_copy_g2s(smem_base + idx_off + (uint32_t)b * p.idx_bytes,
                                  p.tile_table + (int64_t)tile * (p.kv + 1) * 128, blk_bytes, &idx_full[b]);
                }
                mbar_arrive(&info_full[e]);          // release: publishes the record written above
            }
            tile = __shfl_sync(0xffffffffu, tile, 0);
            if (tile < 0) break;
        }
        // the last CTA to run dry leaves the scheduler state zeroed for the next launch
        if (lane == 0) {
            __threadfence();
            const int done = atomicAdd(p.sched_state + 1, 1);
            if (done == (int)gridDim.x - 1) {
                p.sched_state[0] = 0;
                p.sched_state[1] = 0;
                __threadfence();
            }
        }
        __syncwarp();
    } else if (warp < TC_CONS_WARPS) {
        // ================================================= consumers: warpgroup wg owns tile rows 64 wg .. 64 wg + 63
        const int wg = warp >> 2;
        int stage = 0; uint32_t phase = 0;
        const uint64_t a_hi = gmma_desc_hi(16u, 8u * SPAN_A, SPAN_A);
        // MN-major B: LBO = distance between swizzle-wide column blocks (sub-tiles), SBO = 8 K rows
        const uint64_t b_hi = p.b_mn_major ? gmma_desc_hi((uint32_t)p.b_sub_bytes, 8u * p.span_b, p.span_b)
                                           : gmma_desc_hi(16u, 8u * p.span_b, p.span_b);
        const uint32_t b_sub16 = (uint32_t)p.b_sub_bytes >> 4;
        Acc acc[N / 2];
        // e4m3: the FP8 MMA adds each k-step's products with about 14 bits kept, aligned to the largest
        // addend, so a large running sum would swallow the small products of later offsets.  Each offset's
        // k-steps (at most 8) therefore start from zero in `acc`, and the finished offset is added into `sum`
        // in fp32 registers (DeepSeek-V3 report section 3.3.2 promotes every 128 channels the same way).
        float sum[KIND == KIND_E4M3 ? N / 2 : 1];
        for (int local = 0;; ++local) {
            uint32_t tm[4];
            const int tile = read_info(local, tm);
            if (tile < 0) break;
            // destination rows of this thread's two fragment rows: row kv of the tile's index block is
            // the argsort row (-1 past the end); the block is released right after
            int32_t d_lo, d_hi;
            {
                const int buf = local & 1;
                mbar_wait_silent(&idx_full[buf], (uint32_t)((local >> 1) & 1));
                const int32_t *dst = reinterpret_cast<const int32_t *>(smem + idx_off + (size_t)buf * p.idx_bytes) +
                                     p.kv * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
                d_lo = dst[0];
                d_hi = dst[8];
                __syncwarp();
                if (lane == 0) mbar_arrive(&idx_empty[buf]);
            }
#pragma unroll
            for (int i = 0; i < N / 2; ++i) acc[i] = (Acc)0;
            if constexpr (KIND == KIND_E4M3) {
#pragma unroll
                for (int i = 0; i < N / 2; ++i) sum[i] = 0.f;
            }
            BitIter it(tm);
            // One wgmma group stays in flight across stages: stage s is released once the group of
            // stage s+1 is issued (wait_group 1), so the next stage's full-barrier wait and MMA issue
            // overlap the current MMAs.  Groups of one warpgroup retire in issue order, so every row
            // still sums its offsets in ascending order.
            int held = -1;                    // stage whose wgmma group may still be reading it
            for (int k = it.next(); k >= 0; k = it.next()) {
                mbar_wait_silent(&full[stage], phase);
                fence_proxy_async_smem();     // cp.async (generic proxy) writes -> wgmma operand reads
                const uint32_t a16 = (smem_base + (uint32_t)stage * p.stage_bytes + (uint32_t)(wg * 64 * SPAN_A)) >> 4;
                const uint32_t b16 = (smem_base + (uint32_t)stage * p.stage_bytes + (uint32_t)p.a_stage_bytes) >> 4;
                fence_regs(acc);
                wgmma_fence();
                if (!p.b_mn_major) {
#pragma unroll
                    for (int sub = 0; sub < A_SUBTILES; ++sub) {
                        const uint32_t as = a16 + (uint32_t)sub * (uint32_t)(A_SUB_BYTES >> 4);
                        const uint32_t bs = b16 + (uint32_t)sub * b_sub16;
#pragma unroll
                        for (int jr = 0; jr < Q_A; ++jr)
                            mma_step<KIND, N>(acc, a_hi | (uint64_t)((as + 2u * jr) & 0x3FFFu),
                                              b_hi | (uint64_t)((bs + 2u * jr) & 0x3FFFu), 0, p.ab_bf16);
                    }
                } else {
#pragma unroll
                    for (int sub = 0; sub < A_SUBTILES; ++sub) {
                        const uint32_t as = a16 + (uint32_t)sub * (uint32_t)(A_SUB_BYTES >> 4);
#pragma unroll
                        for (int jr = 0; jr < Q_A; ++jr) {
                            const uint32_t j = (uint32_t)(sub * Q_A + jr);
                            mma_step<KIND, N>(acc, a_hi | (uint64_t)((as + 2u * jr) & 0x3FFFu),
                                              b_hi | (uint64_t)((b16 + j * (uint32_t)p.b_kstep16_mn) & 0x3FFFu), 1,
                                              p.ab_bf16);
                        }
                    }
                }
                wgmma_commit();
                if constexpr (KIND == KIND_E4M3) {
                    // promote: the offset's group must finish before its sum leaves the accumulator
                    wgmma_wait<0>();
                    fence_regs(acc);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[stage]);
#pragma unroll
                    for (int i = 0; i < N / 2; ++i) {
                        sum[i] = __fadd_rn(sum[i], acc[i]);
                        acc[i] = 0.f;
                    }
                } else {
                    wgmma_wait<1>();
                    fence_regs(acc);
                    if (held >= 0) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty[held]);      // this warp is done reading that stage
                    }
                    held = stage;
                }
                if (++stage == p.stages) { stage = 0; phase ^= 1u; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (held >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[held]);
            }
            if constexpr (KIND == KIND_F16) {
                if (p.out_dtype == SPX_F16) epilogue_frag<SPX_F16, false, N, Acc, false, GROUPED>(p, ec, acc, d_lo, d_hi, lane);
                else epilogue_frag<SPX_BF16, false, N, Acc, false, GROUPED>(p, ec, acc, d_lo, d_hi, lane);
            } else if constexpr (KIND == KIND_TF32) {
                epilogue_frag<SPX_F32, false, N>(p, ec, acc, d_lo, d_hi, lane);
            } else if constexpr (KIND == KIND_I8) {
                if (p.out_dtype == SPX_I8) epilogue_frag<SPX_I8, true, N>(p, ec, acc, d_lo, d_hi, lane);
                else if (p.out_dtype == SPX_F32) epilogue_frag<SPX_F32, true, N>(p, ec, acc, d_lo, d_hi, lane);
                else epilogue_frag<SPX_F16, true, N>(p, ec, acc, d_lo, d_hi, lane);
            } else {
                const float add_s = p.add_scale ? __ldg(p.add_scale) : 1.f;
                const float out_s = p.out_dtype == SPX_E4M3 ? __ldg(p.out_scale) : 1.f;
                if (p.out_dtype == SPX_E4M3) epilogue_fp8<SPX_E4M3, N>(p, ec, sum, d_lo, d_hi, lane, add_s, out_s);
                else if (p.out_dtype == SPX_F32) epilogue_fp8<SPX_F32, N>(p, ec, sum, d_lo, d_hi, lane, add_s, out_s);
                else if (p.out_dtype == SPX_F16) epilogue_fp8<SPX_F16, N>(p, ec, sum, d_lo, d_hi, lane, add_s, out_s);
                else epilogue_fp8<SPX_BF16, N>(p, ec, sum, d_lo, d_hi, lane, add_s, out_s);
            }
        }
    }

    __syncthreads();
}

template <int KIND, int CPR, int N>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gather_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const TcParams p) {
    tc_gather_gemm_body<KIND, CPR, N>(tmap_w, p);
}

template <int CPR, int N>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gather_gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_w, const TcParams p) {
    tc_gather_gemm_body<KIND_E4M3, CPR, N>(tmap_w, p);
}

template <int CPR, int N>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_grouped_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const TcParams p) {
    tc_gather_gemm_body<KIND_F16, CPR, N, true>(tmap_w, p);
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}

// 2-D view of the KRSC filter: inner = kv*c_in elements, outer = c_out rows
int make_weight_tmap(CUtensorMap *tm, const void *w, int dtype, int kv, int c_in, int c_out, int span_bytes) {
    EncodeTiledFn fn = get_encode_fn();
    SPX_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (driver too old?)");
    const int e = dtype_bytes(dtype);
    CUtensorMapDataType dt = dtype == SPX_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                           : dtype == SPX_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                           : dtype == SPX_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                              : CU_TENSOR_MAP_DATA_TYPE_UINT8;
    cuuint64_t dims[2] = {(cuuint64_t)kv * c_in, (cuuint64_t)c_out};
    cuuint64_t strides[1] = {(cuuint64_t)kv * c_in * e};
    cuuint32_t box[2] = {(cuuint32_t)(span_bytes / e), (cuuint32_t)c_out};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMapSwizzle sw = span_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : span_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                             : CU_TENSOR_MAP_SWIZZLE_32B;
    CUresult r = fn(tm, dt, 2, const_cast<void *>(w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SPX_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with %d (kv=%d C=%d K=%d span=%d)", (int)r, kv, c_in,
                c_out, span_bytes);
    return 0;
}

// row bytes the kernels tile: one swizzle span (32/64/128 B) or a power-of-two multiple of 128 B
static bool span_ok(int bytes) { return bytes == 32 || bytes == 64 || bytes == 128 || bytes == 256 || bytes == 512; }

static bool tc_shape_ok(int dtype, int kv, int c_in, int c_out, int transpose_w) {
    const int e = dtype_bytes(dtype);
    if (e == 0) return false;
    if (c_in > 256 || c_out > 256) return false;
    if (c_in % 16 || c_out % 16) return false;
    if (!span_ok(c_in * e) || !span_ok(c_out * e)) return false;
    const int cy = transpose_w ? c_in : c_out;
    if (cy % 16 || cy > 256) return false;
    const int xb = (transpose_w ? c_out : c_in) * e;
    if ((dtype == SPX_I8 || dtype == SPX_E4M3) && (c_in % 32 || c_out % 32)) return false;   // docs/INT8_GUIDE.md:10; wgmma e4m3: K = 32
    size_t stage = align_up((size_t)TC_TILE_M * xb, 1024) + align_up((size_t)c_in * c_out * e, 1024);
    const size_t idx = align_up((size_t)(kv + 1) * 512, 1024);
    if (2 * idx + 2 * stage > (size_t)TC_SMEM_BUDGET) return false;
    return true;
}

// The producers gather x rows with 16-byte cp.async, the weight slice comes through a tensor map (or as
// float4 for the fp32 input gradient) and the epilogue stores column pairs: a call whose x, w or y is not
// 16-byte aligned runs on the FMA kernels, which access them element by element.
static bool tc_operands_aligned(const GatherGemmArgs &a) { return aligned16(a.x) && aligned16(a.w) && aligned16(a.y); }

bool tc_gather_gemm_supported(const GatherGemmArgs &a) {
    if (a.dtype == SPX_I8) return false;
    if (!a.tile_table || !a.tile_mask) return false;   // built by spx_build_tile_table
    if (!tc_operands_aligned(a)) return false;
    // tf32 input gradient: the weight loader writes the filter slice transposed (tf32 wgmma reads K-major
    // operands only); it is served for whole 128-byte filter rows, otherwise fp32 dgrad runs on the FMA
    // kernel; spx_debug_configure bit 256 switches the tensor-core route off (A/B against the FMA kernel).
    if (a.dtype == SPX_F32 && a.transpose_w && (runtime_cfg().tf32_dgrad_fma || (a.c_in * 4) % 128)) return false;
    if (((size_t)a.kv * a.c_in * dtype_bytes(a.dtype)) % 16) return false;
    return tc_shape_ok(a.dtype, a.kv, a.c_in, a.c_out, a.transpose_w);
}
bool tc_gather_gemm_int8_supported(const Int8Args &q) {
    if (!q.g.tile_table || !q.g.tile_mask) return false;
    if (!tc_operands_aligned(q.g)) return false;
    if (((size_t)q.g.kv * q.g.c_in) % 16) return false;
    return tc_shape_ok(SPX_I8, q.g.kv, q.g.c_in, q.g.c_out, 0);
}

bool tc_gather_gemm_fp8_supported(const Fp8Args &q) {
    if (!q.g.tile_table || !q.g.tile_mask) return false;
    if (!tc_operands_aligned(q.g)) return false;
    if (((size_t)q.g.kv * q.g.c_in) % 16) return false;
    return tc_shape_ok(SPX_E4M3, q.g.kv, q.g.c_in, q.g.c_out, 0);
}

static int fill_params(const GatherGemmArgs &a, TcParams &p) {
    memset(&p, 0, sizeof(p));
    const int e = dtype_bytes(a.dtype);
    const int cx = a.cx(), cy = a.cy();
    p.x = (const uint8_t *)a.x;
    p.xb = cx * e;
    const int span_a = p.xb < 128 ? p.xb : 128;
    const int wb = a.c_in * e;                 // inner (contiguous) bytes of one weight slice row
    p.b_transposed = (a.dtype == SPX_F32 && a.transpose_w) ? 1 : 0;
    if (p.b_transposed) {
        // K-major [c_in rows x c_out] written by the weight loader, cut into the A operand's K sub-tiles
        p.span_b = span_a;
        p.b_subtiles = p.xb / span_a;
        p.b_sub_bytes = cy * span_a;
        p.b_mn_major = 0;
    } else {
        p.span_b = wb < 128 ? wb : 128;
        p.b_subtiles = wb / p.span_b;
        p.b_sub_bytes = a.c_out * p.span_b;
        p.b_mn_major = a.transpose_w;
    }
    p.b_bytes = a.c_out * wb;
    p.b_kstep16_mn = ((32 / e) * p.span_b) >> 4;   // one k-step = 32 bytes of contraction = 32/e rows of the weight box
    p.w = (const float *)a.w;
    p.c_in = a.c_in; p.c_out = a.c_out;
    p.w_inner_elems = a.c_in;
    p.span_b_elems = p.span_b / e;
    p.n = cy;
    p.ab_bf16 = a.dtype == SPX_BF16;
    p.a_stage_bytes = (int)align_up((size_t)TC_TILE_M * p.xb, 1024);
    p.stage_bytes = p.a_stage_bytes + (int)align_up((size_t)p.b_bytes, 1024);
    p.idx_bytes = (int)align_up((size_t)(a.kv + 1) * 512, 1024);
    p.stages = (TC_SMEM_BUDGET - 2 * p.idx_bytes) / p.stage_bytes;
    if (p.stages > TC_MAX_STAGES) p.stages = TC_MAX_STAGES;
    SPX_REQUIRE(p.stages >= 2, "tc_gather_gemm: tile does not fit shared memory (stage %d bytes)", p.stage_bytes);
    p.rows = a.rows; p.tile_table = a.tile_table; p.argsort = a.argsort;
    {
        const int64_t tiles = div_up64(a.rows, TC_TILE_M);
        p.sched_rec = a.tile_table + tt_blocks_elems(tiles, a.kv);
        // scheduler scratch lives in the caller's tile-table buffer (include/spconv_b200.h): TT_STATE_INTS / 2
        // {ticket, finished} pairs.  Every launch takes the next pair, so launches that overlap on the
        // same rulebook (two layers sharing an indice_key on different streams, graph branches) never
        // draw from one counter; a pair is zero when its launch ends.
        static std::atomic<unsigned> next_slot{0};
        const unsigned slot = next_slot.fetch_add(1, std::memory_order_relaxed) % (TT_STATE_INTS / 2);
        p.sched_state = const_cast<int *>(reinterpret_cast<const int *>(p.sched_rec + tiles * TT_REC_INTS)) + 2 * slot;
    }
    p.kv = a.kv; p.words = (a.kv + 31) / 32; p.reverse = a.reverse;
    p.y = a.y; p.out_dtype = a.dtype; p.epi_mode = 0; p.bias = a.bias; p.act = a.act; p.alpha = a.alpha;
    return 0;
}

template <int KIND, int CPR, int N, bool GROUPED>
static int launch_tc_n(const CUtensorMap &tm, const TcParams &p, cudaStream_t stream) {
    void (*kernel)(const CUtensorMap, const TcParams);
    if constexpr (GROUPED) kernel = tc_grouped_gemm_kernel<CPR, N>;
    else if constexpr (KIND == KIND_E4M3) kernel = tc_gather_gemm_fp8_kernel<CPR, N>;
    else kernel = tc_gather_gemm_kernel<KIND, CPR, N>;
    const size_t smem = (size_t)p.stages * p.stage_bytes + 2 * (size_t)p.idx_bytes + 1024 /*align slack*/ + 1024 /*barriers, tile-info ring*/ +
                        2 * N * sizeof(float) /*epilogue constants*/;
    // the opt-in is a per-DEVICE attribute: one process may drive several GPUs
    if (!func_configured((const void *)kernel, current_device())) {
        SPX_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)(TC_SMEM_BUDGET + 2048 + 2 * N * sizeof(float))));
        SPX_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    }
    const int64_t tiles = div_up64(p.rows, TC_TILE_M);
    const int64_t max_ctas = (int64_t)sm_count();
    const int grid = (int)(tiles < max_ctas ? tiles : max_ctas);
    kernel<<<grid, TC_THREADS, smem, stream>>>(tm, p);
    SPX_CHECK_LAUNCH(GROUPED ? "tc_grouped_gemm_kernel" : KIND == KIND_E4M3 ? "tc_gather_gemm_fp8_kernel" : "tc_gather_gemm_kernel");
    return 0;
}

// instantiated (channels x element bytes) combinations: rows of 32..512 bytes, N = 16..256 output
// channels (tf32: 16..128, int8: 32..256, e4m3: 32..128).  512-byte rows (CPR = 32) stop at N = 64: a 64 KB
// gathered tile plus a weight slice of 128 or more rows puts two stages over TC_SMEM_BUDGET.  The grouped
// (16-bit) instances cover the same (CPR, N) set as the dense 16-bit ones.
template <int KIND, int CPR, bool GROUPED>
static int launch_tc_cpr(const CUtensorMap &tm, const TcParams &p, cudaStream_t stream) {
    switch (p.n) {
        case 16: if constexpr (KIND != KIND_I8 && KIND != KIND_E4M3) return launch_tc_n<KIND, CPR, 16, GROUPED>(tm, p, stream); break;
        case 32: return launch_tc_n<KIND, CPR, 32, GROUPED>(tm, p, stream);
        case 64: return launch_tc_n<KIND, CPR, 64, GROUPED>(tm, p, stream);
        case 128: if constexpr (CPR != 32) return launch_tc_n<KIND, CPR, 128, GROUPED>(tm, p, stream); break;
        case 256: if constexpr (KIND != KIND_TF32 && KIND != KIND_E4M3 && CPR != 32) return launch_tc_n<KIND, CPR, 256, GROUPED>(tm, p, stream); break;
    }
    set_error("tc_gather_gemm: unsupported output channel count %d", p.n);
    return 2;
}

template <int KIND, bool GROUPED = false>
static int launch_tc(const CUtensorMap &tm, const TcParams &p, cudaStream_t stream) {
    static_assert(!GROUPED || KIND == KIND_F16, "grouped instances are 16-bit only");
    switch (p.xb >> 4) {
        case 2: if constexpr (KIND != KIND_TF32) return launch_tc_cpr<KIND, 2, GROUPED>(tm, p, stream); break;
        case 4: return launch_tc_cpr<KIND, 4, GROUPED>(tm, p, stream);
        case 8: return launch_tc_cpr<KIND, 8, GROUPED>(tm, p, stream);
        case 16: return launch_tc_cpr<KIND, 16, GROUPED>(tm, p, stream);
        case 32: if constexpr (KIND != KIND_I8 && KIND != KIND_E4M3) return launch_tc_cpr<KIND, 32, GROUPED>(tm, p, stream); break;
    }
    set_error("tc_gather_gemm: unsupported row bytes %d", p.xb);
    return 2;
}

// ldx != 0: one group of a grouped conv (16-bit only); the tensor map covers the group's [c_out, kv * c_in] filter
// block, which is contiguous in the grouped filter
int tc_gather_gemm(const GatherGemmArgs &a, cudaStream_t stream, int64_t ldx, int64_t ldy) {
    TcParams p;
    if (fill_params(a, p)) return 2;
    CUtensorMap tm;
    if (make_weight_tmap(&tm, a.w, a.dtype, a.kv, a.c_in, a.c_out, p.b_transposed ? 128 : p.span_b)) return 2;
    if (ldx) {
        SPX_REQUIRE(a.dtype == SPX_F16 || a.dtype == SPX_BF16, "tc_gather_gemm: grouped calls are 16-bit only");
        p.ldx = (int)ldx * dtype_bytes(a.dtype);
        p.ldy = (int)ldy;
        return launch_tc<KIND_F16, true>(tm, p, stream);
    }
    if (a.dtype == SPX_F32) return launch_tc<KIND_TF32>(tm, p, stream);
    return launch_tc<KIND_F16>(tm, p, stream);
}

int tc_gather_gemm_int8(const Int8Args &q, cudaStream_t stream) {
    TcParams p;
    if (fill_params(q.g, p)) return 2;
    p.out_dtype = q.out_dtype;
    p.epi_mode = 1;
    p.scale = q.scale; p.bias_f32 = q.bias_f32; p.output_add = q.output_add;
    p.output_add_scale = q.output_add_scale;
    CUtensorMap tm;
    if (make_weight_tmap(&tm, q.g.w, SPX_I8, q.g.kv, q.g.c_in, q.g.c_out, p.span_b)) return 2;
    return launch_tc<KIND_I8>(tm, p, stream);
}

// e4m3 operands take the int8 operand path (1-byte K-major rows, UINT8 tensor map) with fp32 accumulators.
// The fp32 sum beside the wgmma accumulator takes N / 2 more registers per consumer thread, which N = 256
// cannot spare: 256 output channels run as two passes of 128, each over its half of the filter rows, scales,
// biases, output and residual columns.
int tc_gather_gemm_fp8(const Fp8Args &q, cudaStream_t stream) {
    const int half = q.g.c_out > 128 ? 2 : 1;
    const int n = q.g.c_out / half;
    const int ob = dtype_bytes(q.out_dtype);
    for (int h = 0; h < half; ++h) {
        GatherGemmArgs g = q.g;
        g.c_out = n;
        g.w = (const uint8_t *)q.g.w + (size_t)h * n * q.g.kv * q.g.c_in;
        g.y = (uint8_t *)q.g.y + (size_t)h * n * ob;
        TcParams p;
        if (fill_params(g, p)) return 2;
        p.out_dtype = q.out_dtype;
        p.epi_mode = 2;
        p.scale = q.w_scale + h * n;
        p.bias_f32 = q.bias_f32 ? q.bias_f32 + h * n : nullptr;
        p.output_add = q.output_add ? (const int8_t *)q.output_add + (size_t)h * n * ob : nullptr;
        p.in_scale = q.in_scale; p.add_scale = q.add_scale; p.out_scale = q.out_scale;
        p.ldy = q.g.c_out;
        CUtensorMap tm;
        if (make_weight_tmap(&tm, g.w, SPX_E4M3, g.kv, g.c_in, g.c_out, p.span_b)) return 2;
        if (int rc = launch_tc<KIND_E4M3>(tm, p, stream)) return rc;
    }
    return 0;
}

}  // namespace spx
