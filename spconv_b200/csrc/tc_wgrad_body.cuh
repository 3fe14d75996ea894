// Not a header: included inside the two kernels below, see gemm_tc_wgrad.cu.
// The body of tc_wgrad_kernel (dense) and tc_grouped_wgrad_kernel (16-bit, one group of a grouped conv), included
// inside both so the dense kernel is compiled exactly as a kernel of its own.  In scope: CPA, CPD, TF32, the
// parameters p, and GROUPED: with GROUPED, x rows are p.ldx bytes apart and dout rows p.ldd; everything else is the
// dense instance.
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
                    cp_async_16(dstb + off, d_lane + (int64_t)max(rsrc[itc], 0) * (GROUPED ? p.ldd : DB), rsrc[itc] >= 0 ? 16u : 0u);
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
                            cp_async_16(atom_base + dst_off[itc], x_atom + (int64_t)max(ridx[itc], 0) * (GROUPED ? p.ldx : p.xb),
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
