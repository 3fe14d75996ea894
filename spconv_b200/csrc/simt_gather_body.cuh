// Not a header: included inside the two kernels below, see gemm_simt.cu.
// The body of simt_gather_gemm_kernel (dense) and simt_grouped_gemm_kernel (one group of a grouped conv), included
// inside both (gemm_simt.cu) so the dense kernel is compiled exactly as a kernel of its own.  In scope: T, the
// arguments a and ep, and GROUPED / ldx / ldy: with GROUPED, gathered rows are ldx elements apart and output rows
// ldy (a column block of wider rows).
    typedef typename AccT<T>::type acc_t;
    __shared__ acc_t As[S_TM][S_TK + 1];
    __shared__ acc_t Bs[S_TK][S_TN + 1];
    __shared__ int32_t row_src[S_TM];     // source row (after argsort) of each tile row, -1 = out of range
    __shared__ int32_t row_idx[S_TM];     // gathered X row for the current offset
    __shared__ uint32_t tile_mask[4];

    const int tid = threadIdx.x;
    const int words = (a.kv + 31) / 32;
    const int cx = a.cx(), cy = a.cy();
    const T *X = (const T *)a.x;
    const T *W = (const T *)a.w;
    const int64_t w_sx = a.transpose_w ? (int64_t)a.kv * a.c_in : 1;   // stride of contraction channel
    const int64_t w_sy = a.transpose_w ? 1 : (int64_t)a.kv * a.c_in;   // stride of output channel
    const int64_t base = (int64_t)blockIdx.x * S_TM;

    if (tid < 4) tile_mask[tid] = 0;
    if (tid < S_TM) {
        int64_t r = base + tid;
        row_src[tid] = r < a.rows ? (a.argsort ? a.argsort[r] : (int32_t)r) : -1;
    }
    __syncthreads();
    if (tid < S_TM * words && tid / words < S_TM) {
        int r = tid / words, w = tid % words;
        if (base + r < a.rows) {
            uint32_t m;
            if (a.mask) m = a.mask[(base + r) * words + w];
            else {
                int hi = a.kv - 32 * w;
                m = hi >= 32 ? 0xffffffffu : ((1u << hi) - 1u);
            }
            atomicOr(&tile_mask[w], m);
        }
    }
    __syncthreads();

    const int trow = tid / 8;          // 0..31
    const int tcg = tid % 8;           // column group: columns tcg*8 .. tcg*8+7
    for (int n0 = 0; n0 < cy; n0 += S_TN) {
        acc_t acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0;
        for (int k = 0; k < a.kv; ++k) {
            if (!((tile_mask[k >> 5] >> (k & 31)) & 1u)) continue;
            const int kw = a.reverse ? a.kv - 1 - k : k;
            __syncthreads();
            if (tid < S_TM) {
                int32_t s = row_src[tid];
                row_idx[tid] = s >= 0 ? a.pair[(int64_t)k * a.pair_stride + s] : -1;
            }
            __syncthreads();
            for (int x0 = 0; x0 < cx; x0 += S_TK) {
                for (int e = tid; e < S_TM * S_TK; e += S_THREADS) {
                    int r = e / S_TK, x = e % S_TK;
                    int32_t idx = row_idx[r];
                    acc_t v = 0;
                    if (idx >= 0 && x0 + x < cx) v = load_acc<T>(X + (int64_t)idx * (GROUPED ? ldx : cx) + x0 + x);
                    As[r][x] = v;
                }
                for (int e = tid; e < S_TK * S_TN; e += S_THREADS) {
                    int x, y;
                    if (a.transpose_w) { x = e / S_TN; y = e % S_TN; }   // y contiguous in memory
                    else { y = e / S_TK; x = e % S_TK; }                 // x contiguous in memory
                    acc_t v = 0;
                    if (x0 + x < cx && n0 + y < cy)
                        v = load_acc<T>(W + (int64_t)(x0 + x) * w_sx + (int64_t)(n0 + y) * w_sy + (int64_t)kw * a.c_in);
                    Bs[x][y] = v;
                }
                __syncthreads();
#pragma unroll 8
                for (int x = 0; x < S_TK; ++x) {
                    acc_t av = As[trow][x];
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] += av * Bs[x][tcg * 8 + j];
                }
                __syncthreads();
            }
        }
        int32_t dst = row_src[trow];
        if constexpr (std::is_same<T, __nv_fp8_e4m3>::value) {
            if (dst >= 0) {
                switch (ep.out_dtype) {
                    case SPX_E4M3: simt_fp8_cols<SPX_E4M3>(ep, a.y, acc, dst, n0 + tcg * 8, cy); break;
                    case SPX_F32: simt_fp8_cols<SPX_F32>(ep, a.y, acc, dst, n0 + tcg * 8, cy); break;
                    case SPX_F16: simt_fp8_cols<SPX_F16>(ep, a.y, acc, dst, n0 + tcg * 8, cy); break;
                    default: simt_fp8_cols<SPX_BF16>(ep, a.y, acc, dst, n0 + tcg * 8, cy); break;
                }
            }
        } else if (dst >= 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                int y = n0 + tcg * 8 + j;
                if (y >= cy) continue;
                int64_t o = (int64_t)dst * (GROUPED ? ldy : cy) + y;
                if (ep.mode == 0) {
                    float v = (float)acc[j];
                    if (ep.bias) v += to_float(((const T *)ep.bias)[y]);
                    v = apply_act(v, ep.act, ep.alpha);
                    if constexpr (!std::is_same<T, int8_t>::value) ((T *)a.y)[o] = from_float<T>(v);
                } else {
                    // int8 inference epilogue: test/test_all_algo.py:272-287
                    float v = (float)acc[j] * ep.scale[y] + (ep.bias_f32 ? ep.bias_f32[y] : 0.f);
                    if (ep.output_add) v += (float)ep.output_add[o] * ep.output_add_scale;
                    v = apply_act(v, ep.act, ep.alpha);
                    if (ep.out_dtype == SPX_I8) {
                        float q = rintf(v);                         // round-half-even, as numpy
                        q = fminf(fmaxf(q, -128.f), 127.f);
                        ((int8_t *)a.y)[o] = (int8_t)q;
                    } else if (ep.out_dtype == SPX_F32) {
                        ((float *)a.y)[o] = v;
                    } else {
                        ((__half *)a.y)[o] = __float2half_rn(v);
                    }
                }
            }
        }
    }
