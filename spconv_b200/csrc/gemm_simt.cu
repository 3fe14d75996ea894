// Generic fp32-FMA kernels for the gather-GEMM-scatter path: any channel counts, any of
// fp32 / fp16 / bf16 / int8 / e4m3, fp32 (int32 for int8) accumulation.
//
// These serve (a) exact fp32 arithmetic, the reference default for fp32 tensors
// (SPCONV_ALLOW_TF32=False, spconv/constants.py:117), and (b) layer shapes the tcgen05
// kernels in gemm_tc.cu do not tile (e.g. the C_in = 3..5 stem layer).  They implement the
// same masked implicit-GEMM contract as ConvMain::implicit_gemm2's call sites
// (spconv/csrc/sparse/convops.py:2196-2235, :2394-2436): visit rows in mask_argsort order,
// skip kernel offsets whose bit is clear in the OR of the tile's masks, gather through the
// pair table (-1 = zero row).
#include "gemm.cuh"

namespace spx {

constexpr int S_TM = 32;    // rows per block
constexpr int S_TN = 64;    // output channels per pass
constexpr int S_TK = 32;    // contraction chunk
constexpr int S_THREADS = 256;

template <typename T> struct AccT { typedef float type; };
template <> struct AccT<int8_t> { typedef int type; };

template <typename T> __device__ __forceinline__ typename AccT<T>::type load_acc(const T *p) { return to_float(*p); }
template <> __device__ __forceinline__ int load_acc<int8_t>(const int8_t *p) { return (int)*p; }
template <> __device__ __forceinline__ float load_acc<__nv_fp8_e4m3>(const __nv_fp8_e4m3 *p) {
    return e4m3_to_float(p->__x);
}

struct SimtEpilogue {   // float path: bias+act ; int8 path: scale/bias/add/act/round
    int mode;           // 0 float, 1 int8, 2 fp8
    const void *bias;
    int act;
    float alpha;
    const float *scale, *bias_f32;
    const int8_t *output_add;
    float output_add_scale;
    int out_dtype;
    // fp8 (T = __nv_fp8_e4m3): scale = w_scale, bias_f32 = bias; the residual in out_dtype
    const float *in_scale, *add_scale, *out_scale;
    const void *add;
};

// the fp8 epilogue (gemm.cuh fp8_epilogue) of one thread's 8 columns y0.. of output row dst, stored as out_dtype
template <int OUT>
__device__ __forceinline__ void simt_fp8_cols(const SimtEpilogue &ep, void *y, const float (&acc)[8], int64_t dst, int y0,
                                           int cy) {
    const float add_s = ep.add_scale ? *ep.add_scale : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int col = y0 + j;
        if (col >= cy) continue;
        const int64_t o = dst * cy + col;
        const float s = __fmul_rn(*ep.in_scale, ep.scale[col]);      // s_j = in_scale * w_scale[j]
        const float a = ep.add ? load_out_elem<OUT>(ep.add, o) : 0.f;
        const float v = fp8_epilogue(acc[j], s, ep.bias_f32, col, ep.add != nullptr, a, add_s, ep.act, ep.alpha);
        if constexpr (OUT == SPX_E4M3) ((uint8_t *)y)[o] = float_to_e4m3(__fdiv_rn(v, *ep.out_scale));
        else if constexpr (OUT == SPX_F32) ((float *)y)[o] = v;
        else if constexpr (OUT == SPX_F16) ((__half *)y)[o] = __float2half_rn(v);
        else ((__nv_bfloat16 *)y)[o] = __float2bfloat16_rn(v);
    }
}

template <typename T>
__global__ void __launch_bounds__(S_THREADS)
simt_gather_gemm_kernel(GatherGemmArgs a, SimtEpilogue ep) {
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
                    if (idx >= 0 && x0 + x < cx) v = load_acc<T>(X + (int64_t)idx * cx + x0 + x);
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
                int64_t o = (int64_t)dst * cy + y;
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
}

template <typename T>
static int launch_simt(const GatherGemmArgs &a, const SimtEpilogue &ep, cudaStream_t stream) {
    if (a.rows == 0) return 0;
    unsigned nblk = (unsigned)div_up64(a.rows, S_TM);
    simt_gather_gemm_kernel<T><<<nblk, S_THREADS, 0, stream>>>(a, ep);
    SPX_CHECK_LAUNCH("simt_gather_gemm_kernel");
    return 0;
}

int simt_gather_gemm(const GatherGemmArgs &a, cudaStream_t stream) {
    SimtEpilogue ep;
    memset(&ep, 0, sizeof(ep));
    ep.mode = 0; ep.bias = a.bias; ep.act = a.act; ep.alpha = a.alpha;
    switch (a.dtype) {
        case SPX_F32: return launch_simt<float>(a, ep, stream);
        case SPX_F16: return launch_simt<__half>(a, ep, stream);
        case SPX_BF16: return launch_simt<__nv_bfloat16>(a, ep, stream);
        default: set_error("simt_gather_gemm: unsupported dtype %d", a.dtype); return 2;
    }
}

int simt_gather_gemm_int8(const Int8Args &q, cudaStream_t stream) {
    SimtEpilogue ep;
    memset(&ep, 0, sizeof(ep));
    ep.mode = 1; ep.act = q.g.act; ep.alpha = q.g.alpha;
    ep.scale = q.scale; ep.bias_f32 = q.bias_f32; ep.output_add = q.output_add;
    ep.output_add_scale = q.output_add_scale; ep.out_dtype = q.out_dtype;
    return launch_simt<int8_t>(q.g, ep, stream);
}

int simt_gather_gemm_fp8(const Fp8Args &q, cudaStream_t stream) {
    SimtEpilogue ep;
    memset(&ep, 0, sizeof(ep));
    ep.mode = 2; ep.act = q.g.act; ep.alpha = q.g.alpha; ep.out_dtype = q.out_dtype;
    ep.scale = q.w_scale; ep.bias_f32 = q.bias_f32; ep.in_scale = q.in_scale;
    ep.add = q.output_add; ep.add_scale = q.add_scale; ep.out_scale = q.out_scale;
    return launch_simt<__nv_fp8_e4m3>(q.g, ep, stream);
}

// ------------------------------------------------------------------ weight gradient
// dW[n][k][c] = sum_o dout[o][n] * x[pair[k][o]][c]; one block per (k, 16x16 (n,c) tile),
// fp32 accumulation over all rows in ascending order (deterministic).
constexpr int WG_T = 16;
constexpr int WG_ROWS = 64;

template <typename T>
__global__ void __launch_bounds__(WG_T *WG_T)
simt_wgrad_kernel(WgradArgs a) {
    __shared__ float Ds[WG_ROWS][WG_T + 1];
    __shared__ float Xs[WG_ROWS][WG_T + 1];
    __shared__ int32_t idx_s[WG_ROWS];
    const int k = blockIdx.z;
    const int n0 = blockIdx.y * WG_T, c0 = blockIdx.x * WG_T;
    const int tn = threadIdx.y, tc = threadIdx.x;
    const int tid = tn * WG_T + tc;
    const T *X = (const T *)a.x;
    const T *D = (const T *)a.dout;
    float acc = 0.f;
    for (int64_t r0 = 0; r0 < a.n_out; r0 += WG_ROWS) {
        if (tid < WG_ROWS) {
            int64_t r = r0 + tid;
            idx_s[tid] = r < a.n_out ? a.pair[(int64_t)k * a.pair_stride + r] : -1;
        }
        __syncthreads();
        for (int e = tid; e < WG_ROWS * WG_T; e += WG_T * WG_T) {
            int r = e / WG_T, j = e % WG_T;
            int32_t idx = idx_s[r];
            float dv = 0.f, xv = 0.f;
            if (idx >= 0) {
                if (n0 + j < a.c_out) dv = to_float(D[(r0 + r) * a.c_out + n0 + j]);
                if (c0 + j < a.c_in) xv = to_float(X[(int64_t)idx * a.c_in + c0 + j]);
            }
            Ds[r][j] = dv;
            Xs[r][j] = xv;
        }
        __syncthreads();
#pragma unroll 16
        for (int r = 0; r < WG_ROWS; ++r) acc += Ds[r][tn] * Xs[r][tc];
        __syncthreads();
    }
    if (n0 + tn < a.c_out && c0 + tc < a.c_in)
        ((T *)a.dw)[((int64_t)(n0 + tn) * a.kv + k) * a.c_in + c0 + tc] = from_float<T>(acc);
}

int simt_wgrad(const WgradArgs &a, cudaStream_t stream) {
    dim3 grid((a.c_in + WG_T - 1) / WG_T, (a.c_out + WG_T - 1) / WG_T, a.kv);
    dim3 block(WG_T, WG_T);
    switch (a.dtype) {
        case SPX_F32: simt_wgrad_kernel<float><<<grid, block, 0, stream>>>(a); break;
        case SPX_F16: simt_wgrad_kernel<__half><<<grid, block, 0, stream>>>(a); break;
        case SPX_BF16: simt_wgrad_kernel<__nv_bfloat16><<<grid, block, 0, stream>>>(a); break;
        default: set_error("simt_wgrad: unsupported dtype %d", a.dtype); return 2;
    }
    SPX_CHECK_LAUNCH("simt_wgrad_kernel");
    return 0;
}

}  // namespace spx
