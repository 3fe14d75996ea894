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
    constexpr bool GROUPED = false;
    constexpr int64_t ldx = 0, ldy = 0;
#include "simt_gather_body.cuh"
}

template <typename T>
__global__ void __launch_bounds__(S_THREADS)
simt_grouped_gemm_kernel(GatherGemmArgs a, SimtEpilogue ep, int ldx, int ldy) {
    constexpr bool GROUPED = true;
#include "simt_gather_body.cuh"
}

template <typename T>
static int launch_simt(const GatherGemmArgs &a, const SimtEpilogue &ep, cudaStream_t stream, int64_t ldx = 0,
                       int64_t ldy = 0) {
    if (a.rows == 0) return 0;
    unsigned nblk = (unsigned)div_up64(a.rows, S_TM);
    if constexpr (std::is_same<T, float>::value || std::is_same<T, __half>::value ||
                  std::is_same<T, __nv_bfloat16>::value) {
        if (ldx) {
            simt_grouped_gemm_kernel<T><<<nblk, S_THREADS, 0, stream>>>(a, ep, (int)ldx, (int)ldy);
            SPX_CHECK_LAUNCH("simt_grouped_gemm_kernel");
            return 0;
        }
    }
    simt_gather_gemm_kernel<T><<<nblk, S_THREADS, 0, stream>>>(a, ep);
    SPX_CHECK_LAUNCH("simt_gather_gemm_kernel");
    return 0;
}

int simt_gather_gemm(const GatherGemmArgs &a, cudaStream_t stream, int64_t ldx, int64_t ldy) {
    SimtEpilogue ep;
    memset(&ep, 0, sizeof(ep));
    ep.mode = 0; ep.bias = a.bias; ep.act = a.act; ep.alpha = a.alpha;
    switch (a.dtype) {
        case SPX_F32: return launch_simt<float>(a, ep, stream, ldx, ldy);
        case SPX_F16: return launch_simt<__half>(a, ep, stream, ldx, ldy);
        case SPX_BF16: return launch_simt<__nv_bfloat16>(a, ep, stream, ldx, ldy);
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

// GROUPED: x rows are ldx elements apart and dout rows ldd (simt_grouped_wgrad_kernel, one group of a grouped conv)
template <typename T, bool GROUPED>
__device__ __forceinline__ void simt_wgrad_body(WgradArgs a, int64_t ldx, int64_t ldd) {
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
                if (n0 + j < a.c_out) dv = to_float(D[(r0 + r) * (GROUPED ? ldd : a.c_out) + n0 + j]);
                if (c0 + j < a.c_in) xv = to_float(X[(int64_t)idx * (GROUPED ? ldx : a.c_in) + c0 + j]);
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

template <typename T>
__global__ void __launch_bounds__(WG_T *WG_T)
simt_wgrad_kernel(WgradArgs a) {
    simt_wgrad_body<T, false>(a, 0, 0);
}

template <typename T>
__global__ void __launch_bounds__(WG_T *WG_T)
simt_grouped_wgrad_kernel(WgradArgs a, int64_t ldx, int64_t ldd) {
    simt_wgrad_body<T, true>(a, ldx, ldd);
}

template <typename T>
static void launch_simt_wgrad(const WgradArgs &a, dim3 grid, dim3 block, int64_t ldx, int64_t ldd, cudaStream_t stream) {
    if (ldx) simt_grouped_wgrad_kernel<T><<<grid, block, 0, stream>>>(a, ldx, ldd);
    else simt_wgrad_kernel<T><<<grid, block, 0, stream>>>(a);
}

int simt_wgrad(const WgradArgs &a, cudaStream_t stream, int64_t ldx, int64_t ldd) {
    dim3 grid((a.c_in + WG_T - 1) / WG_T, (a.c_out + WG_T - 1) / WG_T, a.kv);
    dim3 block(WG_T, WG_T);
    switch (a.dtype) {
        case SPX_F32: launch_simt_wgrad<float>(a, grid, block, ldx, ldd, stream); break;
        case SPX_F16: launch_simt_wgrad<__half>(a, grid, block, ldx, ldd, stream); break;
        case SPX_BF16: launch_simt_wgrad<__nv_bfloat16>(a, grid, block, ldx, ldd, stream); break;
        default: set_error("simt_wgrad: unsupported dtype %d", a.dtype); return 2;
    }
    SPX_CHECK_LAUNCH(ldx ? "simt_grouped_wgrad_kernel" : "simt_wgrad_kernel");
    return 0;
}

}  // namespace spx
