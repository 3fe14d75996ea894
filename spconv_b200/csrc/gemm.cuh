// Internal interface between the C-ABI dispatcher (api_gemm.cu) and the two kernel families
// (gemm_simt.cu: generic fp32-FMA kernels; gemm_tc.cu: tcgen05 / TMEM / TMA kernels).
#pragma once
#include "common.cuh"
#include <cuda_fp8.h>

namespace spx {

// y[r, :] = act( sum_k  X[pair[k][row(r)], :] * W_k'  + bias )        r in [0, rows)
//   row(r) = argsort ? argsort[r] : r ;  y row written = row(r)
//   W is the KRSC filter [c_out, kv, c_in]:
//     transpose_w == 0 (forward): X has c_in channels, y has c_out:  W_k'[x][y] = W[y][k'][x]
//     transpose_w == 1 (dgrad)  : X has c_out channels, y has c_in:  W_k'[x][y] = W[x][k'][y]
//   k' = reverse ? kv-1-k : k
struct GatherGemmArgs {
    int dtype, f32_mode, kv, c_in, c_out, transpose_w, reverse, act;
    float alpha;
    int64_t rows, x_rows;
    const void *x, *w, *bias;
    void *y;
    const int32_t *pair;
    int64_t pair_stride;
    const uint32_t *mask;      // [rows, words] in visiting order, or NULL
    const int32_t *argsort;    // [rows] or NULL
    const int32_t *tile_table; // [tiles][kv+1][128] or NULL (spx_build_tile_table)
    const uint32_t *tile_mask; // [tiles][words] or NULL
    __host__ __device__ int cx() const { return transpose_w ? c_out : c_in; }
    __host__ __device__ int cy() const { return transpose_w ? c_in : c_out; }
};

// dW[:, k, :] = sum_o dout[o, :]^T x[pair[k][o], :]
struct WgradArgs {
    int dtype, f32_mode, kv, c_in, c_out;
    int64_t n_in, n_out;
    const void *x, *dout;
    void *dw;
    const int32_t *pair;       // forward table [kv, n_out]
    int64_t pair_stride;
    const uint32_t *mask;      // [n_out, words] in visiting order or NULL
    const int32_t *argsort;    // [n_out] or NULL
    const int32_t *tile_table; // [tiles][kv+1][128] or NULL
    const uint32_t *tile_mask; // [tiles][words] or NULL
    void *workspace;
    size_t workspace_bytes;
    const spx_peer_group *peers;   // NULL, or: push this rank's fp32 dW to these ranks instead of writing dw
};

// Layout of the buffer spx_build_tile_table fills (int32 elements):
//   [tiles][kv+1][128]              gather blocks
//   [tiles][TT_REC_INTS]            schedule records {tile, mask[4], 0, 0, 0}, heaviest tile first
//   [TT_STATE_INTS]                 scheduler scratch: [0] ticket counter, [1] finished CTAs
//                                   (zero between launches; a launch leaves it zero again)
constexpr int TT_REC_INTS = 8;
constexpr int TT_STATE_INTS = 64;
__host__ __device__ inline int64_t tt_blocks_elems(int64_t tiles, int kv) { return tiles * (int64_t)(kv + 1) * 128; }
__host__ __device__ inline int64_t tt_total_elems(int64_t tiles, int kv) {
    return tt_blocks_elems(tiles, kv) + tiles * TT_REC_INTS + TT_STATE_INTS;
}

// ldx / ldy / ldd != 0: one group of a grouped conv (api_gemm.cu).  The args describe the group's dense
// (C / groups -> K / groups) GEMM, with x, w, y (bias, dout, dw) already at the group's column block, filter rows
// and bias; gathered x rows are ldx elements apart, output rows ldy and dout rows ldd.  The grouped instances
// run the dense instance's schedule and summation order: only the row addressing differs.
int simt_gather_gemm(const GatherGemmArgs &a, cudaStream_t stream, int64_t ldx = 0, int64_t ldy = 0);
int simt_wgrad(const WgradArgs &a, cudaStream_t stream, int64_t ldx = 0, int64_t ldd = 0);

bool tc_gather_gemm_supported(const GatherGemmArgs &a);
int tc_gather_gemm(const GatherGemmArgs &a, cudaStream_t stream, int64_t ldx = 0, int64_t ldy = 0);
bool tc_wgrad_supported(const WgradArgs &a);
size_t tc_wgrad_workspace_size(const WgradArgs &a);
int tc_wgrad(const WgradArgs &a, cudaStream_t stream, int64_t ldx = 0, int64_t ldd = 0);

struct Int8Args {
    GatherGemmArgs g;          // dtype = SPX_I8; bias / act fields unused
    int out_dtype;
    const float *scale, *bias_f32;
    const int8_t *output_add;
    float output_add_scale;
};
int simt_gather_gemm_int8(const Int8Args &a, cudaStream_t stream);
bool tc_gather_gemm_int8_supported(const Int8Args &a);
int tc_gather_gemm_int8(const Int8Args &a, cudaStream_t stream);

// FP8 (e4m3) inference forward: the epilogue of include/spconv_b200.h (spx_implicit_gemm_fwd_fp8)
struct Fp8Args {
    GatherGemmArgs g;          // dtype = SPX_E4M3; bias field unused
    int out_dtype;             // SPX_F32 / SPX_F16 / SPX_BF16 / SPX_E4M3
    const float *in_scale, *w_scale, *bias_f32, *add_scale, *out_scale;
    const void *output_add;    // [rows, c_out] in out_dtype, or NULL
};
int simt_gather_gemm_fp8(const Fp8Args &a, cudaStream_t stream);
bool tc_gather_gemm_fp8_supported(const Fp8Args &a);
int tc_gather_gemm_fp8(const Fp8Args &a, cudaStream_t stream);

#ifdef __CUDACC__
// ---- the fp8 epilogue, shared by the tensor-core and FMA kernels.  One IEEE fp32 operation per step (the
// explicit _rn intrinsics keep the compiler from fusing them), in this order:
//   y = acc * s;  y = y + bias;  y = y + add * add_scale;  y = act(y)        s = in_scale * w_scale[j]
__device__ __forceinline__ float fp8_epilogue(float acc, float s, const float *bias, int j, bool has_add, float add,
                                              float add_scale, int act, float alpha) {
    float y = __fmul_rn(acc, s);
    if (bias) y = __fadd_rn(y, bias[j]);
    if (has_add) y = __fadd_rn(y, __fmul_rn(add, add_scale));
    return apply_act(y, act, alpha);
}
// e4m3 byte -> float (exact)
__device__ __forceinline__ float e4m3_to_float(uint8_t v) {
    return __half2float(__half(__nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)v, __NV_E4M3)));
}
// two floats -> two e4m3 bytes (a in the low byte): cvt.rn.satfinite.e4m3x2.f32
__device__ __forceinline__ uint16_t float2_to_e4m3x2(float a, float b) {
    return (uint16_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
}
__device__ __forceinline__ uint8_t float_to_e4m3(float a) {
    return (uint8_t)__nv_cvt_float_to_fp8(a, __NV_SATFINITE, __NV_E4M3);
}
// one element of a row of out_dtype (OUT, an spx_dtype code) as float
template <int OUT> __device__ __forceinline__ float load_out_elem(const void *p, int64_t i) {
    if constexpr (OUT == SPX_F32) return ((const float *)p)[i];
    else if constexpr (OUT == SPX_F16) return __half2float(((const __half *)p)[i]);
    else if constexpr (OUT == SPX_BF16) return __bfloat162float(((const __nv_bfloat16 *)p)[i]);
    else return e4m3_to_float(((const uint8_t *)p)[i]);
}
#endif

}  // namespace spx
