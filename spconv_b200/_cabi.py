"""ctypes binding of ``include/spconv_b200.h`` (the C-ABI shared library).

This is the only place Python touches native code; it replaces the reference's pybind bridge
``spconv/pytorch/cppcore.py:65-109`` (raw ``data_ptr`` + stream integer).  There is no CPU
fallback: a missing library raises immediately.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import (POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_size_t,
                    c_ubyte, c_uint32, c_uint64, c_void_p)

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libspconv_b200.so")

SPX_MAX_NDIM = 4
SPX_F32, SPX_F16, SPX_BF16, SPX_I8, SPX_E4M3 = 0, 1, 2, 3, 4
SPX_ACT_NONE, SPX_ACT_RELU, SPX_ACT_SIGMOID, SPX_ACT_LEAKY_RELU = 0, 1, 2, 3
SPX_GN_ACT_NONE, SPX_GN_ACT_RELU, SPX_GN_ACT_SILU = 0, 1, 2
SPX_F32_EXACT, SPX_F32_TF32 = 0, 1


class ConvGeometry(Structure):
    _fields_ = [
        ("ndim", c_int), ("batch_size", c_int),
        ("in_dims", c_int * SPX_MAX_NDIM), ("out_dims", c_int * SPX_MAX_NDIM),
        ("ksize", c_int * SPX_MAX_NDIM), ("stride", c_int * SPX_MAX_NDIM),
        ("padding", c_int * SPX_MAX_NDIM), ("dilation", c_int * SPX_MAX_NDIM),
        ("transposed", c_int),
    ]


class GemmDesc(Structure):
    _fields_ = [
        ("dtype", c_int), ("f32_mode", c_int), ("kv", c_int), ("c_in", c_int), ("c_out", c_int),
        ("n_in", c_int64), ("n_out", c_int64),
        ("pair", c_void_p), ("pair_stride", c_int64),
        ("mask", c_void_p), ("argsort", c_void_p),
        ("reverse_offsets", c_int),
        ("tile_table", c_void_p), ("tile_mask", c_void_p),
    ]


SPX_MAX_PEERS = 16
SPX_P2V_MAX_BATCH = 65536


class PeerGroup(Structure):
    """``spx_peer_group``: the exchange buffers of a data-parallel group as mapped in this process."""
    _fields_ = [
        ("world", c_int), ("rank", c_int), ("timeout_ms", c_int), ("colocated", c_int),
        ("capacity_bytes", c_uint64),
        ("buffers", c_void_p * SPX_MAX_PEERS),
    ]


SPX_SPARSE_ADD_MAX_OPERANDS = 64


class SparseAddOperands(Structure):
    """``spx_sparse_add_operands``: the operands of a sparse add in visit order."""
    _fields_ = [
        ("count", c_int),
        ("rows", c_int64 * SPX_SPARSE_ADD_MAX_OPERANDS),
        ("features", c_void_p * SPX_SPARSE_ADD_MAX_OPERANDS),
        ("grads", c_void_p * SPX_SPARSE_ADD_MAX_OPERANDS),
    ]


class MaskedSyncBN(Structure):
    """``spx_masked_sync_bn``: the operands of one MaskedSyncBatchNorm1d pass on this rank."""
    _fields_ = [
        ("rows", c_int64), ("channels", c_int), ("dtype", c_int), ("param_dtype", c_int), ("world", c_int),
        ("num_valid", c_void_p), ("x", c_void_p), ("y", c_void_p), ("dy", c_void_p), ("dx", c_void_p),
        ("weight", c_void_p), ("bias", c_void_p), ("running_mean", c_void_p), ("running_var", c_void_p),
        ("num_batches_tracked", c_void_p), ("momentum", c_float), ("cumulative", c_int), ("eps", c_float),
        ("save_mean", c_void_p), ("save_invstd", c_void_p), ("dweight", c_void_p), ("dbias", c_void_p),
        ("local", c_void_p), ("gathered", c_void_p),
    ]


class MaskedGroupNorm(Structure):
    """``spx_masked_group_norm``: the operands of one MaskedGroupNorm call (forward and backward)."""
    _fields_ = [
        ("rows", c_int64), ("row_ints", c_int), ("batch_size", c_int), ("channels", c_int), ("groups", c_int),
        ("dtype", c_int), ("param_dtype", c_int), ("eps", c_float),
        ("coords", c_void_p), ("num_valid", c_void_p), ("x", c_void_p), ("y", c_void_p), ("dy", c_void_p),
        ("dx", c_void_p), ("weight", c_void_p), ("bias", c_void_p), ("dweight", c_void_p), ("dbias", c_void_p),
        ("mean", c_void_p), ("invstd", c_void_p), ("order", c_void_p), ("offsets", c_void_p), ("cstart", c_void_p),
    ]


class MaskedGroupNormMod(Structure):
    """``spx_masked_group_norm_mod``: a MaskedGroupNorm call with per-sample scale / shift and an activation."""
    _fields_ = [
        ("norm", MaskedGroupNorm), ("scale", c_void_p), ("shift", c_void_p), ("act", c_int), ("dscale", c_void_p),
        ("dshift", c_void_p),
    ]


class PointInterp(Structure):
    """``spx_point_interp``: the operands of a voxel -> point interpolation (plan, forward and backward)."""
    _fields_ = [
        ("ndim", c_int), ("batch_size", c_int), ("mode", c_int), ("normalize", c_int), ("channels", c_int),
        ("dtype", c_int), ("spatial_shape", c_int * SPX_MAX_NDIM), ("rows", c_int64), ("num_points", c_int64),
        ("indices", c_void_p), ("num_valid", c_void_p), ("pos", c_void_p), ("batch_ids", c_void_p),
        ("index", c_void_p), ("weight", c_void_p), ("order", c_void_p), ("offsets", c_void_p),
        ("x", c_void_p), ("y", c_void_p), ("dy", c_void_p), ("dx", c_void_p),
    ]


class Fp8Gemm(Structure):
    """``spx_fp8_gemm``: the operands of one fp8 (e4m3) forward."""
    _fields_ = [
        ("features", c_void_p), ("filters", c_void_p), ("in_scale", c_void_p), ("w_scale", c_void_p),
        ("bias", c_void_p), ("output_add", c_void_p), ("add_scale", c_void_p), ("out", c_void_p),
        ("out_dtype", c_int), ("out_scale", c_void_p), ("act", c_int), ("act_alpha", c_float),
    ]


class GroupedGemm(Structure):
    """``spx_grouped_gemm``: the operands of one grouped-conv GEMM (forward, input or weight gradient)."""
    _fields_ = [
        ("features", c_void_p), ("filters", c_void_p), ("out_bp", c_void_p), ("bias", c_void_p), ("out", c_void_p),
        ("din", c_void_p), ("dfilters", c_void_p), ("workspace", c_void_p), ("workspace_bytes", c_size_t),
        ("act", c_int), ("act_alpha", c_float),
    ]


class Fp8Quant(Structure):
    """``spx_fp8_quant``: the operands of one e4m3 quantisation."""
    _fields_ = [
        ("x", c_void_p), ("dtype", c_int), ("rows", c_int64), ("channels", c_int), ("num_valid", c_void_p),
        ("scale_in", c_void_p), ("out", c_void_p), ("scale_out", c_void_p),
    ]


# name -> (restype, argtypes); also the list the CPU test checks against the header
SIGNATURES = {
    "spx_last_error": (c_char_p, []),
    "spx_version": (c_int, []),
    "spx_device_check": (c_int, [c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "spx_rulebook_workspace_size": (c_size_t, [POINTER(ConvGeometry), c_int64, c_int64, c_int]),
    "spx_conv_max_out": (c_int64, [POINTER(ConvGeometry), c_int64]),
    "spx_subm_rulebook": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_conv_rulebook_stage1": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64,
                                         POINTER(c_int64), c_void_p, c_size_t, c_void_p]),
    "spx_conv_rulebook_stage2": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64, c_int64,
                                         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_size_t, c_void_p]),
    "spx_subm_rulebook_all_workspace_size": (c_size_t, [POINTER(ConvGeometry), c_int64]),
    "spx_subm_rulebook_all": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_conv_rulebook_all_workspace_size": (c_size_t, [POINTER(ConvGeometry), c_int64]),
    "spx_conv_rulebook_stage2_all": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64, c_int64, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_conv_rulebook_bounded_workspace_size": (c_size_t, [POINTER(ConvGeometry), c_int64, c_int64]),
    "spx_conv_rulebook_bounded_all": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64, c_int64, c_void_p, c_void_p,
                                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                              c_void_p]),
    "spx_cross_rulebook_all_workspace_size": (c_size_t, [POINTER(ConvGeometry), c_int64, c_int64]),
    "spx_cross_rulebook_all": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_zero_rows_from_count": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    "spx_native_pairs": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                 c_size_t, c_void_p]),
    "spx_native_pairs_workspace_size": (c_size_t, [c_int64, c_int]),
    "spx_pairs_to_table": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_int64, c_int,
                                   c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "spx_mask_argsort_workspace_size": (c_size_t, [c_int64, c_int]),
    "spx_mask_argsort": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p,
                                 c_size_t, c_void_p]),
    "spx_tile_table_elems": (c_size_t, [c_int64, c_int]),
    "spx_build_tile_table": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_int64,
                                     c_void_p, c_void_p, c_void_p]),
    "spx_implicit_gemm_fwd": (c_int, [POINTER(GemmDesc), c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_int, c_float, c_void_p]),
    "spx_implicit_gemm_dgrad": (c_int, [POINTER(GemmDesc), c_void_p, c_void_p, c_void_p,
                                        c_void_p]),
    "spx_implicit_gemm_wgrad_workspace_size": (c_size_t, [POINTER(GemmDesc)]),
    "spx_implicit_gemm_wgrad": (c_int, [POINTER(GemmDesc), c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_size_t, c_void_p]),
    "spx_peer_buffer_bytes": (c_size_t, [c_size_t, c_int]),
    "spx_peer_buffer_create": (c_int, [c_size_t, c_int, POINTER(c_void_p), POINTER(c_ubyte)]),
    "spx_peer_buffer_open": (c_int, [POINTER(c_ubyte), POINTER(c_void_p)]),
    "spx_peer_buffer_close": (c_int, [c_void_p]),
    "spx_peer_buffer_destroy": (c_int, [c_void_p]),
    "spx_peer_error": (c_int, [POINTER(PeerGroup), POINTER(c_int)]),
    "spx_implicit_gemm_wgrad_push": (c_int, [POINTER(GemmDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                             POINTER(PeerGroup), c_void_p]),
    "spx_peer_push": (c_int, [POINTER(PeerGroup), c_void_p, c_int64, c_int, c_void_p]),
    "spx_peer_finish": (c_int, [POINTER(PeerGroup), c_void_p, c_int64, c_int, c_float, c_void_p]),
    "spx_peer_allreduce": (c_int, [POINTER(PeerGroup), c_void_p, c_int64, c_int, c_float, c_void_p]),
    "spx_peer_allgather": (c_int, [POINTER(PeerGroup), c_void_p, c_int64, c_void_p, c_void_p]),
    "spx_bias_act_inplace": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_float,
                                     c_void_p]),
    "spx_implicit_gemm_fwd_int8": (c_int, [POINTER(GemmDesc), c_void_p, c_void_p, c_void_p,
                                           c_int, c_void_p, c_void_p, c_void_p, c_float, c_int,
                                           c_float, c_void_p]),
    "spx_implicit_gemm_fwd_fp8": (c_int, [POINTER(GemmDesc), POINTER(Fp8Gemm), c_void_p]),
    "spx_grouped_gemm_fwd": (c_int, [POINTER(GemmDesc), c_int, POINTER(GroupedGemm), c_void_p]),
    "spx_grouped_gemm_dgrad": (c_int, [POINTER(GemmDesc), c_int, POINTER(GroupedGemm), c_void_p]),
    "spx_grouped_gemm_wgrad_workspace_size": (c_size_t, [POINTER(GemmDesc), c_int]),
    "spx_grouped_gemm_wgrad": (c_int, [POINTER(GemmDesc), c_int, POINTER(GroupedGemm), c_void_p]),
    "spx_grouped_gemm_wgrad_push": (c_int, [POINTER(GemmDesc), c_int, POINTER(GroupedGemm), POINTER(PeerGroup),
                                            c_void_p]),
    "spx_fp8_quantize_workspace_size": (c_size_t, [c_int64, c_int]),
    "spx_fp8_quantize": (c_int, [POINTER(Fp8Quant), c_void_p, c_size_t, c_void_p]),
    "spx_point2voxel_workspace_size": (c_size_t, [c_int64, c_int]),
    "spx_point2voxel_stage1": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, POINTER(c_float), POINTER(c_int),
                                       POINTER(c_float), c_int64, POINTER(c_int64), POINTER(c_int64), c_void_p,
                                       c_size_t, c_void_p]),
    "spx_point2voxel_stage2": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, POINTER(c_float), POINTER(c_int),
                                       POINTER(c_float), c_int64, c_int64, c_int, c_int, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_point2voxel_bounded_workspace_size": (c_size_t, [c_int64, c_int, c_int64]),
    "spx_point2voxel_bounded": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, POINTER(c_float), POINTER(c_int),
                                        POINTER(c_float), c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_void_p,
                                        c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                        c_void_p]),
    "spx_indice_pool_fwd": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_int,
                                    c_void_p, c_void_p]),
    "spx_indice_pool_bwd": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int,
                                    c_int64, c_int, c_int, c_void_p, c_void_p]),
    "spx_global_pool_rearrange": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "spx_global_pool_workspace_size": (c_size_t, [c_int64, c_int, c_int]),
    "spx_global_pool_fwd": (c_int, [c_int, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_global_pool_bwd": (c_int, [c_int, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p]),
    "spx_sparse_add_group_workspace_size": (c_size_t, [c_int64]),
    "spx_sparse_add_group": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_sparse_add_fwd": (c_int, [POINTER(SparseAddOperands), c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p,
                                   c_void_p]),
    "spx_sparse_add_gather": (c_int, [c_void_p, c_void_p, c_int64, POINTER(SparseAddOperands), c_int, c_int,
                                      c_void_p]),
    "spx_sparse_add_union_workspace_size": (c_size_t, [POINTER(ConvGeometry), c_int64, c_int64]),
    "spx_sparse_add_union": (c_int, [POINTER(ConvGeometry), c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_masked_sparse_add_workspace_size": (c_size_t, [POINTER(ConvGeometry), c_int64, c_int64]),
    "spx_masked_sparse_add_plan": (c_int, [POINTER(ConvGeometry), POINTER(SparseAddOperands), POINTER(c_void_p),
                                           c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_masked_sparse_add_heads": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p,
                                            c_void_p]),
    "spx_point_scatter_group_workspace_size": (c_size_t, [c_int64]),
    "spx_point_scatter_group": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_size_t, c_void_p]),
    "spx_point_scatter_fwd": (c_int, [c_int, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int64, c_void_p,
                                      c_void_p, c_void_p]),
    "spx_point_scatter_bwd": (c_int, [c_int, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    "spx_point_interp_plan_workspace_size": (c_size_t, [POINTER(PointInterp)]),
    "spx_point_interp_plan": (c_int, [POINTER(PointInterp), c_void_p, c_size_t, c_void_p]),
    **{f"spx_point_interp_{p}": (c_int, [POINTER(PointInterp), c_void_p]) for p in ("fwd", "bwd")},
    "spx_depthwise_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int,
                                  c_int, c_int, c_float, c_void_p]),
    "spx_depthwise_dgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_int,
                                    c_int, c_void_p]),
    "spx_depthwise_wgrad_workspace_size": (c_size_t, [c_int64, c_int, c_int]),
    "spx_depthwise_wgrad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_int,
                                    c_void_p, c_size_t, c_void_p]),
    "spx_masked_bn_fwd_train_workspace_size": (c_size_t, [c_int64, c_int]),
    "spx_masked_bn_fwd_train": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_float, c_void_p,
                                        c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_masked_bn_bwd_workspace_size": (c_size_t, [c_int64, c_int]),
    "spx_masked_bn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_masked_sync_bn_workspace_size": (c_size_t, [c_int64, c_int]),
    **{f"spx_masked_sync_bn_{p}": (c_int, [POINTER(MaskedSyncBN), c_void_p, c_size_t, c_void_p])
       for p in ("fwd_local", "fwd_merge", "bwd_local", "bwd_merge")},
    "spx_masked_group_norm_workspace_size": (c_size_t, [c_int64, c_int, c_int]),
    **{f"spx_masked_group_norm_{p}": (c_int, [POINTER(MaskedGroupNorm), c_void_p, c_size_t, c_void_p])
       for p in ("fwd", "bwd")},
    **{f"spx_masked_group_norm_mod_{p}": (c_int, [POINTER(MaskedGroupNormMod), c_void_p, c_size_t, c_void_p])
       for p in ("fwd", "bwd")},
    "spx_hash_workspace_size": (c_size_t, [c_int64, c_int64]),
    "spx_hash_clear": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p]),
    "spx_hash_insert": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int64,
                                c_int64, c_void_p, c_size_t, c_void_p]),
    "spx_hash_query": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int64,
                               c_void_p]),
    "spx_hash_insert_exist": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_int64, c_int64, c_void_p, c_size_t, c_void_p]),
    "spx_hash_rank": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int64, c_int, c_void_p,
                              c_void_p, c_int64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "spx_last_kernel_family": (c_int, []),
    "spx_launch_count": (c_int64, [c_int]),
    "spx_debug_configure": (c_int, [c_int, c_int, c_int, c_void_p, c_size_t]),
}

_lib = None


def load() -> ctypes.CDLL:
    """Load the shared library (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"spconv_b200 native library not found at {LIB_PATH}. Build it with "
            "`python -m spconv_b200.build` (needs nvcc, no GPU). There is no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError here == header / library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    msg = load().spx_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int, what: str = "") -> None:
    """Reference convention: native failures surface as RuntimeError with the C++ text
    (TV_ASSERT_RT_ERR -> std::runtime_error -> Python exception)."""
    if rc != 0:
        raise RuntimeError(f"spconv_b200::{what} failed ({rc}): {last_error()}")


def make_geometry(ndim, batch_size, in_dims, out_dims, ksize, stride, padding, dilation,
                  transposed=False) -> ConvGeometry:
    g = ConvGeometry()
    g.ndim = int(ndim)
    g.batch_size = int(batch_size)
    for i in range(ndim):
        g.in_dims[i] = int(in_dims[i])
        g.out_dims[i] = int(out_dims[i])
        g.ksize[i] = int(ksize[i])
        g.stride[i] = int(stride[i])
        g.padding[i] = int(padding[i])
        g.dilation[i] = int(dilation[i])
    g.transposed = int(bool(transposed))
    return g
