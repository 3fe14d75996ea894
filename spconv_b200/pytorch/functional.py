"""Autograd layer over :mod:`spconv_b200.pytorch.ops`.

Public entry points keep the reference's names and positional argument order
(``spconv/pytorch/functional.py:423-429``): ``indice_conv``, ``indice_inverse_conv``,
``indice_subm_conv``, ``implicit_gemm``.  One generic :class:`_NativeConv` serves the three
ConvAlgo.Native variants (they differ only in the ``inverse`` / ``subm`` flags,
reference classes at ``functional.py:59-189,293-357``).
"""
from __future__ import annotations

import functools
import sys
from typing import List, Optional

import numpy as np
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from ..core import Activation
from . import ops
from .core import CUDAKernelTimer, SparseConvTensor

# AMP: inputs are cast to fp16 inside autocast regions, like the reference (functional.py:44-56)
_amp_fwd = torch.amp.custom_fwd(cast_inputs=torch.float16, device_type="cuda")
_amp_bwd = torch.amp.custom_bwd(device_type="cuda")


def _report(tag: str, **shapes) -> None:
    """Reference convention: print a one-line context to stderr before re-raising."""
    info = ",".join(f"{k}={v}" for k, v in shapes.items())
    print(f"[Exception|{tag}]{info}", file=sys.stderr)


class _NativeConv(Function):
    """features, filters, indice_pairs, indice_pair_num, num_activate_out, algo, timer, bias,
    act_alpha, act_beta, act_type, inverse, subm, groups"""

    @staticmethod
    @_amp_fwd
    def forward(ctx, features, filters, indice_pairs, indice_pair_num, num_activate_out, algo,
                timer, bias, act_alpha, act_beta, act_type, inverse, subm, groups=1):
        ctx.save_for_backward(indice_pairs, indice_pair_num, features, filters)
        ctx.spx = (algo, timer, inverse, subm, groups)
        ctx.spx_scope = timer.snapshot()
        try:
            return ops.indice_conv(features, filters, indice_pairs, indice_pair_num,
                                   num_activate_out, inverse, subm, algo=algo, timer=timer,
                                   bias=bias, act_alpha=act_alpha, act_beta=act_beta,
                                   act_type=act_type, groups=groups)
        except Exception:
            _report("indice_conv", feat=tuple(features.shape), w=tuple(filters.shape),
                    pair=tuple(indice_pairs.shape), act=num_activate_out, algo=algo,
                    inverse=inverse, subm=subm)
            raise

    @staticmethod
    @once_differentiable
    @_amp_bwd
    def backward(ctx, grad_output):
        indice_pairs, indice_pair_num, features, filters = ctx.saved_tensors
        algo, timer, inverse, subm, groups = ctx.spx
        try:
            with timer.scoped(ctx.spx_scope):
                din, dw = ops.indice_conv_backward(features, filters, grad_output, indice_pairs,
                                                   indice_pair_num, inverse, subm, algo=algo,
                                                   timer=timer, groups=groups)
        except Exception:
            _report("indice_conv_backward", feat=tuple(features.shape), w=tuple(filters.shape),
                    pair=tuple(indice_pairs.shape), do=tuple(grad_output.shape))
            raise
        return (din, dw) + (None,) * 12


class SparseImplicitGemmFunction(Function):
    """Masked implicit GEMM with autograd (reference ``functional.py:191-290``)."""

    @staticmethod
    @_amp_fwd
    def forward(ctx, features: torch.Tensor, filters: torch.Tensor, pair_fwd: torch.Tensor,
                pair_bwd: torch.Tensor, pair_mask_fwd_splits: List[torch.Tensor],
                pair_mask_bwd_splits: List[torch.Tensor],
                mask_argsort_fwd_splits: List[torch.Tensor],
                mask_argsort_bwd_splits: List[torch.Tensor], num_activate_out: int,
                masks: List[np.ndarray], is_train: bool, is_subm: bool,
                timer: CUDAKernelTimer = CUDAKernelTimer(False),
                fp32_accum: Optional[bool] = None, bias: Optional[torch.Tensor] = None,
                act_alpha: float = 0.0, act_beta: float = 0.0, act_type=Activation.None_, groups: int = 1):
        try:
            out, mask_out, mask_width = ops.implicit_gemm(
                features, filters, pair_fwd, pair_mask_fwd_splits, mask_argsort_fwd_splits,
                num_activate_out, masks, is_train, is_subm, timer, fp32_accum, bias, act_alpha,
                act_beta, act_type, groups=groups)
        except Exception:
            _report("implicit_gemm", feat=tuple(features.shape), w=tuple(filters.shape),
                    pair=tuple(pair_fwd.shape), act=num_activate_out, issubm=is_subm,
                    istrain=is_train)
            raise
        ctx.save_for_backward(features, filters, pair_fwd, pair_bwd)
        ctx.spx = dict(mask_width=mask_width, mask_out=mask_out, timer=timer, masks=masks,
                       scope=timer.snapshot(),
                       is_subm=is_subm, fp32_accum=fp32_accum, groups=groups,
                       mask_fwd=pair_mask_fwd_splits, mask_bwd=pair_mask_bwd_splits,
                       sort_fwd=mask_argsort_fwd_splits, sort_bwd=mask_argsort_bwd_splits)
        return out

    @staticmethod
    @once_differentiable
    @_amp_bwd
    def backward(ctx, grad_output):
        features, filters, pair_fwd, pair_bwd = ctx.saved_tensors
        s = ctx.spx
        try:
            with s["timer"].scoped(s["scope"]):
                din, dw = ops.implicit_gemm_backward(
                    features, filters, grad_output, pair_fwd, pair_bwd, s["mask_fwd"], s["mask_bwd"],
                    s["sort_fwd"], s["sort_bwd"], mask_output_fwd=s["mask_out"], masks=s["masks"],
                    mask_width=s["mask_width"], is_subm=s["is_subm"], timer=s["timer"],
                    fp32_accum=s["fp32_accum"], groups=s["groups"])
        except Exception:
            _report("implicit_gemm_backward", feat=tuple(features.shape), w=tuple(filters.shape),
                    pair=tuple(pair_fwd.shape), issubm=s["is_subm"], do=tuple(grad_output.shape))
            raise
        return (din, dw) + (None,) * 17


class ZeroPaddingGrad(Function):
    """Identity on the features of a padded tensor whose backward zeroes the gradient rows at and beyond
    ``num_valid``.  The conv modules put it behind every layer that produces a padded tensor (after the bias
    add), so the bias gradient ``dout.sum(0)`` and the weight gradient of a SubM layer (whose centre tap
    pairs a padding row with itself) are exact whatever the loss did with the padding rows."""

    @staticmethod
    def forward(ctx, features, num_valid):
        ctx.save_for_backward(num_valid)
        return features.view_as(features)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        num_valid, = ctx.saved_tensors
        grad = grad_output.contiguous().clone()      # the incoming gradient may be shared: never zero it in place
        return ops.zero_rows_from_count_(grad, num_valid), None


class SparseMaxPoolFunction(Function):
    """ConvAlgo.Native max pooling (reference ``functional.py:360-378``)."""

    @staticmethod
    @_amp_fwd
    def forward(ctx, features, indice_pairs, indice_pair_num, num_activate_out):
        out = ops.indice_maxpool(features, indice_pairs, indice_pair_num, num_activate_out)
        ctx.save_for_backward(indice_pairs, indice_pair_num, features, out)
        return out

    @staticmethod
    @once_differentiable
    @_amp_bwd
    def backward(ctx, grad_output):
        indice_pairs, indice_pair_num, features, out = ctx.saved_tensors
        return ops.indice_maxpool_backward(features, out, grad_output, indice_pairs,
                                           indice_pair_num), None, None, None


class SparseMaxPoolImplicitGemmFunction(Function):
    """Reference ``functional.py:381-400``."""

    @staticmethod
    @_amp_fwd
    def forward(ctx, features, indice_pairs_fwd, indice_pairs_bwd, num_activate_out, num_valid=None):
        out = ops.indice_maxpool_implicit_gemm(features, indice_pairs_fwd, num_activate_out)
        if num_valid is not None:                 # padding rows of a bounded rulebook: 0, not the lowest value
            ops.zero_rows_from_count_(out, num_valid)
        ctx.save_for_backward(indice_pairs_bwd, features, out)
        return out

    @staticmethod
    @once_differentiable
    @_amp_bwd
    def backward(ctx, grad_output):
        indice_pairs_bwd, features, out = ctx.saved_tensors
        return ops.indice_maxpool_implicit_gemm_backward(features, out, grad_output,
                                                         indice_pairs_bwd), None, None, None, None


class SparseAvgPoolImplicitGemmFunction(Function):
    """Reference ``functional.py:403-423``."""

    @staticmethod
    @_amp_fwd
    def forward(ctx, features, indice_pairs_fwd, indice_pairs_bwd, num_activate_out, calc_count):
        out, count = ops.indice_avgpool_implicit_gemm(features, indice_pairs_fwd, num_activate_out,
                                                      calc_count)
        ctx.save_for_backward(indice_pairs_bwd, count)
        return out

    @staticmethod
    @once_differentiable
    @_amp_bwd
    def backward(ctx, grad_output):
        indice_pairs_bwd, count = ctx.saved_tensors
        return ops.indice_avgpool_implicit_gemm_backward(grad_output, indice_pairs_bwd,
                                                         count), None, None, None, None


def _native(features, filters, indice_pairs, indice_pair_num, num_activate_out, algo, timer, bias,
            act_alpha, act_beta, act_type, inverse, subm, groups=1):
    if timer is None:
        timer = CUDAKernelTimer(False)
    if groups == 1:
        return _NativeConv.apply(features, filters, indice_pairs, indice_pair_num, num_activate_out,
                                 algo, timer, bias, act_alpha, act_beta, act_type, inverse, subm)
    return _NativeConv.apply(features, filters, indice_pairs, indice_pair_num, num_activate_out,
                             algo, timer, bias, act_alpha, act_beta, act_type, inverse, subm, groups)


def indice_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out, algo,
                timer=None, bias=None, act_alpha=0.0, act_beta=0.0, act_type=Activation.None_, groups=1):
    return _native(features, filters, indice_pairs, indice_pair_num, num_activate_out, algo, timer,
                   bias, act_alpha, act_beta, act_type, False, False, groups)


def indice_inverse_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out, algo,
                        timer=None, bias=None, act_alpha=0.0, act_beta=0.0,
                        act_type=Activation.None_, groups=1):
    return _native(features, filters, indice_pairs, indice_pair_num, num_activate_out, algo, timer,
                   bias, act_alpha, act_beta, act_type, True, False, groups)


def indice_subm_conv(features, filters, indice_pairs, indice_pair_num, num_activate_out, algo,
                     timer=None, bias=None, act_alpha=0.0, act_beta=0.0,
                     act_type=Activation.None_, groups=1):
    return _native(features, filters, indice_pairs, indice_pair_num, num_activate_out, algo, timer,
                   bias, act_alpha, act_beta, act_type, False, True, groups)


class DepthwiseConvFunction(Function):
    """``features, filters [C, *ksize, 1], table_fwd, table_bwd, num_activate_out, timer, bias, act_alpha,
    act_type`` -> depthwise conv over the dense tables (:func:`ops.depthwise_conv`); ``table_bwd`` None walks the
    forward table with mirrored offsets in the backward (SubM)."""

    @staticmethod
    @_amp_fwd
    def forward(ctx, features, filters, table_fwd, table_bwd, num_activate_out, timer, bias, act_alpha, act_type):
        try:
            out = ops.depthwise_conv(features, filters, table_fwd, num_activate_out, bias, act_type, act_alpha,
                                     timer=timer)
        except Exception:
            _report("depthwise_conv", feat=tuple(features.shape), w=tuple(filters.shape),
                    pair=tuple(table_fwd.shape), act=num_activate_out)
            raise
        ctx.save_for_backward(features, filters, table_fwd, table_bwd)
        ctx.spx = (timer, timer.snapshot())
        return out

    @staticmethod
    @once_differentiable
    @_amp_bwd
    def backward(ctx, grad_output):
        features, filters, table_fwd, table_bwd = ctx.saved_tensors
        timer, scope = ctx.spx
        try:
            with timer.scoped(scope):
                din, dw = ops.depthwise_conv_backward(features, filters, grad_output, table_fwd, table_bwd,
                                                      timer=timer)
        except Exception:
            _report("depthwise_conv_backward", feat=tuple(features.shape), w=tuple(filters.shape),
                    pair=tuple(table_fwd.shape), do=tuple(grad_output.shape))
            raise
        return (din, dw) + (None,) * 7


def depthwise_conv(features, filters, table_fwd, table_bwd, num_activate_out, timer=None, bias=None,
                   act_alpha=0.0, act_type=Activation.None_):
    if timer is None:
        timer = CUDAKernelTimer(False)
    return DepthwiseConvFunction.apply(features, filters, table_fwd, table_bwd, num_activate_out, timer, bias,
                                       act_alpha, act_type)


implicit_gemm = SparseImplicitGemmFunction.apply
zero_padding_grad = ZeroPaddingGrad.apply
indice_maxpool = SparseMaxPoolFunction.apply
indice_maxpool_implicit_gemm = SparseMaxPoolImplicitGemmFunction.apply
indice_avgpool_implicit_gemm = SparseAvgPoolImplicitGemmFunction.apply


# ---------------------------------------------------------------------------- sparse add
class SparseAddFunction(Function):
    """``dst, order, offsets, m, *features`` (operands in visit order) -> their sum over the union of the
    coordinates (:func:`ops.sparse_add_forward`); the gradient of operand row ``g`` is ``dout[dst[g]]``, or 0
    for a dropped row, and is computed only for the operands that need it."""

    @staticmethod
    def forward(ctx, dst, order, offsets, m, *features):
        ctx.save_for_backward(dst)
        ctx.rows = [f.shape[0] for f in features]
        return ops.sparse_add_forward(features, order, offsets, m)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        dst, = ctx.saved_tensors
        grads = ops.sparse_add_gather(dst, grad_output, ctx.rows, ctx.needs_input_grad[4:])
        return (None, None, None, None, *grads)


def _sparse_add(tens) -> SparseConvTensor:
    assert len(tens) >= 1, "sparse_add needs at least one operand"
    for ten in tens:
        ten.require_unpadded("sparse_add")
    first = tens[0]
    largest = 0
    for i, ten in enumerate(tens):
        assert ten.spatial_shape == first.spatial_shape
        assert ten.batch_size == first.batch_size
        assert ten.features.shape[1] == first.features.shape[1]
        ops._sparse_add_dtype(ten.features.dtype)
        if ten.features.shape[0] > tens[largest].features.shape[0]:     # ties: the earliest operand
            largest = i
    dtype = functools.reduce(torch.promote_types, [t.features.dtype for t in tens])
    visit = [largest] + [i for i in range(len(tens)) if i != largest]
    out_inds, dst = ops.sparse_add_union([tens[i].indices for i in visit], first.batch_size, first.spatial_shape)
    m = out_inds.shape[0]
    order, offsets = ops.sparse_add_group(dst, m)
    feats = [tens[i].features if tens[i].features.dtype == dtype else tens[i].features.to(dtype) for i in visit]
    res = SparseConvTensor(SparseAddFunction.apply(dst, order, offsets, m, *feats), out_inds, first.spatial_shape,
                           first.batch_size, benchmark=first.benchmark)
    # The largest operand is visited first, so its rows are output rows 0, 1, .. in order exactly when they
    # are all distinct and in range, i.e. when its last row is output row N - 1.  Only then do the output
    # coordinates equal its coordinates row for row and its rulebooks stay valid (a second host sync).
    n_l = tens[largest].features.shape[0]
    if m == n_l and (n_l == 0 or int(dst[n_l - 1]) == n_l - 1):
        res.indice_dict = tens[largest].indice_dict
    res.benchmark_record = first.benchmark_record
    res._timer = first._timer
    res.thrust_allocator = first.thrust_allocator
    return res


def sparse_add(*tens: SparseConvTensor) -> SparseConvTensor:
    """Sum of sparse tensors with the same shape, batch size and channels but different coordinates
    (``spconv/pytorch/functional.py:517-544``).

    Every distinct in-range coordinate appears once in the result.  Rows are in first-touch order: the
    largest operand (ties: the earliest) is visited first, then the others in argument order, each row by
    row, and an output row's rank is that of the first visited row carrying its coordinate.  Each output
    row is the sum of every row with its coordinate, duplicates within one operand included, accumulated in
    fp32 in visit order and rounded once: the result is bit-reproducible.  Rows whose batch index or
    coordinate is out of range are dropped and get a zero gradient.  Operands of different dtypes are
    promoted as ``+`` would.  The largest operand's ``indice_dict`` is kept exactly when the result's
    coordinates equal its coordinates row for row, so a following ``SparseInverseConv`` on one of its keys
    gathers the right rows.

    Differences from the reference: the reference orders rows by ``torch.sparse`` coalesce (sorted linear
    index), which is not the row order of the operand whose ``indice_dict`` it keeps; here the order above
    makes that documented usage correct.  Host syncs: one for the output count, plus one 4-byte read when
    the output count equals the largest operand's row count (to decide on ``indice_dict``)."""
    return _sparse_add(tens)


def sparse_add_hash_based(*tens: SparseConvTensor) -> SparseConvTensor:
    """The same result as :func:`sparse_add` (``spconv/pytorch/functional.py:441-514``).  Unlike the
    reference, whose ``index_put`` keeps one arbitrary row of duplicate coordinates within one operand, every
    such row is summed, and rows come in first-touch order rather than hash-slot order."""
    return _sparse_add(tens)


class _RowGather(Function):
    """``out[o] = features[heads[o]]``; gradient ``din[i] = dout[inverse[i]]`` (0 where ``inverse[i] < 0``)."""

    @staticmethod
    def forward(ctx, features, heads, inverse):
        ctx.save_for_backward(inverse)
        return ops.sparse_add_gather(heads, features, [heads.shape[0]])[0]

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        inverse, = ctx.saved_tensors
        return ops.sparse_add_gather(inverse, grad_output, [inverse.shape[0]])[0], None, None


def remove_duplicate(x: SparseConvTensor) -> SparseConvTensor:
    """Keep the first row of every coordinate (rows in first-touch order) and drop rows whose batch index or
    coordinate is out of range; see :class:`spconv_b200.pytorch.spatial.RemoveDuplicate`."""
    x.require_unpadded("remove_duplicate")
    ops._sparse_add_dtype(x.features.dtype)
    out_inds, dst = ops.sparse_add_union([x.indices], x.batch_size, x.spatial_shape)
    m = out_inds.shape[0]
    order, offsets = ops.sparse_add_group(dst, m)
    heads = order[offsets[:m].long()]
    inverse = torch.full_like(dst, -1)
    inverse[heads.long()] = torch.arange(m, dtype=torch.int32, device=dst.device)
    feats = _RowGather.apply(x.features, heads, inverse)
    return SparseConvTensor(feats, out_inds, x.spatial_shape, x.batch_size, x.grid)


# ---------------------------------------------------------------------------- padding-aware sparse add
def _masked_bound(rows: int, num_out_act_bound: Optional[int]) -> int:
    if num_out_act_bound is None:
        return rows
    if int(num_out_act_bound) < 1:
        raise ValueError(f"num_out_act_bound must be positive, got {num_out_act_bound}")
    return min(int(num_out_act_bound), rows)            # the union never has more rows than its operands


def _merged_status(tens, name: Optional[str], status: Optional[torch.Tensor]):
    words = {}
    for ten in tens:
        words.update(ten.bound_status or {})
    if name is not None:
        words[name] = status
    return words or None


def _masked_sparse_add(tens, num_out_act_bound=None, status=None, name=None) -> SparseConvTensor:
    assert len(tens) >= 1, "masked_sparse_add needs at least one operand"
    first = tens[0]
    bound = _masked_bound(sum(t.features.shape[0] for t in tens), num_out_act_bound)
    for ten in tens:
        assert ten.spatial_shape == first.spatial_shape
        assert ten.batch_size == first.batch_size
        assert ten.features.shape[1] == first.features.shape[1]
        ops._sparse_add_dtype(ten.features.dtype)
        ops._require_cuda(ten.features, "features")
    dtype = functools.reduce(torch.promote_types, [t.features.dtype for t in tens])
    out_inds, dst, order, offsets, num_out, status = ops.masked_sparse_add_plan(
        [t.indices for t in tens], [t.num_valid for t in tens], first.batch_size, first.spatial_shape, bound, status)
    feats = [t.features if t.features.dtype == dtype else t.features.to(dtype) for t in tens]
    res = SparseConvTensor(SparseAddFunction.apply(dst, order, offsets, bound, *feats), out_inds, first.spatial_shape,
                           first.batch_size, benchmark=first.benchmark)
    res.num_valid = num_out
    res.bound_status = _merged_status(tens, name, status)
    res.benchmark_record = first.benchmark_record
    res._timer = first._timer
    res.thrust_allocator = first.thrust_allocator
    return res


def masked_sparse_add(*tens: SparseConvTensor, num_out_act_bound: Optional[int] = None) -> SparseConvTensor:
    """:func:`sparse_add` of padded and / or unpadded operands, with no host synchronisation (CUDA-graph capturable).

    Operand ``t``'s valid rows are ``[0, t.num_valid)`` (every row when ``num_valid`` is None); rows beyond are never
    read, neither features nor indices.  The result has ``bound`` rows and ``num_valid`` = M (device int32 ``[1]``):
    rows ``[0, M)`` of its indices and features, M, and every operand's gradient rows ``[0, valid_t)`` equal
    :func:`sparse_add` of the valid rows bit for bit, whatever the padding.  The visit order is decided on the device
    from the valid counts (the largest valid count first, ties: the earliest operand, then the others in argument
    order), as :func:`sparse_add` decides it from the row counts.  Rows ``[M, bound)`` have indices -1 and features 0;
    padding and dropped rows get a zero gradient.

    ``bound`` defaults to the operands' total row count, which the union can never exceed; a larger
    ``num_out_act_bound`` is clamped to it.  A smaller one truncates deterministically: the outputs ranked >= bound
    are dropped, their rows get a zero gradient, and bit 0 of the result's ``bound_status`` word is set
    (:func:`spconv.check_bounds`).  An empty union gives M = 0.  ``indice_dict`` is not kept: deciding whether the
    result's rows are an operand's rows would need a host read-back.  float32, float16 and bfloat16, CUDA only."""
    return _masked_sparse_add(tens, num_out_act_bound, name="masked_sparse_add")


def masked_remove_duplicate(x: SparseConvTensor, num_out_act_bound: Optional[int] = None) -> SparseConvTensor:
    """:func:`remove_duplicate` of the valid rows ``[0, x.num_valid)``, with no host synchronisation.  The result has
    ``bound`` rows (default and upper limit: ``x``'s row count) and ``num_valid`` = M; rows ``[0, M)`` equal
    :func:`remove_duplicate` of the valid rows bit for bit, rows ``[M, bound)`` have indices -1 and features 0, and
    the gradient goes to the kept rows only.  Truncation and ``bound_status`` as :func:`masked_sparse_add`."""
    return _masked_remove_duplicate(x, num_out_act_bound, name="masked_remove_duplicate")


def _masked_remove_duplicate(x: SparseConvTensor, num_out_act_bound=None, status=None, name=None) -> SparseConvTensor:
    bound = _masked_bound(x.features.shape[0], num_out_act_bound)
    ops._sparse_add_dtype(x.features.dtype)
    ops._require_cuda(x.features, "features")
    out_inds, dst, order, offsets, num_out, status = ops.masked_sparse_add_plan(
        [x.indices], [x.num_valid], x.batch_size, x.spatial_shape, bound, status)
    heads, inverse = ops.masked_sparse_add_heads(order, offsets, num_out)
    res = SparseConvTensor(_RowGather.apply(x.features, heads, inverse), out_inds, x.spatial_shape, x.batch_size,
                           x.grid)
    res.num_valid = num_out
    res.bound_status = _merged_status([x], name, status)
    return res


# ---------------------------------------------------------------------------- padding-aware BatchNorm
class MaskedBatchNormFunction(Function):
    """``x, weight, bias, running_mean, running_var, num_batches_tracked, num_valid, momentum, eps`` -> training-mode
    BatchNorm over rows ``[0, num_valid)`` (:func:`ops.masked_batch_norm_forward`); the running stats are updated
    in place.  The backward gives dx (0 on padding rows), dweight and dbias."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, num_batches_tracked, num_valid, momentum, eps):
        y, mean, invstd = ops.masked_batch_norm_forward(x, num_valid, weight, bias, running_mean, running_var,
                                                        num_batches_tracked, momentum, eps)
        ctx.save_for_backward(x, weight, mean, invstd, num_valid)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        x, weight, mean, invstd, num_valid = ctx.saved_tensors
        dx, dw, db = ops.masked_batch_norm_backward(x, grad_output, num_valid, weight, mean, invstd,
                                                    ctx.needs_input_grad[1], ctx.needs_input_grad[2])
        return dx, dw, db, None, None, None, None, None, None


masked_batch_norm = MaskedBatchNormFunction.apply


class MaskedSyncBatchNormFunction(Function):
    """``x, weight, bias, running_mean, running_var, num_batches_tracked, num_valid, momentum, eps, transport`` ->
    training-mode BatchNorm whose statistics cover rows ``[0, num_valid)`` of every rank of ``transport``
    (:func:`ops.masked_sync_batch_norm_forward`).  The backward exchanges again over the same transport and gives
    dx (0 on padding rows) and this rank's dweight and dbias."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, num_batches_tracked, num_valid, momentum, eps,
                transport):
        y, mean, invstd = ops.masked_sync_batch_norm_forward(x, num_valid, weight, bias, running_mean, running_var,
                                                             num_batches_tracked, momentum, eps, transport)
        ctx.save_for_backward(x, weight, mean, invstd, num_valid)
        ctx.transport = transport
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        x, weight, mean, invstd, num_valid = ctx.saved_tensors
        dx, dw, db = ops.masked_sync_batch_norm_backward(x, grad_output, num_valid, weight, mean, invstd,
                                                         ctx.transport, ctx.needs_input_grad[1],
                                                         ctx.needs_input_grad[2])
        return dx, dw, db, None, None, None, None, None, None, None


def masked_sync_batch_norm(x, weight, bias, running_mean, running_var, num_batches_tracked, num_valid, momentum, eps,
                           process_group=None):
    """:class:`MaskedSyncBatchNormFunction` over the transport :func:`ops.sync_bn_transport` picks for
    ``process_group``: the installed peer group, else ``torch.distributed``, else this rank alone."""
    return MaskedSyncBatchNormFunction.apply(x, weight, bias, running_mean, running_var, num_batches_tracked,
                                             num_valid, momentum, eps, ops.sync_bn_transport(process_group))


# ---------------------------------------------------------------------------- per-sample GroupNorm
class MaskedGroupNormFunction(Function):
    """``x, weight, bias, indices, batch_size, num_valid, num_groups, eps, scale, shift, act`` -> per-sample GroupNorm
    over the rows ``[0, num_valid)`` whose batch index is in range, modulated by fp32 ``scale`` / ``shift`` and
    followed by ``act`` (:func:`ops.masked_group_norm_forward`).  The backward reuses the forward's grouping and
    gives dx (0 on padding and dropped rows), dweight, dbias, dscale and dshift."""

    @staticmethod
    def forward(ctx, x, weight, bias, indices, batch_size, num_valid, num_groups, eps, scale=None, shift=None,
                act=None):
        y, mean, invstd, order, offsets, cstart = ops.masked_group_norm_forward(
            x, indices, batch_size, num_valid, num_groups, weight, bias, eps, scale, shift, act)
        ctx.save_for_backward(x, weight, bias, indices, num_valid, mean, invstd, order, offsets, cstart, scale, shift)
        ctx.batch_size, ctx.num_groups, ctx.act = batch_size, num_groups, act
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        x, weight, bias, indices, num_valid, mean, invstd, order, offsets, cstart, scale, shift = ctx.saved_tensors
        given = len(ctx.needs_input_grad)                   # 8 when called without scale, shift and act
        need = tuple(ctx.needs_input_grad) + (False,) * (11 - given)
        dx, dw, db, ds, dt = ops.masked_group_norm_backward(
            x, grad_output, indices, ctx.batch_size, num_valid, ctx.num_groups, weight, mean, invstd, order, offsets,
            cstart, need[1], need[2], bias, scale, shift, ctx.act, need[8], need[9])
        return (dx, dw, db, None, None, None, None, None, ds, dt, None)[:given]


def _fp32(t):
    # the kernels read scale / shift in fp32: another float dtype runs on an fp32 copy, whose gradient autograd
    # casts back; anything else reaches the checks of ops unchanged
    return t.float() if t is not None and t.is_floating_point() and t.dtype != torch.float32 else t


def masked_group_norm(x, weight, bias, indices, batch_size, num_valid, num_groups, eps, scale=None, shift=None,
                      act=None):
    """Per-sample GroupNorm of ``x`` (:class:`MaskedGroupNormFunction`); with ``scale`` / ``shift``
    (``[batch_size, C]``) the normalised value of sample b becomes ``h * (1 + scale[b]) + shift[b]``, then ``act``
    (None, ``"relu"`` or ``"silu"``) is applied, all in one kernel."""
    return MaskedGroupNormFunction.apply(x, weight, bias, indices, batch_size, num_valid, num_groups, eps,
                                         _fp32(scale), _fp32(shift), act)


# ---------------------------------------------------------------------------- padding-aware global pooling
class MaskedGlobalPoolFunction(Function):
    """``features, indices, batch_size, num_valid, is_mean`` -> ``[batch_size, C]``: per-sample max or mean over
    the rows ``[0, num_valid)`` whose batch index is in range (:func:`ops.masked_global_pool_fwd`).  The backward
    gives the features' gradient: ``dy`` at the argmax row (max) or ``dy / count`` (mean), 0 on the other rows."""

    @staticmethod
    def forward(ctx, features, indices, batch_size, num_valid, is_mean):
        out, aux = ops.masked_global_pool_fwd(features, indices, batch_size, num_valid, is_mean)
        ctx.save_for_backward(indices, num_valid, aux)
        ctx.batch_size = batch_size
        ctx.is_mean = is_mean
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        indices, num_valid, aux = ctx.saved_tensors
        din = ops.masked_global_pool_bwd(grad_output, indices, ctx.batch_size, num_valid, aux, ctx.is_mean)
        return din, None, None, None, None


masked_global_pool = MaskedGlobalPoolFunction.apply


# ---------------------------------------------------------------------------- point -> voxel reductions
class PointScatterFunction(Function):
    """``x, row32, order, offsets, count, mode`` -> ``[rows, C]``: per-row max, mean or sum of the points
    (:func:`ops.point_scatter_fwd`).  The backward gives ``x``'s gradient: ``dy`` at the argmax point (max),
    ``dy / count`` (mean) or ``dy`` (sum) on the row's points, 0 on dropped points."""

    @staticmethod
    def forward(ctx, x, row32, order, offsets, count, mode):
        out, argmax = ops.point_scatter_fwd(x, order, offsets, mode)
        ctx.save_for_backward(row32, argmax if mode == "max" else (count if mode == "mean" else None))
        ctx.mode = mode
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        row32, aux = ctx.saved_tensors
        return ops.point_scatter_bwd(grad_output, row32, aux, ctx.mode), None, None, None, None, None


point_scatter = PointScatterFunction.apply


# ---------------------------------------------------------------------------- voxel -> point interpolation
class PointInterpFunction(Function):
    """``features, index, weight, order, offsets`` -> ``[P, C]``: the interpolation of the rows ``features [rows, C]``
    at the points of a plan (:func:`ops.point_interp_plan`, :func:`ops.point_interp_fwd`).  The backward gives the
    features' gradient (:func:`ops.point_interp_bwd`): a weighted segment sum per row, no atomics.  The plan is
    constant: there is no gradient to the positions or the weights."""

    @staticmethod
    def forward(ctx, features, index, weight, order, offsets):
        ctx.save_for_backward(weight, order, offsets)
        return ops.point_interp_fwd(features, index, weight)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        weight, order, offsets = ctx.saved_tensors
        return ops.point_interp_bwd(grad_output, weight, order, offsets), None, None, None, None


point_interp = PointInterpFunction.apply
