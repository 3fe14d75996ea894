"""Sparse convolution modules: ``SparseConv{1..4}d``, ``SubMConv{1..4}d``,
``SparseInverseConv{1..4}d``, ``SparseConvTranspose{1..4}d``.

Behavioural contract follows ``spconv/pytorch/conv.py`` (constructor kwargs :63-84, algo default
:110-120, KRSC weight :136-139, ``indice_key`` caching and its error messages :247-319,
:345-444, :519-560, bias outside the op in training :492-493, kaiming-uniform init :705-750).
"""
from __future__ import annotations

import math
import sys
from typing import List, Optional, Tuple, Union

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F
from torch.nn import init
from torch.nn.parameter import Parameter

from .. import constants as _constants
from ..core import Activation, ConvAlgo
from . import functional as Fsp
from . import ops
from .core import (ImplicitGemmIndiceData, IndiceData, SparseConvTensor, expand_nd, rulebook_num_valid)
from .modules import SparseModule

_MAX_NUM_VOXELS_DURING_TRAINING = "max_num_voxels_during_training"
IntOrSeq = Union[int, List[int], Tuple[int, ...]]


def _activate(x: torch.Tensor, act_type: Activation, alpha: float, beta: float) -> torch.Tensor:
    if act_type == Activation.None_:
        return x
    if act_type == Activation.ReLU:
        return F.relu(x)
    if act_type == Activation.Sigmoid:
        return torch.sigmoid(x)
    if act_type == Activation.LeakyReLU:
        return F.leaky_relu(x, alpha)
    raise NotImplementedError(act_type)


class SparseConvolution(SparseModule):
    """Base of every sparse conv module.  Weight layout is KRSC ``[K, *ksize, C]``."""

    __constants__ = ["stride", "padding", "dilation", "groups", "bias", "subm", "inverse",
                     "transposed", "output_padding"]

    def __init__(self, ndim: int, in_channels: int, out_channels: int, kernel_size: IntOrSeq = 3,
                 stride: IntOrSeq = 1, padding: IntOrSeq = 0, dilation: IntOrSeq = 1,
                 groups: int = 1, bias: bool = True, subm: bool = False,
                 output_padding: IntOrSeq = 0, transposed: bool = False, inverse: bool = False,
                 indice_key: Optional[str] = None, algo: Optional[ConvAlgo] = None,
                 fp32_accum: Optional[bool] = None, record_voxel_count: bool = False,
                 act_type: Activation = Activation.None_, act_alpha: float = 0,
                 act_beta: float = 0, large_kernel_fast_algo: bool = False,
                 name=None, device=None, dtype=None):
        super().__init__(name=name)
        # groups: 1, depthwise (groups == in_channels == out_channels > 1), or grouped: both group widths
        # in_channels / groups and out_channels / groups multiples of 16 (every group is a dense GEMM of that width)
        grouped = (groups > 1 and in_channels % groups == 0 and out_channels % groups == 0
                   and (in_channels // groups) % 16 == 0 and (out_channels // groups) % 16 == 0)
        assert groups == 1 or (groups > 1 and groups == in_channels == out_channels) or grouped, \
            f"groups must be 1, in_channels == out_channels (depthwise), or leave group widths in_channels / groups " \
            f"and out_channels / groups that are multiples of 16; got groups={groups} for " \
            f"{in_channels} -> {out_channels} channels"
        self.ndim = ndim
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = expand_nd(ndim, kernel_size)
        self.stride = expand_nd(ndim, stride)
        self.dilation = expand_nd(ndim, dilation)
        self.padding = expand_nd(ndim, padding)
        self.output_padding = expand_nd(ndim, output_padding)
        self.groups = groups
        self.depthwise = groups > 1 and groups == in_channels == out_channels
        self.subm = subm
        self.transposed = transposed
        self.inverse = inverse
        self.indice_key = indice_key
        self.record_voxel_count = record_voxel_count
        # strided / transposed layers with the masked implicit-GEMM algo: an upper limit on the output count.
        # When set the rulebook runs without a host read-back, the output has exactly this many rows and
        # carries ``num_valid`` (spconv.set_output_bounds finds the value).  None: exact shapes, one sync.
        self.num_out_act_bound: Optional[int] = None
        self.fp32_accum = fp32_accum
        self.act_type, self.act_alpha, self.act_beta = act_type, act_alpha, act_beta
        kv = int(np.prod(self.kernel_size))
        # a 1x1(x1) stride-1 kernel is a plain matmul on the features
        self.conv1x1 = kv == 1 and (subm or int(np.prod(self.stride)) == 1)
        if self.conv1x1 and not subm:
            assert self.padding == [0] * ndim, "padding must be zero for 1x1 conv (k=1,s=1)"
        if self.conv1x1:
            assert act_type == Activation.None_, "conv1x1 don't support fused act"
        if algo is None:
            # reference default: masked implicit GEMM whenever the mask fits (kv <= 32, or <= 128
            # with large_kernel_fast_algo), else Native
            algo = (ConvAlgo.MaskImplicitGemm if kv <= (128 if large_kernel_fast_algo else 32)
                    else ConvAlgo.Native)
        self.algo = algo
        self.weight_shape = [out_channels, *self.kernel_size, in_channels // groups]
        factory = {"device": device, "dtype": dtype}
        self.weight = Parameter(torch.empty(*self.weight_shape, **factory))
        if bias:
            self.bias = Parameter(torch.empty(out_channels, **factory))
        else:
            self.register_parameter("bias", None)
        if record_voxel_count and not subm and not inverse:
            self.register_buffer(_MAX_NUM_VOXELS_DURING_TRAINING, torch.zeros(1, dtype=torch.int32))
        self.reset_parameters()
        self._register_load_state_dict_pre_hook(self._load_weight_different_layout)

    # ------------------------------------------------------------------ checkpoints
    def get_max_num_voxels(self) -> Optional[torch.Tensor]:
        return getattr(self, _MAX_NUM_VOXELS_DURING_TRAINING, None)

    def _load_weight_different_layout(self, state_dict, prefix, local_metadata, strict, missing_keys,
                                      unexpected_keys, error_msgs):
        """``load_state_dict`` pre-hook (``spconv/pytorch/conv.py:648-683``): checkpoints written by
        spconv 1.x / 2.1 hold filters as RSKC ``[*ksize, K, C]`` or RSCK ``[*ksize, C, K]``; with
        ``SPCONV_SAVED_WEIGHT_LAYOUT`` set to that layout they are permuted to this engine's (and
        spconv >= 2.2's) KRSC ``[K, *ksize, C]`` while loading.  Also supplies the voxel-count buffer
        when an older checkpoint lacks it.

        (The reference applies its permutation twice when ``ALL_WEIGHT_IS_KRSC`` -- :661-673 -- which
        only round-trips for degenerate shapes; the conversion here is applied once.)"""
        name = prefix + _MAX_NUM_VOXELS_DURING_TRAINING
        if self.record_voxel_count and not self.subm and not self.inverse and name not in state_dict:
            state_dict[name] = torch.zeros(1, dtype=torch.int32)
        layout = _constants.SAVED_WEIGHT_LAYOUT
        if not layout or layout == "KRSC":
            return
        key = prefix + "weight"
        if key not in state_dict:
            return
        nd = self.ndim
        w = state_dict[key]
        if layout == "RSKC":
            state_dict[key] = w.permute(nd, *range(nd), nd + 1).contiguous()
        elif layout == "RSCK":
            state_dict[key] = w.permute(nd + 1, *range(nd), nd).contiguous()
        else:
            raise ValueError(f"SPCONV_SAVED_WEIGHT_LAYOUT must be KRSC, RSKC or RSCK, got {layout!r}")

    # ------------------------------------------------------------------ parameters
    def reset_parameters(self):
        """kaiming-uniform(a=sqrt(5)) on fan_in = (C / groups) * kv, bias U(+-1/sqrt(fan_in))."""
        fan_in = self.in_channels // self.groups * int(np.prod(self.kernel_size))
        gain = math.sqrt(2.0 / (1 + 5.0))
        bound = gain * math.sqrt(3.0 / fan_in)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)
            if self.bias is not None:
                b = 1 / math.sqrt(fan_in)
                self.bias.uniform_(-b, b)

    def extra_repr(self):
        parts = [f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}",
                 f"stride={self.stride}"]
        if self.padding != [0] * self.ndim:
            parts.append(f"padding={self.padding}")
        if self.dilation != [1] * self.ndim:
            parts.append(f"dilation={self.dilation}")
        if self.output_padding != [0] * self.ndim:
            parts.append(f"output_padding={self.output_padding}")
        if self.groups != 1:
            parts.append(f"groups={self.groups}")
        if self.bias is None:
            parts.append("bias=False")
        parts.append(f"algo={self.algo}")
        return ", ".join(parts)

    def is_inverseable(self):
        return self.indice_key is not None and not self.subm

    def _bounded(self, algo: ConvAlgo) -> bool:
        return (self.num_out_act_bound is not None and self.num_out_act_bound > 0 and not self.subm
                and not self.inverse and algo == ConvAlgo.MaskImplicitGemm)

    # ------------------------------------------------------------------ cache validity
    def _check_subm_reuse_valid(self, inp: SparseConvTensor, spatial_shape: List[int], datas):
        assert datas.is_subm, "only support reuse subm indices"
        if self.kernel_size != datas.ksize:
            raise ValueError(f"subm with same indice_key must have same kernel size, "
                             f"expect {datas.ksize}, this layer {self.kernel_size}")
        if self.dilation != datas.dilation:
            raise ValueError(f"subm with same indice_key must have same dilation, "
                             f"expect {datas.dilation}, this layer {self.dilation}")
        if inp.spatial_shape != datas.spatial_shape:
            raise ValueError(f"subm with same indice_key must have same spatial structure, "
                             f"expect {datas.spatial_shape}, input {spatial_shape}")
        if inp.indices.shape[0] != datas.indices.shape[0]:
            raise ValueError(f"subm with same indice_key must have same num of indices, "
                             f"expect {datas.indices.shape[0]}, input {inp.indices.shape[0]}")

    def _check_prefetched_valid(self, inp: SparseConvTensor, datas):
        """A strided conv may only consume a rulebook that RulebookPrefetcher built for exactly this
        layer geometry and this input coordinate set."""
        assert getattr(datas, "prefetched", False), "only support reuse subm indices"
        same = (self.kernel_size == datas.ksize and self.stride == datas.stride and self.padding == datas.padding
                and self.dilation == datas.dilation and inp.spatial_shape == datas.spatial_shape
                and inp.indices.shape[0] == datas.indices.shape[0]
                and inp.indices.data_ptr() == datas.indices.data_ptr())
        if not same:
            raise ValueError(f"prefetched rulebook of indice_key {self.indice_key} does not match this layer / input: "
                             f"expect ksize {datas.ksize} stride {datas.stride} padding {datas.padding} dilation "
                             f"{datas.dilation} on {datas.indices.shape[0]} voxels in {datas.spatial_shape}")

    def _check_inverse_reuse_valid(self, inp: SparseConvTensor, spatial_shape: List[int], datas):
        if self.kernel_size != datas.ksize:
            raise ValueError(f"Inverse with same indice_key must have same kernel size, "
                             f"expect {datas.ksize}, this layer {self.kernel_size}, "
                             "please check Inverse Convolution in docs/USAGE.md.")
        if inp.spatial_shape != datas.out_spatial_shape:
            raise ValueError(f"Inverse with same indice_key must have same spatial structure "
                             f"(spatial shape), expect {datas.out_spatial_shape}, input "
                             f"{spatial_shape}, please check Inverse Convolution in docs/USAGE.md.")
        if inp.indices.shape[0] != datas.out_indices.shape[0]:
            raise ValueError(f"Inverse with same indice_key must have same num of indices, "
                             f"expect {datas.out_indices.shape[0]}, input {inp.indices.shape[0]}, "
                             "please check Inverse Convolution in docs/USAGE.md.")

    # ------------------------------------------------------------------ forward
    def _depthwise_native(self, features, weight, indice_pairs, indice_pair_num, n_out, timer, bias, act_alpha,
                          act_type):
        """Depthwise conv on ConvAlgo.Native compact pairs: scattered into the dense tables the kernels walk (the
        backward table only when a gradient can flow; SubM mirrors the forward table instead)."""
        kv = int(indice_pairs.shape[1])
        need_bwd = (not self.subm and torch.is_grad_enabled()
                    and (features.requires_grad or weight.requires_grad))
        with timer.record("depthwise_conv_table", ops._stream()):
            t_fwd, _, t_bwd, _ = ops._native_tables(indice_pairs.contiguous(), indice_pair_num, features.shape[0],
                                                    int(n_out), kv, self.subm, self.inverse, True, need_bwd)
        if not self.subm and t_bwd is None:
            t_bwd = torch.empty((kv, 0), dtype=torch.int32, device=features.device)     # no backward will run
        return Fsp.depthwise_conv(features, weight, t_fwd, t_bwd, n_out, timer, bias, act_alpha, act_type)

    def forward(self, input: SparseConvTensor, add_input: Optional[SparseConvTensor] = None, *,
                target: Optional[SparseConvTensor] = None):
        """``target``: convolve onto the coordinates of this tensor instead of the layer's own output set (SubM,
        strided and transposed layers, depthwise included).  It must have the input's ``batch_size`` and the layer's
        output spatial shape; the output takes its ``indices``, ``spatial_shape``, ``num_valid`` and a copy of its
        ``indice_dict``.  Only the input features, the weight and the bias get gradients.  The rulebook is
        registered under ``indice_key``: a later layer of the same geometry on the same input and target index tensors,
        given a target that carries the key, reuses it, and an inverse conv with the key walks it back to the input's coordinates."""
        return self._conv_forward(self.training, input, self.weight, self.bias, add_input,
                                  name=self.name, sparse_unique_name=self._sparse_unique_name,
                                  act_type=self.act_type, act_alpha=self.act_alpha,
                                  act_beta=self.act_beta, target=target)

    def _out_spatial_shape(self, spatial_shape):
        if self.subm:
            return spatial_shape
        if self.transposed:
            return ops.get_deconv_output_size(spatial_shape, self.kernel_size, self.stride,
                                              self.padding, self.dilation, self.output_padding)
        return ops.get_conv_output_size(spatial_shape, self.kernel_size, self.stride,
                                        self.padding, self.dilation)

    # ------------------------------------------------------------------ convolution onto given coordinates
    def _check_target(self, input: SparseConvTensor, target: SparseConvTensor, algo: ConvAlgo) -> None:
        """Every refusal of a ``target`` happens here, on the host, before any launch."""
        if not isinstance(target, SparseConvTensor):
            raise TypeError(f"target must be a SparseConvTensor, got {type(target).__name__}")
        if self.inverse:
            raise ValueError("an inverse conv restores the coordinates of the conv sharing its indice_key: it takes "
                             "no target")
        if algo == ConvAlgo.MaskSplitImplicitGemm:
            raise NotImplementedError("a conv onto given coordinates does not support ConvAlgo.MaskSplitImplicitGemm: "
                                      "use ConvAlgo.MaskImplicitGemm or ConvAlgo.Native")
        if int(np.prod(self.kernel_size)) > 128:
            raise NotImplementedError(f"a conv onto given coordinates supports kernel volume <= 128, this layer has "
                                      f"{self.kernel_size}")
        if target.batch_size != input.batch_size:
            raise ValueError(f"target batch_size {target.batch_size} differs from the input's {input.batch_size}")
        want = self._out_spatial_shape(input.spatial_shape)
        if target.indices.shape[1] != input.indices.shape[1] or list(target.spatial_shape) != list(want):
            raise ValueError(f"target spatial shape {target.spatial_shape} (indices {tuple(target.indices.shape)}) "
                             f"must be this layer's output shape {want} for the input's {input.spatial_shape}")

    def _cross_geometry(self) -> Tuple[List[int], List[int], bool]:
        """(stride, padding, transposed) of the relation a target is read through; SubM is stride 1, pad (k//2)*d."""
        if self.subm:
            return [1] * self.ndim, [(k // 2) * d for k, d in zip(self.kernel_size, self.dilation)], False
        return list(self.stride), list(self.padding), bool(self.transposed)

    def _cross_rulebook(self, input: SparseConvTensor, target: Optional[SparseConvTensor], algo: ConvAlgo):
        """The rulebook onto ``target``'s coordinates (``ops.get_indice_pairs_to``), reused from ``target``'s
        ``indice_dict`` under ``indice_key`` when present (built on the same input and target index tensors); with ``target`` None, the one under ``indice_key`` in the
        input's dict walked back by an inverse conv.  Returns ``_rulebook``'s 4-tuple in the implicit-GEMM form."""
        if target is None:
            datas = input.find_indice_pair(self.indice_key)
            self._check_inverse_reuse_valid(input, input.spatial_shape, datas)
            rb = (datas.indices, datas.pair_bwd, datas.pair_fwd, datas.pair_mask_bwd_splits,
                  datas.pair_mask_fwd_splits, datas.mask_argsort_bwd_splits, datas.mask_argsort_fwd_splits, datas.masks)
            return rb, input.indice_dict.copy(), datas.spatial_shape, datas.in_voxel_num
        stride, padding, transposed = self._cross_geometry()
        indice_dict = target.indice_dict.copy()
        datas = target.find_indice_pair(self.indice_key)
        if datas is not None:
            same = (getattr(datas, "cross", False) and self.kernel_size == datas.ksize and stride == datas.stride
                    and padding == datas.padding and self.dilation == datas.dilation
                    and transposed == datas.transposed and input.spatial_shape == datas.spatial_shape
                    and target.spatial_shape == datas.out_spatial_shape
                    and input.indices.shape[0] == datas.indices.shape[0]
                    and target.indices.shape[0] == datas.out_indices.shape[0]
                    # the same coordinate tensors, not only the same row counts (padded tensors all share theirs)
                    and input.indices.data_ptr() == datas.indices.data_ptr()
                    and target.indices.data_ptr() == datas.out_indices.data_ptr())
            if not same:
                raise ValueError(f"the rulebook under indice_key {self.indice_key} in the target does not match this "
                                 f"layer and input: expect a conv onto given coordinates with ksize {datas.ksize} "
                                 f"stride {datas.stride} padding {datas.padding} dilation {datas.dilation} from the "
                                 f"{datas.indices.shape[0]} voxels in {datas.spatial_shape} it was built on onto its "
                                 f"{datas.out_indices.shape[0]} target voxels in {datas.out_spatial_shape}")
        else:
            with input._timer.namespace("gen_pairs"):
                res = ops.get_indice_pairs_to(input.indices, target.indices, input.batch_size, input.spatial_shape,
                                              target.spatial_shape, self.kernel_size, stride, padding, self.dilation,
                                              transposed, True, input.num_valid, target.num_valid)
            # the record keeps the target's own index tensor (res[0] may be an aligned copy of it)
            datas = ImplicitGemmIndiceData.from_rulebook(
                (target.indices, *res[1:]), input.indices, input.num_valid, False, spatial_shape=input.spatial_shape,
                out_spatial_shape=target.spatial_shape, algo=algo, ksize=self.kernel_size, stride=stride,
                dilation=self.dilation, padding=padding, cross=True, transposed=transposed)
            datas.out_voxel_num = target.num_valid
            if self.indice_key is not None:
                indice_dict[self.indice_key] = datas
        rb = (target.indices, datas.pair_fwd, datas.pair_bwd, datas.pair_mask_fwd_splits, datas.pair_mask_bwd_splits,
              datas.mask_argsort_fwd_splits, datas.mask_argsort_bwd_splits, datas.masks)
        return rb, indice_dict, target.spatial_shape, target.num_valid

    def _rulebook_error(self, tag, indices, batch_size, spatial_shape, algo):
        print(f"[Exception|{tag}]indices={indices.shape},bs={batch_size},ss={spatial_shape},"
              f"algo={algo},ksize={self.kernel_size},stride={self.stride},padding={self.padding},"
              f"dilation={self.dilation},subm={self.subm},transpose={self.transposed}",
              file=sys.stderr)

    def _rulebook(self, input: SparseConvTensor, training: bool, algo: ConvAlgo, out_tensor: SparseConvTensor):
        """This layer's rulebook on ``input``: taken from ``input.indice_dict`` under ``indice_key`` (SubM reuse,
        a prefetched strided rulebook, or the paired conv's rulebook walked backwards by an inverse conv) or built
        and registered there.  Returns ``(rb, indice_dict, out_spatial_shape, num_valid)`` with ``rb`` =
        ``(outids, indice_pairs, indice_pair_num)`` for ConvAlgo.Native and ``(outids, pair_fwd, pair_bwd,
        mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks)`` for the implicit-GEMM algos.  A bounded rulebook's
        status word joins ``out_tensor.bound_status``.  The float and the fp8 convs share it."""
        indices = input.indices
        spatial_shape = input.spatial_shape
        batch_size = input.batch_size
        timer = input._timer
        out_spatial_shape = self._out_spatial_shape(spatial_shape)
        # SubM inherits the padding of its input; strided and inverse layers set it below
        num_valid = input.num_valid
        indice_dict = input.indice_dict.copy()
        datas = input.find_indice_pair(self.indice_key)
        if getattr(datas, "cross", False):
            raise ValueError(f"indice_key {self.indice_key} holds the rulebook of a conv onto given coordinates: only a "
                             "layer given a target carrying it or a float inverse conv can use it")
        if datas is not None:
            assert algo == datas.algo, ("due to limitation of pytorch, you must provide same algo "
                                        "to layers share same indice key.")

        if algo == ConvAlgo.Native:
            if datas is not None:
                assert isinstance(datas, IndiceData)
            if self.inverse:
                assert datas is not None and self.indice_key is not None
                assert datas.is_subm is False, \
                    "inverse conv can only be used with standard conv and pool ops."
                outids, indice_pairs, indice_pair_num = (datas.indices, datas.indice_pairs,
                                                         datas.indice_pair_num)
                out_spatial_shape = datas.spatial_shape
                self._check_inverse_reuse_valid(input, spatial_shape, datas)
            elif self.indice_key is not None and datas is not None:
                outids, indice_pairs, indice_pair_num = (datas.out_indices, datas.indice_pairs,
                                                         datas.indice_pair_num)
                assert self.subm, "only support reuse subm indices"
                self._check_subm_reuse_valid(input, spatial_shape, datas)
            else:
                try:
                    outids, indice_pairs, indice_pair_num = ops.get_indice_pairs(
                        indices, batch_size, spatial_shape, algo, self.kernel_size, self.stride,
                        self.padding, self.dilation, self.output_padding, self.subm,
                        self.transposed)
                except Exception:
                    self._rulebook_error("native_pair", indices, batch_size, spatial_shape, algo)
                    raise
                if self.indice_key is not None:
                    assert self.indice_key not in indice_dict, \
                        f"your indice key {self.indice_key} already exists in this sparse tensor."
                    indice_dict[self.indice_key] = IndiceData(
                        outids, indices, indice_pairs, indice_pair_num, spatial_shape,
                        out_spatial_shape, is_subm=self.subm, algo=algo, ksize=self.kernel_size,
                        stride=self.stride, padding=self.padding, dilation=self.dilation)
            if indice_pairs.device != input.features.device:
                indice_pairs = indice_pairs.to(input.features.device)
            return (outids, indice_pairs, indice_pair_num), indice_dict, out_spatial_shape, num_valid
        if datas is not None:
            assert isinstance(datas, ImplicitGemmIndiceData)
        if self.inverse:
            assert datas is not None and self.indice_key is not None
            assert datas.is_subm is False, \
                "inverse conv can only be used with standard conv and pool ops."
            # the inverse conv walks the paired conv's rulebook backwards
            outids = datas.indices
            num_valid = datas.in_voxel_num
            pair_fwd, pair_bwd = datas.pair_bwd, datas.pair_fwd
            mask_fwd, mask_bwd = datas.pair_mask_bwd_splits, datas.pair_mask_fwd_splits
            sort_fwd, sort_bwd = datas.mask_argsort_bwd_splits, datas.mask_argsort_fwd_splits
            masks = datas.masks
            out_spatial_shape = datas.spatial_shape
            self._check_inverse_reuse_valid(input, spatial_shape, datas)
        elif self.indice_key is not None and datas is not None:
            outids = datas.out_indices
            pair_fwd, pair_bwd = datas.pair_fwd, datas.pair_bwd
            mask_fwd, mask_bwd = datas.pair_mask_fwd_splits, datas.pair_mask_bwd_splits
            sort_fwd, sort_bwd = datas.mask_argsort_fwd_splits, datas.mask_argsort_bwd_splits
            masks = datas.masks
            if self.subm:
                self._check_subm_reuse_valid(input, spatial_shape, datas)
            else:
                self._check_prefetched_valid(input, datas)
                num_valid = datas.out_voxel_num
        else:
            with timer.namespace("gen_pairs"):
                try:
                    # regular convs always build the backward table: an inverse conv may
                    # consume it later
                    res = ops.get_indice_pairs_implicit_gemm(
                        indices, batch_size, spatial_shape, algo, ksize=self.kernel_size,
                        stride=self.stride, padding=self.padding, dilation=self.dilation,
                        out_padding=self.output_padding, subm=self.subm,
                        transpose=self.transposed, is_train=(not self.subm) or training,
                        alloc=input.thrust_allocator, timer=timer,
                        num_out_act_bound=self.num_out_act_bound if self._bounded(algo) else -1,
                        bound_status=self._status_word(indices.device) if self._bounded(algo) else None)
                except Exception:
                    self._rulebook_error("implicit_gemm_pair", indices, batch_size,
                                         spatial_shape, algo)
                    raise
            (outids, _num_per_loc, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd,
             masks) = res
            num_valid = rulebook_num_valid(outids, input, out_tensor, self.subm, self)
            if self.indice_key is not None:
                assert self.indice_key not in indice_dict, \
                    f"your indice key {self.indice_key} already exists in this sparse tensor."
                indice_dict[self.indice_key] = ImplicitGemmIndiceData.from_rulebook(
                    res, indices, input.num_valid, self.subm, spatial_shape=spatial_shape,
                    out_spatial_shape=out_spatial_shape, algo=algo, ksize=self.kernel_size,
                    stride=self.stride, dilation=self.dilation, padding=self.padding)
        return ((outids, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks), indice_dict,
                out_spatial_shape, num_valid)

    def _conv_forward(self, training: bool, input: SparseConvTensor, weight: torch.Tensor,
                      bias: Optional[torch.Tensor], add_input: Optional[SparseConvTensor] = None,
                      channel_scale: Optional[torch.Tensor] = None,
                      output_scale: Optional[float] = None, name: Optional[str] = None,
                      sparse_unique_name: str = "", act_type: Activation = Activation.None_,
                      act_alpha: float = 0, act_beta: float = 0,
                      target: Optional[SparseConvTensor] = None):
        assert isinstance(input, SparseConvTensor)
        assert input.features.shape[1] == self.in_channels, "channel size mismatch"
        if training:
            assert self.act_type == Activation.None_, \
                "act don't support backward, only used in inference"
        features = input.features
        # training: bias is added outside the op (it needs its own gradient);
        # inference: bias and activation ride in the kernel epilogue
        bias_train = bias if training else None
        bias_infer = None if training else bias
        out_spatial_shape = self._out_spatial_shape(input.spatial_shape)
        out_tensor = input.shadow_copy()
        algo = self.algo if input.force_algo is None else input.force_algo
        if target is not None:
            self._check_target(input, target, algo)
        # a conv onto given coordinates, or an inverse conv walking one back: dense tables whatever the algo
        cross = target is not None or (self.inverse and getattr(input.find_indice_pair(self.indice_key), "cross",
                                                                False))

        if self.conv1x1 and not cross:
            if self.depthwise:
                feats = features * weight.view(self.out_channels)
            elif self.groups > 1:
                # one batched matmul over the groups: [g, N, C/g] x [g, C/g, K/g]
                g = self.groups
                x3 = features.reshape(-1, g, self.in_channels // g).transpose(0, 1)
                w3 = weight.reshape(g, self.out_channels // g, self.in_channels // g)
                feats = torch.bmm(x3, w3.transpose(1, 2)).transpose(0, 1).reshape(-1, self.out_channels)
            else:
                w2d = weight.view(self.out_channels, self.in_channels)
                feats = torch.mm(features, w2d.t())
            if bias is not None:
                feats = feats + bias
            out_tensor = out_tensor.replace_feature(feats)
            out_tensor.spatial_shape = out_spatial_shape
            return out_tensor

        if not features.is_contiguous():
            features = features.contiguous()
        timer = input._timer
        if cross:
            rb, indice_dict, out_spatial_shape, num_valid = self._cross_rulebook(input, target, algo)
        else:
            rb, indice_dict, out_spatial_shape, num_valid = self._rulebook(input, training, algo, out_tensor)
        is_subm = self.subm and not cross          # cross tables are not symmetric

        if algo == ConvAlgo.Native and not cross:
            outids, indice_pairs, indice_pair_num = rb
            if self.depthwise:
                out_features = self._depthwise_native(features, weight, indice_pairs, indice_pair_num,
                                                      outids.shape[0], timer, bias_infer, act_alpha, act_type)
            else:
                conv_fn = (Fsp.indice_subm_conv if self.subm else
                           Fsp.indice_inverse_conv if self.inverse else Fsp.indice_conv)
                out_features = conv_fn(features, weight, indice_pairs, indice_pair_num,
                                       outids.shape[0], algo, timer, bias_infer, act_alpha, act_beta,
                                       act_type, groups=self.groups)
        else:
            outids, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks = rb
            num_activate_out = outids.shape[0]
            if self.depthwise:
                # the whole dense table is walked: no tile table, mask sort or split is needed.  SubM (whose
                # inference rulebook has no pair_bwd) walks pair_fwd with mirrored offsets in the backward
                out_features = Fsp.depthwise_conv(features, weight, pair_fwd, None if is_subm else pair_bwd,
                                                  num_activate_out, timer, bias_infer, act_alpha, act_type)
            elif training:
                out_features = Fsp.implicit_gemm(features, weight, pair_fwd, pair_bwd, mask_fwd,
                                                 mask_bwd, sort_fwd, sort_bwd, num_activate_out,
                                                 masks, training, is_subm, timer,
                                                 self.fp32_accum, bias_infer, act_alpha, act_beta,
                                                 act_type, self.groups)
            else:
                out_features, _, _ = ops.implicit_gemm(
                    features, weight, pair_fwd, mask_fwd, sort_fwd, num_activate_out, masks,
                    training, is_subm, timer, self.fp32_accum, bias_infer, act_alpha, act_beta,
                    act_type, 1.0 if output_scale is None else output_scale, channel_scale,
                    output_add=None, output_add_scale=0.0,
                    output_dtype=weight.dtype if output_scale is None else None, groups=self.groups)

        if bias_train is not None:
            out_features = out_features + bias_train.to(out_features.dtype)
        if not self.subm and not self.inverse and self.record_voxel_count:
            if hasattr(self, _MAX_NUM_VOXELS_DURING_TRAINING):
                ops.maximum_value_int_(getattr(self, _MAX_NUM_VOXELS_DURING_TRAINING),
                                       outids.shape[0] if num_valid is None else num_valid)
        if num_valid is not None and out_features.requires_grad:
            out_features = Fsp.zero_padding_grad(out_features, num_valid)
        out_tensor = out_tensor.replace_feature(out_features)
        out_tensor.num_valid = num_valid
        out_tensor.indices = outids
        out_tensor.indice_dict = indice_dict
        out_tensor.spatial_shape = out_spatial_shape
        if target is not None and (input.bound_status or target.bound_status):
            out_tensor.bound_status = {**(input.bound_status or {}), **(target.bound_status or {})}
        if add_input is not None:
            out_tensor = out_tensor.replace_feature(
                _activate(out_tensor.features + add_input.features, self.act_type, self.act_alpha,
                          self.act_beta))
        return out_tensor


def _make_variant(cls_name: str, ndim: int, kind: str, doc: str):
    """Build one public module class; ``kind`` in {conv, subm, inverse, transpose}."""

    if kind == "conv":
        def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                     groups=1, bias=True, indice_key=None, algo: Optional[ConvAlgo] = None,
                     fp32_accum: Optional[bool] = None, record_voxel_count: bool = False,
                     large_kernel_fast_algo: bool = False, name=None, **kw):
            SparseConvolution.__init__(self, ndim, in_channels, out_channels, kernel_size, stride,
                                       padding, dilation, groups, bias, indice_key=indice_key,
                                       algo=algo, fp32_accum=fp32_accum,
                                       record_voxel_count=record_voxel_count,
                                       large_kernel_fast_algo=large_kernel_fast_algo, name=name,
                                       **kw)
    elif kind == "subm":
        def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                     groups=1, bias=True, indice_key=None, algo: Optional[ConvAlgo] = None,
                     fp32_accum: Optional[bool] = None, large_kernel_fast_algo: bool = False,
                     name=None, **kw):
            SparseConvolution.__init__(self, ndim, in_channels, out_channels, kernel_size, stride,
                                       padding, dilation, groups, bias, True,
                                       indice_key=indice_key, algo=algo, fp32_accum=fp32_accum,
                                       large_kernel_fast_algo=large_kernel_fast_algo, name=name,
                                       **kw)
    elif kind == "inverse":
        def __init__(self, in_channels, out_channels, kernel_size, indice_key, bias=True,
                     algo: Optional[ConvAlgo] = None, fp32_accum: Optional[bool] = None,
                     large_kernel_fast_algo: bool = False, name=None, **kw):
            SparseConvolution.__init__(self, ndim, in_channels, out_channels, kernel_size,
                                       bias=bias, inverse=True, indice_key=indice_key, algo=algo,
                                       fp32_accum=fp32_accum,
                                       large_kernel_fast_algo=large_kernel_fast_algo, name=name,
                                       **kw)
    else:
        def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1,
                     groups=1, bias=True, indice_key=None, algo: Optional[ConvAlgo] = None,
                     fp32_accum: Optional[bool] = None, record_voxel_count: bool = False,
                     large_kernel_fast_algo: bool = False, name=None, **kw):
            SparseConvolution.__init__(self, ndim, in_channels, out_channels, kernel_size, stride,
                                       padding, dilation, groups, bias, transposed=True,
                                       indice_key=indice_key, algo=algo, fp32_accum=fp32_accum,
                                       record_voxel_count=record_voxel_count,
                                       large_kernel_fast_algo=large_kernel_fast_algo, name=name,
                                       **kw)
    return type(cls_name, (SparseConvolution,), {"__init__": __init__, "__doc__": doc,
                                                 "__module__": __name__})


for _nd in (1, 2, 3, 4):
    globals()[f"SparseConv{_nd}d"] = _make_variant(
        f"SparseConv{_nd}d", _nd, "conv", f"{_nd}-D strided sparse convolution (new active set).")
    globals()[f"SubMConv{_nd}d"] = _make_variant(
        f"SubMConv{_nd}d", _nd, "subm",
        f"{_nd}-D submanifold convolution (active set unchanged; stride/padding ignored).")
    globals()[f"SparseInverseConv{_nd}d"] = _make_variant(
        f"SparseInverseConv{_nd}d", _nd, "inverse",
        f"{_nd}-D inverse of the SparseConv sharing ``indice_key`` (restores its input set).")
    globals()[f"SparseConvTranspose{_nd}d"] = _make_variant(
        f"SparseConvTranspose{_nd}d", _nd, "transpose", f"{_nd}-D transposed sparse convolution.")
