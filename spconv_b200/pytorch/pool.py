"""Sparse pooling modules on the conv rulebooks: ``SparseMaxPool{1..4}d``, ``SparseAvgPool{1..3}d``,
``SparseGlobalMaxPool`` / ``SparseGlobalAvgPool``, and the padding-aware, capturable global pools
``MaskedGlobalMaxPool`` / ``MaskedGlobalAvgPool`` (``spx_global_pool_fwd/bwd``).

Behaviour follows ``spconv/pytorch/pool.py``: constructor arguments :36-81 / :288-318 (``stride=None``
means ``kernel_size``), algo default :66-80, rulebook caching under ``indice_key`` :144-230, the
pooled tensor takes the output coordinate set of a regular conv with the same geometry
(``subm=True`` keeps the input set).  The reductions run in ``spx_indice_pool_fwd/bwd``.
"""
from __future__ import annotations

from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from ..core import ConvAlgo
from . import functional as Fsp
from . import ops
from .core import ImplicitGemmIndiceData, IndiceData, SparseConvTensor, expand_nd, rulebook_num_valid
from .modules import SparseModule

_MAX_NUM_VOXELS_DURING_TRAINING = "max_num_voxels_during_training"
IntOrSeq = Union[int, List[int], Tuple[int, ...]]


class _SparsePool(SparseModule):
    """Shared geometry / rulebook handling of the max and average pools."""

    def __init__(self, ndim: int, kernel_size: IntOrSeq = 3, stride: Optional[IntOrSeq] = 1,
                 padding: IntOrSeq = 0, dilation: IntOrSeq = 1, indice_key: Optional[str] = None,
                 subm: bool = False, algo: Optional[ConvAlgo] = None, record_voxel_count: bool = False,
                 name=None):
        super().__init__(name=name)
        self.ndim = ndim
        self.kernel_size = expand_nd(ndim, kernel_size)
        self.stride = list(self.kernel_size) if stride is None else expand_nd(ndim, stride)
        self.padding = expand_nd(ndim, padding)
        self.dilation = expand_nd(ndim, dilation)
        self.subm = subm
        self.indice_key = indice_key
        self.record_voxel_count = record_voxel_count
        # as SparseConvolution.num_out_act_bound: bounded implicit-GEMM rulebook, padded output, no host sync
        self.num_out_act_bound: Optional[int] = None
        if record_voxel_count and not subm:
            self.register_buffer(_MAX_NUM_VOXELS_DURING_TRAINING, torch.zeros(1, dtype=torch.int32))
        self.algo = algo

    def extra_repr(self):
        s = f"kernel_size={self.kernel_size}, stride={self.stride}"
        if self.padding != [0] * self.ndim:
            s += f", padding={self.padding}"
        if self.dilation != [1] * self.ndim:
            s += f", dilation={self.dilation}"
        return s + f", algo={self.algo}"

    def get_max_num_voxels(self) -> Optional[torch.Tensor]:
        return getattr(self, _MAX_NUM_VOXELS_DURING_TRAINING, None)

    def _out_shape(self, spatial_shape):
        if self.subm:
            return spatial_shape
        return ops.get_conv_output_size(spatial_shape, self.kernel_size, self.stride, self.padding, self.dilation)

    def _implicit_rulebook(self, input: SparseConvTensor, out_spatial_shape, indice_dict):
        bounded = (self.num_out_act_bound is not None and self.num_out_act_bound > 0 and not self.subm
                   and self.algo == ConvAlgo.MaskImplicitGemm)
        with input._timer.namespace("gen_pairs"):
            res = ops.get_indice_pairs_implicit_gemm(
                input.indices, input.batch_size, input.spatial_shape, self.algo, ksize=self.kernel_size,
                stride=self.stride, padding=self.padding, dilation=self.dilation,
                out_padding=[0] * self.ndim, subm=self.subm, is_train=(not self.subm) or self.training,
                alloc=input.thrust_allocator, timer=input._timer,
                num_out_act_bound=self.num_out_act_bound if bounded else -1,
                bound_status=self._status_word(input.indices.device) if bounded else None)
        if self.indice_key is not None:
            assert self.indice_key not in indice_dict, \
                f"your indice key {self.indice_key} already exists in this sparse tensor."
            indice_dict[self.indice_key] = ImplicitGemmIndiceData.from_rulebook(
                res, input.indices, input.num_valid, self.subm, spatial_shape=input.spatial_shape,
                out_spatial_shape=out_spatial_shape, algo=self.algo, ksize=self.kernel_size, stride=self.stride,
                dilation=self.dilation, padding=self.padding)
        return res[0], res[2], res[3]                       # out_inds, pair_fwd, pair_bwd

    def _finish(self, input: SparseConvTensor, out_features, outids, indice_dict, out_spatial_shape):
        out = input.shadow_copy().replace_feature(out_features)
        num_valid = rulebook_num_valid(outids, input, out, self.subm, self)
        if not self.subm and self.record_voxel_count and hasattr(self, _MAX_NUM_VOXELS_DURING_TRAINING):
            ops.maximum_value_int_(getattr(self, _MAX_NUM_VOXELS_DURING_TRAINING),
                                   outids.shape[0] if num_valid is None else num_valid)
        out.num_valid = num_valid
        out.indices = outids
        out.indice_dict = indice_dict
        out.spatial_shape = out_spatial_shape
        return out


class SparseMaxPool(_SparsePool):
    def __init__(self, ndim, kernel_size: IntOrSeq = 3, stride: Optional[IntOrSeq] = 1, padding: IntOrSeq = 0,
                 dilation: IntOrSeq = 1, indice_key: Optional[str] = None, subm: bool = False,
                 algo: Optional[ConvAlgo] = None, record_voxel_count: bool = False, name=None):
        super().__init__(ndim, kernel_size, stride, padding, dilation, indice_key, subm, algo,
                         record_voxel_count, name)
        kv = int(np.prod(self.kernel_size))
        if self.algo is None:
            # the implicit-GEMM rulebook is what a paired SparseInverseConv consumes (pool.py:66-76)
            self.algo = ConvAlgo.MaskImplicitGemm if kv <= 128 else ConvAlgo.Native
        if kv > 128:
            assert self.algo == ConvAlgo.Native, "implicit gemm don't support kv >= 32 for now"

    def forward(self, input: SparseConvTensor):
        assert isinstance(input, SparseConvTensor)
        out_spatial_shape = self._out_shape(input.spatial_shape)
        indice_dict = input.indice_dict.copy()
        if self.algo == ConvAlgo.Native:
            outids, indice_pairs, indice_pairs_num = ops.get_indice_pairs(
                input.indices, input.batch_size, input.spatial_shape, ConvAlgo.Native, self.kernel_size,
                self.stride, self.padding, self.dilation, [0] * self.ndim, False)
            if self.indice_key is not None:
                if input.find_indice_pair(self.indice_key) is not None:
                    raise ValueError(f"indice key {self.indice_key} exists")
                indice_dict[self.indice_key] = IndiceData(
                    outids, input.indices, indice_pairs, indice_pairs_num, input.spatial_shape,
                    out_spatial_shape, is_subm=False, algo=self.algo, ksize=self.kernel_size,
                    stride=self.stride, padding=self.padding, dilation=self.dilation)
            out_features = Fsp.indice_maxpool(input.features, indice_pairs, indice_pairs_num, outids.shape[0])
        else:
            outids, pair_fwd, pair_bwd = self._implicit_rulebook(input, out_spatial_shape, indice_dict)
            out_features = Fsp.indice_maxpool_implicit_gemm(input.features, pair_fwd, pair_bwd, outids.shape[0],
                                                            getattr(outids, "_spx_num_valid", None))
        return self._finish(input, out_features, outids, indice_dict, out_spatial_shape)


class SparseAvgPool(_SparsePool):
    def __init__(self, ndim, kernel_size: IntOrSeq = 3, stride: Optional[IntOrSeq] = 1, padding: IntOrSeq = 0,
                 dilation: IntOrSeq = 1, indice_key: Optional[str] = None, subm: bool = False,
                 algo: Optional[ConvAlgo] = None, record_voxel_count: bool = False, name=None):
        super().__init__(ndim, kernel_size, stride, padding, dilation, indice_key, subm, algo,
                         record_voxel_count, name)
        kv = int(np.prod(self.kernel_size))
        assert kv <= 32, "avg pool only support implicit-gemm style indice gen with kv <= 32 limit"
        self.algo = ConvAlgo.MaskImplicitGemm

    def forward(self, input: SparseConvTensor):
        assert isinstance(input, SparseConvTensor)
        out_spatial_shape = self._out_shape(input.spatial_shape)
        indice_dict = input.indice_dict.copy()
        outids, pair_fwd, pair_bwd = self._implicit_rulebook(input, out_spatial_shape, indice_dict)
        out_features = Fsp.indice_avgpool_implicit_gemm(input.features, pair_fwd, pair_bwd, outids.shape[0],
                                                        self.training)
        return self._finish(input, out_features, outids, indice_dict, out_spatial_shape)


class SparseGlobalMaxOrAvgPool(SparseModule):
    """Per-sample reduction over all active voxels -> dense ``[batch, C]`` (``pool.py:251-278``).
    Rows are grouped on the device (``spx_global_pool_rearrange``); the reductions are torch ops so
    autograd provides the backward, as in the reference."""

    def __init__(self, is_mean: bool, name=None):
        super().__init__(name=name)
        self.is_mean = is_mean

    def forward(self, input: SparseConvTensor):
        assert isinstance(input, SparseConvTensor)
        input.require_unpadded("global pooling")
        out_indices, counts = ops.global_pool_rearrange(input.indices, input.batch_size)
        counts_cpu = counts.cpu().tolist()
        rows = []
        for b in range(input.batch_size):
            feats = input.features[out_indices[b, :counts_cpu[b]].long()]
            rows.append(feats.mean(dim=0) if self.is_mean else feats.max(dim=0)[0])
        return torch.stack(rows)


class SparseGlobalAvgPool(SparseGlobalMaxOrAvgPool):
    def __init__(self, name=None):
        super().__init__(is_mean=True, name=name)


class SparseGlobalMaxPool(SparseGlobalMaxOrAvgPool):
    def __init__(self, name=None):
        super().__init__(is_mean=False, name=name)


class MaskedGlobalMaxOrAvgPool(SparseModule):
    """Per-sample reduction over the valid rows -> dense ``[batch, C]``, in CUDA (``csrc/global_pool.cu``) with no
    host synchronisation, so a net that ends in a global pool captures as one CUDA graph.  Accepts padded and
    unpadded tensors: only rows below ``x.num_valid`` count, and they are never read beyond it.  Rows whose batch
    index is outside ``[0, batch_size)`` are dropped.  float32, float16 and bfloat16 features.

    Max returns the value of the first row (in row order) that attains the maximum, bit for bit; a NaN counts as
    the maximum and -0 / +0 tie.  Its gradient goes to that one row, as ``torch.max(dim)``'s does.  Mean is the
    fp32 sum of the sample's rows divided by their count, rounded once; its gradient is ``dy / count`` on every
    row of the sample.  Padding and dropped rows get a zero gradient.

    Differences from the reference's global pools (``spconv/pytorch/pool.py:251-278``):
      * an empty sample gives 0 (the reference's max raises, its mean gives NaN);
      * the output is ``[batch, C]`` for the mean too (the reference's average pool returns channel 0 only);
      * results are deterministic: the rows of a sample are reduced in a fixed order, whatever the padding."""

    def __init__(self, is_mean: bool, name=None):
        super().__init__(name=name)
        self.is_mean = is_mean

    def forward(self, input: SparseConvTensor):
        assert isinstance(input, SparseConvTensor)
        return Fsp.masked_global_pool(input.features, input.indices, input.batch_size, input.num_valid,
                                      self.is_mean)


class MaskedGlobalAvgPool(MaskedGlobalMaxOrAvgPool):
    def __init__(self, name=None):
        super().__init__(is_mean=True, name=name)


class MaskedGlobalMaxPool(MaskedGlobalMaxOrAvgPool):
    def __init__(self, name=None):
        super().__init__(is_mean=False, name=name)


def _variant(base, cls_name: str, ndim: int):
    def __init__(self, kernel_size, stride=None, padding=0, dilation=1, indice_key=None, algo=None,
                 record_voxel_count=False, name=None):
        base.__init__(self, ndim, kernel_size, stride, padding, dilation, indice_key=indice_key, algo=algo,
                      record_voxel_count=record_voxel_count, name=name)
    return type(cls_name, (base,), {"__init__": __init__, "__module__": __name__,
                                    "__doc__": f"{ndim}-D sparse {'max' if base is SparseMaxPool else 'average'} "
                                               "pooling (stride=None means kernel_size)."})


for _nd in (1, 2, 3, 4):
    globals()[f"SparseMaxPool{_nd}d"] = _variant(SparseMaxPool, f"SparseMaxPool{_nd}d", _nd)
for _nd in (1, 2, 3):
    globals()[f"SparseAvgPool{_nd}d"] = _variant(SparseAvgPool, f"SparseAvgPool{_nd}d", _nd)
