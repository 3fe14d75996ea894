"""Static int8 inference hookup for sparse convs -- the hot-path part of the reference's quantization
toolchain (``spconv/pytorch/quantization/quantized/conv.py``): a conv whose filter is per-channel
symmetric int8, fed int8 features with a per-tensor scale, producing int8 features with the
layer's output scale through the int8 tensor-core kernel (``spx_implicit_gemm_fwd_int8``).

The per-channel epilogue scale is derived exactly as the reference does (``quantized/conv.py:368-377``)::

    channel_scale[k] = input_scale * weight_scale[k] / output_scale
    bias_q[k]        = bias[k] / output_scale
    y_q              = clip(rint(acc_i32 * channel_scale + bias_q [+ add_q * add_scale]), -128, 127)

The torch.ao FX tooling around it (observers, QAT modules, backend config; ``quantization/*.py``, 2 k
lines of framework glue) is out of this engine's scope: scales are given by the caller or taken
from calibration with :func:`calibrate_output_scale`.  CUDA per-tensor ``qint8`` tensors are not a
reliable carrier, so quantized activations travel as plain ``torch.int8`` features with the scale in
``SparseConvTensor.int8_scale``.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from ..core import Activation
from .conv import SparseConvolution
from .core import SparseConvTensor


def quantize_per_channel_weight(weight: torch.Tensor):
    """Symmetric per-output-channel int8 quantisation of a KRSC filter -> ``(w_int8, scales [K])``
    (what ``torch.ao``'s per-channel weight observer yields for qint8 symmetric)."""
    k = weight.shape[0]
    amax = weight.detach().float().abs().reshape(k, -1).amax(dim=1).clamp_min(1e-12)
    scales = amax / 127.0
    q = torch.clamp(torch.round(weight.detach().float() / scales.view(-1, *[1] * (weight.ndim - 1))), -127, 127)
    return q.to(torch.int8).contiguous(), scales


def quantize_tensor(x: SparseConvTensor, scale: float) -> SparseConvTensor:
    """float features -> int8 features with per-tensor ``scale`` (zero point 0)."""
    q = torch.clamp(torch.round(x.features.float() / scale), -128, 127).to(torch.int8)
    out = x.replace_feature(q)
    out.int8_scale = float(scale)
    return out


def dequantize_tensor(x: SparseConvTensor) -> SparseConvTensor:
    assert x.features.dtype == torch.int8 and x.int8_scale is not None, "not a quantized SparseConvTensor"
    out = x.replace_feature(x.features.float() * float(x.int8_scale))
    out.int8_scale = None
    return out


def calibrate_output_scale(conv: SparseConvolution, x: SparseConvTensor) -> float:
    """max-abs calibration of a float conv's output on one batch (a MinMax observer)."""
    with torch.no_grad():
        y = conv(x)
    return float(y.features.float().abs().max()) / 127.0


class QuantizedSparseConv(SparseConvolution):
    """Int8 inference twin of a float :class:`SparseConvolution` (same geometry, ``indice_key`` and
    fused activation).  Build with :meth:`from_float`."""

    @classmethod
    def from_float(cls, mod: SparseConvolution, output_scale: float) -> "QuantizedSparseConv":
        assert isinstance(mod, SparseConvolution) and not mod.conv1x1
        if getattr(mod, "depthwise", False):
            raise NotImplementedError(f"int8 depthwise convolution is not supported (groups={mod.groups}); "
                                      "keep this layer in floating point")
        if mod.groups != 1:
            raise NotImplementedError(f"int8 grouped convolution is not supported (groups={mod.groups}); "
                                      "keep this layer in floating point")
        q = cls(mod.ndim, mod.in_channels, mod.out_channels, mod.kernel_size, mod.stride, mod.padding,
                mod.dilation, mod.groups, mod.bias is not None, subm=mod.subm,
                output_padding=mod.output_padding, transposed=mod.transposed, inverse=mod.inverse,
                indice_key=mod.indice_key, algo=mod.algo, record_voxel_count=mod.record_voxel_count,
                act_type=mod.act_type, act_alpha=mod.act_alpha, act_beta=mod.act_beta)
        w_q, w_scales = quantize_per_channel_weight(mod.weight)
        del q.weight
        q.register_buffer("weight", w_q.to(mod.weight.device))
        q.register_buffer("weight_scales", w_scales.to(mod.weight.device))
        bias = mod.bias.detach().float() if mod.bias is not None else torch.zeros(mod.out_channels, device=mod.weight.device)
        q._parameters.pop("bias", None)               # Parameter or the registered None placeholder
        q.register_buffer("bias", bias.to(mod.weight.device))        # the reference requires a bias tensor
        q.scale = float(output_scale)
        q.zero_point = 0
        return q.eval()

    def reset_parameters(self):          # parameters are replaced by buffers in from_float
        return

    def forward(self, input: SparseConvTensor, add_input: Optional[SparseConvTensor] = None):
        assert input.features.dtype == torch.int8 and input.int8_scale is not None, \
            "int8 must be called in static quantized module"          # reference assertion text
        inp_scale = float(input.int8_scale)
        channel_scale = (inp_scale * self.weight_scales) / self.scale         # quantized/conv.py:372
        bias = self.bias / self.scale                                         # :373
        out = self._int8_forward(input, channel_scale, bias, add_input)
        out.int8_scale = self.scale
        return out

    def _int8_forward(self, input, channel_scale, bias, add_input):
        from . import ops
        from .core import ImplicitGemmIndiceData
        assert not self.inverse, "inverse conv has no int8 path"
        indice_dict = input.indice_dict.copy()
        datas = input.find_indice_pair(self.indice_key)
        out_spatial_shape = self._out_spatial_shape(input.spatial_shape)
        if self.indice_key is not None and datas is not None:
            assert self.subm, "only support reuse subm indices"
            self._check_subm_reuse_valid(input, input.spatial_shape, datas)
            outids, pair_fwd = datas.out_indices, datas.pair_fwd
            mask_fwd, sort_fwd, masks = datas.pair_mask_fwd_splits, datas.mask_argsort_fwd_splits, datas.masks
        else:
            res = ops.get_indice_pairs_implicit_gemm(
                input.indices, input.batch_size, input.spatial_shape, self.algo, ksize=self.kernel_size,
                stride=self.stride, padding=self.padding, dilation=self.dilation, out_padding=self.output_padding,
                subm=self.subm, transpose=self.transposed, is_train=not self.subm, alloc=input.thrust_allocator,
                timer=input._timer)
            outids, _, pair_fwd, _, mask_fwd, _, sort_fwd, _, masks = res
            if self.indice_key is not None:
                indice_dict[self.indice_key] = ImplicitGemmIndiceData.from_rulebook(
                    res, input.indices, None, self.subm, spatial_shape=input.spatial_shape,
                    out_spatial_shape=out_spatial_shape, algo=self.algo, ksize=self.kernel_size, stride=self.stride,
                    dilation=self.dilation, padding=self.padding)
        add_scale = 0.0
        add_feats = None
        if add_input is not None:                 # residual enters the epilogue (conv.py:511-512)
            add_feats = add_input.features
            add_scale = float(add_input.int8_scale)
        out_features, _, _ = ops.implicit_gemm(
            input.features, self.weight, pair_fwd, mask_fwd, sort_fwd, outids.shape[0], masks, False, self.subm,
            input._timer, None, bias, self.act_alpha, self.act_beta, self.act_type, self.scale, channel_scale,
            output_add=add_feats, output_add_scale=add_scale, output_dtype=torch.int8)
        out = input.shadow_copy().replace_feature(out_features)
        out.indices = outids
        out.indice_dict = indice_dict
        out.spatial_shape = out_spatial_shape
        return out
