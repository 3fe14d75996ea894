"""FP8 (e4m3) sparse convolution inference on the Hopper tensor cores.

e4m3 (``torch.float8_e4m3fn``: finite range +-448, no infinities) keeps about two decades of dynamic range inside
one per-tensor scale, so unlike the static int8 path (:mod:`.quantized`) a layer needs no calibrated input scale:
float features are quantised with a scale computed on the device (amax / 448 over the valid rows), and every scale
stays a device tensor, so no call reads anything back and a bounded fp8 network captures as one CUDA graph.

* filters: per-output-channel scale ``w_scale[k] = amax(|W[k]|) / 448`` (:func:`quantize_fp8_weight`);
* features: e4m3 rows with the per-tensor device scale in ``SparseConvTensor.fp8_scale`` (:func:`quantize_fp8`);
* epilogue (``spx_implicit_gemm_fwd_fp8`` in ``include/spconv_b200.h``), fp32 in registers, one IEEE operation
  per step: ``y = act(acc * (in_scale * w_scale[k]) + bias[k] [+ add * add_scale])``, stored as fp32 / fp16 /
  bf16 (rounded once) or as e4m3 ``satfinite_rne(y / out_scale)``.

torch's own cast to float8_e4m3fn does not saturate (470.0 becomes NaN), so quantisation here clamps to +-448
first or uses the CUDA kernel.  FP8 is inference only.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from ..core import ConvAlgo
from . import ops
from .conv import SparseConvolution
from .core import SparseConvTensor

E4M3_MAX = 448.0


def quantize_fp8_weight(weight: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """KRSC filter ``[K, *ksize, C]`` -> ``(w_e4m3, scale [K] fp32)``: per-output-channel ``amax / 448`` (1 for an
    all-zero channel), ``w_e4m3 = satfinite_rne(w / scale)``."""
    k = weight.shape[0]
    w = weight.detach().float()
    amax = w.abs().reshape(k, -1).amax(dim=1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    q = (w / scale.view(-1, *[1] * (w.dim() - 1))).clamp(-E4M3_MAX, E4M3_MAX)
    return q.to(torch.float8_e4m3fn).contiguous(), scale


def quantize_fp8(x: SparseConvTensor, scale: Optional[torch.Tensor] = None) -> SparseConvTensor:
    """float features -> e4m3 features with the per-tensor device scale in ``fp8_scale``.  Without ``scale`` it is
    dynamic: amax / 448 over the rows below ``x.num_valid`` (padding rows are never read and come out 0), NaN and
    +-Inf left out of the amax.  One CUDA kernel pair, no host read-back."""
    q, s = ops.fp8_quantize(x.features, x.num_valid, scale)
    out = x.replace_feature(q)
    out.fp8_scale = s
    return out


def dequantize_fp8(x: SparseConvTensor, dtype: torch.dtype = torch.float32) -> SparseConvTensor:
    """e4m3 features -> ``dtype`` features ``x_e4m3 * fp8_scale``."""
    assert x.features.dtype == torch.float8_e4m3fn and x.fp8_scale is not None, "not an fp8 SparseConvTensor"
    out = x.replace_feature((x.features.float() * x.fp8_scale.float()).to(dtype))
    out.fp8_scale = None
    return out


def calibrate_fp8_output_scale(conv: SparseConvolution, x: SparseConvTensor) -> torch.Tensor:
    """amax / 448 of a float conv's output on one batch (its valid rows), as a device fp32 ``[1]`` tensor: the
    static ``output_scale`` that lets fp8 layers chain e4m3 -> e4m3."""
    with torch.no_grad():
        y = conv(x)
    f = y.features.float()
    keep = torch.isfinite(f) & y.valid_mask().unsqueeze(1)
    f = torch.where(keep, f.abs(), torch.zeros_like(f))
    amax = f.amax() if f.numel() else torch.zeros((), device=f.device)
    return torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax)).reshape(1).float()


def fp8_refusal(mod: nn.Module) -> Optional[str]:
    """Why ``mod`` cannot run in fp8, or None when it can."""
    if not isinstance(mod, SparseConvolution):
        return "not a sparse convolution"
    if isinstance(mod, Fp8SparseConv):
        return "already an fp8 layer (its filter is e4m3 with its own scale)"
    if getattr(mod, "depthwise", False):
        return f"depthwise convolution (groups={mod.groups}) has no fp8 kernel"
    if mod.groups != 1:
        return f"grouped convolution (groups={mod.groups}) has no fp8 kernel"
    if mod.conv1x1:
        return "a 1x1 convolution is a dense matmul, not a sparse conv kernel"
    if mod.algo == ConvAlgo.MaskSplitImplicitGemm:
        return "ConvAlgo.MaskSplitImplicitGemm has no fp8 path (use MaskImplicitGemm)"
    return None


class Fp8SparseConv(SparseConvolution):
    """FP8 inference twin of a float :class:`SparseConvolution`: same geometry, ``indice_key``, output bound and
    fused activation, so it shares rulebooks with float layers.  Build with :meth:`from_float`.

    ``forward(input, add_input=None)`` takes float features (quantised dynamically) or e4m3 features with
    ``fp8_scale``; ``add_input`` is a residual in the output dtype (e4m3 with its ``fp8_scale``) added before the
    activation.  The output is ``output_dtype`` (e4m3 with ``fp8_scale = output_scale``)."""

    @classmethod
    def from_float(cls, mod: SparseConvolution, output_dtype: Optional[torch.dtype] = None,
                   output_scale: Optional[torch.Tensor] = None) -> "Fp8SparseConv":
        why = fp8_refusal(mod)
        if why is not None:
            raise NotImplementedError(f"fp8 conversion refused: {why}; keep this layer in floating point")
        output_dtype = mod.weight.dtype if output_dtype is None else output_dtype
        if output_dtype not in (torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn):
            raise ValueError(f"fp8 conv: output dtype {output_dtype} not supported")
        if output_dtype == torch.float8_e4m3fn and output_scale is None:
            raise ValueError("fp8 conv: an e4m3 output needs a static output_scale (calibrate_fp8_output_scale)")
        dev = mod.weight.device
        q = cls(mod.ndim, mod.in_channels, mod.out_channels, mod.kernel_size, mod.stride, mod.padding,
                mod.dilation, mod.groups, mod.bias is not None, subm=mod.subm,
                output_padding=mod.output_padding, transposed=mod.transposed, inverse=mod.inverse,
                indice_key=mod.indice_key, algo=mod.algo, act_type=mod.act_type, act_alpha=mod.act_alpha,
                act_beta=mod.act_beta, name=mod.name)
        q.num_out_act_bound = mod.num_out_act_bound
        q._sparse_unique_name = mod._sparse_unique_name
        w_q, w_scale = quantize_fp8_weight(mod.weight)
        del q.weight
        q.register_buffer("weight", w_q.to(dev))
        q.register_buffer("weight_scale", w_scale.to(dev))
        q._parameters.pop("bias", None)
        q.register_buffer("bias", mod.bias.detach().float().to(dev) if mod.bias is not None else None)
        q.output_dtype = output_dtype
        q.register_buffer("output_scale", None if output_scale is None else
                          torch.as_tensor(output_scale, dtype=torch.float32, device=dev).reshape(1).clone())
        return q.eval()

    def reset_parameters(self):          # parameters are replaced by buffers in from_float
        return

    def forward(self, input: SparseConvTensor, add_input: Optional[SparseConvTensor] = None):
        if self.training:
            raise RuntimeError("Fp8SparseConv is inference only: call .eval() (fp8 training is not supported)")
        assert input.features.shape[1] == self.in_channels, "channel size mismatch"
        algo = self.algo if input.force_algo is None else input.force_algo
        if algo == ConvAlgo.MaskSplitImplicitGemm:
            # the split rulebook needs one pass per split; a single fp8 pass would drop the second split's offsets
            raise NotImplementedError("fp8 + ConvAlgo.MaskSplitImplicitGemm (from SparseConvTensor.force_algo) is "
                                      "not supported: use ConvAlgo.MaskImplicitGemm or keep this layer in float")
        if input.features.dtype != torch.float8_e4m3fn:
            input = quantize_fp8(input)
        elif input.fp8_scale is None:
            raise RuntimeError("e4m3 features need their scale in SparseConvTensor.fp8_scale (see quantize_fp8)")
        out_tensor = input.shadow_copy()
        rb, indice_dict, out_spatial_shape, num_valid = self._rulebook(input, False, algo, out_tensor)
        features = input.features
        if algo == ConvAlgo.Native:
            outids, indice_pairs, indice_pair_num = rb
            n_out = outids.shape[0]
            kv = int(indice_pairs.shape[1])
            pair, mask, _, _ = ops._native_tables(indice_pairs.contiguous(), indice_pair_num, features.shape[0],
                                                  n_out, kv, self.subm, self.inverse, True, False)
            argsort = None
        else:
            outids, pair, _, mask, _, argsort, _, masks = rb
            mask, argsort = ops._first(mask), ops._first(argsort)
            n_out = outids.shape[0]
        add = add_scale = None
        if add_input is not None:
            add = add_input.features
            add_scale = add_input.fp8_scale if add.dtype == torch.float8_e4m3fn else None
        out_features, _, _ = ops.implicit_gemm(
            features, self.weight, pair, mask, argsort, n_out, None, False, self.subm, input._timer, None,
            self.bias, self.act_alpha, self.act_beta, self.act_type, scale=self.weight_scale, output_add=add,
            output_dtype=self.output_dtype, in_scale=input.fp8_scale, out_scale=self.output_scale,
            add_scale=add_scale)
        out_tensor = out_tensor.replace_feature(out_features)
        out_tensor.num_valid = num_valid
        out_tensor.indices = outids
        out_tensor.indice_dict = indice_dict
        out_tensor.spatial_shape = out_spatial_shape
        out_tensor.fp8_scale = self.output_scale if self.output_dtype == torch.float8_e4m3fn else None
        return out_tensor


def convert_to_fp8(module: nn.Module, output_dtype: Optional[torch.dtype] = None) -> List[Tuple[str, str]]:
    """Replace, in place, every sparse conv of ``module`` that fp8 can run by its :class:`Fp8SparseConv`
    (``output_dtype`` as in :meth:`Fp8SparseConv.from_float`, default each layer's weight dtype).  Returns the
    ``(name, reason)`` of every sparse conv left in floating point.

    A converted layer adds ``add_input`` before its fused activation, ``act(conv + bias + add)``, where the float
    module applies the activation first and then adds, ``act(act(conv + bias) + add)``: a network that passes
    ``add_input`` to a conv with ``act_type`` set computes something else after conversion, not only with less
    precision."""
    skipped: List[Tuple[str, str]] = []
    for parent_name, parent in list(module.named_modules()):
        for name, child in list(parent.named_children()):
            if not isinstance(child, SparseConvolution) or isinstance(child, Fp8SparseConv):
                continue
            full = f"{parent_name}.{name}" if parent_name else name
            why = fp8_refusal(child)
            if why is not None:
                skipped.append((full, why))
                continue
            setattr(parent, name, Fp8SparseConv.from_float(child, output_dtype))
    return skipped
