"""The int8 conv epilogue of both kernel families and QuantizedSparseConv against the exact formula in
float64:

    y = clip(round_half_even(act(acc * scale + bias + add * add_scale)), -128, 127)

with acc the int32 sum over the oracle's rulebook (exact: integers far below 2^24).  The kernels evaluate
the epilogue in fp32, whose rounding may move a value across a .5 tie: an int8 output may differ by 1
only where the float64 value lies within the fp32 error bound of a tie.  fp16 and fp32 outputs are
checked with the bound of test_conv_tc_coverage_gpu.py plus that fp32 error.

The tensor cores serve int8 with C and K multiples of 32; C 16, K 48 runs on the FMA kernel by shape and
C = K = 64 with the FMA kernels pinned.  With SPX_FORCE_SIMT=1 or SPX_FORCE_TC=1 in the environment the
calls behave as in the coverage file.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_conv_tc_coverage_gpu import (Conv, _check, _conv, _lib, _launch, _nan, _reference,
                                             gemm_instance)
from tests.test_conv_tc_coverage_gpu import _restore_forced_family  # noqa: F401  (autouse fixture)
from tests.util import random_cloud

gpu = pytest.mark.gpu

ACTS = ["none", "relu", "leaky_relu", "sigmoid"]
OUTS = ["i8", "f16", "f32"]
ALPHA = 0.25
# (C, K, FMA kernels pinned): tensor cores, FMA kernel by shape, FMA kernels pinned
SHAPES = {"tc32x64": (32, 64, False), "tc64x32": (64, 32, False), "fma16x48": (16, 48, False),
          "fma64x64-forced": (64, 64, True)}
SENTINEL = -77          # int8 outputs are pre-filled with it; NaN for the float outputs


def _matrix():
    """every activation x output type on every shape; bias and residual cycle through their four
    combinations, the residual scale is negative with no activation"""
    out, i = [], 0
    for shape in SHAPES:
        for act in ACTS:
            for o in OUTS:
                out.append((shape, act, o, i % 2 == 0, (i // 2) % 2 == 0))
                i += 1
    return out


def _act_code(act):
    from spconv_b200.core import Activation
    return {"none": Activation.None_, "relu": Activation.ReLU, "leaky_relu": Activation.LeakyReLU,
            "sigmoid": Activation.Sigmoid}[act].value


def _apply_act(v, act):
    return {"none": lambda t: t, "relu": lambda t: t.clamp_min(0),
            "leaky_relu": lambda t: torch.where(t >= 0, t, t * ALPHA), "sigmoid": torch.sigmoid}[act](v)


def _int8_fwd(conv, x, w, scale, bias, add, add_scale, act, out_dt, fma, dev):
    """spx_implicit_gemm_fwd_int8 on the family the shape (or `fma`) says; returns the output as float64"""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    K, C = w.shape[0], w.shape[-1]
    xd, wd, sd = x.to(dev), w.to(dev), scale.to(dev)
    bd = None if bias is None else bias.to(dev)
    ad = None if add is None else add.to(dev)
    d = conv.desc(torch.int8, C, K, conv.fwd)
    code = {"i8": _cabi.SPX_I8, "f16": _cabi.SPX_F16, "f32": _cabi.SPX_F32}[out_dt]

    def launch():
        out = (torch.full((conv.n_out, K), SENTINEL, dtype=torch.int8, device=dev) if out_dt == "i8"
               else _nan((conv.n_out, K), torch.float16 if out_dt == "f16" else torch.float32, dev))
        _cabi.check(_lib().spx_implicit_gemm_fwd_int8(
            ctypes.byref(d), xd.data_ptr(), wd.data_ptr(), out.data_ptr(), code, sd.data_ptr(),
            None if bd is None else bd.data_ptr(), None if ad is None else ad.data_ptr(), add_scale,
            _act_code(act), ALPHA, ops._stream()), "implicit_gemm_fwd_int8")
        return out
    return _launch("int8 fwd", gemm_instance("i8", conv.kv, C, K), launch, fma).double()


def _formula(acc, scale, bias, add, add_scale, act, dev, u=4):
    """float64 epilogue value after the activation, and the bound of its fp32 evaluation (u roundings of
    the largest term, through the activation's Lipschitz constant; sigmoid adds the error of __expf)"""
    s64 = scale.to(dev, torch.float64)
    b64 = torch.zeros_like(s64) if bias is None else bias.to(dev, torch.float64)
    a64 = torch.zeros_like(acc) if add is None else add.to(dev, torch.float64) * add_scale
    pre = acc * s64 + b64 + a64
    err = u * 2.0 ** -24 * ((acc * s64).abs() + b64.abs() + a64.abs()) + 1e-30
    lip = 0.25 if act == "sigmoid" else 1.0
    return _apply_act(pre, act), lip * err + (2.0 ** -20 if act == "sigmoid" else 0.0)


def _check_int8(name, got, val, err):
    assert not (got == SENTINEL).all(1).any(), f"{name}: rows never written"
    ref = torch.round(val).clamp(-128, 127)                     # torch.round: half to even
    diff = (got - ref).abs()
    tie = ((val - val.floor()) - 0.5).abs() <= err
    off = diff > 0
    assert not (diff > 1).any() and not (off & ~tie).any(), (
        f"{name}: {int(off.sum())} outputs differ, {int((off & ~tie).sum())} of them away from a .5 tie, "
        f"max diff {float(diff.max())}")


def _check_out(name, got, val, err, out_dt):
    if out_dt == "i8":
        _check_int8(name, got, val, err)
    else:
        z = torch.zeros_like(val)
        _check(name, got, val, z, z, "f16" if out_dt == "f16" else "tf32", extra=err)


def _ints(rng, shape, lo, hi):
    return torch.from_numpy(rng.integers(lo, hi, size=shape).astype(np.int8))


# ------------------------------------------------------------------ the epilogue matrix
@gpu
@pytest.mark.parametrize("case", _matrix(),
                         ids=lambda c: f"{c[0]}-{c[1]}-{c[2]}out{'-bias' if c[3] else ''}{'-add' if c[4] else ''}")
def test_int8_epilogue(case, oracle, cuda_dev):
    shape, act, out_dt, with_bias, with_add = case
    C, K, fma = SHAPES[shape]
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    rng = np.random.default_rng(C * 7 + K + ACTS.index(act))
    x, w = _ints(rng, (conv.n_in, C), -4, 4), _ints(rng, (K, conv.kv, C), -4, 4)
    scale = torch.from_numpy((rng.uniform(0.5, 1.5, size=K) * 0.2).astype(np.float32))
    bias = torch.from_numpy(rng.uniform(-5, 5, size=K).astype(np.float32)) if with_bias else None
    add = _ints(rng, (conv.n_out, K), -3, 4) if with_add else None
    add_scale = -0.625 if act == "none" else 0.375
    acc = _reference(x.float(), w.float(), torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)["out"]
    val, err = _formula(acc, scale, bias, add, add_scale, act, cuda_dev)
    if act == "leaky_relu":
        assert (val < -2).any(), "no negative outputs: the slope would not be checked"
    got = _int8_fwd(conv, x, w, scale, bias, add, add_scale, act, out_dt, fma, cuda_dev)
    _check_out(f"{shape} {act} -> {out_dt}", got, val, err, out_dt)


def test_matrix_covers_every_combination():
    """No GPU needed: per shape every activation meets every output type, every bias / residual
    combination occurs, and the shapes run where their names say"""
    cases = _matrix()
    for shape in SHAPES:
        mine = [c for c in cases if c[0] == shape]
        assert {(a, o) for _, a, o, _, _ in mine} == {(a, o) for a in ACTS for o in OUTS}
        assert {(b, r) for _, _, _, b, r in mine} == {(b, r) for b in (True, False) for r in (True, False)}
    for name, (C, K, fma) in SHAPES.items():
        assert (gemm_instance("i8", 27, C, K) is not None) == (name.startswith("tc") or fma)
        assert fma == name.endswith("forced")


@gpu
def test_int8_bf16_output_is_refused(oracle, cuda_dev):
    """bf16 is not an int8 output type: the C ABI refuses the call and writes nothing"""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    rng = np.random.default_rng(1)
    x, w = _ints(rng, (conv.n_in, 32), -4, 4).to(cuda_dev), _ints(rng, (32, 27, 32), -4, 4).to(cuda_dev)
    scale = torch.ones(32, device=cuda_dev)
    d = conv.desc(torch.int8, 32, 32, conv.fwd)
    out = torch.full((conv.n_out, 32), 3.0, dtype=torch.bfloat16, device=cuda_dev)
    with pytest.raises(RuntimeError, match=f"out dtype {_cabi.SPX_BF16} not supported"):
        _cabi.check(_lib().spx_implicit_gemm_fwd_int8(
            ctypes.byref(d), x.data_ptr(), w.data_ptr(), out.data_ptr(), _cabi.SPX_BF16, scale.data_ptr(), None,
            None, 0.0, _act_code("none"), 0.0, ops._stream()), "implicit_gemm_fwd_int8")
    torch.cuda.synchronize()
    assert (out == 3.0).all()


# ------------------------------------------------------------------ saturation and ties
FAMS = {"tc": (32, 32, False), "fma": (16, 48, False), "fma-forced": (32, 32, True)}


@gpu
@pytest.mark.parametrize("fam", list(FAMS))
def test_int8_saturates_at_both_ends(fam, oracle, cuda_dev):
    """scale 4: accumulators of several hundred land far outside [-128, 127] on both sides"""
    C, K, fma = FAMS[fam]
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    rng = np.random.default_rng(40)
    x, w = _ints(rng, (conv.n_in, C), -4, 4), _ints(rng, (K, conv.kv, C), -4, 4)
    scale = torch.full((K,), 4.0)
    acc = _reference(x.float(), w.float(), torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)["out"]
    val, err = _formula(acc, scale, None, None, 0.0, "none", cuda_dev)
    assert (val < -129).sum() > 100 and (val > 128).sum() > 100
    got = _int8_fwd(conv, x, w, scale, None, None, 0.0, "none", "i8", fma, cuda_dev)
    _check_int8(f"{fam} saturation", got, val, err)
    assert (got == -128).any() and (got == 127).any()
    assert (got[val < -129] == -128).all() and (got[val > 128] == 127).all()


@gpu
@pytest.mark.parametrize("fam", list(FAMS))
def test_int8_round_half_even_ties(fam, oracle, cuda_dev):
    """integer accumulators times 0.5, no bias: every odd accumulator is an exact .5 tie in fp32 as well,
    so the result must be round-half-even with no slack (+2.5 -> 2, -2.5 -> -2)"""
    C, K, fma = FAMS[fam]
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    rng = np.random.default_rng(41)
    x, w = _ints(rng, (conv.n_in, C), -2, 3), _ints(rng, (K, conv.kv, C), -1, 2)
    scale = torch.full((K,), 0.5)
    acc = _reference(x.float(), w.float(), torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)["out"]
    val = acc * 0.5
    for t in (2.5, -2.5, 0.5, -0.5, 3.5, -3.5):
        assert (val == t).any(), f"no element at {t}"
    got = _int8_fwd(conv, x, w, scale, None, None, 0.0, "none", "i8", fma, cuda_dev)
    ref = torch.round(val).clamp(-128, 127)
    bad = got != ref
    assert not bad.any(), (f"{int(bad.sum())} outputs differ from round-half-even, e.g. {float(val[bad][0])} -> "
                           f"{float(got[bad][0])}")
    assert (got[val == 2.5] == 2).all() and (got[val == -2.5] == -2).all()


# ------------------------------------------------------------------ QuantizedSparseConv
SHAPE = [20, 20, 20]


def _cloud_tensor(dev, C, seed=8):
    import spconv_b200.pytorch as spconv
    rng = np.random.default_rng(seed)
    feats, inds = random_cloud(rng, SHAPE, [2500], C)
    return spconv.SparseConvTensor(torch.from_numpy(feats).to(dev), torch.from_numpy(inds).to(dev), SHAPE, 1), inds


def _float_layer(kind, C, K, dev, seed, **kw):
    import spconv_b200.pytorch as spconv
    if kind == "subm":
        m = spconv.SubMConv3d(C, K, 3, bias=True, **kw)
    elif kind == "conv":
        m = spconv.SparseConv3d(C, K, 3, 2, 1, bias=True, **kw)
    else:
        m = spconv.SparseInverseConv3d(C, K, 3, bias=True, **kw)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.weight.copy_(torch.rand(m.weight.shape, generator=g) * 2 - 1)
        m.bias.copy_(torch.rand(K, generator=g) * 2 - 1)
    m.act_type = spconv.Activation.ReLU
    return m.to(dev).eval()


def _quantized_reference(oracle, dev, inds, kind, fconv, q, xq, add=None):
    """float64 value of QuantizedSparseConv's docstring formula and its fp32 error bound, from the
    oracle's rulebook, quantize_per_channel_weight and the float layer's bias"""
    from spconv_b200.pytorch.quantized import quantize_per_channel_weight
    subm = kind == "subm"
    st, pd = (1, 0) if subm else (2, 1)
    conv = Conv(oracle, dev, inds, 1, SHAPE, 3, st, pd, 1, subm)
    ref_out = oracle.get_indice_pairs(inds, 1, SHAPE, [3] * 3, [st] * 3, [pd] * 3, [1] * 3, [0] * 3, subm)[0]
    w_q, w_s = quantize_per_channel_weight(fconv.weight)
    assert torch.equal(q.weight, w_q) and torch.equal(q.weight_scales, w_s)
    K, C = w_q.shape[0], w_q.shape[-1]
    acc = _reference(xq.features.float(), w_q.float().reshape(K, -1, C), torch.zeros((conv.n_out, K)),
                     conv.ref_pair, dev)["out"]
    out_scale = float(q.scale)
    channel_scale = float(xq.int8_scale) * w_s.double() / out_scale
    bias_q = fconv.bias.detach().double() / out_scale
    add_feats = None if add is None else add.features
    add_scale = 0.0 if add is None else float(add.int8_scale) / out_scale
    # channel_scale and bias_q are rounded to fp32 on the host as well: two more roundings
    val, err = _formula(acc, channel_scale, bias_q, add_feats, add_scale, "relu", dev, u=8)
    return ref_out, val, err


@gpu
@pytest.mark.parametrize("kind", ["subm", "conv"])
def test_quantized_conv_from_float(kind, oracle, cuda_dev):
    from spconv_b200.pytorch import quantized as Q
    x, inds = _cloud_tensor(cuda_dev, 32)
    fconv = _float_layer(kind, 32, 64, cuda_dev, seed=1)
    q = Q.QuantizedSparseConv.from_float(fconv, 0.04)
    xq = Q.quantize_tensor(x, 1.0 / 127.0)
    with torch.no_grad():
        y = q(xq)
    ref_out, val, err = _quantized_reference(oracle, cuda_dev, inds, kind, fconv, q, xq)
    assert y.features.dtype == torch.int8 and y.int8_scale == 0.04
    assert np.array_equal(y.indices.cpu().numpy(), ref_out), "output coordinates differ from the oracle"
    assert (val > 127.5).any() and (val == 0).any(), "the scales exercise neither the clamp nor the ReLU"
    _check_int8(f"{kind} QuantizedSparseConv", y.features.double(), val, err)


@gpu
def test_quantized_conv_residual(oracle, cuda_dev):
    """add_input with a scale different from the output's enters the epilogue as add * add_scale / out_scale"""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import quantized as Q
    x, inds = _cloud_tensor(cuda_dev, 32)
    fconv = _float_layer("subm", 32, 64, cuda_dev, seed=2)
    q = Q.QuantizedSparseConv.from_float(fconv, 0.05)
    xq = Q.quantize_tensor(x, 1.0 / 127.0)
    rng = np.random.default_rng(3)
    res = spconv.SparseConvTensor(torch.from_numpy(rng.uniform(-3, 3, size=(len(inds), 64)).astype(np.float32))
                                  .to(cuda_dev), x.indices, SHAPE, 1)
    addq = Q.quantize_tensor(res, 0.03)
    with torch.no_grad():
        y = q(xq, add_input=addq)
        y0 = q(xq)
    _, val, err = _quantized_reference(oracle, cuda_dev, inds, "subm", fconv, q, xq, add=addq)
    _check_int8("residual", y.features.double(), val, err)
    assert not torch.equal(y.features, y0.features)


@gpu
def test_quantized_conv_shared_indice_key(oracle, cuda_dev, monkeypatch):
    """a second SubM layer on the same indice_key reuses the first one's rulebook"""
    from spconv_b200.pytorch import ops
    from spconv_b200.pytorch import quantized as Q
    built = []
    real = ops.get_indice_pairs_implicit_gemm
    monkeypatch.setattr(ops, "get_indice_pairs_implicit_gemm", lambda *a, **k: built.append(1) or real(*a, **k))
    x, inds = _cloud_tensor(cuda_dev, 32)
    f1 = _float_layer("subm", 32, 64, cuda_dev, seed=4, indice_key="s")
    f2 = _float_layer("subm", 64, 32, cuda_dev, seed=5, indice_key="s")
    q1 = Q.QuantizedSparseConv.from_float(f1, 0.04)
    q2 = Q.QuantizedSparseConv.from_float(f2, 0.1)
    xq = Q.quantize_tensor(x, 1.0 / 127.0)
    with torch.no_grad():
        y1 = q1(xq)
        y2 = q2(y1)
    assert len(built) == 1, f"{len(built)} rulebooks built for two layers on one indice_key"
    assert y2.indice_dict["s"] is y1.indice_dict["s"]
    _, val1, err1 = _quantized_reference(oracle, cuda_dev, inds, "subm", f1, q1, xq)
    _check_int8("first layer", y1.features.double(), val1, err1)
    _, val2, err2 = _quantized_reference(oracle, cuda_dev, inds, "subm", f2, q2, y1)
    _check_int8("second layer", y2.features.double(), val2, err2)


@gpu
def test_quantized_conv_refusals(cuda_dev):
    """int8 has no mask-split path and no inverse conv"""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import quantized as Q
    x, _ = _cloud_tensor(cuda_dev, 32)
    xq = Q.quantize_tensor(x, 1.0 / 127.0)
    split = Q.QuantizedSparseConv.from_float(
        _float_layer("subm", 32, 32, cuda_dev, seed=6, algo=ConvAlgo.MaskSplitImplicitGemm), 0.05)
    with pytest.raises(NotImplementedError, match="MaskSplitImplicitGemm"), torch.no_grad():
        split(xq)
    inv = Q.QuantizedSparseConv.from_float(_float_layer("inverse", 32, 32, cuda_dev, seed=7, indice_key="d"), 0.05)
    with pytest.raises(AssertionError, match="inverse"), torch.no_grad():
        inv(xq)


def test_quantize_per_channel_weight_against_numpy():
    """half-even ties and the symmetric clamp at +-127: with power-of-two scales every value below is exact"""
    from spconv_b200.pytorch.quantized import quantize_per_channel_weight
    steps = np.array([-127, -126.5, -2.5, -1.5, -0.5, 0.5, 1.5, 2.5, 125.5, 126.5, 127, 3], np.float64)
    w = np.stack([steps * 2.0 ** -e for e in (0, 3, 7)]).reshape(3, 1, 2, 6).astype(np.float32)   # KRSC, kv 2
    q, s = quantize_per_channel_weight(torch.from_numpy(w))
    amax = np.abs(w).reshape(3, -1).max(1)
    s_np = (amax / np.float32(127)).astype(np.float32)
    q_np = np.clip(np.round(w / s_np.reshape(-1, 1, 1, 1)), -127, 127).astype(np.int8)
    assert np.array_equal(s.numpy(), s_np) and np.array_equal(s_np, 2.0 ** -np.array([0, 3, 7]))
    assert q.dtype == torch.int8 and np.array_equal(q.numpy(), q_np)
    assert np.array_equal(q.numpy()[0].reshape(-1), [-127, -126, -2, -2, 0, 0, 2, 2, 126, 126, 127, 3])


def test_quantize_tensor_against_numpy():
    """half-even ties, clamp to [-128, 127]"""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch.quantized import quantize_tensor
    scale = 2.0 ** -5
    v = np.array([-300, -128.5, -128, -127.5, -2.5, -1.5, -0.5, 0.5, 1.5, 2.5, 126.5, 127.5, 300, 7.25], np.float64)
    f = (v * scale).astype(np.float32).reshape(-1, 1)
    x = spconv.SparseConvTensor(torch.from_numpy(f), torch.zeros((len(f), 4), dtype=torch.int32), [4, 4, 4], 1)
    q = quantize_tensor(x, scale)
    want = np.clip(np.round(f / np.float32(scale)), -128, 127).astype(np.int8)
    assert q.features.dtype == torch.int8 and q.int8_scale == scale
    assert np.array_equal(q.features.numpy(), want)
    assert np.array_equal(want.reshape(-1), [-128, -128, -128, -128, -2, -2, 0, 0, 2, 2, 126, 127, 127, 7])
