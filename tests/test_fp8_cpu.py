"""FP8 (e4m3) inference without a GPU: a numpy restatement of e4m3 rounding (round to nearest, ties to even,
saturating at +-448) checked against torch's own cast, the per-channel weight quantisation, and the argument
checks of the new C entry points, which run before any launch."""
import ctypes

import numpy as np
import pytest
import torch

E4M3_MAX = 448.0


def e4m3_rne(v):
    """float64 values -> the nearest e4m3 value (ties to even), +-Inf and |v| > 448 saturated, NaN kept:
    what cvt.rn.satfinite.e4m3x2.f32 gives.  3 mantissa bits, exponent bias 7, subnormal spacing 2^-9."""
    v = np.asarray(v, dtype=np.float64)
    a = np.abs(v)
    _, ex = np.frexp(np.where(np.isfinite(a) & (a > 0), a, 1.0))     # a = m * 2^ex, m in [0.5, 1)
    ulp = np.ldexp(1.0, np.maximum(ex - 1, -6) - 3)
    q = np.rint(np.where(np.isfinite(a), a, 0.0) / ulp) * ulp          # exact scaling, rint = half to even
    q = np.where(np.isinf(a) | (q > E4M3_MAX), E4M3_MAX, q)
    return np.where(np.isnan(v), np.nan, np.copysign(q, v))


def test_e4m3_rounding_against_torch_over_every_fp16_pattern():
    x = np.arange(1 << 16, dtype=np.uint16).view(np.float16).astype(np.float64)
    x = x[np.isfinite(x)]
    clamped = np.clip(x, -E4M3_MAX, E4M3_MAX)
    got = torch.from_numpy(clamped).float().to(torch.float8_e4m3fn).double().numpy()
    ref = e4m3_rne(clamped)
    assert np.array_equal(got, ref), np.flatnonzero(got != ref)[:10]
    # beyond the range and at infinity the restatement saturates where torch's cast gives NaN
    assert e4m3_rne(470.0) == 448.0 and e4m3_rne(-np.inf) == -448.0 and np.isnan(e4m3_rne(np.nan))
    assert np.isnan(torch.tensor([470.0]).to(torch.float8_e4m3fn).float().item())


@pytest.mark.parametrize("v,want", [(1.0625, 1.0), (1.1875, 1.25), (-1.0625, -1.0), (3.125, 3.0), (3.375, 3.5),
                                    (2.0 ** -10, 0.0), (3 * 2.0 ** -10, 2.0 ** -8), (464.0, 448.0), (0.0, 0.0)])
def test_e4m3_ties_to_even(v, want):
    assert e4m3_rne(v) == want
    if abs(v) <= E4M3_MAX:
        assert torch.tensor([v]).to(torch.float8_e4m3fn).double().item() == want


def test_quantize_fp8_weight_against_numpy():
    from spconv_b200.pytorch import quantize_fp8_weight
    rng = np.random.default_rng(3)
    w = rng.standard_normal((8, 3, 3, 3, 16)).astype(np.float32) * rng.uniform(0.01, 10, size=(8, 1, 1, 1, 1))
    w = w.astype(np.float32)
    w[5] = 0.0                                        # an all-zero channel gets scale 1
    q, scale = quantize_fp8_weight(torch.from_numpy(w))
    assert q.dtype == torch.float8_e4m3fn and q.shape == w.shape and scale.dtype == torch.float32
    amax = np.abs(w).reshape(8, -1).max(1)
    ref_scale = np.where(amax > 0, amax / np.float32(E4M3_MAX), np.float32(1)).astype(np.float32)
    assert np.array_equal(scale.numpy(), ref_scale)
    ref_q = e4m3_rne(np.clip((w / ref_scale.reshape(-1, 1, 1, 1, 1)).astype(np.float32), -E4M3_MAX, E4M3_MAX))
    assert np.array_equal(q.double().numpy(), ref_q)
    assert np.abs(q.double().numpy()).reshape(8, -1).max(1)[[0, 1, 2, 3, 4, 6, 7]].tolist() == [E4M3_MAX] * 7


# ------------------------------------------------------------------ C entry points: checks before any launch
@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def _desc(dtype, n_out=10):
    from spconv_b200 import _cabi
    d = _cabi.GemmDesc()
    d.dtype, d.kv, d.c_in, d.c_out, d.n_in, d.n_out = dtype, 27, 32, 32, 10, n_out
    d.pair = 16
    return d


FAKE = 4096      # never dereferenced: every call below fails its checks first


def _fwd(lib, d, out_dtype, in_scale=FAKE, w_scale=FAKE, out_scale=None, add=None, add_scale=None, act=0):
    from spconv_b200 import _cabi
    a = _cabi.Fp8Gemm(FAKE, FAKE, in_scale, w_scale, None, add, add_scale, FAKE, out_dtype, out_scale, act, 0.0)
    return lib.spx_implicit_gemm_fwd_fp8(ctypes.byref(d), ctypes.byref(a), None)


def test_fp8_gemm_argument_checks(lib):
    from spconv_b200 import _cabi
    E4M3, F16, I8 = _cabi.SPX_E4M3, _cabi.SPX_F16, _cabi.SPX_I8
    cases = [
        (lambda: _fwd(lib, _desc(F16), F16), "descriptor dtype must be SPX_E4M3"),
        (lambda: _fwd(lib, _desc(E4M3), I8), "out dtype 3 not supported"),
        (lambda: _fwd(lib, _desc(E4M3), F16, act=9), "unknown activation 9"),
        (lambda: _fwd(lib, _desc(E4M3), F16, in_scale=None), "NULL tensor"),
        (lambda: _fwd(lib, _desc(E4M3), F16, w_scale=None), "NULL tensor"),
        (lambda: _fwd(lib, _desc(E4M3), E4M3), "e4m3 output needs out_scale"),
        (lambda: _fwd(lib, _desc(E4M3), E4M3, out_scale=FAKE, add=FAKE), "e4m3 residual needs add_scale"),
    ]
    for call, text in cases:
        assert call() == 2
        assert text in _cabi.last_error(), (text, _cabi.last_error())
    bad = _desc(E4M3)
    bad.kv = 129
    assert _fwd(lib, bad, F16) == 2 and "kernel volume 129" in _cabi.last_error()
    assert _fwd(lib, _desc(E4M3, n_out=0), F16) == 0           # nothing to compute: no launch
    assert lib.spx_implicit_gemm_fwd_fp8(ctypes.byref(_desc(E4M3)), None, None) == 2
    assert "argument block is NULL" in _cabi.last_error()


def test_fp8_quantize_argument_checks(lib):
    from spconv_b200 import _cabi
    ws = lib.spx_fp8_quantize_workspace_size(1000, 64)
    assert ws >= 4

    def q(dtype=_cabi.SPX_F16, rows=1000, ch=64, x=FAKE, scale_in=None, out=FAKE, scale_out=FAKE, w=FAKE, wb=ws):
        a = _cabi.Fp8Quant(x, dtype, rows, ch, None, scale_in, out, scale_out)
        return lib.spx_fp8_quantize(ctypes.byref(a), w, wb, None)

    cases = [(lambda: q(dtype=_cabi.SPX_I8), "dtype 3 not supported"),
             (lambda: q(dtype=_cabi.SPX_E4M3), "dtype 4 not supported"),
             (lambda: q(ch=0), "bad shape"), (lambda: q(rows=-1), "bad shape"),
             (lambda: q(x=None), "NULL tensor"), (lambda: q(out=None), "NULL tensor"),
             (lambda: q(scale_out=None), "needs scale_out"),
             (lambda: q(wb=ws - 1), "workspace too small"), (lambda: q(w=None), "workspace too small")]
    for call, text in cases:
        assert call() == 2
        assert text in _cabi.last_error(), (text, _cabi.last_error())
    assert lib.spx_fp8_quantize(None, None, 0, None) == 2 and "argument block is NULL" in _cabi.last_error()


def test_fp8_exports():
    import spconv_b200.pytorch as spconv
    for name in ("Fp8SparseConv", "quantize_fp8", "quantize_fp8_weight", "dequantize_fp8", "convert_to_fp8",
                 "calibrate_fp8_output_scale"):
        assert getattr(spconv, name).__doc__


def test_module_refusals_before_any_launch():
    """Re-converting an fp8 layer, and a split rulebook asked for by the input tensor, are refused on the host."""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import fp8
    q = fp8.Fp8SparseConv.from_float(spconv.SubMConv3d(32, 32, 3).eval())
    with pytest.raises(NotImplementedError, match="already an fp8 layer"):
        fp8.Fp8SparseConv.from_float(q)
    net = spconv.SparseSequential(q, spconv.SubMConv3d(32, 32, 3))
    assert fp8.convert_to_fp8(net) == [] and isinstance(net[1], fp8.Fp8SparseConv) and net[0] is q
    x = spconv.SparseConvTensor(torch.zeros(4, 32), torch.zeros(4, 4, dtype=torch.int32), [8, 8, 8], 1)
    x.force_algo = spconv.ConvAlgo.MaskSplitImplicitGemm
    with pytest.raises(NotImplementedError, match="MaskSplitImplicitGemm"):
        q(x)
