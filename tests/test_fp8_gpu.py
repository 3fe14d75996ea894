"""FP8 (e4m3) inference on the GPU: every tensor-core instance and the FMA kernel bit for bit against float64, the
quantise kernel, the modules, graph capture and the refusals.

The epilogue under test (include/spconv_b200.h, spx_implicit_gemm_fwd_fp8), one IEEE fp32 operation per step:

    y = act(acc * (in_scale * w_scale[k]) + bias[k] + add * add_scale)
    out = y (fp32), rne(y) (fp16 / bf16), satfinite_rne(y / out_scale) (e4m3)

The exact cases use integer operands in [-2, 2] (e4m3-exact) and power-of-two scales, with biases on a 1/8 grid:
every product is exact, every sum an integer far below 2^11, and every epilogue step exact, so the float64
reference rounded once to the output type must equal the kernel's output bit for bit, whatever order the sums are
taken in.  (The Hopper FP8 tensor cores add a k-step's products with only about 14 bits kept, DeepSeek-V3 technical
report section 3.3.2; integer sums below 2^11 are exact there too.)
"""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_conv_tc_coverage_gpu import _configure, _conv, _launch, _lib, _reference
from tests.test_conv_tc_coverage_gpu import _restore_forced_family  # noqa: F401  (autouse fixture)
from tests.test_fp8_cpu import E4M3_MAX, e4m3_rne

gpu = pytest.mark.gpu

F8 = torch.float8_e4m3fn
OUT_DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "e4m3": F8}
ACTS = {"none": 0, "relu": 1, "sigmoid": 2, "leaky_relu": 3}
ALPHA = 0.25


def fp8_instance(kv, C, K):
    """("gemm", KIND_E4M3, CPR, N) of the tensor-core instance serving an fp8 call, None for the FMA kernel
    (tc_shape_ok / tc_gather_gemm_fp8_supported of gemm_tc.cu).  K = 256 runs as two passes of N = 128."""
    if C % 32 or K % 32 or C > 256 or K > 256:
        return None
    al = lambda n: (n + 1023) // 1024 * 1024       # noqa: E731
    if 2 * al((kv + 1) * 512) + 2 * (al(128 * C) + al(C * K)) > 200 * 1024:
        return None
    return ("gemm", 3, C // 16, min(K, 128))


def _round_out(y, out, out_scale):
    """float64 epilogue value -> the output type, as float64 (NaN kept)"""
    if out == "f32":
        return y.float().double()
    if out in ("f16", "bf16"):
        return y.to(OUT_DT[out]).double()
    return torch.from_numpy(e4m3_rne((y / out_scale).cpu().numpy())).to(y.device)


def _act(y, act):
    return {"none": lambda t: t, "relu": lambda t: t.clamp_min(0), "leaky_relu": lambda t: torch.where(t >= 0, t, t * ALPHA),
            "sigmoid": torch.sigmoid}[act](y)


def _fp8_fwd(conv, x, w, in_scale, w_scale, bias, add, add_scale, out, out_scale, act, dev, fma=False, x_view=None):
    """spx_implicit_gemm_fwd_fp8 on the family the shape (or `fma`) says -> output as float64"""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    K, C = w.shape[0], w.shape[-1]
    xd = x_view if x_view is not None else x.to(dev).to(F8)
    wd = w.to(dev).to(F8)
    f32 = lambda t: None if t is None else torch.as_tensor(t, dtype=torch.float32).reshape(-1).to(dev)   # noqa: E731
    s_in, s_w, b, s_add, s_out = f32(in_scale), f32(w_scale), f32(bias), f32(add_scale), f32(out_scale)
    ad = None if add is None else add.to(dev).to(OUT_DT[out])
    d = conv.desc(F8, C, K, conv.fwd)
    p = lambda t: None if t is None else t.data_ptr()     # noqa: E731

    def launch():
        y = torch.full((conv.n_out, K), float("nan"), device=dev).to(OUT_DT[out])
        a = _cabi.Fp8Gemm(xd.data_ptr(), wd.data_ptr(), p(s_in), p(s_w), p(b), p(ad), p(s_add), y.data_ptr(),
                          {"f32": _cabi.SPX_F32, "f16": _cabi.SPX_F16, "bf16": _cabi.SPX_BF16,
                           "e4m3": _cabi.SPX_E4M3}[out], p(s_out), ACTS[act], ALPHA)
        _cabi.check(_lib().spx_implicit_gemm_fwd_fp8(ctypes.byref(d), ctypes.byref(a), ops._stream()),
                    "implicit_gemm_fwd_fp8")
        return y
    inst = None if fma else fp8_instance(conv.kv, C, K)
    return _launch("fp8 fwd", inst, launch, fma).double()


def _ints(rng, shape, lo=-2, hi=2):
    return torch.from_numpy(rng.integers(lo, hi + 1, size=shape).astype(np.float32))


def _exact_case(conv, C, K, out, act, with_bias, with_add, seed, dev, fma=False):
    rng = np.random.default_rng(seed)
    x, w = _ints(rng, (conv.n_in, C)), _ints(rng, (K, conv.kv, C))
    in_scale = 2.0 ** -3
    w_scale = torch.from_numpy((2.0 ** rng.integers(-2, 2, size=K)).astype(np.float32))
    bias = torch.from_numpy((rng.integers(-16, 17, size=K) / 8).astype(np.float32)) if with_bias else None
    add = _ints(rng, (conv.n_out, K), -3, 3) if with_add else None
    add_scale = 0.5 if (with_add and out == "e4m3") else None
    out_scale = 2.0 ** -2 if out == "e4m3" else None
    acc = _reference(x, w, torch.zeros((conv.n_out, K)), conv.ref_pair, dev)["out"]
    y = acc * (in_scale * w_scale.to(dev, torch.float64))
    if bias is not None:
        y = y + bias.to(dev, torch.float64)
    if add is not None:
        y = y + add.to(dev, torch.float64) * (add_scale if add_scale is not None else 1.0)
    y = _act(y, act)
    got = _fp8_fwd(conv, x, w, in_scale, w_scale, bias, add, add_scale, out, out_scale, act, dev, fma)
    return got, y, out_scale


def _same(name, got, ref):
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), f"{name}: NaN pattern differs"
    bad = (got != ref) & ~nan
    assert not bad.any(), f"{name}: {int(bad.sum())} of {got.numel()} outputs differ, max {float((got - ref)[bad].abs().max())}"


# ------------------------------------------------------------------ every kernel instance, bit for bit
CHANNELS = (32, 64, 128, 256)
OUTS = ("f32", "f16", "bf16", "e4m3")
INSTANCES = [(C, K) for C in CHANNELS for K in CHANNELS]


@gpu
@pytest.mark.parametrize("ck", INSTANCES, ids=lambda c: f"C{c[0]}-K{c[1]}")
def test_every_tensor_core_instance(ck, oracle, cuda_dev):
    C, K = ck
    # C = K = 256 at kv 27 does not fit two stages in shared memory (FMA kernel): its instance serves kv 1
    geom = "k3" if fp8_instance(27, C, K) else "k1"
    conv = _conv(oracle, cuda_dev, geom, "subm")
    assert fp8_instance(conv.kv, C, K) is not None
    i = INSTANCES.index(ck)
    out = OUTS[i % 4]
    act = ("none", "relu", "leaky_relu")[i % 3]
    got, y, out_scale = _exact_case(conv, C, K, out, act, i % 2 == 0, (i // 2) % 2 == 0, 100 + i, cuda_dev)
    _same(f"C{C} K{K} {out} {act}", got, _round_out(y, out, out_scale))


# (geometry, mode, C, K, fma): a strided conv, kernel volumes up to 125 (several mask words), the FMA kernel by
# shape and pinned
FAMS = {"strided-tc": ("k3", "conv", 64, 32, False), "k5-tc": ("k5", "subm", 32, 64, False),
        "k533-tc": ("k533", "conv", 32, 32, False), "fma-shape": ("k3", "subm", 48, 40, False),
        "fma-forced": ("k3", "subm", 64, 64, True), "fma-k5": ("k5", "conv", 16, 32, False)}


@gpu
@pytest.mark.parametrize("fam", list(FAMS))
@pytest.mark.parametrize("out", OUTS)
def test_families_and_outputs(fam, out, oracle, cuda_dev):
    geom, mode, C, K, fma = FAMS[fam]
    conv = _conv(oracle, cuda_dev, geom, mode)
    for j, act in enumerate(("none", "relu", "leaky_relu")):
        got, y, out_scale = _exact_case(conv, C, K, out, act, j != 1, j != 0, 7 + j + OUTS.index(out), cuda_dev, fma)
        _same(f"{fam} {out} {act}", got, _round_out(y, out, out_scale))


@gpu
@pytest.mark.parametrize("fma", [False, True], ids=["tc", "fma"])
def test_sigmoid_and_every_residual_dtype(fma, oracle, cuda_dev):
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    for out in OUTS:
        got, y, out_scale = _exact_case(conv, 32, 64, out, "sigmoid", True, True, 31, cuda_dev, fma)
        ref = _round_out(y, out, out_scale)
        # __expf: a few ulp of fp32 before the one rounding to the output type
        tol = {"f32": 2.0 ** -20, "f16": 2.0 ** -11, "bf16": 2.0 ** -8, "e4m3": 2.0 ** -3 * out_scale if out_scale else 0}[out]
        assert (got - ref).abs().max() <= tol + 2.0 ** -20, out


@gpu
@pytest.mark.parametrize("fma", [False, True], ids=["tc", "fma"])
def test_e4m3_output_saturation_nan_and_ties(fma, oracle, cuda_dev):
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    C, K = 32, 32
    rng = np.random.default_rng(5)
    x, w = _ints(rng, (conv.n_in, C)), _ints(rng, (K, conv.kv, C))
    x[3] = float("nan")                                   # NaN input row: every output reading it is NaN
    acc = _reference(torch.nan_to_num(x), w, torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)["out"]
    pair = torch.from_numpy(conv.ref_pair).to(cuda_dev)
    reads_nan = (pair == 3).any(0)
    for out_scale in (1.0, 2.0 ** -4, 2.0 ** -1):
        y = acc.clone()
        y[reads_nan] = float("nan")
        ref = _round_out(y, "e4m3", out_scale)
        got = _fp8_fwd(conv, x, w, 1.0, torch.ones(K), None, None, None, "e4m3", out_scale, "none", cuda_dev, fma)
        _same(f"e4m3 out_scale {out_scale}", got, ref)
    q = (acc / 2.0 ** -4)[~reads_nan]
    assert (q.abs() > E4M3_MAX).any(), "no output saturated"
    t = (acc / 1.0)[~reads_nan].abs()
    assert ((t >= 16) & (t < 32) & (t % 2 == 1)).any(), "no round-half-even tie at the e4m3 output"
    assert reads_nan.any()


@gpu
def test_misaligned_features_run_on_the_fma_kernel_with_the_same_bits(oracle, cuda_dev):
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    C, K = 64, 64
    rng = np.random.default_rng(9)
    x, w = _ints(rng, (conv.n_in, C)), _ints(rng, (K, conv.kv, C))
    want = _fp8_fwd(conv, x, w, 1.0, torch.ones(K), None, None, None, "f32", None, "none", cuda_dev)
    buf = torch.zeros(conv.n_in * C + 16, dtype=torch.uint8, device=cuda_dev)
    view = buf[1:1 + conv.n_in * C].view(F8).view(conv.n_in, C)
    view.copy_(x.to(cuda_dev).to(F8))
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    d = conv.desc(F8, C, K, conv.fwd)
    y = torch.full((conv.n_out, K), float("nan"), device=cuda_dev)
    _configure(0)
    one = torch.ones(1, device=cuda_dev)
    ws = torch.ones(K, device=cuda_dev)
    wd = w.to(cuda_dev).to(F8)
    a = _cabi.Fp8Gemm(view.data_ptr(), wd.data_ptr(), one.data_ptr(), ws.data_ptr(), None, None, None, y.data_ptr(),
                      _cabi.SPX_F32, None, 0, 0.0)
    _cabi.check(_lib().spx_implicit_gemm_fwd_fp8(ctypes.byref(d), ctypes.byref(a), ops._stream()),
                "implicit_gemm_fwd_fp8")
    assert _lib().spx_last_kernel_family() == 1
    assert torch.equal(y.double(), want)


# ------------------------------------------------------------------ the quantise kernel
def _quant_ref(x, m, scale=None):
    """numpy: (e4m3 values as float64, scale) of spx_fp8_quantize"""
    xv = x.float().cpu().numpy()
    if scale is None:
        v = np.abs(xv[:m])
        v = v[np.isfinite(v)]
        amax = np.float32(v.max()) if v.size else np.float32(0)
        scale = np.float32(amax / np.float32(448)) if amax > 0 else np.float32(1)
    q = e4m3_rne((xv[:m] / np.float32(scale)).astype(np.float32))
    out = np.zeros(xv.shape)
    out[:m] = q
    return out, np.float32(scale)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("C", [64, 3])
def test_dynamic_quantise_ignores_padding(dtype, C, cuda_dev):
    from spconv_b200.pytorch import ops
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(5000, C, generator=g) * 3).to(dtype)
    x[17, 0], x[18, min(1, C - 1)], x[19, 0] = float("nan"), float("inf"), -float("inf")
    x[4000:] = 1e4                                         # padding rows with garbage: never read
    x[4100, 0] = float("nan")
    nv = torch.tensor([4000], dtype=torch.int32, device=cuda_dev)
    q, s = ops.fp8_quantize(x.to(cuda_dev), nv)
    ref, rs = _quant_ref(x, 4000)
    assert s.item() == rs
    got = q.double().cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[~np.isnan(ref)], ref[~np.isnan(ref)])
    assert (got[4000:] == 0).all() and np.isnan(got[17, 0]) and got[18, min(1, C - 1)] == E4M3_MAX
    # given scale: the cast alone; repeat runs are bit-identical
    q2, s2 = ops.fp8_quantize(x.to(cuda_dev), nv, torch.tensor([0.5], device=cuda_dev))
    ref2, _ = _quant_ref(x, 4000, 0.5)
    got2 = q2.double().cpu().numpy()
    assert np.array_equal(got2[~np.isnan(ref2)], ref2[~np.isnan(ref2)]) and s2.item() == 0.5
    q3, _ = ops.fp8_quantize(x.to(cuda_dev), nv)
    assert torch.equal(q.view(torch.uint8), q3.view(torch.uint8))
    # a misaligned input takes the element-wise path with the same bits
    buf = torch.empty(5000 * C + 8, dtype=dtype, device=cuda_dev)
    xv = buf[1:1 + 5000 * C].view(5000, C)
    xv.copy_(x.to(cuda_dev))
    lib, ws = _lib(), torch.empty(4096, dtype=torch.uint8, device=cuda_dev)
    q4, s4 = torch.empty((5000, C), dtype=F8, device=cuda_dev), torch.empty(1, device=cuda_dev)
    code = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}[dtype]
    from spconv_b200 import _cabi
    args = _cabi.Fp8Quant(xv.data_ptr(), code, 5000, C, nv.data_ptr(), None, q4.data_ptr(), s4.data_ptr())
    assert lib.spx_fp8_quantize(ctypes.byref(args), ws.data_ptr(), 4096, ops._stream()) == 0
    assert torch.equal(q.view(torch.uint8), q4.view(torch.uint8)) and s4.item() == rs


@gpu
def test_quantise_edges(cuda_dev):
    from spconv_b200.pytorch import ops
    q, s = ops.fp8_quantize(torch.zeros(300, 32, device=cuda_dev))
    assert s.item() == 1.0 and (q.float() == 0).all()
    x = torch.full((10, 16), float("nan"), device=cuda_dev)
    x[2, 3] = float("inf")
    q, s = ops.fp8_quantize(x)
    assert s.item() == 1.0 and q.float().isnan().sum() == 159 and q.float()[2, 3] == E4M3_MAX
    q, s = ops.fp8_quantize(torch.zeros(0, 64, device=cuda_dev, dtype=torch.float16))
    assert q.shape == (0, 64) and s.item() == 1.0
    q, s = ops.fp8_quantize(torch.ones(50, 8, device=cuda_dev), torch.zeros(1, dtype=torch.int32, device=cuda_dev))
    assert s.item() == 1.0 and (q.float() == 0).all()


# ------------------------------------------------------------------ modules
def _unet(dev, C=32):
    import spconv_b200.pytorch as spconv
    torch.manual_seed(0)
    return spconv.SparseSequential(
        spconv.SubMConv3d(C, C, 3, indice_key="s1"),
        spconv.SubMConv3d(C, C, 3, indice_key="s1", groups=C, bias=False),        # depthwise: stays float
        spconv.SparseConv3d(C, 64, 3, 2, 1, indice_key="d1"),
        spconv.SubMConv3d(64, 64, 3, indice_key="s2"),
        spconv.SparseInverseConv3d(64, C, 3, indice_key="d1"),
        spconv.SubMConv3d(C, C, 3, indice_key="s1"),
        spconv.SparseConvTranspose3d(C, 32, 3, 2, 1),
    ).to(dev).half().eval()


def _cloud(dev, C=32, n=3000, shape=(24, 24, 24)):
    import spconv_b200.pytorch as spconv
    rng = np.random.default_rng(4)
    flat = rng.choice(int(np.prod(shape)), size=n, replace=False)
    coords = np.stack(np.unravel_index(flat, shape), 1)
    inds = torch.from_numpy(np.concatenate([np.zeros((n, 1), np.int64), coords], 1).astype(np.int32)).to(dev)
    f = torch.randn(n, C, generator=torch.Generator().manual_seed(1)).half().to(dev)
    return spconv.SparseConvTensor(f, inds, list(shape), 1)


@gpu
def test_convert_unet_layer_by_layer(cuda_dev):
    """Each fp8 layer of a converted U-Net against a float64 conv of its dequantised e4m3 operands over the layer's
    own gather table (pair[k, o]: the input row of output row o at offset k, -1 none).

    Bound: a product of two e4m3 values is exact in fp32.  The FP8 tensor cores add a k-step (32 channels of one
    offset) to the accumulator keeping about 14 significant bits (DeepSeek-V3 report section 3.3.2): each of the
    step's 33 addends (32 products and the running sum) loses less than 2^-13 of the largest.  The kernel sums
    each offset's ceil(C / 32) k-steps from zero and adds them into an fp32 sum, so offset k loses less than
    33 * ceil(C / 32) * 2^-13 * S_k (S_k = sum over the offset of |x| |w|, which bounds every addend) and
    the kv fp32 additions 2^-24 * S each, S = sum_k S_k (the FMA kernel's kv * C fp32 additions lose less).  The
    epilogue's fp32 steps (in_scale * w_scale, * s, + bias) add 3 * 2^-24 of (S + |bias|), and the fp16 output one
    rounding: half an ulp, 2^-11 of the value, or 2^-25 among the subnormals."""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import fp8
    net = _unet(cuda_dev)
    skipped = spconv.convert_to_fp8(net)
    assert [n for n, _ in skipped] == ["1"] and "depthwise" in skipped[0][1]
    assert [type(m).__name__ for m in net].count("Fp8SparseConv") == 6
    x = _cloud(cuda_dev)
    checked = 0
    with torch.no_grad():
        for i, layer in enumerate(net):
            y = layer(x)
            if isinstance(layer, fp8.Fp8SparseConv):
                xq = fp8.quantize_fp8(x)              # what the layer quantises its float input to (deterministic)
                rb = layer._rulebook(xq, False, layer.algo, xq.shadow_copy())[0]
                outids, pair = rb[0], rb[1]
                assert torch.equal(outids, y.indices)
                x64 = xq.features.double() * xq.fp8_scale.double()
                w64 = (layer.weight.double() * layer.weight_scale.double().view(-1, *[1] * (layer.weight.dim() - 1)))
                kv, C = layer.weight[0].numel() // layer.in_channels, layer.in_channels
                w64 = w64.reshape(layer.out_channels, kv, C)
                n_out = outids.shape[0]
                want = torch.zeros((n_out, layer.out_channels), dtype=torch.float64, device=cuda_dev)
                S = torch.zeros_like(want)
                for k in range(kv):
                    idx = pair[k, :n_out].long()
                    g = torch.where((idx >= 0)[:, None], x64[idx.clamp_min(0)], 0.0)
                    want += g @ w64[:, k].T
                    S += g.abs() @ w64[:, k].abs().T
                b = layer.bias.double() if layer.bias is not None else torch.zeros_like(want[0])
                want += b
                acc_err = (33 * -(-C // 32) * 2.0 ** -13 + kv * 2.0 ** -24) * S + 3 * 2.0 ** -24 * (S + b.abs())
                tol = acc_err + 2.0 ** -11 * (want.abs() + acc_err) + 2.0 ** -25
                err = (y.features.double() - want).abs()
                assert (err <= tol).all(), f"layer {i}: max err {float(err.max())}, worst err / bound {float((err / tol).max())}"
                checked += 1
            x = y
    assert checked == 6


@gpu
def test_e4m3_chain_and_inference_only(cuda_dev):
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import fp8
    torch.manual_seed(2)
    a = spconv.SubMConv3d(32, 32, 3, indice_key="s").to(cuda_dev).half().eval()
    b = spconv.SubMConv3d(32, 32, 3, indice_key="s").to(cuda_dev).half().eval()
    x = _cloud(cuda_dev)
    s = fp8.calibrate_fp8_output_scale(a, x)
    qa = fp8.Fp8SparseConv.from_float(a, output_dtype=F8, output_scale=s)
    qb = fp8.Fp8SparseConv.from_float(b)
    with torch.no_grad():
        ya = qa(x)
        assert ya.features.dtype == F8 and torch.equal(ya.fp8_scale, s.reshape(1))
        yb = qb(ya, add_input=x)                           # e4m3 in, fp16 residual, fp16 out
        assert yb.features.dtype == torch.float16 and torch.isfinite(yb.features).all()
        yc = qa(x, add_input=ya)                           # fp16 in, e4m3 residual with its scale, e4m3 out
        assert yc.features.dtype == F8 and not torch.isnan(yc.features.float()).any()
        with pytest.raises(RuntimeError, match="output_add must be"):
            qb(ya, add_input=ya)
    qa.train()
    with pytest.raises(RuntimeError, match="inference only"):
        qa(x)
    for bad in (spconv.SubMConv3d(32, 32, 3, groups=32), spconv.SubMConv3d(32, 32, 1),
                spconv.SubMConv3d(32, 32, 3, algo=spconv.ConvAlgo.MaskSplitImplicitGemm)):
        with pytest.raises(NotImplementedError, match="fp8 conversion refused"):
            fp8.Fp8SparseConv.from_float(bad)
    with pytest.raises(NotImplementedError, match="already an fp8 layer"):
        fp8.Fp8SparseConv.from_float(qb)
    # a split rulebook asked for by the tensor, not by the layer: refused, not computed over the first split only
    xs = x.replace_feature(x.features)
    xs.force_algo = spconv.ConvAlgo.MaskSplitImplicitGemm
    q = fp8.Fp8SparseConv.from_float(spconv.SubMConv3d(32, 32, 3).to(cuda_dev).half().eval())
    with torch.no_grad(), pytest.raises(NotImplementedError, match="MaskSplitImplicitGemm"):
        q(xs)


@gpu
def test_native_algo(cuda_dev):
    import spconv_b200.pytorch as spconv
    torch.manual_seed(3)
    net = spconv.SparseSequential(spconv.SubMConv3d(32, 32, 3, algo=spconv.ConvAlgo.Native),
                                  spconv.SparseConv3d(32, 32, 3, 2, 1, algo=spconv.ConvAlgo.Native)).to(cuda_dev).half().eval()
    x = _cloud(cuda_dev)
    with torch.no_grad():
        want = net(x)
        spconv.convert_to_fp8(net)
        got = net(x)
    assert torch.equal(got.indices, want.indices)
    rel = (got.features.float() - want.features.float()).norm() / want.features.float().norm()
    assert rel < 0.1, float(rel)


@gpu
def test_bounded_encoder_captures(cuda_dev):
    import spconv_b200.pytorch as spconv
    torch.manual_seed(5)
    # no biases: a padding row sums no offsets, so it comes out 0
    net = spconv.SparseSequential(spconv.SubMConv3d(32, 32, 3, indice_key="a", bias=False),
                                  spconv.SparseConv3d(32, 64, 3, 2, 1, bias=False),
                                  spconv.SubMConv3d(64, 64, 3, indice_key="b", bias=False)).to(cuda_dev).half().eval()
    x0 = _cloud(cuda_dev)
    spconv.set_output_bounds(net, x0, margin=1.5)
    assert spconv.convert_to_fp8(net) == []
    padded = x0.pad_to(3500)

    def step(f, i, nv):
        x = spconv.SparseConvTensor(f, i, x0.spatial_shape, 1)
        x.num_valid = nv
        y = net(x)
        return y.features, y.num_valid

    with torch.no_grad():
        eager = step(padded.features, padded.indices, padded.num_valid)
        eager = (eager[0].clone(), eager[1].clone())
        graphed = spconv.graph_capture(step, padded.features, padded.indices, padded.num_valid)
        got = graphed(padded.features, padded.indices, padded.num_valid)
    assert torch.equal(got[0].view(torch.int16), eager[0].view(torch.int16))
    m = int(got[1].item())
    assert m < got[0].shape[0] and (got[0][m:] == 0).all()
