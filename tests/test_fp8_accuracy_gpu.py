"""FP8 (e4m3) inference off the exact grid: real-valued scales bit for bit, full-depth real-valued sums and
magnitude-skewed rows against the documented accumulation bound, and converted layers at full width.

The exact-grid tests (tests/test_fp8_gpu.py) use power-of-two scales, where a fused multiply-add, a reassociated
scale product or a multiply by 1 / out_scale give the same bits as the documented epilogue.  Here:

1. Integer operands (so the accumulator is exact) with real scales, biases and residuals: the kernel's output
   must equal a numpy float32 restatement of the epilogue (tests/fp8_epilogue_ref.py) bit for bit, and every case
   asserts that it contains elements where each wrong variant gives different bits.
2. Real-valued features and filters quantised the way the library does it, at every e4m3 tensor-core instance,
   at kernel volumes 27, 81 and 125 and through a strided conv, against float64 over the dequantised operands.
   Bound on the tensor cores: the FP8 MMA adds one k-step (32 channels) to its accumulator keeping about 14 bits,
   DeepSeek-V3 report section 3.3.2; each of the step's 33 addends (32 products, the running sum) loses less than
   2^-13 of the largest.  The kernel starts every kernel offset (window of ceil(C / 32) k-steps) from zero and
   adds the finished window into an fp32 sum, so a window w loses less than 33 ceil(C / 32) 2^-13 S_w, and the
   windows' S_w add up to S:
       |got - ref| <= (33 ceil(C / 32) 2^-13 + A 2^-24) S + 3 2^-24 (S + |bias|)
   and on the FMA kernel (T fp32 additions):
       |got - ref| <= (T + 1) 2^-23 S + 3 2^-24 (S + |bias|)
   S = sum |x| |w| of the row, A its active offsets (one fp32 addition each), T = A * C.  The epilogue term
   covers s = in_scale * w_scale, y = acc * s and y + bias, one fp32 rounding each.
3. Rows whose first active offset (the MMA visits offsets in ascending order) carries a term 2^9 to 2^12 times
   larger than every later product, with the later products together far above the bound: a tensor core that
   lets the large running sum swallow the small products of later offsets fails here (without the per-offset
   fp32 sum it does, by up to 9 times the bound).
4. Converted 128- and 256-channel layers, unpadded and padded, each against float64 of its own operands.

Sections 2 and 3 print the worst error / S of each case (pytest -s).
"""
import re

import numpy as np
import pytest
import torch

from tests.fp8_epilogue_ref import F32, differ, discriminating_bias, epilogue, reciprocal_trap_scale
from tests.test_conv_tc_coverage_gpu import KV, SIMT, _conv, _reference, library_symbols
from tests.test_conv_tc_coverage_gpu import _restore_forced_family  # noqa: F401  (autouse fixture)
from tests.test_fp8_cpu import e4m3_rne
from tests.test_fp8_gpu import ALPHA, OUTS, _cloud, _fp8_fwd, _ints, fp8_instance

gpu = pytest.mark.gpu


# ------------------------------------------------------------------ 1. the epilogue with real scales, bit for bit
# (name, C, K, fma): every tensor-core N (K = 256: two passes of N = 128 over the column halves), the FMA kernel
# pinned and by shape (C, K not multiples of 32)
EPI = ([(f"tc-N{n}", 64, n, False) for n in (32, 64, 128, 256)]
       + [("fma-forced", 64, 64, True), ("fma-shape", 48, 40, False)])


def _scales(C, K, kv, seed, dev):
    """in_scale = amax / 448 of a Gaussian feature tensor (the quantise kernel), w_scale of a Gaussian filter"""
    from spconv_b200.pytorch import ops, quantize_fp8_weight
    g = torch.Generator().manual_seed(seed)
    _, s_in = ops.fp8_quantize((torch.randn(4096, C, generator=g) * 2.3).to(dev))
    _, w_scale = quantize_fp8_weight(torch.randn(K, kv, C, generator=g) * 0.05)
    return F32(s_in.item()), w_scale.numpy().astype(F32)


def _residual(rng, n, K, out, mag):
    """(residual values of the output type as float64 [n, K], add_scale): a NaN and, for float types, an Inf"""
    if out == "e4m3":
        add = e4m3_rne(rng.standard_normal((n, K)) * 60)
        add[0, 0] = np.nan
        return add, F32(mag / 37.3)
    v = rng.standard_normal((n, K)) * mag
    add = {"f32": lambda a: a.astype(F32), "f16": lambda a: a.astype(np.float16),
           "bf16": lambda a: torch.from_numpy(a.astype(F32)).bfloat16().float().numpy()}[out](v).astype(np.float64)
    add[0, 0], add[1, 1] = np.nan, np.inf
    return add, F32(0.7071)


@gpu
@pytest.mark.parametrize("case", EPI, ids=lambda c: c[0])
@pytest.mark.parametrize("out", OUTS)
def test_epilogue_with_real_scales_bit_for_bit(case, out, oracle, cuda_dev):
    name, C, K, fma = case
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    seed = 1000 + 10 * EPI.index(case) + OUTS.index(out)
    rng = np.random.default_rng(seed)
    x, w = _ints(rng, (conv.n_in, C)), _ints(rng, (K, conv.kv, C))
    in_scale, w_scale = _scales(C, K, conv.kv, seed, cuda_dev)
    acc = _reference(x, w, torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)["out"].cpu().numpy()
    mag = float(np.abs(acc).mean() * in_scale * w_scale.mean())
    bias0 = (rng.standard_normal(K) * mag).astype(F32)
    add, add_scale = _residual(rng, conv.n_out, K, out, mag)
    y0 = acc * (float(in_scale) * w_scale.astype(np.float64)) + bias0
    out_scale = reciprocal_trap_scale(np.abs(y0).max() / 448) if out == "e4m3" else None
    variants = ("fma", "assoc", "recip") if out == "e4m3" else ("fma", "assoc")
    for act in ("none", "relu", "leaky_relu"):
        kw = dict(in_scale=in_scale, w_scale=w_scale, add=add, add_scale=add_scale, act=act, alpha=ALPHA, out=out,
                  out_scale=out_scale)
        bias = bias0.copy()
        # fp16 / bf16 / e4m3 outputs round most one-ulp fp32 differences away: channels K-1, K-2, ... get a bias
        # that puts some of their rows on a rounding boundary of the output type where the wrong variant lands on
        # the other side (fp32 outputs show every difference)
        for j, v in enumerate(variants if out != "f32" else ()):
            c = K - 1 - j
            bias[c], _ = discriminating_bias(acc[:, c], in_scale, w_scale[c], bias0[c], add[:, c], add_scale, act,
                                             ALPHA, out, out_scale, v)
        ref = epilogue(acc, bias=bias, **kw)
        for v in variants:
            n = int(differ(ref, epilogue(acc, bias=bias, variant=v, **kw)).sum())
            assert n > 0, f"{name} {out} {act}: no element tells the '{v}' epilogue from the documented one"
        got = _fp8_fwd(conv, x, w, in_scale, torch.from_numpy(w_scale), torch.from_numpy(bias), torch.from_numpy(add),
                       add_scale, out, out_scale, act, cuda_dev, fma).cpu().numpy()
        bad = differ(got, ref)
        if bad.any():
            r, c = np.argwhere(bad)[0]
            raise AssertionError(f"{name} {out} {act}: {int(bad.sum())} of {bad.size} outputs differ from the "
                                 f"float32 epilogue; first at ({r}, {c}): got {got[r, c]!r} want {ref[r, c]!r} "
                                 f"(acc {acc[r, c]:.0f})")


# ------------------------------------------------------------------ 2. full-depth real-valued sums
def tc_bound(S, bias, C, active):
    """the documented error bound of the tensor cores' f32 output (float64 tensors; active [rows, 1])"""
    return (33 * -(-C // 32) * 2.0 ** -13 + active * 2.0 ** -24) * S + 3 * 2.0 ** -24 * (S + bias.abs())


def _bound(r, bias, C, fma):
    """the documented error bound of every output element on the family that runs the call (float64 tensor)"""
    S, active = r["out_abs"], r["t_out"][:, None]
    if fma or SIMT:
        return (active * C + 1) * 2.0 ** -23 * S + 3 * 2.0 ** -24 * (S + bias.abs())
    return tc_bound(S, bias, C, active)


def _real_run(conv, xf, wf, bias, dev, fma=False):
    """quantise xf (ops.fp8_quantize) and wf (quantize_fp8_weight), run the f32-output fp8 conv -> (got, float64
    reference dict over the dequantised operands, dequantised features, dequantised filter)"""
    from spconv_b200.pytorch import ops, quantize_fp8_weight
    q, s_in = ops.fp8_quantize(xf.to(dev))
    wq, w_scale = quantize_fp8_weight(wf)
    x64 = q.double() * s_in.double()
    w64 = (wq.double() * w_scale.double().view(-1, 1, 1)).to(dev)
    K = wf.shape[0]
    r = _reference(x64, w64, torch.zeros((conv.n_out, K)), conv.ref_pair, dev)
    got = _fp8_fwd(conv, None, wq.float(), s_in, w_scale, bias, None, None, "f32", None, "none", dev, fma, x_view=q)
    return got, r, x64, w64


def _check_bound(name, got, want, S, bound):
    err = (got - want).abs()
    rel = torch.where(S > 0, err / S, torch.zeros_like(err))
    worst = int(rel.reshape(-1).argmax())
    row = worst // rel.shape[1]
    ratio = float((err / bound.clamp_min(1e-300)).max())
    print(f"\n{name}: worst err / S {float(rel.reshape(-1)[worst]):.3e} (row {row}), worst err / bound {ratio:.3f}")
    assert not torch.isnan(got).any(), f"{name}: NaN in the output"
    bad = err > bound
    assert not bad.any(), (f"{name}: {int(bad.sum())} elements beyond the documented bound; worst err / S "
                           f"{float(rel.reshape(-1)[worst]):.3e} at row {row} (S {float(S.reshape(-1)[worst]):.4g}), "
                           f"worst err / bound {ratio:.2f}")


CHANNELS = (32, 64, 128, 256)
# (geometry, mode, C, K): every e4m3 tensor-core instance at kv 27 (kv 1 where kv 27 does not fit), kv 81 and 125,
# a strided conv
DEPTH = ([("k3" if fp8_instance(27, C, K) else "k1", "subm", C, K) for C in CHANNELS for K in CHANNELS]
         + [("4d_k3", "subm", 128, 256), ("k5", "subm", 128, 128), ("k3", "conv", 256, 128)])


@gpu
@pytest.mark.parametrize("case", DEPTH, ids=lambda c: f"{c[0]}-{c[1]}-C{c[2]}K{c[3]}")
def test_full_depth_real_valued_sums(case, oracle, cuda_dev):
    geom, mode, C, K = case
    conv = _conv(oracle, cuda_dev, geom, mode)
    assert fp8_instance(conv.kv, C, K) is not None
    i = DEPTH.index(case)
    g = torch.Generator().manual_seed(200 + i)
    xf = torch.randn(conv.n_in, C, generator=g) * 1.7
    if i % 2:
        xf = xf.clamp_min(0)                        # post-ReLU: half-normal, half the features 0
    wf = torch.randn(K, conv.kv, C, generator=g) * 0.05
    bias = torch.randn(K, generator=g) * 0.5
    got, r, _, _ = _real_run(conv, xf, wf, bias, cuda_dev)
    b = bias.to(cuda_dev, torch.float64)
    _check_bound(f"C{C} K{K} kv{conv.kv} {mode} {'relu' if i % 2 else 'gauss'}", got, r["out"] + b, r["out_abs"],
                 _bound(r, b, C, False))


# ------------------------------------------------------------------ 3. magnitude-skewed rows
# the widest C each kernel volume allows on the tensor cores, and the FMA kernel
SKEW = [("k3", 256, 128, False), ("k5", 128, 128, False), ("k3", 256, 128, True)]


@gpu
@pytest.mark.parametrize("case", SKEW, ids=lambda c: f"{c[0]}-C{c[1]}K{c[2]}-{'fma' if c[3] else 'tc'}")
def test_magnitude_skewed_rows(case, oracle, cuda_dev):
    """Channel 0 of every feature row is 1 and the rest lie in [1/4, 1/2]; the filter is 1 at (offset 0, channel
    0) of every output channel and in [2^-10, 2^-9] elsewhere.  A row with offset 0 active thus starts with the
    product 1 and every later product lies in [2^-12, 2^-9]; all terms are positive, so nothing cancels."""
    geom, C, K, fma = case
    conv = _conv(oracle, cuda_dev, geom, "subm")
    assert fma or fp8_instance(conv.kv, C, K) is not None
    g = torch.Generator().manual_seed(C + conv.kv)
    xf = 0.25 + 0.25 * torch.rand(conv.n_in, C, generator=g)
    xf[:, 0] = 1.0
    wf = 2.0 ** -10 * (1 + torch.rand(K, conv.kv, C, generator=g))
    wf[:, 0, 0] = 1.0
    bias = torch.zeros(K)
    got, r, x64, w64 = _real_run(conv, xf, wf, bias, cuda_dev, fma)
    b = bias.to(cuda_dev, torch.float64)
    bound = _bound(r, b, C, fma)
    # the skewed rows and their first term; every later product against it
    pair = torch.from_numpy(conv.ref_pair).to(cuda_dev).long()
    skewed = pair[0] >= 0
    assert int(skewed.sum()) >= 100, "too few rows with offset 0 active"
    first = x64[pair[0, skewed], 0][:, None] * w64[:, 0, 0][None, :]
    w_small = w64.reshape(K, -1)[:, 1:]                 # every filter entry but (offset 0, channel 0)
    later_max, later_min = x64.max() * w_small.max(), x64.min() * w_small.min()
    assert float(later_max) <= 2.0 ** -8 * float(first.min()) and float(later_min) >= 2.0 ** -12 * float(first.max())
    # the later terms together are far above the bound: losing them cannot pass
    small = r["out_abs"][skewed] - first
    margin = small / bound[skewed]
    assert float(margin.min()) > 2 and float(margin.median()) > 10, (
        f"the small terms are only {float(margin.min()):.2f} x the bound on some row, "
        f"{float(margin.median()):.2f} x on the median row")
    _check_bound(f"skewed C{C} K{K} kv{conv.kv} {'fma' if fma else 'tc'}", got, r["out"] + b, r["out_abs"], bound)


# ------------------------------------------------------------------ 4. converted layers at full width
def _wide_net(dev, C):
    import spconv_b200.pytorch as spconv
    torch.manual_seed(C)
    return spconv.SparseSequential(
        spconv.SubMConv3d(C, C, 3, indice_key="s1"),
        spconv.SparseConv3d(C, C, 3, 2, 1, indice_key="d1"),
        spconv.SubMConv3d(C, C, 3, indice_key="s2"),
        spconv.SparseInverseConv3d(C, C, 3, indice_key="d1"),
        spconv.SubMConv3d(C, C, 5, indice_key="s5", algo=spconv.ConvAlgo.Native),     # kv 125
    ).to(dev).half().eval()


def _gather_table(layer, rb, n_in, n_out):
    """pair[k, o]: the input row of output row o at offset k (-1 none), from the layer's own rulebook.  A Native
    rulebook holds compact pairs [2, kv, L] (input rows, output rows); a SubM one counts only the offsets below
    the centre, the mirrored offset has the same count and the centre pairs every input row."""
    from spconv_b200.core import ConvAlgo
    if layer.algo != ConvAlgo.Native:
        return rb[1][:, :n_out].long()
    ip, ipn = rb[1], rb[2].cpu()
    kv = ip.shape[1]
    pair = torch.full((kv, n_out), -1, dtype=torch.long, device=ip.device)
    for k in range(kv):
        n = int(ipn[k]) if not layer.subm else n_in if k == kv // 2 else int(ipn[min(k, kv - 1 - k)])
        i, o = ip[0, k, :n].long(), ip[1, k, :n].long()
        keep = (i >= 0) & (i < n_in) & (o >= 0) & (o < n_out)
        pair[k, o[keep]] = i[keep]
    return pair


@gpu
@pytest.mark.parametrize("padded", [False, True], ids=["unpadded", "padded"])
@pytest.mark.parametrize("C", [128, 256])
def test_converted_wide_layers(C, padded, cuda_dev):
    """Each converted layer against float64 of its dequantised operands over its own gather table, bound as in
    section 2 (the tensor-core bound, which covers the FMA kernel's) plus the fp16 output rounding.  C = 256 at
    kernel volume 27 and 125 runs on the FMA kernel, the rest on the tensor cores."""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import fp8
    net = _wide_net(cuda_dev, C)
    x = _cloud(cuda_dev, C)
    if padded:
        spconv.set_output_bounds(net, x, margin=1.5)
        x = x.pad_to(3500)
    assert spconv.convert_to_fp8(net) == []
    checked = 0
    with torch.no_grad():
        for i, layer in enumerate(net):
            y = layer(x)
            xq = fp8.quantize_fp8(x)
            rb = layer._rulebook(xq, False, layer.algo, xq.shadow_copy())[0]
            n_out = y.features.shape[0] if y.num_valid is None else int(y.num_valid.item())
            assert torch.equal(rb[0][:n_out], y.indices[:n_out])
            n_in = x.features.shape[0] if x.num_valid is None else int(x.num_valid.item())
            pair = _gather_table(layer, rb, n_in, n_out)
            kv = pair.shape[0]
            x64 = xq.features.double() * xq.fp8_scale.double()
            w64 = (layer.weight.double() * layer.weight_scale.double().view(-1, *[1] * (layer.weight.dim() - 1)))
            w64 = w64.reshape(layer.out_channels, kv, C)
            want = torch.zeros((n_out, layer.out_channels), dtype=torch.float64, device=cuda_dev)
            S = torch.zeros_like(want)
            for k in range(kv):
                idx = pair[k]
                gk = torch.where((idx >= 0)[:, None], x64[idx.clamp_min(0)], 0.0)
                want += gk @ w64[:, k].T
                S += gk.abs() @ w64[:, k].abs().T
            b = layer.bias.double()
            want += b
            acc_err = tc_bound(S, b, C, (pair >= 0).sum(0)[:, None])
            tol = acc_err + 2.0 ** -11 * (want.abs() + acc_err) + 2.0 ** -25
            err = (y.features[:n_out].double() - want).abs()
            rel = torch.where(S > 0, err / S, torch.zeros_like(err))
            print(f"\nC{C} {'padded' if padded else 'unpadded'} layer {i} kv{kv}: worst err / S {float(rel.max()):.3e}")
            assert (err <= tol).all(), f"layer {i}: max err {float(err.max())}, worst err / bound {float((err / tol).max())}"
            checked += 1
            x = y
    assert checked == len(net)


# ------------------------------------------------------------------ every compiled e4m3 instance is reached
def _cases_instances():
    seen = {fp8_instance(27, C, K) for _, C, K, fma in EPI if not fma}
    seen |= {fp8_instance(KV[geom], C, K) for geom, _, C, K in DEPTH}
    seen |= {fp8_instance(KV[geom], C, K) for geom, C, K, fma in SKEW if not fma}
    seen.discard(None)
    return {(cpr, n) for _, _, cpr, n in seen}


def test_every_fp8_instance_is_reached():
    """No GPU needed: each tc_gather_gemm_fp8_kernel<CPR, N> in the library is served by a case of this file."""
    found = re.findall(r"tc_gather_gemm_fp8_kernel<(\d+), (\d+)>", library_symbols())
    compiled = {(int(a), int(b)) for a, b in found}
    assert compiled, "no tc_gather_gemm_fp8_kernel instance in the library's symbol table"
    reached = _cases_instances()
    assert not compiled - reached, f"compiled but reached by no case: {sorted(compiled - reached)}"
    assert not reached - compiled, f"expected by a case but not compiled: {sorted(reached - compiled)}"
