"""Every kernel with operands at unaligned and strided addresses.

The caching allocator hands out 512-byte aligned blocks, but the public API also produces contiguous tensors at
odd element offsets: the gradient autograd slices out of a ``torch.cat``, a parameter living in a flat buffer, a
``view`` of a larger buffer.  The tensor-core GEMMs, the pooling and the rulebook kernels read rows as 16-byte
vectors; the C entry points keep a misaligned GEMM operand off the tensor cores and refuse a misaligned pool or
rulebook pointer, and the Python operators realign such an operand, so that a public call runs the same kernel
as an aligned one and returns the same bits.

Every case moves one operand (then all of them) to each byte offset in (0, 16) that the element type allows and
to the aligned offsets 16, 48, 112 and 512, relative to a 1024-byte boundary, plus a column slice, a
transposed-back tensor and a stride-0 expanded gradient.  Each result is compared bit for bit with the same call
on 1024-byte aligned copies, and one case per family against a float64 reference on exact-grid inputs.  Direct
C-ABI calls fill their outputs with NaN first, so a row a kernel never writes cannot pass.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from tests.test_conv_tc_coverage_gpu import (ELEM, ENV_FAMILY, REFUSED, SIMT, TORCH_DT, _calls, _check, _configure,
                                             _conv, _exact, _lib, _reference)
from tests.test_conv_tc_coverage_gpu import _restore_forced_family  # noqa: F401  (autouse fixture)
from tests.test_int8_gpu import _check_out, _formula
from tests.util import random_cloud

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALIGNED_OFFSETS = [16, 48, 112, 512]


def offsets(elem):
    """every multiple of the element size in (0, 16), then aligned offsets that are not 128- or 1024-aligned"""
    return list(range(elem, 16, elem)) + ALIGNED_OFFSETS


def at_offset(t, nbytes):
    """a contiguous copy of ``t`` whose ``data_ptr() % 1024 == nbytes``"""
    size = t.numel() * t.element_size()
    raw = torch.empty(size + 2048, dtype=torch.uint8, device=t.device)
    skip = (nbytes - raw.data_ptr()) % 1024
    out = raw[skip:skip + size].view(t.dtype).view(t.shape)
    out.copy_(t)
    assert out.is_contiguous() and out.data_ptr() % 1024 == nbytes
    return out


def near_offset(t, nbytes):
    """at_offset at the largest multiple of the element size not above ``nbytes`` (one offset for mixed dtypes)"""
    return at_offset(t, nbytes - nbytes % t.element_size())


def column_slice(t):
    """the same values as a column slice of a wider tensor (row stride > columns; a 1-D tensor: a strided view)"""
    cols = t.shape[1] if t.dim() == 2 else 1
    wide = torch.zeros((t.shape[0], cols + 3), dtype=t.dtype, device=t.device)
    wide[:, 1:1 + cols] = t.reshape(t.shape[0], cols)
    out = wide[:, 1:1 + cols] if t.dim() == 2 else wide[:, 1]
    assert not out.is_contiguous()
    return out


def transposed_back(t):
    out = t.t().contiguous().t()
    assert not out.is_contiguous() and torch.equal(out, t)
    return out


def _bits(t):
    t = t.contiguous()
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.int8}[t.element_size()])


def _same(got, want, what):
    """bit-for-bit equality of two lists of tensors (NaN included)"""
    assert len(got) == len(want), what
    for j, (a, b) in enumerate(zip(got, want)):
        if a is None or b is None:
            assert a is None and b is None, f"{what}: output {j}"
            continue
        assert a.dtype == b.dtype and a.shape == b.shape, f"{what}: output {j} {a.dtype}{tuple(a.shape)}"
        assert torch.equal(_bits(a), _bits(b)), f"{what}: output {j} differs from the aligned call"


def _auto_unless_tc(tc_able):
    """with the tensor cores forced from the environment, a case they cannot tile at all (aligned or not) runs
    with the automatic choice instead"""
    if ENV_FAMILY == 2 and not tc_able:
        _configure(0)


# ============================================================================ C ABI: the conv GEMMs
# (dtype, geometry, mode, C, K): one shape per compiled row-byte span of the gathered rows (32 .. 512 bytes), the
# fp32 input gradient's float4 weight path (C * 4 % 128 == 0), a strided conv, an inverse conv and odd channels
GEMM_CASES = [("f16", "k3", "subm", 16, 16), ("bf16", "k3", "conv", 32, 32), ("f16", "k3", "subm", 64, 64),
              ("bf16", "k3", "inverse", 128, 32), ("f16", "k1", "conv", 256, 16), ("tf32", "k3", "subm", 32, 32),
              ("tf32", "k3", "conv", 64, 16), ("f16", "k3", "subm", 31, 17)]


def _pinned(family, launch):
    """run on `family` (1 FMA, 2 tensor cores) and check that it ran there; a call that must leave the tensor
    cores is refused while they are forced"""
    if SIMT or family == 1:
        if not SIMT:
            _configure(2)
            with pytest.raises(RuntimeError, match=REFUSED):
                launch()
        _configure(0 if not SIMT else 1)
    else:
        _configure(2)
    out = launch()
    assert _lib().spx_last_kernel_family() == (1 if SIMT else family)
    return out


def _fma(launch):
    _configure(1)
    out = launch()
    assert _lib().spx_last_kernel_family() == 1
    return out


def _gemm_calls(conv, C, K):
    """launchers of fwd / dgrad / wgrad taking the operands as tensors (outputs NaN-filled, aligned)"""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    lib = _lib()

    def fwd(x, w, bias=None):
        d = conv.desc(x.dtype, C, K, conv.fwd)
        out = torch.full((conv.n_out, K), float("nan"), dtype=x.dtype, device=x.device)
        _cabi.check(lib.spx_implicit_gemm_fwd(ctypes.byref(d), x.data_ptr(), w.data_ptr(), out.data_ptr(),
                                              None if bias is None else bias.data_ptr(), 0, 0.0, ops._stream()), "fwd")
        return out

    def dgrad(dout, w):
        d = conv.desc(dout.dtype, C, K, conv.fwd, reverse=True) if conv.subm else conv.desc(dout.dtype, C, K, conv.bwd)
        din = torch.full((conv.n_in, C), float("nan"), dtype=dout.dtype, device=dout.device)
        _cabi.check(lib.spx_implicit_gemm_dgrad(ctypes.byref(d), dout.data_ptr(), w.data_ptr(), din.data_ptr(),
                                                ops._stream()), "dgrad")
        return din

    def wgrad(x, dout):
        d = conv.desc(x.dtype, C, K, conv.fwd)
        ws = torch.empty(lib.spx_implicit_gemm_wgrad_workspace_size(ctypes.byref(d)), dtype=torch.uint8,
                         device=x.device)
        dw = torch.full((K, conv.kv, C), float("nan"), dtype=x.dtype, device=x.device)
        _cabi.check(lib.spx_implicit_gemm_wgrad(ctypes.byref(d), x.data_ptr(), dout.data_ptr(), dw.data_ptr(),
                                                ws.data_ptr(), ws.numel(), ops._stream()), "wgrad")
        return dw
    return fwd, dgrad, wgrad


@gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: f"{c[0]}-{c[1]}-{c[2]}-C{c[3]}K{c[4]}")
def test_gemm_c_abi_operands_at_every_offset(case, oracle, cuda_dev):
    """A misaligned operand runs on the FMA kernels (refused while the tensor cores are forced) and equals the
    aligned call pinned there bit for bit; an operand at an aligned offset stays on the family of the aligned call
    and equals it bit for bit.  Both baselines are checked against the float64 reference."""
    dt, geom, mode, C, K = case
    conv = _conv(oracle, cuda_dev, geom, mode)
    rng = np.random.default_rng(C * 100 + K)
    tdt = TORCH_DT[dt]
    x = _exact(rng, (conv.n_in, C), dt).to(cuda_dev, tdt)
    w = _exact(rng, (K, conv.kv, C), dt).to(cuda_dev, tdt)
    dout = _exact(rng, (conv.n_out, K), dt).to(cuda_dev, tdt)
    bias = _exact(rng, (K,), dt).to(cuda_dev, tdt)
    inst = _calls(dt, conv.kv, C, K)
    fam = {k: 2 if v is not None else 1 for k, v in inst.items()}
    fwd, dgrad, wgrad = _gemm_calls(conv, C, K)
    a = {n: at_offset(t, 0) for n, t in (("x", x), ("w", w), ("dout", dout), ("bias", bias))}
    calls = {"fwd": (fwd, ("x", "w")), "fwd+bias": (lambda x_, w_, b_: fwd(x_, w_, b_), ("x", "w", "bias")),
             "dgrad": (dgrad, ("dout", "w")), "wgrad": (wgrad, ("x", "dout"))}
    base, base_fma = {}, {}
    for name, (fn, ops_) in calls.items():
        base[name] = _pinned(fam[name.split("+")[0]], lambda: fn(*[a[o] for o in ops_]))
        base_fma[name] = _fma(lambda: fn(*[a[o] for o in ops_]))
    torch.cuda.synchronize()
    r = _reference(x.float(), w.float(), dout.float(), conv.ref_pair, cuda_dev)
    for res in (base, base_fma):
        _check("out", res["fwd"], r["out"], r["out_abs"], r["t_out"][:, None] * C, dt, zero=r["t_out"] == 0)
        _check("din", res["dgrad"], r["din"], r["din_abs"], r["t_in"][:, None] * K, dt, zero=r["t_in"] == 0)
        _check("dw", res["wgrad"], r["dw"], r["dw_abs"], r["t_k"][None, :, None], dt,
               zero=(r["t_k"] == 0)[None, :, None].expand(K, conv.kv, C))
    for name, (fn, ops_) in calls.items():
        moves = [(o, off) for o in ops_ for off in offsets(ELEM[dt])] + [("all", ELEM[dt]), ("all", 16)]
        for what, off in moves:
            args = [at_offset(a[o], off) if what in (o, "all") else a[o] for o in ops_]
            # the bias is read element by element: it alone never moves a call off the tensor cores
            misaligned = off % 16 != 0 and what != "bias"
            got = _pinned(1 if misaligned else fam[name.split("+")[0]], lambda: fn(*args))
            _same([got], [(base_fma if misaligned else base)[name]], f"{name}: {what} at {off} bytes")


@gpu
@pytest.mark.parametrize("out_dtype", [torch.int8, torch.float16])
def test_int8_operands_at_every_offset(out_dtype, oracle, cuda_dev):
    """int8 forward through ops.implicit_gemm on the tensor cores and on the FMA kernels: features, filters,
    scale, bias and the int8 residual moved; the result is the aligned call's, on the aligned call's family"""
    from spconv_b200.pytorch import ops
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    rng = np.random.default_rng(8)
    pf, mask, argsort, n_out = conv.fwd
    for C, K in ((64, 64), (48, 24)):             # tensor-core shape, FMA shape
        _auto_unless_tc(C == 64)
        x = torch.from_numpy(rng.integers(-8, 8, (conv.n_in, C)).astype(np.int8)).to(cuda_dev)
        w = torch.from_numpy(rng.integers(-8, 8, (K, 3, 3, 3, C)).astype(np.int8)).to(cuda_dev)
        scale = torch.from_numpy(rng.uniform(0.001, 0.01, K).astype(np.float32)).to(cuda_dev)
        bias = torch.from_numpy(rng.uniform(-1, 1, K).astype(np.float32)).to(cuda_dev)
        add = torch.from_numpy(rng.integers(-100, 100, (n_out, K)).astype(np.int8)).to(cuda_dev)

        def call(x_, w_, s_, b_, a_):
            out = ops.implicit_gemm(x_, w_, pf, [mask], [argsort], n_out, [np.full(1, 0xFFFFFFFF, np.uint32)], False, True,
                                    bias=b_, scale=s_, output_add=a_, output_add_scale=0.5, output_dtype=out_dtype)[0]
            return out, ops.last_kernel_family()
        want, fam = call(x, w, scale, bias, add)
        assert fam == (1 if SIMT or C == 48 else 2)
        # float64 reference: the exact int32 accumulator, then the epilogue (scale, bias, residual x 0.5)
        acc = _reference(x.float(), w.float().reshape(K, -1, C), torch.zeros((n_out, K)), conv.ref_pair,
                         cuda_dev)["out"]
        val, err = _formula(acc, scale, bias, add, 0.5, "none", cuda_dev)
        _check_out("int8 fwd", want.double(), val, err, "i8" if out_dtype == torch.int8 else "f16")
        ops_ = {"x": x, "w": w, "scale": scale, "bias": bias, "add": add}
        for name, t in ops_.items():
            for off in offsets(t.element_size()):
                args = {k: (at_offset(v, off) if k == name else v) for k, v in ops_.items()}
                got, f = call(*args.values())
                assert f == fam, (name, off)
                _same([got], [want], f"int8 {name} at {off} bytes")
        got, f = call(x, w, scale, bias, column_slice(add))
        _same([got], [want], "int8 residual as a column slice")
        with pytest.raises(RuntimeError, match="output_add must be int8"):
            call(x, w, scale, bias, add.half())
        with pytest.raises(RuntimeError, match="output_add must be int8"):
            call(x, w, scale, bias, add[:-1])


# ============================================================================ public API: conv, pool, depthwise
def _values(rng, shape, dev, dt, exact):
    """exact: small integers, every sum exact in fp32 (for the float64 checks); otherwise normal values, whose sums
    round differently in any other order (for the bit-for-bit comparisons of two calls)"""
    v = rng.integers(-2, 3, shape) if exact else rng.standard_normal(shape)
    return torch.from_numpy(v.astype(np.float32)).to(dev, dt)


def _cloud_tensor(dev, dt, C, seed, shape=(24, 24, 24), counts=(1500, 1300), exact=False):
    rng = np.random.default_rng(seed)
    _, inds = random_cloud(rng, list(shape), list(counts), 1)
    return _values(rng, (inds.shape[0], C), dev, dt, exact), torch.from_numpy(inds).to(dev)


def _module_net(kind, algo_name, C, K):
    import spconv_b200.pytorch as spconv
    from spconv_b200.core import ConvAlgo
    algo = ConvAlgo[algo_name]
    if kind == "subm":
        return spconv.SparseSequential(spconv.SubMConv3d(C, K, 3, indice_key="s", algo=algo))
    if kind == "conv":
        return spconv.SparseSequential(spconv.SparseConv3d(C, K, 3, 2, 1, algo=algo))
    if kind == "transpose":
        return spconv.SparseSequential(spconv.SparseConvTranspose3d(C, K, 2, 2, algo=algo))
    if kind == "inverse":
        return spconv.SparseSequential(spconv.SparseConv3d(C, C, 3, 2, 1, indice_key="d", algo=algo),
                                       spconv.SparseInverseConv3d(C, K, 3, indice_key="d", algo=algo))
    if kind == "depthwise":
        return spconv.SparseSequential(spconv.SubMConv3d(C, C, 3, groups=C, indice_key="s", algo=algo))
    if kind == "maxpool":
        return spconv.SparseSequential(spconv.SparseMaxPool3d(2, 2, algo=algo))
    if kind == "avgpool":
        return spconv.SparseSequential(spconv.SparseAvgPool3d(2, 2))
    raise ValueError(kind)


def _run_module(net, params, f, inds, g, moves, dev):
    """forward + backward with the operands placed as `moves` says; -> (outputs, kernel families)"""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    place = lambda t, what: moves.get(what, lambda v: at_offset(v, 0))(t)     # noqa: E731
    for p, v in zip(net.parameters(), params):
        p.data = place(v, "bias" if p.dim() == 1 else "weight")
        p.grad = None
    x = spconv.SparseConvTensor(place(f, "features").requires_grad_(True), place(inds, "indices"), [24, 24, 24], 2)
    y = net(x)
    fam_fwd = ops.last_kernel_family()
    if "expand" in moves:
        y.features.sum().backward()
    else:
        y.features.backward(place(g, "grad"))
    fam_bwd = ops.last_kernel_family()
    torch.cuda.synchronize()
    return [y.features.detach(), y.indices, x.features.grad] + [p.grad for p in net.parameters()], (fam_fwd, fam_bwd)


# (kind, algo, dtype, C, K): every conv route, the fp32 routes, odd channels, depthwise and the pools
MODULE_CASES = [("subm", "MaskImplicitGemm", "f16", 64, 64), ("conv", "MaskImplicitGemm", "bf16", 32, 64),
                ("transpose", "MaskImplicitGemm", "f16", 32, 32), ("inverse", "MaskImplicitGemm", "f16", 64, 32),
                ("subm", "MaskSplitImplicitGemm", "f16", 32, 32), ("conv", "MaskSplitImplicitGemm", "bf16", 32, 16),
                ("subm", "Native", "f16", 32, 32), ("conv", "Native", "bf16", 64, 32),
                ("subm", "MaskImplicitGemm", "tf32", 32, 32), ("conv", "MaskImplicitGemm", "f32", 32, 32),
                ("subm", "MaskImplicitGemm", "f16", 31, 17), ("depthwise", "MaskImplicitGemm", "f16", 32, 32),
                ("depthwise", "Native", "f32", 20, 20),
                ("maxpool", "MaskImplicitGemm", "f16", 32, 32), ("maxpool", "MaskImplicitGemm", "f32", 8, 8),
                ("maxpool", "MaskImplicitGemm", "bf16", 16, 16), ("maxpool", "Native", "f16", 16, 16),
                ("avgpool", "MaskImplicitGemm", "f32", 12, 12), ("avgpool", "MaskImplicitGemm", "bf16", 24, 24)]


@gpu
@pytest.mark.parametrize("case", MODULE_CASES, ids=lambda c: "-".join(map(str, c)))
def test_public_api_operands_at_every_offset(case, cuda_dev, monkeypatch):
    """Through the modules: features, indices, every weight, every bias and the output gradient moved one at a
    time and all together, as a column slice, transposed back, and the stride-0 gradient of a sum.  Every
    output, the input gradient and every parameter gradient equal the aligned run's bits, on the same kernel
    family, forward and backward."""
    from spconv_b200.pytorch import ops
    kind, algo, dt, C, K = case
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", dt == "tf32")
    tdt = TORCH_DT["tf32" if dt == "f32" else dt]
    conv_kind = kind in ("subm", "conv", "transpose", "inverse")
    _auto_unless_tc(not conv_kind or (dt != "f32" and C % 16 == 0 and K % 16 == 0))
    torch.manual_seed(0)
    net = _module_net(kind, algo, C, K).to(cuda_dev).to(tdt)
    rng = np.random.default_rng(1)
    params = [_values(rng, tuple(p.shape), cuda_dev, tdt, False) * 0.2 for p in net.parameters()]
    f, inds = _cloud_tensor(cuda_dev, tdt, C, seed=C + K)
    probe, _ = _run_module(net, params, f, inds, None, {"expand": True}, cuda_dev)
    g = _values(rng, tuple(probe[0].shape), cuda_dev, tdt, False)
    want, fams = _run_module(net, params, f, inds, g, {}, cuda_dev)
    if conv_kind:
        assert fams[0] in (1, 2) and fams[1] in (1, 2)
    e = f.element_size()
    runs = []
    for what in ("features", "weight", "bias", "grad"):
        for off in offsets(e):
            runs.append((f"{what} at {off}", {what: lambda t, off=off: at_offset(t, off)}))
    for off in (4, 8, 12):
        runs.append((f"indices at {off}", {"indices": lambda t, off=off: at_offset(t, off)}))
    runs.append(("all at one element", {w: (lambda t: at_offset(t, t.element_size()))
                                        for w in ("features", "weight", "bias", "grad", "indices")}))
    runs.append(("all at 16", {w: (lambda t: at_offset(t, 16)) for w in ("features", "weight", "bias", "grad")}))
    runs.append(("column slices", {"features": column_slice, "grad": column_slice, "indices": column_slice}))
    runs.append(("transposed back", {"features": transposed_back, "grad": transposed_back}))
    # the bias gradient is torch's own sum of the output gradient (the bias is added outside the op), and torch
    # sums a column-major gradient in another order: for that layout it is left out of the comparison
    keep = [True] * 3 + [p.dim() > 1 for p in net.parameters()]
    for name, moves in runs:
        got, gf = _run_module(net, params, f, inds, g, moves, cuda_dev)
        assert gf == fams, f"{name}: kernel families {gf}, aligned {fams}"
        if name == "transposed back":
            _same([t for t, k in zip(got, keep) if k], [t for t, k in zip(want, keep) if k], name)
        else:
            _same(got, want, name)
    ones = torch.ones_like(g)
    want1, fams1 = _run_module(net, params, f, inds, ones, {}, cuda_dev)
    got1, gf1 = _run_module(net, params, f, inds, ones, {"expand": True}, cuda_dev)
    assert gf1 == fams1
    _same(got1, want1, "stride-0 expanded gradient")
    if kind in ("maxpool", "depthwise", "subm") and algo == "MaskImplicitGemm":
        params = [_values(rng, tuple(p.shape), cuda_dev, tdt, True) for p in net.parameters()]
        f = _values(rng, tuple(f.shape), cuda_dev, tdt, True)
        g = _values(rng, tuple(g.shape), cuda_dev, tdt, True)
        got, _ = _run_module(net, params, f, inds, g, {}, cuda_dev)
        _float64_check(kind, net, params, f, inds, g, got)


def _float64_check(kind, net, params, f, inds, g, got):
    """exact-grid inputs: every sum is exact in fp32, so the outputs equal the float64 reference exactly"""
    from tests.conv_ref import SparseConvRef
    m = net[0]
    sub = kind != "maxpool"
    ref = SparseConvRef(inds.cpu().numpy(), 2, [24, 24, 24], [m.kernel_size[0]] * 3 if hasattr(m, "kernel_size")
                        else [2] * 3, [1 if sub else 2] * 3, [1 if sub else 0] * 3, [1] * 3, kind="subm" if sub else "conv")
    x = f.double().cpu()
    dt = f.dtype
    cast = lambda a: torch.as_tensor(a).to(dt).cpu()        # noqa: E731  (the exact sum, rounded once)
    if kind == "maxpool":
        out = torch.full((ref.n_out, x.shape[1]), -float("inf"), dtype=torch.float64)
        for i, o in ref.pairs:
            out.index_reduce_(0, torch.from_numpy(o), x[torch.from_numpy(i)], "amax")
        _same([got[0].cpu()], [cast(out)], "max pool forward against the float64 reference")
        return
    w = params[0].double().cpu()
    if kind == "depthwise":                    # [C, *ksize, 1] -> the dense KRSC [C, kv, C] with a diagonal
        C = w.shape[0]
        wfull = torch.zeros((C, w[0].numel(), C), dtype=torch.float64)
        wfull[torch.arange(C), :, torch.arange(C)] = w.reshape(C, -1)
    else:
        wfull = w.reshape(w.shape[0], -1, w.shape[-1])
    bias = params[1].double().cpu().numpy() if len(params) > 1 else None
    out = ref.forward(x.numpy(), wfull.numpy(), bias)[0]
    _same([got[0].cpu()], [cast(out)], f"{kind}: forward against the float64 reference")
    dx = ref.backward(x.numpy(), wfull.numpy(), g.double().cpu().numpy())[0]
    _same([got[2].cpu()], [cast(dx)], f"{kind}: input gradient against the float64 reference")


# ============================================================================ rulebooks
# (name, shape, ksize, stride, padding, subm, transposed, bound): 1-D to 4-D, SubM 3x3x3 probe, generic SubM,
# regular k3, FAST3 (3-D, not 3x3x3), generic (2-D / 4-D), transposed, bounded
RULEBOOKS = [("1d-subm", [3000], [5], [1], [2], True, False, -1), ("1d-conv", [3000], [5], [2], [2], False, False, -1),
             ("2d-conv", [60, 50], [3, 3], [2, 2], [1, 1], False, False, -1),
             ("3d-subm-k3", [24, 24, 24], [3] * 3, [1] * 3, [1] * 3, True, False, -1),
             ("3d-subm-k5", [24, 24, 24], [5] * 3, [1] * 3, [2] * 3, True, False, -1),
             ("3d-conv-k3", [24, 24, 24], [3] * 3, [2] * 3, [1] * 3, False, False, -1),
             ("3d-fast3-k2", [24, 24, 24], [2] * 3, [2] * 3, [0] * 3, False, False, -1),
             ("3d-transposed", [12, 12, 12], [2] * 3, [2] * 3, [0] * 3, False, True, -1),
             ("3d-bounded", [24, 24, 24], [3] * 3, [2] * 3, [1] * 3, False, False, 4096),
             ("4d-conv", [9, 10, 11, 12], [3] * 4, [2] * 4, [1] * 4, False, False, -1)]


@gpu
@pytest.mark.parametrize("case", RULEBOOKS, ids=lambda c: c[0])
def test_rulebook_indices_at_every_offset(case, cuda_dev):
    """indices at 4, 8 and 12 bytes past a 16-byte boundary, and as a column slice: every table of the masked
    implicit-GEMM rulebook (out indices, pairs, masks, argsorts, tile tables) and of the Native one equals the
    aligned build bit for bit"""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    name, shape, ks, st, pd, subm, tr, bound = case
    nd = len(shape)
    _, inds = random_cloud(np.random.default_rng(len(name)), shape, [1500, 1200] if nd < 4 else [2000], 1)
    inds = torch.from_numpy(inds).to(cuda_dev)
    dil, op = [1] * nd, [0] * nd
    kv = int(np.prod(ks))

    def build(i):
        res = ops.get_indice_pairs_implicit_gemm(i, 2, shape, ConvAlgo.MaskImplicitGemm, ks, st, pd, dil, op, subm, tr,
                                                 is_train=True, num_out_act_bound=bound)
        out_inds, num, pf, pb, mf, mb, sf, sb, _ = res
        tables = [out_inds, num, pf, pb, *mf, *mb, *sf, *sb]
        tables += list(ops._tile_tables(pf, mf[0], sf[0], pf.shape[1], kv))
        if not subm:
            tables += list(ops._tile_tables(pb, mb[0], sb[0], pb.shape[1], kv))
        if bound > 0:
            tables += [out_inds._spx_num_valid, out_inds._spx_bound_status]
        else:
            tables += list(ops.get_indice_pairs(i, 2, shape, ConvAlgo.Native, ks, st, pd, dil, op, subm, tr))
        torch.cuda.synchronize()
        return [t.clone() for t in tables]

    want = build(at_offset(inds, 0))
    for off in (4, 8, 12, 16, 48):
        _same(build(at_offset(inds, off)), want, f"{name}: indices at {off} bytes")
    _same(build(column_slice(inds)), want, f"{name}: indices as a column slice")


# ============================================================================ the guarded families
GUARDED = ["batchnorm", "global_max", "global_avg", "sparse_add", "masked_sparse_add", "scatter_max", "scatter_mean",
           "scatter_sum"]


@gpu
@pytest.mark.parametrize("family", GUARDED)
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_guarded_kernels_agree_on_both_paths(family, dt, cuda_dev):
    """MaskedBatchNorm1d, the masked global pools, sparse_add, masked_sparse_add and PointVoxelScatter check their
    pointers and take a per-element path when one is not 16-byte aligned: on normal (not exact-grid) values both
    paths give the same bits, forward and backward"""
    import spconv_b200.pytorch as spconv
    tdt = TORCH_DT["tf32" if dt == "f32" else dt]
    C = 32
    f, inds = _cloud_tensor(cuda_dev, tdt, C, seed=3)
    f2, inds2 = _cloud_tensor(cuda_dev, tdt, C, seed=4)
    rows = 700
    ids = torch.from_numpy(np.random.default_rng(6).integers(-1, rows, f.shape[0]).astype(np.int32)).to(cuda_dev)

    def run(place):
        rng = np.random.default_rng(5)
        x = spconv.SparseConvTensor(place(f).requires_grad_(True), inds, [24, 24, 24], 2)
        x2 = spconv.SparseConvTensor(place(f2).requires_grad_(True), inds2, [24, 24, 24], 2)
        if family == "batchnorm":
            y = spconv.MaskedBatchNorm1d(C).to(cuda_dev).to(tdt)(x).features
        elif family == "sparse_add":
            y = spconv.functional.sparse_add(x, x2).features
        elif family == "masked_sparse_add":
            y = spconv.functional.masked_sparse_add(x, x2).features
        elif family.startswith("scatter"):
            sc = spconv.PointVoxelScatter(place(ids), rows)
            y = getattr(sc, family.split("_")[1])(x.features)
        else:
            y = (spconv.MaskedGlobalMaxPool() if family == "global_max" else spconv.MaskedGlobalAvgPool())(x)
        y.backward(place(_values(rng, tuple(y.shape), cuda_dev, tdt, False)))
        torch.cuda.synchronize()
        return [y.detach(), x.features.grad, x2.features.grad]

    want = run(lambda t: at_offset(t, 0))
    for off in offsets(f.element_size()):
        _same(run(lambda t: near_offset(t, off)), want, f"{family}: operands at {off} bytes")
    _same(run(column_slice), want, f"{family}: operands as column slices")


@gpu
def test_point_to_voxel_and_hash_table_operands_at_every_offset(cuda_dev):
    """PointToVoxel, MaskedPointToVoxel and HashTable read their inputs element by element: points, point offsets,
    keys and values at every offset give the aligned call's bits"""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch.hash import HashTable
    rng = np.random.default_rng(12)
    vs, cr = [0.4, 0.4, 0.5], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0]
    sizes = [6000, 4000]
    pts = torch.from_numpy(np.stack([rng.random(sum(sizes)) * 30, rng.random(sum(sizes)) * 20 - 10,
                                     rng.random(sum(sizes)) * 3 - 2.5, rng.random(sum(sizes))], 1)
                           .astype(np.float32)).to(cuda_dev)
    off = torch.tensor([0, sizes[0], sum(sizes)], dtype=torch.int32, device=cuda_dev)
    keys = torch.from_numpy(rng.permutation(1 << 20)[:5000].astype(np.int32)).to(cuda_dev)
    vals = _values(rng, (5000,), cuda_dev, torch.float32, False)

    def run(place):
        gen = spconv.PointToVoxel(vs, cr, 4, 8000, 5, device=cuda_dev)
        out = [t.clone() for t in gen.generate_voxel_with_id(place(pts))]
        mgen = spconv.MaskedPointToVoxel(vs, cr, 4, 8000, 5, 2, device=cuda_dev)
        out += [t.clone() for t in mgen(place(pts), place(off))]
        for kdt in (torch.int32, torch.int64):
            table = HashTable(cuda_dev, kdt, torch.float32, max_size=2 * keys.numel())
            table.insert(place(keys.to(kdt)), place(vals))
            table.insert_exist_keys(place(keys[::2].to(kdt)), place(vals[::2] * 2))
            out += list(table.query(place(keys.to(kdt))))
        torch.cuda.synchronize()
        return out

    want = run(lambda t: at_offset(t, 0))
    for o in (4, 8, 12, 16, 48, 112, 512):
        _same(run(lambda t: near_offset(t, o)), want, f"points, offsets, keys and values at {o} bytes")


@gpu
@pytest.mark.parametrize("case", [("subm", "MaskImplicitGemm", "f16", 64, 64), ("conv", "Native", "bf16", 32, 32),
                                  ("subm", "MaskImplicitGemm", "f32", 24, 40), ("depthwise", "MaskImplicitGemm",
                                                                                "f16", 32, 32)],
                         ids=lambda c: "-".join(map(str, c)))
def test_weight_gradient_under_the_wgrad_hook(case, cuda_dev):
    """with ops.set_wgrad_hook installed the weight gradient runs first and the hook sees dW: misaligned features
    and output gradients give the aligned call's dW, as the hook sees it and as the op returns it"""
    from spconv_b200.pytorch import ops
    kind, algo, dt, C, K = case
    _auto_unless_tc(dt != "f32")
    tdt = TORCH_DT["tf32" if dt == "f32" else dt]
    torch.manual_seed(0)
    net = _module_net(kind, algo, C, K).to(cuda_dev).to(tdt)
    rng = np.random.default_rng(2)
    params = [_values(rng, tuple(p.shape), cuda_dev, tdt, False) * 0.2 for p in net.parameters()]
    f, inds = _cloud_tensor(cuda_dev, tdt, C, seed=7)
    probe, _ = _run_module(net, params, f, inds, None, {"expand": True}, cuda_dev)
    g = _values(rng, tuple(probe[0].shape), cuda_dev, tdt, False)
    seen = []
    ops.set_wgrad_hook(lambda dw: seen.append(dw.clone()))
    try:
        want, fams = _run_module(net, params, f, inds, g, {}, cuda_dev)
        want_seen, seen[:] = list(seen), []
        assert want_seen, "the hook was not called"
        for off in offsets(f.element_size()):
            got, gf = _run_module(net, params, f, inds, g, {"features": lambda t, o=off: at_offset(t, o),
                                                            "grad": lambda t, o=off: at_offset(t, o)}, cuda_dev)
            assert gf == fams
            _same(got, want, f"outputs, features and gradient at {off} bytes")
            _same(seen, want_seen, f"dW seen by the hook, features and gradient at {off} bytes")
            seen[:] = []
    finally:
        ops.set_wgrad_hook(None)


# ============================================================================ end to end through autograd
@gpu
def test_misaligned_gradients_from_autograd(cuda_dev):
    """fp16 SubMConv3d and SparseMaxPool3d with tensor-core channel counts under a loss on
    ``torch.cat([aux.flatten(), y.features.flatten()])``: with 7 fp16 elements of aux autograd hands both layers a
    gradient 14 bytes past a 16-byte boundary.  Every gradient equals the run with 8 elements of aux."""
    import spconv_b200.pytorch as spconv
    torch.manual_seed(0)
    conv = spconv.SubMConv3d(64, 64, 3, indice_key="s").to(cuda_dev).half()
    pool = spconv.SparseMaxPool3d(2, 2)
    f, inds = _cloud_tensor(cuda_dev, torch.float16, 64, seed=9)

    def run(n_aux):
        conv.weight.grad = conv.bias.grad = None
        x = spconv.SparseConvTensor(f.clone().requires_grad_(True), inds, [24, 24, 24], 2)
        x2 = spconv.SparseConvTensor(f.clone().requires_grad_(True), inds, [24, 24, 24], 2)
        y1, y2 = conv(x), pool(x2)
        seen = []
        for y in (y1, y2):
            y.features.register_hook(lambda gr: seen.append(gr.data_ptr() % 16))
        aux = torch.ones(n_aux, dtype=torch.float16, device=cuda_dev, requires_grad=True)
        cat = torch.cat([aux.flatten(), y1.features.flatten(), y2.features.flatten()])
        gen = np.random.default_rng(11)
        wts = torch.from_numpy(gen.integers(-2, 3, cat.numel() - n_aux).astype(np.float32)).to(cuda_dev)
        (cat.float() * torch.cat([torch.ones(n_aux, device=cuda_dev), wts])).sum().backward()
        torch.cuda.synchronize()
        return seen, [y1.features.detach(), y2.features.detach(), x.features.grad, x2.features.grad,
                      conv.weight.grad, conv.bias.grad]

    seen_odd, got = run(7)
    seen_even, want = run(8)
    assert all(s != 0 for s in seen_odd), f"autograd delivered aligned gradients: {seen_odd}"
    assert all(s == 0 for s in seen_even), seen_even
    _same(got, want, "gradients delivered 14 bytes off")


def _flat_params(net, prefix):
    """move every parameter into one flat buffer behind `prefix` elements (vector_to_parameters)"""
    params = list(net.mods.parameters())
    vec = torch.nn.utils.parameters_to_vector(params)
    buf = torch.cat([torch.zeros(prefix, dtype=vec.dtype, device=vec.device), vec])
    torch.nn.utils.vector_to_parameters(buf[prefix:], params)
    return params


@gpu
@pytest.mark.parametrize("name", ["unet", "encoder"])
def test_misaligned_weights_from_a_flat_buffer(name, cuda_dev):
    """A U-Net and an encoder whose parameters live in one flat buffer behind a 3-element parameter: every conv
    weight sits 6 bytes off a 16-byte boundary.  Forward and backward equal the aligned model bit for bit, eagerly
    and replayed through graph_capture on padded inputs with output bounds."""
    import spconv_b200.pytorch as spconv
    from tests.test_networks_gpu import BATCH, SHAPE, _pad_rows, _Seq, clouds, flat, inputs, make_g, run, setup
    _auto_unless_tc(False)          # the U-Net ends in a 5-channel layer
    cl = clouds(cuda_dev)
    nets = []
    for moved in (False, True):
        net, c_in = setup(name, "MaskImplicitGemm", "f16", True, cuda_dev, seed=1)
        if moved:
            _flat_params(net, 3)
            convs = [m for m in net.mods.modules() if isinstance(m, spconv.SparseConvolution)]
            assert convs and all(m.weight.data_ptr() % 16 for m in convs), "a conv weight is still aligned"
        nets.append(net)
    rows = _pad_rows(cl)
    for net in nets:
        spconv.set_output_bounds(_Seq(net), inputs(net, c_in, cl[1], "f16", cuda_dev), margin=1.3)
    xs = [inputs(nets[0], c_in, c, "f16", cuda_dev, rows, seed=k) for k, c in enumerate(cl)]
    probe = run(nets[0], xs[0], 0.0)
    Gs = [make_g(probe["y"][nets[0].steps[-1][0]], 100 + k) for k in range(3)]
    probe = None
    results = []
    for net in nets:
        eager = []
        for k in range(3):
            x = xs[k].replace_feature(xs[k].features.detach().clone().requires_grad_(True))
            eager.append([t.detach().clone() for t in flat(net, run(net, x, Gs[k]))])

        def step(f, i, nv, g, net=net):
            x = spconv.SparseConvTensor(f.detach().requires_grad_(True), i, SHAPE, BATCH)
            x.num_valid = nv
            return flat(net, run(net, x, g))
        args = [(x.features.detach(), x.indices, x.num_valid, g) for x, g in zip(xs, Gs)]
        graphed = spconv.graph_capture(step, *args[0])
        replay = [[t.clone() for t in graphed(*args[k])] for k in (0, 1, 2)]
        results.append((eager, replay))
    (e0, r0), (e1, r1) = results
    for k in range(3):
        _same(e1[k], e0[k], f"{name}: eager step on cloud {k}")
        _same(r1[k], e0[k], f"{name}: flat-buffer replay of cloud {k}")
        _same(r0[k], e0[k], f"{name}: aligned replay of cloud {k}")


# ============================================================================ coverage of the C ABI
# (entry point, pointer parameter) -> the test above that moves it
_GEMM, _INT8, _MOD = ("test_gemm_c_abi_operands_at_every_offset", "test_int8_operands_at_every_offset",
                      "test_public_api_operands_at_every_offset")
_GUARD, _RB = "test_guarded_kernels_agree_on_both_paths", "test_rulebook_indices_at_every_offset"
SWEPT = {
    ("spx_implicit_gemm_fwd", "features"): _GEMM, ("spx_implicit_gemm_fwd", "filters"): _GEMM,
    ("spx_implicit_gemm_fwd", "bias"): _GEMM, ("spx_implicit_gemm_dgrad", "out_bp"): _GEMM,
    ("spx_implicit_gemm_dgrad", "filters"): _GEMM, ("spx_implicit_gemm_wgrad", "features"): _GEMM,
    ("spx_implicit_gemm_wgrad", "out_bp"): _GEMM,
    ("spx_implicit_gemm_fwd_int8", "features"): _INT8, ("spx_implicit_gemm_fwd_int8", "filters"): _INT8,
    ("spx_implicit_gemm_fwd_int8", "scale"): _INT8, ("spx_implicit_gemm_fwd_int8", "bias"): _INT8,
    ("spx_implicit_gemm_fwd_int8", "output_add"): _INT8,
    ("spx_indice_pool_fwd", "features"): _MOD, ("spx_indice_pool_bwd", "features"): _MOD,
    ("spx_indice_pool_bwd", "out_bp"): _MOD,
    ("spx_depthwise_fwd", "features"): _MOD, ("spx_depthwise_fwd", "weight"): _MOD, ("spx_depthwise_fwd", "bias"): _MOD,
    ("spx_depthwise_dgrad", "out_bp"): _MOD, ("spx_depthwise_dgrad", "weight"): _MOD,
    ("spx_depthwise_wgrad", "features"): _MOD, ("spx_depthwise_wgrad", "out_bp"): _MOD,
    ("spx_global_pool_fwd", "features"): _GUARD, ("spx_global_pool_bwd", "dy"): _GUARD,
    ("spx_masked_bn_fwd_train", "x"): _GUARD, ("spx_masked_bn_bwd", "x"): _GUARD, ("spx_masked_bn_bwd", "dy"): _GUARD,
    ("spx_sparse_add_gather", "src"): _GUARD,
    ("spx_point_scatter_group", "ids"): _GUARD, ("spx_point_scatter_fwd", "x"): _GUARD,
    ("spx_point_scatter_bwd", "dy"): _GUARD,
    ("spx_point2voxel_stage1", "points"): "test_point_to_voxel_and_hash_table_operands_at_every_offset",
    ("spx_point2voxel_stage2", "points"): "test_point_to_voxel_and_hash_table_operands_at_every_offset",
    ("spx_point2voxel_bounded", "points"): "test_point_to_voxel_and_hash_table_operands_at_every_offset",
    **{(f, "indices"): _RB for f in ("spx_subm_rulebook", "spx_conv_rulebook_stage1", "spx_conv_rulebook_stage2",
                                     "spx_subm_rulebook_all", "spx_conv_rulebook_stage2_all",
                                     "spx_conv_rulebook_bounded_all")},
    **{("spx_hash_" + f, p): "test_point_to_voxel_and_hash_table_operands_at_every_offset"
       for f, ps in (("insert", ("keys", "values")), ("query", ("keys",)), ("insert_exist", ("keys", "values")))
       for p in ps},
}
LIBRARY_OUTPUT = "output allocated by the library"
EXPLAINED = {
    "workspace": "workspace, allocated by the library",
    ("spx_implicit_gemm_fwd", "out"): LIBRARY_OUTPUT,
    ("spx_implicit_gemm_fwd_int8", "out"): LIBRARY_OUTPUT,
    ("spx_implicit_gemm_dgrad", "din"): LIBRARY_OUTPUT,
    ("spx_implicit_gemm_wgrad", "dfilters"): "written element by element (wgrad_reduce_kernel, the FMA kernel)",
    ("spx_implicit_gemm_wgrad_push", "features"): "the data-parallel twin of spx_implicit_gemm_wgrad: same predicate",
    ("spx_implicit_gemm_wgrad_push", "out_bp"): "the data-parallel twin of spx_implicit_gemm_wgrad: same predicate",
    ("spx_implicit_gemm_wgrad_push", "dfilters"): "written element by element (peer_finish_kernel)",
    ("spx_indice_pool_fwd", "out"): LIBRARY_OUTPUT,
    ("spx_indice_pool_bwd", "din"): LIBRARY_OUTPUT,
    ("spx_indice_pool_bwd", "out_features"): "the forward's output, allocated by the library",
    ("spx_sparse_add_fwd", "out"): LIBRARY_OUTPUT,
    ("spx_zero_rows_from_count", "ptr"): "16-byte stores only when aligned, 2-byte stores otherwise",
    ("spx_peer_buffer_create", "buffer"): "out-parameter: a peer buffer handle, not tensor data",
    ("spx_peer_buffer_open", "mapped"): "out-parameter: a peer buffer handle, not tensor data",
    ("spx_peer_buffer_close", "mapped"): "a peer buffer handle, not tensor data",
    ("spx_peer_buffer_destroy", "buffer"): "a peer buffer handle, not tensor data",
    ("spx_peer_push", "data"): "read element by element (peer_push_kernel)",
    ("spx_peer_finish", "out"): "written element by element (peer_finish_kernel)",
    ("spx_peer_allreduce", "data"): "read and written element by element (peer_push_kernel, peer_finish_kernel)",
    ("spx_bias_act_inplace", "x"): "read and written element by element (bias_act_kernel)",
    ("spx_bias_act_inplace", "bias"): "read element by element (bias_act_kernel)",
    ("spx_global_pool_fwd", "out"): LIBRARY_OUTPUT,
    ("spx_global_pool_bwd", "din"): LIBRARY_OUTPUT,
    ("spx_sparse_add_union", "indices"): "its callers pass a library-made torch.cat of the operands' indices; "
                                         "refused when misaligned like the other rulebooks",
    ("spx_masked_sparse_add_plan", "indices"): "read element by element (sa_pack_kernel) into a library buffer",
    ("spx_point_scatter_fwd", "out"): LIBRARY_OUTPUT,
    ("spx_point_scatter_bwd", "dx"): LIBRARY_OUTPUT,
    ("spx_depthwise_fwd", "out"): LIBRARY_OUTPUT,
    ("spx_depthwise_dgrad", "din"): LIBRARY_OUTPUT,
    ("spx_depthwise_wgrad", "dweight"): LIBRARY_OUTPUT,
    ("spx_masked_bn_fwd_train", "y"): LIBRARY_OUTPUT,
    ("spx_masked_bn_fwd_train", "weight"): "a per-channel vector read element by element",
    ("spx_masked_bn_fwd_train", "bias"): "a per-channel vector read element by element",
    ("spx_masked_bn_bwd", "weight"): "a per-channel vector read element by element",
    ("spx_masked_bn_fwd_train", "running_mean"): "a per-channel vector read and written element by element",
    ("spx_masked_bn_fwd_train", "running_var"): "a per-channel vector read and written element by element",
    ("spx_masked_bn_bwd", "dx"): LIBRARY_OUTPUT,
    ("spx_masked_bn_bwd", "dweight"): LIBRARY_OUTPUT,
    ("spx_masked_bn_bwd", "dbias"): LIBRARY_OUTPUT,
    **{("spx_hash_" + f, p): "the table's own storage, allocated by HashTable"
       for f in ("clear", "insert", "query", "insert_exist", "rank") for p in ("table_keys", "table_values")},
    ("spx_hash_query", "values"): LIBRARY_OUTPUT,
    ("spx_hash_rank", "out_keys"): LIBRARY_OUTPUT,
    ("spx_hash_rank", "out_values"): LIBRARY_OUTPUT,
    ("spx_hash_rank", "count"): LIBRARY_OUTPUT,
    **{(f, p): "a host array of the grid geometry, not device data"
       for f in ("spx_point2voxel_stage1", "spx_point2voxel_stage2", "spx_point2voxel_bounded")
       for p in ("vsize_host", "coors_range_host")},
    ("spx_point2voxel_stage2", "voxels"): LIBRARY_OUTPUT,
    ("spx_point2voxel_bounded", "voxels"): LIBRARY_OUTPUT,
    ("spx_masked_bn_fwd_train", "save_mean"): LIBRARY_OUTPUT,
    ("spx_masked_bn_fwd_train", "save_invstd"): LIBRARY_OUTPUT,
    ("spx_masked_bn_bwd", "save_mean"): "per-channel statistics the forward saved, allocated by the library",
    ("spx_masked_bn_bwd", "save_invstd"): "per-channel statistics the forward saved, allocated by the library",
    ("spx_debug_configure", "trace_buf"): "test switch, not tensor data",
}


def _header_pointer_params():
    s = open(os.path.join(ROOT, "include", "spconv_b200.h")).read()
    s = re.sub(r"/\*.*?\*/", "", s, flags=re.S)
    out = []
    for m in re.finditer(r"\bint\s+(spx_\w+)\s*\(([^;]*?)\)\s*;", s, re.S):
        for p in (q.strip() for q in m.group(2).replace("\n", " ").split(",")):
            if re.match(r"(const\s+)?(void|int8_t|float)\s*\*", p) or re.match(r"const\s+int32_t\s*\*\s*indices$", p):
                out.append((m.group(1), p.split("*")[-1].strip()))
    return out


def test_every_pointer_of_the_c_abi_is_swept_or_explained():
    """needs no GPU: every pointer parameter of include/spconv_b200.h (untyped, int8 / float data, rulebook indices)
    is moved by a named test of this file or explained; every swept entry names a test that exists"""
    found = _header_pointer_params()
    assert len(found) > 100 and ("spx_implicit_gemm_fwd_int8", "features") in found
    missing = [(f, p) for f, p in found if (f, p) not in SWEPT and (f, p) not in EXPLAINED and p != "workspace"]
    assert not missing, f"pointer parameters neither swept nor explained: {missing}"
    for (f, p), test in SWEPT.items():
        assert (f, p) in found, f"{f}({p}): not a pointer parameter of the header"
        assert callable(globals().get(test)), f"{f}({p}): no test {test}"
    stale = [k for k in EXPLAINED if k != "workspace" and (k in SWEPT or k not in found)]
    assert not stale, f"explanations of swept or unknown parameters: {stale}"
