"""The tensor-core forward / input-gradient epilogue, bit for bit.

After a tile's last offset the consumer warps add the bias (or apply the int8 scale and bias), apply
the activation, convert and store their rows.  The destination rows come from the argsort row of the
tile's index block, and bias and scales from shared memory.  These tests pin what that must not change:

* every output type (f16, bf16, f32, int8 with and without output_add) and N = 16 ... 256;
* row counts that leave a partial last tile, destinations of -1 (padding rows of bounded
  rulebooks: never written) and the identity order (no argsort);
* the same call with y as a view that is not 16-byte aligned, which runs on the FMA kernels, must
  equal the aligned call bit for bit.

Inputs are small integers times a power of two, so every partial sum is exact in fp32 whatever the
order, and each output must be the float64 result rounded once (as in test_bench_workloads_gpu.py).
Outputs are pre-filled with NaN, so a row that is never written cannot pass.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_bench_workloads_gpu import _assert_exact
from tests.test_conv_tc_coverage_gpu import ENV_FAMILY, SIMT, _conv, _configure, _lib, _reference

pytestmark = pytest.mark.gpu

SCALE = 0.125
TDT = {"f16": torch.float16, "bf16": torch.bfloat16, "tf32": torch.float32}
CODE = {"f16": 1, "bf16": 2, "f32": 0, "i8": 3}


@pytest.fixture(autouse=True)
def _restore_forced_family():
    yield
    if torch.cuda.is_available():
        _configure(ENV_FAMILY)


def _grid(gen, shape, dev, lo=-2, hi=2, scale=SCALE):
    return torch.randint(lo, hi + 1, shape, generator=gen, device=dev).float() * scale


def _unaligned(shape, dtype, dev):
    """a NaN-filled view one element past a 16-byte boundary"""
    flat = torch.full((int(np.prod(shape)) + 16,), float("nan") if dtype.is_floating_point else 0, dtype=dtype,
                      device=dev)
    v = flat[1:1 + int(np.prod(shape))].view(shape)
    assert v.data_ptr() % 16
    return v


def _table(conv, order):
    """(pair, mask, argsort, rows) of the forward table: as built, as the identity order, or with every
    seventh destination replaced by -1 (a padding row)"""
    pair, mask, argsort, rows = conv.fwd
    if order == "identity":
        return pair, None, None, rows
    if order == "padded":
        argsort = argsort.clone()
        argsort[::7] = -1
    return pair, mask, argsort, rows


def _desc(conv, dtype, C, K, table, reverse=False):
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    pair, mask, argsort, rows = table
    tiles = ops._tile_tables(pair, mask, argsort, rows, conv.kv)
    d = ops._desc(dtype, conv.kv, C, K, conv.n_in, conv.n_out, pair, mask, argsort, reverse=reverse, tiles=tiles)
    d.f32_mode = _cabi.SPX_F32_TF32
    return d, tiles


def _run(out, fn, family):
    """fn(out) on the expected kernel family (2 tensor cores, 1 FMA kernels)"""
    _configure(1 if SIMT else 0)
    fn(out)
    torch.cuda.synchronize()
    got = _lib().spx_last_kernel_family()
    assert got == (1 if SIMT else family), f"kernel family {got}, expected {family}"
    return out


def _fwd(conv, d, x, w, bias, out):
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    _cabi.check(_lib().spx_implicit_gemm_fwd(ctypes.byref(d), x.data_ptr(), w.data_ptr(), out.data_ptr(),
                                             bias.data_ptr(), _cabi.SPX_ACT_RELU, 0.0, ops._stream()),
                "implicit_gemm_fwd")


def _dgrad(conv, d, dout, w, din):
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    _cabi.check(_lib().spx_implicit_gemm_dgrad(ctypes.byref(d), dout.data_ptr(), w.data_ptr(), din.data_ptr(),
                                               ops._stream()), "implicit_gemm_dgrad")


# (dtype, C, K): forward N = K, input gradient N = C
FLOAT_CASES = [("f16", 64, 64), ("f16", 16, 32), ("f16", 32, 256), ("f16", 256, 16),
               ("bf16", 64, 128), ("bf16", 128, 128), ("tf32", 32, 16), ("tf32", 32, 128)]


@pytest.mark.parametrize("case", FLOAT_CASES, ids=lambda c: f"{c[0]}-C{c[1]}K{c[2]}")
def test_float_epilogue_exact(case, oracle, cuda_dev):
    dt, C, K = case
    tdt = TDT[dt]
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    assert conv.n_out % 128, "the cloud must leave a partial last tile"
    gen = torch.Generator(device=cuda_dev).manual_seed(C * 1000 + K)
    x = _grid(gen, (conv.n_in, C), cuda_dev)
    w = _grid(gen, (K, conv.kv, C), cuda_dev)
    dout = _grid(gen, (conv.n_out, K), cuda_dev)
    bias = _grid(gen, (K,), cuda_dev, scale=SCALE * SCALE)
    r = _reference(x, w, dout, conv.ref_pair, cuda_dev)
    ref_out = torch.relu(r["out"] + bias.double())
    q = SCALE * SCALE
    xd, wd, dd, bd = x.to(tdt), w.to(tdt), dout.to(tdt), bias.to(tdt)

    for order in ("sorted", "identity", "padded"):
        d, tiles = _desc(conv, tdt, C, K, _table(conv, order))
        nan = torch.full((conv.n_out, K), float("nan"), dtype=tdt, device=cuda_dev)
        out = _run(nan.clone(), lambda o: _fwd(conv, d, xd, wd, bd, o), 2)
        if order == "padded":
            # destinations of -1 are never written; every other row is exact
            skipped = _table(conv, order)[2] < 0
            dropped = conv.fwd[2][skipped].long()
            keep = torch.ones(conv.n_out, dtype=torch.bool, device=cuda_dev)
            keep[dropped] = False
            assert torch.isnan(out[dropped].float()).all(), "a padding row was written"
            _assert_exact(f"fwd {order}", out[keep], ref_out[keep], r["out_abs"][keep], q, tdt)
        else:
            _assert_exact(f"fwd {order}", out, ref_out, r["out_abs"], q, tdt)
        if order == "sorted":
            un = _run(_unaligned((conv.n_out, K), tdt, cuda_dev), lambda o: _fwd(conv, d, xd, wd, bd, o), 1)
            assert torch.equal(un, out), "fwd: unaligned y differs from the aligned call"

    d, _ = _desc(conv, tdt, C, K, conv.fwd, reverse=True)
    din = _run(torch.full((conv.n_in, C), float("nan"), dtype=tdt, device=cuda_dev),
               lambda o: _dgrad(conv, d, dd, wd, o), 2)
    _assert_exact("dgrad", din, r["din"], r["din_abs"], q, tdt)
    un = _run(_unaligned((conv.n_in, C), tdt, cuda_dev), lambda o: _dgrad(conv, d, dd, wd, o), 1)
    assert torch.equal(un, din), "dgrad: unaligned y differs from the aligned call"


INT8_CASES = [(32, 32), (64, 64), (64, 128), (128, 256)]
OUT_I8 = {"i8": torch.int8, "f32": torch.float32, "f16": torch.float16}


def _int8_fwd(d, x, w, out, out_dt, scale, bias, add, add_scale):
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    _cabi.check(_lib().spx_implicit_gemm_fwd_int8(
        ctypes.byref(d), x.data_ptr(), w.data_ptr(), out.data_ptr(), CODE[out_dt],
        scale.data_ptr(), bias.data_ptr(), None if add is None else add.data_ptr(), add_scale, _cabi.SPX_ACT_RELU,
        0.0, ops._stream()), "implicit_gemm_fwd_int8")


@pytest.mark.parametrize("case", INT8_CASES, ids=lambda c: f"C{c[0]}K{c[1]}")
@pytest.mark.parametrize("out_dt", sorted(OUT_I8))
@pytest.mark.parametrize("with_add", [False, True], ids=["plain", "add"])
def test_int8_epilogue_exact(case, out_dt, with_add, oracle, cuda_dev):
    C, K = case
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    gen = torch.Generator(device=cuda_dev).manual_seed(C * 7 + K)
    x = torch.randint(-4, 5, (conv.n_in, C), generator=gen, device=cuda_dev)
    w = torch.randint(-4, 5, (K, conv.kv, C), generator=gen, device=cuda_dev)
    scale = torch.randint(1, 3, (K,), generator=gen, device=cuda_dev).float() * 2.0 ** -8
    bias = _grid(gen, (K,), cuda_dev)
    add = torch.randint(-8, 9, (conv.n_out, K), generator=gen, device=cuda_dev) if with_add else None
    # float64 reference: integer sums, then the fp32 epilogue's steps, each exact on these values
    pair = torch.from_numpy(conv.ref_pair).to(cuda_dev).long()
    acc = torch.zeros((conv.n_out, K), dtype=torch.float64, device=cuda_dev)
    for k in range(conv.kv):
        o = (pair[k] >= 0).nonzero().squeeze(1)
        acc[o] += x[pair[k, o]].double() @ w[:, k].double().T
    y = acc * scale.double() + bias.double()
    if with_add:
        y = y + add.double() * 0.5
    y = torch.relu(y)
    odt = OUT_I8[out_dt]
    want = y.round().clamp(-128, 127).to(torch.int8) if out_dt == "i8" else y.to(odt)

    from spconv_b200.pytorch import ops
    tiles = ops._tile_tables(*conv.fwd[:3], conv.fwd[3], conv.kv)      # kept alive: d holds raw pointers
    d = ops._desc(torch.int8, conv.kv, C, K, conv.n_in, conv.n_out, *conv.fwd[:3], tiles=tiles)
    x8, w8 = x.to(torch.int8), w.to(torch.int8)
    a8 = add.to(torch.int8) if with_add else None
    fill = (lambda: torch.full((conv.n_out, K), 77, dtype=torch.int8, device=cuda_dev)) if out_dt == "i8" else \
        (lambda: torch.full((conv.n_out, K), float("nan"), dtype=odt, device=cuda_dev))
    out = _run(fill(), lambda o: _int8_fwd(d, x8, w8, o, out_dt, scale, bias, a8, 0.5), 2)
    assert torch.equal(out, want), f"int8 -> {out_dt}: {int((out != want).sum())} elements differ"
    un = _unaligned((conv.n_out, K), odt, cuda_dev)
    un = _run(un, lambda o: _int8_fwd(d, x8, w8, o, out_dt, scale, bias, a8, 0.5), 1)
    assert torch.equal(un, out), f"int8 -> {out_dt}: unaligned y differs from the aligned call"
