"""The FMA conv kernels (gemm_simt.cu) and the mask-word edges of both kernel families against a float64
reference.

The FMA kernels run every fp32 layer by default (exact fp32 unless SPCONV_ALLOW_TF32=1) and every shape
the tensor cores do not tile.  They tile rows by 32 (S_TM), the contraction by 32 (S_TK) and output
channels by 64 (S_TN); the weight gradient uses 16 x 16 channel tiles over 64-row chunks (WG_T,
WG_ROWS).  The cases below put C, K and the row count on each side of those edges, forced onto the FMA
kernels in-process, including shapes that by default only run on the tensor cores.

Kernel volumes 31 .. 128 put the last mask bit on each side of the 32-bit word boundaries (the
rulebook's multi-word masks and sort, the tile-mask OR of both families); kv = 128 sets bit 31 of word 3.

Every output element is checked with the bound of test_conv_tc_coverage_gpu.py, outputs pre-filled
with NaN.  Calls on the tensor cores run with them forced, calls the shape sends to the FMA kernels
must be refused when the tensor cores are forced; with SPX_FORCE_SIMT=1 or SPX_FORCE_TC=1 in the
environment those calls behave as in the coverage file.  Calls pinned to the FMA kernels here run there
whatever the environment.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_conv_tc_coverage_gpu import (TORCH_DT, Conv, _check, _configure, _conv, _exact, _launch, _lib, _nan,
                                             _reference, _run_case, gemm_instance, wgrad_instance)
from tests.test_conv_tc_coverage_gpu import _restore_forced_family  # noqa: F401  (autouse fixture)
from tests.util import random_cloud

gpu = pytest.mark.gpu

F32 = "tf32"    # the coverage helpers' name for fp32 operands; with the FMA kernels pinned they stay fp32

# (dtype, C, K): C in {1, 31, 32, 33, 65, 100}, K in {1, 15, 17, 63, 64, 65, 129, 200}; each value once at
# least, as C and as K (the input gradient contracts over K and writes C).  The last four are shapes the
# tensor cores serve by default.
CHANNELS = [(F32, 1, 17), ("f16", 31, 1), ("bf16", 32, 65), (F32, 33, 63), ("f16", 65, 129), ("bf16", 100, 15),
            (F32, 33, 200), ("f16", 100, 64),
            ("f16", 32, 64), ("bf16", 64, 32), (F32, 32, 64), ("f16", 16, 128)]
TC_SHAPED = CHANNELS[-4:]
# rows: forward / input gradient tiles of 32 rows, weight-gradient chunks of 64 rows
ROW_M = [1, 31, 32, 33, 63, 64, 65, 129]
KV_1D = [31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128]
KV_TC = ("f16", 16, 32)         # the tensor cores serve fwd / dgrad at every kv, wgrad up to its smem limit
KV_FMA = (F32, 20, 24)          # never tiled by the tensor cores


def _kv_cases():
    out = []
    for kv in KV_1D:
        for mode in (["subm"] if kv % 2 else []) + ["conv"]:
            out += [(kv, mode, "tc"), (kv, mode, "fma")]
    return out + [(65, "subm", "fma-forced"), (128, "conv", "fma-forced")]


def _block_rows(oracle, dev, m):
    """SubM 3x3x3 on the first m rows of a dense 8 x 8 x 8 block (as test_partial_tiles)"""
    g = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3)[:m]
    inds = np.concatenate([np.zeros((m, 1), np.int32), g.astype(np.int32)], 1)
    return Conv(oracle, dev, inds, 1, [8, 8, 8], 3, 1, 0, 1, True)


def _conv_1d(oracle, dev, kv, mode):
    """1-D conv of kernel size kv on 1200 points of a 3000-cell line: SubM, or stride 2 with padding kv / 2"""
    _, inds = random_cloud(np.random.default_rng(1000 + kv), [3000], [1200], 1)
    if mode == "subm":
        return Conv(oracle, dev, inds, 1, [3000], kv, 1, 0, 1, True)
    return Conv(oracle, dev, inds, 1, [3000], kv, 2, kv // 2, 1, False)


# ------------------------------------------------------------------ channel and row edges
@gpu
@pytest.mark.parametrize("mode", ["subm", "conv"])
@pytest.mark.parametrize("case", CHANNELS, ids=lambda c: f"{c[0]}-C{c[1]}K{c[2]}")
def test_channel_edges_on_fma(case, mode, oracle, cuda_dev):
    dt, C, K = case
    _run_case(oracle, cuda_dev, _conv(oracle, cuda_dev, "k3", mode), dt, C, K, seed=C * 1000 + K, fma=True)


def test_channel_cases_cover_every_edge():
    """No GPU needed: every C / K edge value occurs, and the tensor-core-shaped cases are served there by
    default, so that pinning them to the FMA kernels checks a route they otherwise never take."""
    assert {c for _, c, _ in CHANNELS} >= {1, 31, 32, 33, 65, 100}
    assert {k for _, _, k in CHANNELS} >= {1, 15, 17, 63, 64, 65, 129, 200}
    for dt, C, K in TC_SHAPED:
        assert gemm_instance(dt, 27, C, K) is not None and gemm_instance(dt, 27, C, K, dgrad=True) is not None
        assert wgrad_instance(dt, 27, C, K) is not None
    assert {dt for dt, _, _ in CHANNELS} == {"f16", "bf16", F32}


@gpu
@pytest.mark.parametrize("m", ROW_M)
def test_row_edges_on_fma(m, oracle, cuda_dev):
    """M rows in the forward / input gradient (32-row tiles) and in the weight gradient (64-row chunks)"""
    conv = _block_rows(oracle, cuda_dev, m)
    assert conv.n_in == conv.n_out == m
    _run_case(oracle, cuda_dev, conv, F32, 33, 65, seed=m, fma=True)


# ------------------------------------------------------------------ exact fp32
@gpu
@pytest.mark.parametrize("mode", ["subm", "conv"])
def test_exact_fp32_public_path(mode, oracle, cuda_dev, monkeypatch):
    """fp32 inputs with all 24 mantissa bits through ops.implicit_gemm / implicit_gemm_backward with tf32
    not allowed: the fp32 bound with no output rounding and no tf32 slack.  The shape is one the tensor
    cores serve when tf32 is allowed, so only the exact mode keeps it on the FMA kernels."""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", False)
    assert ops._f32_mode() == _cabi.SPX_F32_EXACT
    C = K = 32
    assert gemm_instance(F32, 3, C, K) and gemm_instance(F32, 3, C, K, dgrad=True) and wgrad_instance(F32, 3, C, K)
    rng = np.random.default_rng(5)
    _, inds = random_cloud(rng, [600], [150], 1)
    subm = mode == "subm"
    conv = Conv(oracle, cuda_dev, inds, 1, [600], 3, 1 if subm else 2, 0 if subm else 1, 1, subm)
    x = _exact(rng, (conv.n_in, C), F32, round_tf32=False)
    w = _exact(rng, (K, conv.kv, C), F32, round_tf32=False)
    dout = _exact(rng, (conv.n_out, K), F32, round_tf32=False)
    assert ((x.view(torch.int32) & 0x1FFF) != 0).float().mean() > 0.99    # bits tf32 would drop
    r = _reference(x, w, dout, conv.ref_pair, cuda_dev)
    # A tf32 route truncates every operand to 11 mantissa bits: each product is off by ~2^-11 of itself,
    # so a sum of T terms is off by ~2^-11 sqrt(sum term^2) >= 2^-11 sum|terms| / sqrt(T).  The fp32 bound
    # (T + 1) 2^-23 sum|terms| lies below that for every element here, so a tf32 route fails it.
    terms = {"out": r["t_out"][:, None] * C, "din": r["t_in"][:, None] * K, "dw": r["t_k"][None, :, None]}
    for name, t in terms.items():
        a = r[name + "_abs"]
        t = t.expand_as(a)
        live = (t > 0) & (a > 0)
        bound = (t + 1) * 2.0 ** -23 * a
        assert (bound < 2.0 ** -11 * a / t.clamp_min(1).sqrt())[live].all(), name
    xd, wd, dd = (v.to(cuda_dev) for v in (x, w, dout))
    pf, mf, sf, _ = conv.fwd
    pb, mb, sb, _ = conv.bwd if conv.bwd is not None else (pf, None, None, None)
    runs = []
    for family in (0, 1):        # the default auto dispatch, then the FMA kernels pinned
        _configure(family)
        out, _, _ = ops.implicit_gemm(xd, wd, pf, [mf], [sf], conv.n_out, [], False, subm)
        fam_fwd = _lib().spx_last_kernel_family()
        din, dw = ops.implicit_gemm_backward(xd, wd, dd, pf, pb, [mf], [] if subm else [mb], [sf],
                                             [] if subm else [sb], None, [], 128, subm)
        fam_bwd = _lib().spx_last_kernel_family()
        torch.cuda.synchronize()
        # the bound before the family: it fails by itself when fp32 runs as tf32
        _check("out", out, r["out"], r["out_abs"], terms["out"], F32, zero=r["t_out"] == 0)
        _check("din", din, r["din"], r["din_abs"], terms["din"], F32, zero=r["t_in"] == 0)
        _check("dw", dw, r["dw"], r["dw_abs"], terms["dw"], F32)
        assert fam_fwd == fam_bwd == 1, f"fp32 ran on kernel families {fam_fwd} / {fam_bwd}, not the FMA kernels"
        runs.append((out, din, dw))
    for name, a, b in zip(("out", "din", "dw"), *runs):
        assert torch.equal(a, b), f"{name}: auto dispatch and pinned FMA kernels differ"


# ------------------------------------------------------------------ kernel volumes on mask-word boundaries
@gpu
@pytest.mark.parametrize("case", _kv_cases(), ids=lambda c: f"kv{c[0]}-{c[1]}-{c[2]}")
def test_kernel_volume_word_edges(case, oracle, cuda_dev):
    """1-D kernels of 31 .. 128 offsets; the rulebook (multi-word masks, their sort, the tile tables) is
    checked bit for bit against the oracle by Conv, every GEMM against the float64 reference.  'tc' runs
    each call where gemm_instance / wgrad_instance put it."""
    kv, mode, fam = case
    conv = _conv_1d(oracle, cuda_dev, kv, mode)
    assert conv.kv == kv
    dt, C, K = KV_FMA if fam == "fma" else KV_TC
    _run_case(oracle, cuda_dev, conv, dt, C, K, seed=kv, fma=fam == "fma-forced")


@gpu
@pytest.mark.parametrize("fam", ["tc", "fma-forced"])
def test_kernel_volume_128_3d(fam, oracle, cuda_dev):
    """[4, 4, 8] stride 2: 128 offsets, the last one bit 31 of mask word 3"""
    _, inds = random_cloud(np.random.default_rng(128), [19, 18, 17], [1500, 1500], 1)
    conv = Conv(oracle, cuda_dev, inds, 2, [19, 18, 17], [4, 4, 8], 2, [1, 1, 3], 1, False)
    assert conv.kv == 128
    dt, C, K = KV_TC
    _run_case(oracle, cuda_dev, conv, dt, C, K, seed=3, fma=fam == "fma-forced")


@gpu
@pytest.mark.parametrize("kv", [32, 33, 64, 65, 96, 97, 128])
def test_fma_without_row_masks(kv, oracle, cuda_dev):
    """A descriptor with no row masks, argsort or tile tables (all optional in the C ABI) visits every
    offset in natural row order: the FMA kernel builds its tile mask from kv alone, full words below
    bit kv and a partial last word.  The tensor cores need the tile tables, so they refuse it."""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    conv = _conv_1d(oracle, cuda_dev, kv, "conv")
    C, K = 33, 17
    rng = np.random.default_rng(kv)
    x, w, dout = (_exact(rng, s, F32) for s in ((conv.n_in, C), (K, kv, C), (conv.n_out, K)))
    r = _reference(x, w, dout, conv.ref_pair, cuda_dev)
    xd, wd, dd = (v.to(cuda_dev) for v in (x, w, dout))
    d_fwd = ops._desc(torch.float32, kv, C, K, conv.n_in, conv.n_out, conv.fwd[0], None, None)
    d_bwd = ops._desc(torch.float32, kv, C, K, conv.n_in, conv.n_out, conv.bwd[0], None, None)

    def fwd():
        out = _nan((conv.n_out, K), torch.float32, cuda_dev)
        _cabi.check(_lib().spx_implicit_gemm_fwd(ctypes.byref(d_fwd), xd.data_ptr(), wd.data_ptr(), out.data_ptr(),
                                                 None, 0, 0.0, ops._stream()), "implicit_gemm_fwd")
        return out

    def dgrad():
        din = _nan((conv.n_in, C), torch.float32, cuda_dev)
        _cabi.check(_lib().spx_implicit_gemm_dgrad(ctypes.byref(d_bwd), dd.data_ptr(), wd.data_ptr(), din.data_ptr(),
                                                   ops._stream()), "implicit_gemm_dgrad")
        return din
    out, din = _launch("fwd", None, fwd), _launch("dgrad", None, dgrad)
    _check("out", out, r["out"], r["out_abs"], r["t_out"][:, None] * C, F32, zero=r["t_out"] == 0)
    _check("din", din, r["din"], r["din_abs"], r["t_in"][:, None] * K, F32, zero=r["t_in"] == 0)


def test_kv_cases_reach_both_families():
    """No GPU needed: at the word edges the 'tc' cases run fwd and dgrad on the tensor cores, and at
    least one weight gradient on each family"""
    dt, C, K = KV_TC
    for kv in KV_1D:
        assert gemm_instance(dt, kv, C, K) is not None and gemm_instance(dt, kv, C, K, dgrad=True) is not None
    wg = {wgrad_instance(dt, kv, C, K) is not None for kv in KV_1D}
    assert wg == {True, False}
    dt, C, K = KV_FMA
    for kv in KV_1D:
        assert gemm_instance(dt, kv, C, K) is None and gemm_instance(dt, kv, C, K, dgrad=True) is None
        assert wgrad_instance(dt, kv, C, K) is None


# ------------------------------------------------------------------ other FMA routes
@gpu
@pytest.mark.parametrize("case", [(F32, 33, 65), ("bf16", 64, 32)], ids=lambda c: f"{c[0]}-C{c[1]}K{c[2]}")
def test_inverse_conv_on_fma(case, oracle, cuda_dev):
    dt, C, K = case
    _run_case(oracle, cuda_dev, _conv(oracle, cuda_dev, "k3", "inverse"), dt, C, K, seed=11, fma=True)


@gpu
@pytest.mark.parametrize("act", ["relu", "leaky_relu", "sigmoid"])
@pytest.mark.parametrize("case", [(F32, 33, 65), ("bf16", 32, 64)], ids=lambda c: f"{c[0]}-C{c[1]}K{c[2]}")
def test_bias_activation_epilogue_on_fma(case, act, oracle, cuda_dev):
    from spconv_b200.core import Activation
    dt, C, K = case
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    rng = np.random.default_rng(22)
    x, w = _exact(rng, (conv.n_in, C), dt), _exact(rng, (K, 27, C), dt)
    bias = _exact(rng, (K,), dt, scale=2.0)
    alpha = 0.25
    code = {"relu": Activation.ReLU, "leaky_relu": Activation.LeakyReLU, "sigmoid": Activation.Sigmoid}[act].value
    tdt = TORCH_DT[dt]
    got = conv.fwd_call(x.to(cuda_dev, tdt), w.to(cuda_dev, tdt), None, bias=bias.to(cuda_dev, tdt), act=code,
                        alpha=alpha, fma=True)
    r = _reference(x, w, torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)
    pre = r["out"] + bias.to(cuda_dev, torch.float64)
    ref = {"relu": pre.clamp_min(0), "leaky_relu": torch.where(pre >= 0, pre, pre * alpha),
           "sigmoid": torch.sigmoid(pre)}[act]
    if act == "leaky_relu":
        assert (pre < -1).any(), "no negative pre-activation: the slope would not be checked"
    lip = 0.25 if act == "sigmoid" else 1.0
    pre_bound = (r["t_out"][:, None] * C + 2) * 2.0 ** -23 * (r["out_abs"] + bias.abs().to(cuda_dev))
    _check(f"{act} out", got, ref, torch.zeros_like(ref), torch.zeros_like(ref), dt,
           extra=lip * pre_bound + (2.0 ** -20 if act == "sigmoid" else 0.0))


@gpu
@pytest.mark.parametrize("name,algo", [("subm3d_k3", "Native"), ("subm3d_k3", "MaskSplitImplicitGemm"),
                                       ("conv3d_k3s2p1", "Native"), ("conv3d_k3s2p1", "MaskSplitImplicitGemm")])
def test_modules_on_fma(name, algo, oracle, cuda_dev):
    """Native and mask-split modules with an fp32 shape the tensor cores never tile (C 33, K 65)"""
    from tests.test_conv_modules_gpu import GEOMS, cloud, run_case
    _configure(0)           # fp32 runs on the FMA kernels by dispatch, also where the environment forces a family
    inds, bs = cloud(name)
    run_case(name, GEOMS[name], inds, bs, algo, "f32", 33, 65, oracle, cuda_dev, seed=4)


@gpu
@pytest.mark.parametrize("case", [(F32, 33, 65), ("bf16", 100, 129)], ids=lambda c: f"{c[0]}-C{c[1]}K{c[2]}")
def test_fma_is_deterministic(case, oracle, cuda_dev):
    """the FMA kernels sum in a fixed order: two identical calls give identical bits"""
    dt, C, K = case
    runs = _run_case(oracle, cuda_dev, _conv(oracle, cuda_dev, "k3", "conv"), dt, C, K, seed=2, repeat=2, fma=True)
    for name, a, b in zip(("out", "din", "dw"), *runs):
        assert torch.equal(a, b), f"{name} differs between two identical runs"
