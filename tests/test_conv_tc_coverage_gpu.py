"""Every tensor-core conv kernel instance against a float64 reference.

The forward, input-gradient (dgrad), int8 forward and weight-gradient (wgrad) kernels are compiled as
template instances over row bytes and output channels.  The cases below reach every compiled instance
(``test_every_compiled_instance_is_reached`` reads them from the library's symbol table), every word
of the tile mask (kernel volumes 1 to 125), partial tiles and the rings that only wrap on long grids.

Each output element is checked against a float64 sum over the oracle's rulebook:
    |got - ref| <= u_out |ref| + T 2^-23 sum|terms| + tiny
where T is the number of terms summed.  The inputs are exactly representable in the operand type, so
every product is exact in fp32 and only the fp32 accumulation (T 2^-23) and the output rounding
(u_out) remain.  Outputs are pre-filled with NaN, so a row a kernel never writes cannot pass.

Every call states the kernel family it must run on.  Calls expected on the tensor cores run with the
tensor cores forced, so a refused call raises instead of falling back.  Calls expected on the FMA
kernels must be refused when forced, and then run there.  With SPX_FORCE_SIMT=1 in the environment
the same cases run on the FMA kernels.
"""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests.util import random_cloud

gpu = pytest.mark.gpu

# kernel family pinned by the environment (core.cu reads these once): 1 FMA, 2 tensor cores, 0 auto
ENV_FAMILY = (1 if os.environ.get("SPX_FORCE_SIMT", "").startswith("1")
              else 2 if os.environ.get("SPX_FORCE_TC", "").startswith("1") else 0)
SIMT = ENV_FAMILY == 1

TORCH_DT = {"f16": torch.float16, "bf16": torch.bfloat16, "tf32": torch.float32, "i8": torch.int8}
ELEM = {"f16": 2, "bf16": 2, "tf32": 4, "i8": 1}
U_OUT = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8, "tf32": 0.0}
TINY = {"f16": 2.0 ** -24, "bf16": 1e-30, "tf32": 1e-30}     # fp16 subnormal spacing
KIND = {"f16": 0, "bf16": 0, "tf32": 1, "i8": 2}             # MmaKind of common.cuh
KIND_NAME = ("F16", "TF32", "I8")
REFUSED = "SPX_FORCE_TC=1 but the tensor-core"


# ------------------------------------------------------------------ which instance serves a call
def _al(n):
    return (n + 1023) // 1024 * 1024


def gemm_instance(dt, kv, c_in, c_out, dgrad=False):
    """("gemm", KIND, CPR, N) of the tc_gather_gemm_kernel that serves this fwd / dgrad / int8 call,
    None when it runs on the FMA kernel (tc_shape_ok, tc_gather_gemm_supported and fill_params of
    gemm_tc.cu)."""
    e = ELEM[dt]
    if dt == "tf32" and dgrad and (c_in * 4) % 128:
        return None
    if any(c % 16 or c * e not in (32, 64, 128, 256, 512) for c in (c_in, c_out)):
        return None
    if dt == "i8" and (c_in % 32 or c_out % 32):
        return None
    cx, cy = (c_out, c_in) if dgrad else (c_in, c_out)
    stage = _al(128 * cx * e) + _al(c_in * c_out * e)
    if 2 * _al((kv + 1) * 512) + 2 * stage > 200 * 1024:
        return None
    return ("gemm", KIND[dt], cx * e // 16, cy)


def wgrad_instance(dt, kv, c_in, c_out):
    """("wgrad", CPA, CPD, TF32) of the tc_wgrad_kernel that serves this call, None for the FMA
    kernel (make_plan of gemm_tc_wgrad.cu)."""
    e, tf32 = ELEM[dt], dt == "tf32"
    if dt == "i8" or c_in % 16 or c_out % 16 or c_in > 256 or c_out > 256:
        return None
    if tf32 and (c_in % 32 or c_out % 32 or c_out > 64):
        return None
    db, xb, span_x = c_out * e, c_in * e, min(c_in * e, 128)
    if db & (db - 1) or xb & (xb - 1):        # whole power-of-two atoms per offset, dout rows of 2^n bytes
        return None
    a_stage = 128 // (span_x // e) * 128 * span_x
    avail = (224 * 1024 - 2048 if tf32 else 200 * 1024) - 2 * 128 * db - 2 * _al((kv + 1) * 512)
    if avail < 2 * a_stage:
        return None
    return ("wgrad", span_x // 16, db // 16, tf32)


def _instance_name(inst):
    if inst[0] == "gemm":
        return f"tc_gather_gemm_kernel<{KIND_NAME[inst[1]]}, {inst[2]}, {inst[3]}>"
    return f"tc_wgrad_kernel<{inst[1]}, {inst[2]}, {str(inst[3]).lower()}>"


# ------------------------------------------------------------------ cases
# name: (spatial shape, points per sample, ksize, dilation, (stride, padding) of the strided conv)
GEOMS = {
    "k3": ([19, 18, 17], [1500, 1500], [3, 3, 3], 1, (2, 1)),
    "k1": ([19, 18, 17], [1500, 1500], [1, 1, 1], 1, (2, 0)),
    "k2s2": ([19, 18, 17], [1500, 1500], [2, 2, 2], 1, (2, 0)),            # kv 8, no centre offset
    "2d_k3": ([40, 50], [900, 800], [3, 3], 1, (2, 1)),                     # kv 9
    "1d_k5": ([3000], [1200], [5], 1, (2, 2)),                              # kv 5
    "k533": ([19, 18, 17], [1500, 1500], [5, 3, 3], 1, (2, [2, 1, 1])),     # kv 45: 2 mask words
    "k4s2": ([19, 18, 17], [1500, 1500], [4, 4, 4], 1, (2, 1)),             # kv 64: 2 full words
    "4d_k3": ([9, 10, 11, 12], [2000], [3, 3, 3, 3], 1, (2, 1)),            # kv 81: 3 words
    "k5": ([19, 18, 17], [1500, 1500], [5, 5, 5], 1, (2, 2)),               # kv 125: bits 96-124
    "dil2": ([19, 18, 17], [1500, 1500], [3, 3, 3], 2, (2, 2)),
}
KV = {g: int(np.prod(v[2])) for g, v in GEOMS.items()}

# (dtype, geometry, C, K): fwd + dgrad + wgrad, as subm (odd kernels) and as a strided conv
CASES = [
    # instance cover at kv = 27
    ("f16", "k3", 16, 16), ("bf16", "k3", 16, 32), ("f16", "k3", 32, 32), ("bf16", "k3", 32, 64),
    ("f16", "k3", 64, 64), ("f16", "k3", 16, 64), ("bf16", "k3", 16, 128), ("f16", "k3", 32, 128),
    ("f16", "k3", 64, 128), ("bf16", "k3", 128, 128), ("f16", "k3", 256, 16), ("bf16", "k3", 256, 32),
    ("f16", "k3", 16, 256),
    # 1x1 convs: 512-byte gathered rows of dgrad, 256-column weight-gradient passes
    ("f16", "k1", 64, 256), ("bf16", "k1", 16, 256), ("f16", "k1", 32, 256), ("f16", "k1", 128, 256),
    ("tf32", "k3", 16, 16), ("tf32", "k3", 32, 16), ("tf32", "k3", 64, 16), ("tf32", "k3", 128, 16),
    ("tf32", "k3", 128, 32), ("tf32", "k3", 32, 32), ("tf32", "k3", 32, 64), ("tf32", "k3", 64, 32),
    ("tf32", "k3", 64, 64), ("tf32", "k1", 64, 128),
    # kernel volumes, every call on the tensor cores
    *[("f16", g, 32, 16) for g in ("k1", "k2s2", "2d_k3", "1d_k5", "k533", "k4s2", "4d_k3", "k5", "dil2")],
    *[("bf16", g, 64, 16) for g in ("k533", "k4s2", "4d_k3", "k5")],
    # just outside the tensor-core envelope: refused when forced, FMA kernels otherwise
    ("f16", "k3", 128, 256), ("f16", "k5", 64, 64), ("tf32", "k3", 32, 128),
    # 384-byte rows (three channel atoms per kernel offset) run the weight gradient on the FMA kernel;
    # 1024-byte fp32 rows take eight atoms per offset on the tensor cores
    ("f16", "k3", 192, 32), ("tf32", "k3", 96, 32), ("tf32", "k3", 256, 32),
]
# inverse convs walk a strided conv's rulebook backwards
INVERSE = [("f16", "k3", 32, 16), ("bf16", "k2s2", 64, 32)]
ROW_EDGE_M = [1, 127, 128, 129, 255]
ROW_EDGE = ("f16", 64, 32)
# (dtype, geometry, C, K, points): more than 4 tiles per SM, so the forward tile-info ring, the index
# double buffer and the weight-gradient index ring wrap, the latter over multi-pass grids
LONG = [("f16", "k5", 32, 16, 70000), ("f16", "k3", 256, 16, 70000)]
EPILOGUE = [("bf16", 32, 16), ("bf16", 16, 256), ("tf32", 32, 16), ("tf32", 32, 128)]
INT8 = ([(c, k, "k3", "i8", True) for c in (32, 64, 128, 256) for k in (32, 64, 128, 256) if (c, k) != (256, 256)]
        + [(256, 256, "k1", "i8", True), (32, 256, "k3", "f16", True), (32, 256, "k3", "f16", False)])


def _modes(geom):
    return (["subm"] if all(k % 2 for k in GEOMS[geom][2]) else []) + ["conv"]


def _calls(dt, kv, C, K, fwd_only=False):
    """instances (None = FMA kernel) of the fwd, dgrad and wgrad calls of one case"""
    if fwd_only:
        return {"fwd": gemm_instance(dt, kv, C, K)}
    return {"fwd": gemm_instance(dt, kv, C, K), "dgrad": gemm_instance(dt, kv, C, K, dgrad=True),
            "wgrad": wgrad_instance(dt, kv, C, K)}


def _all_instances():
    seen = set()
    for dt, g, C, K in CASES + INVERSE:
        seen.update(_calls(dt, KV[g], C, K).values())
    seen.update(_calls(ROW_EDGE[0], 27, *ROW_EDGE[1:]).values())
    for dt, g, C, K, _ in LONG:
        seen.update(_calls(dt, KV[g], C, K).values())
    for dt, C, K in EPILOGUE:
        seen.add(gemm_instance(dt, 27, C, K))
    for C, K, g, _, _ in INT8:
        seen.add(gemm_instance("i8", KV[g], C, K))
    seen.discard(None)
    return seen


# ------------------------------------------------------------------ helpers
def _lib():
    from spconv_b200 import _cabi
    return _cabi.load()


def _configure(family):
    from spconv_b200 import _cabi
    _cabi.check(_lib().spx_debug_configure(family, 0, 0, None, 0), "debug_configure")


@pytest.fixture(autouse=True)
def _restore_forced_family():
    yield
    if torch.cuda.is_available():
        _configure(ENV_FAMILY)


def _launch(what, inst, launch, fma=False):
    """Run `launch` on the family `inst` says (None: FMA kernel) and check that it ran there.
    fma=True pins the FMA kernels whatever the shape."""
    fma = fma or SIMT
    if fma:
        _configure(1)
    elif inst is not None:
        _configure(2)
    else:
        _configure(2)
        with pytest.raises(RuntimeError, match=REFUSED):
            launch()
        _configure(0)
    out = launch()
    fam = _lib().spx_last_kernel_family()
    want = 1 if fma or inst is None else 2
    assert fam == want, f"{what}: kernel family {fam}, expected {want} ({inst and _instance_name(inst)})"
    return out


def _nan(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def _exact(rng, shape, dt, scale=1.0, round_tf32=True):
    """uniform values exactly representable in the operand type, as float32"""
    v = torch.from_numpy(rng.uniform(-scale, scale, size=shape).astype(np.float32))
    if dt in ("f16", "bf16"):
        return v.to(TORCH_DT[dt]).float()
    if round_tf32:     # clear the 13 mantissa bits tf32 wgmma does not read
        return (v.view(torch.int32) & ~0x1FFF).view(torch.float32)
    return v


class Conv:
    """One conv's rulebook: the engine's tables (checked bit for bit against the oracle's) and the
    oracle's pair table the reference is summed over.  `ref_pair[k, o]` is the input row of output
    row o at offset k."""

    def __init__(self, oracle, dev, inds, bs, shape, ks, stride, padding, dilation, subm, inverse=False):
        from spconv_b200.core import ConvAlgo
        from spconv_b200.pytorch import ops
        nd = len(shape)
        ks, st, pd, dl = ([v] * nd if np.isscalar(v) else list(v) for v in (ks, stride, padding, dilation))
        ref_out, pairs, num = oracle.get_indice_pairs(inds, bs, shape, ks, st, pd, dl, [0] * nd, subm)
        n_in, n_out = inds.shape[0], ref_out.shape[0]
        tab = oracle.implicit_gemm_tables(pairs, num, n_in, n_out, subm)
        res = ops.get_indice_pairs_implicit_gemm(torch.from_numpy(inds).to(dev), bs, shape, ConvAlgo.MaskImplicitGemm,
                                                 ks, st, pd, dl, [0] * nd, subm, False, is_train=True)
        out_inds, _, pf, pb, mf, mb, sf, sb, _ = res
        # the rulebook first, so that a failure below is the GEMM's
        assert np.array_equal(out_inds.cpu().numpy(), ref_out), "output coordinates differ from the oracle"
        assert np.array_equal(pf.cpu().numpy(), tab["pair_fwd"]), "pair_fwd differs from the oracle"
        assert np.array_equal(pb.cpu().numpy(), tab["pair_bwd"]), "pair_bwd differs from the oracle"
        assert np.array_equal(mf[0].cpu().numpy().view(np.uint32), tab["mask_fwd"]), "mask_fwd differs"
        assert np.array_equal(sf[0].cpu().numpy(), tab["argsort_fwd"]), "argsort_fwd differs"
        fwd, bwd = (pf, mf[0], sf[0], n_out), None
        if not subm:
            assert np.array_equal(mb[0].cpu().numpy().view(np.uint32), tab["mask_bwd"]), "mask_bwd differs"
            assert np.array_equal(sb[0].cpu().numpy(), tab["argsort_bwd"]), "argsort_bwd differs"
            bwd = (pb, mb[0], sb[0], n_in)
        self.kv, self.subm, self.n_in, self.n_out = int(np.prod(ks)), subm, n_in, n_out
        self.fwd, self.bwd, self.ref_pair = fwd, bwd, tab["pair_fwd"]
        if inverse:
            assert not subm
            self.fwd, self.bwd, self.ref_pair = bwd, fwd, tab["pair_bwd"]
            self.n_in, self.n_out = n_out, n_in

    def desc(self, dtype, C, K, table, reverse=False):
        from spconv_b200 import _cabi
        from spconv_b200.pytorch import ops
        pair, mask, argsort, rows = table
        tiles = ops._tile_tables(pair, mask, argsort, rows, self.kv, owner=argsort)
        d = ops._desc(dtype, self.kv, C, K, self.n_in, self.n_out, pair, mask, argsort, reverse=reverse, tiles=tiles)
        d.f32_mode = _cabi.SPX_F32_TF32
        return d

    def fwd_call(self, x, w, inst, bias=None, act=0, alpha=0.0, fma=False):
        from spconv_b200 import _cabi
        from spconv_b200.pytorch import ops
        K, C = w.shape[0], w.shape[-1]
        d = self.desc(x.dtype, C, K, self.fwd)

        def launch():
            out = _nan((self.n_out, K), x.dtype, x.device)
            _cabi.check(_lib().spx_implicit_gemm_fwd(ctypes.byref(d), x.data_ptr(), w.data_ptr(), out.data_ptr(),
                                                     None if bias is None else bias.data_ptr(), act, alpha,
                                                     ops._stream()), "implicit_gemm_fwd")
            return out
        return _launch("fwd", inst, launch, fma)

    def dgrad_call(self, dout, w, inst, fma=False):
        from spconv_b200 import _cabi
        from spconv_b200.pytorch import ops
        K, C = w.shape[0], w.shape[-1]
        # subm: the forward table walked with mirrored offsets; strided conv: the backward table
        d = self.desc(dout.dtype, C, K, self.fwd, reverse=True) if self.subm else self.desc(dout.dtype, C, K, self.bwd)

        def launch():
            din = _nan((self.n_in, C), dout.dtype, dout.device)
            _cabi.check(_lib().spx_implicit_gemm_dgrad(ctypes.byref(d), dout.data_ptr(), w.data_ptr(), din.data_ptr(),
                                                       ops._stream()), "implicit_gemm_dgrad")
            return din
        return _launch("dgrad", inst, launch, fma)

    def wgrad_call(self, x, dout, w_shape, inst, fma=False):
        from spconv_b200 import _cabi
        from spconv_b200.pytorch import ops
        K, C = w_shape[0], w_shape[-1]
        d = self.desc(x.dtype, C, K, self.fwd)

        def launch():
            lib = _lib()
            ws = _nan(((lib.spx_implicit_gemm_wgrad_workspace_size(ctypes.byref(d)) + 3) // 4,), torch.float32,
                      x.device)
            dw = _nan(tuple(w_shape), x.dtype, x.device)
            _cabi.check(lib.spx_implicit_gemm_wgrad(ctypes.byref(d), x.data_ptr(), dout.data_ptr(), dw.data_ptr(),
                                                    ws.data_ptr(), ws.numel() * 4, ops._stream()), "implicit_gemm_wgrad")
            return dw
        return _launch("wgrad", inst, launch, fma)


def _reference(x, w, dout, ref_pair, dev):
    """float64 out / din / dW, the same sums over absolute values, and the number of terms summed
    into every element (active offsets of a row, contributing voxels of an offset)."""
    x, dout = x.to(dev, torch.float64), dout.to(dev, torch.float64)
    K, C = w.shape[0], w.shape[-1]
    w = w.to(dev, torch.float64).reshape(K, -1, C)
    pair = torch.from_numpy(ref_pair).to(dev).long()
    kv, n_out, n_in = w.shape[1], pair.shape[1], x.shape[0]
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=dev)    # noqa: E731
    r = dict(out=z(n_out, K), out_abs=z(n_out, K), din=z(n_in, C), din_abs=z(n_in, C), dw=z(K, kv, C),
             dw_abs=z(K, kv, C), t_out=z(n_out), t_in=z(n_in), t_k=z(kv))
    for k in range(kv):
        o = (pair[k] >= 0).nonzero().squeeze(1)
        if not len(o):
            continue
        i = pair[k, o]
        xi, do, wk = x[i], dout[o], w[:, k]
        r["out"][o] += xi @ wk.T
        r["out_abs"][o] += xi.abs() @ wk.abs().T
        r["din"].index_add_(0, i, do @ wk)
        r["din_abs"].index_add_(0, i, do.abs() @ wk.abs())
        r["dw"][:, k] = do.T @ xi
        r["dw_abs"][:, k] = do.abs().T @ xi.abs()
        r["t_out"][o] += 1
        r["t_in"].index_add_(0, i, torch.ones_like(i, dtype=torch.float64))
        r["t_k"][k] = len(o)
    return r


def _check(name, got, ref, ref_abs, terms, dt, zero=None, extra=0.0):
    """element-wise bound; `terms` broadcasts against ref, `zero` marks elements that must be exactly 0"""
    g = got.double()
    nan = torch.isnan(g)
    if nan.any():
        rows = nan.reshape(nan.shape[0], -1).any(1).nonzero().squeeze(1)
        raise AssertionError(f"{name}: {int(nan.sum())} NaN in {len(rows)} rows never written "
                             f"(first rows {rows[:8].tolist()})")
    bound = U_OUT[dt] * ref.abs() + (1 + U_OUT[dt]) * ((terms + 1) * 2.0 ** -23 * ref_abs + extra) + TINY[dt]
    err = (g - ref).abs()
    bad = err > bound
    if bad.any():
        flat = (err - bound).reshape(-1).argmax()
        idx = np.unravel_index(int(flat), tuple(err.shape))
        rows = bad.reshape(bad.shape[0], -1).any(1).nonzero().squeeze(1)
        raise AssertionError(
            f"{name}: {int(bad.sum())}/{bad.numel()} elements out of bound in {len(rows)} rows "
            f"(first rows {rows[:8].tolist()}); worst at {idx}: got {float(g[idx]):.6g} ref {float(ref[idx]):.6g} "
            f"bound {float(bound[idx]):.3g}")
    if zero is not None and zero.any():
        nz = (g[zero] != 0).sum()
        assert nz == 0, f"{name}: {int(nz)} elements without any pair are not exactly 0"


def _run_case(oracle, dev, conv, dt, C, K, seed, repeat=1, round_tf32=True, fma=False):
    """fwd + dgrad + wgrad of one conv against the float64 reference; returns the outputs.
    fma=True runs every call on the FMA kernels."""
    rng = np.random.default_rng(seed)
    x = _exact(rng, (conv.n_in, C), dt, round_tf32=round_tf32)
    w = _exact(rng, (K, conv.kv, C), dt, round_tf32=round_tf32)
    dout = _exact(rng, (conv.n_out, K), dt, round_tf32=round_tf32)
    tdt = TORCH_DT[dt]
    xd, wd, dd = x.to(dev, tdt), w.to(dev, tdt), dout.to(dev, tdt)
    inst = _calls(dt, conv.kv, C, K)
    r = _reference(x, w, dout, conv.ref_pair, dev)
    rel = 0.0 if round_tf32 else 2 * 2.0 ** -10             # operands rounded to tf32 by the tensor cores
    runs = []
    for _ in range(repeat):
        out = conv.fwd_call(xd, wd, inst["fwd"], fma=fma)
        din = conv.dgrad_call(dd, wd, inst["dgrad"], fma=fma)
        dw = conv.wgrad_call(xd, dd, wd.shape, inst["wgrad"], fma=fma)
        torch.cuda.synchronize()
        runs.append((out, din, dw))
    out, din, dw = runs[0]
    _check("out", out, r["out"], r["out_abs"], r["t_out"][:, None] * C, dt, zero=r["t_out"] == 0,
           extra=rel * r["out_abs"])
    _check("din", din, r["din"], r["din_abs"], r["t_in"][:, None] * K, dt, zero=r["t_in"] == 0,
           extra=rel * r["din_abs"])
    _check("dw", dw.reshape(K, conv.kv, C), r["dw"], r["dw_abs"], r["t_k"][None, :, None], dt,
           zero=(r["t_k"] == 0)[None, :, None].expand(K, conv.kv, C), extra=rel * r["dw_abs"])
    return runs


def _cloud(geom, seed):
    shape, pts = GEOMS[geom][:2]
    _, inds = random_cloud(np.random.default_rng(seed), shape, pts, 1)
    return inds


def _conv(oracle, dev, geom, mode, inds=None, shape=None, seed=50005):
    shape_g, _, ks, dil, (st, pd) = GEOMS[geom]
    shape = shape_g if shape is None else shape
    inds = _cloud(geom, seed) if inds is None else inds
    bs = int(inds[:, 0].max()) + 1
    if mode == "subm":
        return Conv(oracle, dev, inds, bs, shape, ks, 1, 0, dil, True)
    return Conv(oracle, dev, inds, bs, shape, ks, st, pd, dil, False, inverse=mode == "inverse")


# ------------------------------------------------------------------ tests
@gpu
@pytest.mark.parametrize("case", [(*c, m) for c in CASES for m in _modes(c[1])],
                         ids=lambda c: f"{c[0]}-{c[1]}-C{c[2]}K{c[3]}-{c[4]}")
def test_conv_against_fp64(case, oracle, cuda_dev):
    dt, geom, C, K, mode = case
    _run_case(oracle, cuda_dev, _conv(oracle, cuda_dev, geom, mode), dt, C, K, seed=C * 1000 + K)


@gpu
@pytest.mark.parametrize("case", INVERSE, ids=lambda c: f"{c[0]}-{c[1]}-C{c[2]}K{c[3]}")
def test_inverse_conv_against_fp64(case, oracle, cuda_dev):
    """an inverse conv reuses a strided conv's rulebook: forward over pair_bwd, dgrad over pair_fwd"""
    dt, geom, C, K = case
    _run_case(oracle, cuda_dev, _conv(oracle, cuda_dev, geom, "inverse"), dt, C, K, seed=7)


@gpu
def test_tf32_unrounded_inputs(oracle, cuda_dev):
    """fp32 inputs with all mantissa bits set: the tensor cores read them as tf32"""
    _run_case(oracle, cuda_dev, _conv(oracle, cuda_dev, "k3", "conv"), "tf32", 64, 32, seed=9, round_tf32=False)


@gpu
@pytest.mark.parametrize("m", ROW_EDGE_M)
def test_partial_tiles(m, oracle, cuda_dev):
    """M = 1 .. 255 rows: first rows of a dense 8 x 8 x 8 block, one partial or full 128-row tile"""
    g = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3)[:m]
    inds = np.concatenate([np.zeros((m, 1), np.int32), g.astype(np.int32)], 1)
    conv = Conv(oracle, cuda_dev, inds, 1, [8, 8, 8], 3, 1, 0, 1, True)
    dt, C, K = ROW_EDGE
    _run_case(oracle, cuda_dev, conv, dt, C, K, seed=m)


@gpu
@pytest.mark.parametrize("case", LONG, ids=lambda c: f"{c[0]}-{c[1]}-C{c[2]}K{c[3]}")
def test_long_grids_and_determinism(case, oracle, cuda_dev):
    """More than 4 tiles per SM (the rings wrap); two runs give bit-identical out, din and dW (the
    weight gradient's static schedule; 2 passes at kv 125 C 32 K 16, 4 passes at C 256 K 16)"""
    dt, geom, C, K, n = case
    _, inds = random_cloud(np.random.default_rng(n), [64, 64, 64], [n], 1)
    conv = _conv(oracle, cuda_dev, geom, "subm", inds=inds, shape=[64, 64, 64])
    sms = torch.cuda.get_device_properties(cuda_dev).multi_processor_count
    assert conv.n_out > 4 * sms * 128
    runs = _run_case(oracle, cuda_dev, conv, dt, C, K, seed=3, repeat=2)
    for name, a, b in zip(("out", "din", "dw"), *runs):
        assert torch.equal(a, b), f"{name} differs between two identical runs"


@gpu
@pytest.mark.parametrize("act", ["relu", "leaky_relu", "sigmoid"])
@pytest.mark.parametrize("case", EPILOGUE, ids=lambda c: f"{c[0]}-C{c[1]}K{c[2]}")
def test_bias_activation_epilogue(case, act, oracle, cuda_dev):
    from spconv_b200.core import Activation
    dt, C, K = case
    conv = _conv(oracle, cuda_dev, "k3", "subm")
    rng = np.random.default_rng(21)
    x, w = _exact(rng, (conv.n_in, C), dt), _exact(rng, (K, 27, C), dt)
    bias = _exact(rng, (K,), dt, scale=2.0)
    alpha = 0.25
    code = {"relu": Activation.ReLU, "leaky_relu": Activation.LeakyReLU, "sigmoid": Activation.Sigmoid}[act].value
    tdt = TORCH_DT[dt]
    got = conv.fwd_call(x.to(cuda_dev, tdt), w.to(cuda_dev, tdt), gemm_instance(dt, 27, C, K),
                        bias=bias.to(cuda_dev, tdt), act=code, alpha=alpha)
    r = _reference(x, w, torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)
    pre = r["out"] + bias.to(cuda_dev, torch.float64)
    ref = {"relu": pre.clamp_min(0), "leaky_relu": torch.where(pre >= 0, pre, pre * alpha),
           "sigmoid": torch.sigmoid(pre)}[act]
    lip = 0.25 if act == "sigmoid" else 1.0
    pre_bound = (r["t_out"][:, None] * C + 2) * 2.0 ** -23 * (r["out_abs"] + bias.abs().to(cuda_dev))
    # the accumulation bound passes through the activation scaled by its Lipschitz constant; the
    # sigmoid adds the error of __expf and of the division
    _check(f"{act} out", got, ref, torch.zeros_like(ref), torch.zeros_like(ref), dt,
           extra=lip * pre_bound + (2.0 ** -20 if act == "sigmoid" else 0.0))


@gpu
@pytest.mark.parametrize("case", INT8, ids=lambda c: f"C{c[0]}K{c[1]}-{c[2]}-{c[3]}out{'-add' if c[4] else ''}")
def test_int8_against_exact_reference(case, oracle, cuda_dev):
    """int8 x int8 -> int32 -> scale, bias, residual, ReLU: int8 outputs may be 1 off only where the
    value lies on a round-to-even tie; fp16 outputs are within half an fp16 ulp plus fp32 rounding"""
    from spconv_b200 import _cabi
    from spconv_b200.core import Activation
    from spconv_b200.pytorch import ops
    C, K, geom, out_dt, with_add = case
    conv = _conv(oracle, cuda_dev, geom, "subm")
    rng = np.random.default_rng(C * 7 + K)
    x = torch.from_numpy(rng.integers(-4, 4, size=(conv.n_in, C)).astype(np.int8))
    w = torch.from_numpy(rng.integers(-4, 4, size=(K, conv.kv, C)).astype(np.int8))
    scale = torch.from_numpy((rng.uniform(0.5, 1.5, size=K) * 0.2).astype(np.float32))
    bias = torch.from_numpy(rng.uniform(-5, 5, size=K).astype(np.float32))
    add = torch.from_numpy(rng.integers(-3, 4, size=(conv.n_out, K)).astype(np.int8))
    add_scale = 0.375
    r = _reference(x.float(), w.float(), torch.zeros((conv.n_out, K)), conv.ref_pair, cuda_dev)
    acc = r["out"]                                                    # exact: integers below 2^24
    s64, b64 = scale.to(cuda_dev, torch.float64), bias.to(cuda_dev, torch.float64)
    a64 = add.to(cuda_dev, torch.float64) * add_scale if with_add else torch.zeros_like(acc)
    res = acc * s64 + b64 + a64
    fp32_err = 4 * 2.0 ** -24 * ((acc * s64).abs() + b64.abs() + a64.abs()) + 1e-30
    xd, wd = x.to(cuda_dev), w.to(cuda_dev)
    sd, bd, ad = scale.to(cuda_dev), bias.to(cuda_dev), add.to(cuda_dev) if with_add else None
    d = conv.desc(torch.int8, C, K, conv.fwd)
    code = _cabi.SPX_I8 if out_dt == "i8" else _cabi.SPX_F16

    def launch():
        out = (torch.full((conv.n_out, K), -77, dtype=torch.int8, device=cuda_dev) if out_dt == "i8"
               else _nan((conv.n_out, K), torch.float16, cuda_dev))
        _cabi.check(_lib().spx_implicit_gemm_fwd_int8(
            ctypes.byref(d), xd.data_ptr(), wd.data_ptr(), out.data_ptr(), code, sd.data_ptr(), bd.data_ptr(),
            None if ad is None else ad.data_ptr(), add_scale, Activation.ReLU.value, 0.0, ops._stream()),
            "implicit_gemm_fwd_int8")
        return out
    got = _launch("int8 fwd", gemm_instance("i8", conv.kv, C, K), launch).double()
    relu = res.clamp_min(0)
    if out_dt == "i8":
        ref = torch.round(relu).clamp(-128, 127)                     # torch.round: half to even
        diff = (got - ref).abs()
        tie = ((relu - relu.floor()) - 0.5).abs() <= fp32_err
        off = diff > 0
        assert not (diff > 1).any() and not (off & ~tie).any(), (
            f"{int(off.sum())} outputs differ, {int((off & ~tie).sum())} of them away from a .5 tie, "
            f"max diff {float(diff.max())} (-77 = never written)")
    else:
        _check("int8 -> f16 out", got, relu, torch.zeros_like(relu), torch.zeros_like(relu), "f16", extra=fp32_err)


def library_symbols():
    """the library's demangled symbol names (nm, or cuobjdump's kernel list)"""
    from spconv_b200 import _cabi
    _cabi.load()
    if shutil.which("nm"):
        return subprocess.run(["nm", "-C", "--defined-only", _cabi.LIB_PATH], capture_output=True, text=True,
                              check=True).stdout
    if shutil.which("cuobjdump") and shutil.which("c++filt"):
        dump = subprocess.run(["cuobjdump", "-res-usage", _cabi.LIB_PATH], capture_output=True, text=True,
                              check=True).stdout
        return subprocess.run(["c++filt"], input=dump, capture_output=True, text=True, check=True).stdout
    pytest.skip("neither nm nor cuobjdump is available")


def _compiled_instances():
    text = library_symbols()
    found = {("gemm", int(a), int(b), int(c))
             for a, b, c in re.findall(r"tc_gather_gemm_kernel<(\d+), (\d+), (\d+)>", text)}
    found |= {("wgrad", int(a), int(b), c == "true")
              for a, b, c in re.findall(r"tc_wgrad_kernel<(\d+), (\d+), (true|false)>", text)}
    return found


def test_every_compiled_instance_is_reached():
    """No GPU needed: each tensor-core kernel instance in the library is served by some case of this
    file, and every instance a case expects exists."""
    compiled = _compiled_instances()
    assert compiled, "no tensor-core kernel instance found in the library's symbol table"
    reached = _all_instances()
    missing = sorted(_instance_name(i) for i in compiled - reached)
    absent = sorted(_instance_name(i) for i in reached - compiled)
    assert not missing, f"compiled but reached by no case: {missing}"
    assert not absent, f"expected by a case but not compiled: {absent}"
