"""MaskedGroupNorm with per-sample scale / shift (AdaGN) and a fused ReLU / SiLU on the GPU: against a float64
per-sample reference with autograd for dx, dweight, dbias, dscale and dshift; bit-identical results under padding,
dropped rows, a clamped num_valid, misaligned operands and repeats, where the torch formulation lets the padding
reach the last sample's dshift; neutral modulation equal to the plain call; launch counts; and a small conditioned
net that trains padded and replays as one CUDA graph."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from tests.test_masked_group_norm_gpu import (BATCHES, DTYPES, EPS, _at_offset, _bits, _close_f32, _close_low,
                                              _inputs, _junk_rows, _params)
from tests.util import random_cloud

import spconv_b200.pytorch as spconv
from spconv_b200 import _cabi
from spconv_b200.pytorch import MaskedGlobalAvgPool, MaskedGroupNorm, ops
from spconv_b200.pytorch.functional import masked_group_norm

pytestmark = pytest.mark.gpu

ACTS = [None, "relu", "silu"]
MODS = ["neither", "scale", "shift", "both"]


def _groups(c):
    """G in {1, 8, C}, where G divides C"""
    return sorted({g for g in (1, 8, c) if c % g == 0})


def _mod(b, c, which, dev, seed):
    g = torch.Generator().manual_seed(seed + 7)
    scale = (torch.rand((b, c), generator=g) - 0.5).to(dev) if which in ("scale", "both") else None
    shift = (torch.rand((b, c), generator=g) * 2 - 1).to(dev) if which in ("shift", "both") else None
    return scale, shift


def _run(x, dy, inds, b, groups, w, bias, scale, shift, act, num_valid=None):
    """y, dx, dweight, dbias, dscale, dshift through autograd"""
    leaf = lambda t: None if t is None else t.clone().requires_grad_(True)  # noqa: E731
    xr, wr, br, sr, tr = leaf(x), leaf(w), leaf(bias), leaf(scale), leaf(shift)
    y = masked_group_norm(xr, wr, br, inds, b, num_valid, groups, EPS, sr, tr, act)
    y.backward(dy)
    return tuple([y.detach()] + [None if t is None else t.grad for t in (xr, wr, br, sr, tr)])


def _reference(x, dy, inds, b, groups, w, bias, scale, shift, act):
    """the per-sample loop F.group_norm -> * (1 + scale[b]) + shift[b] -> act in float64 with autograd, on the
    (dtype-rounded) inputs.  Also, per result, the size of the terms that cancel in it, and for ReLU the elements
    whose z is within the fp32 error of 0 (`amb`): there the kernel's z and the float64 z may sit on either side of
    the kink (and a tiny positive y rounds to 0 in fp16), so their dx is not compared and the sums' tolerances
    take in the dy they may or may not add."""
    rows, c = x.shape
    cg = c // groups
    dev = x.device
    f64 = lambda t, d: (t.double() if t is not None else d).clone().requires_grad_(True)  # noqa: E731
    xd = f64(x, None)
    wd = f64(w, torch.ones(c, dtype=torch.float64, device=dev))
    bd = f64(bias, torch.zeros(c, dtype=torch.float64, device=dev))
    sd = f64(scale, torch.zeros((b, c), dtype=torch.float64, device=dev))
    td = f64(shift, torch.zeros((b, c), dtype=torch.float64, device=dev))
    dyd = dy.double()
    ids = inds[:, 0].long()
    y = torch.zeros((rows, c), dtype=torch.float64, device=dev)
    zero = torch.zeros_like(y)
    cond = {k: torch.zeros_like(y) for k in ("y", "dx")}
    sq = {k: torch.zeros(c, dtype=torch.float64, device=dev) for k in ("dw", "db")}
    cond["ds"] = torch.zeros((b, c), dtype=torch.float64, device=dev)
    cond["dt"] = torch.zeros((b, c), dtype=torch.float64, device=dev)
    amb = torch.zeros((rows, c), dtype=torch.bool, device=dev)
    with torch.no_grad():
        w0, b0, s1 = wd.detach(), bd.detach(), 1 + sd.detach()
    for s in range(b):
        sel = (ids == s).nonzero().squeeze(1)
        if sel.numel() == 0:
            continue
        h = F.group_norm(xd[sel].T[None], groups, wd, bd, EPS)[0].T
        z = h * (1 + sd[s]) + td[s]
        ys = z if act is None else (F.relu(z) if act == "relu" else F.silu(z))
        y = y.index_put((sel,), ys)
        with torch.no_grad():
            n = sel.numel() * cg
            xg = xd[sel].detach().view(-1, groups, cg)
            mean_c = xg.mean((0, 2)).repeat_interleave(cg)
            inv_c = (1.0 / torch.sqrt(xg.var((0, 2), unbiased=False) + EPS)).repeat_interleave(cg)
            xhat = (xd[sel].detach() - mean_c) * inv_c
            zs = z.detach()
            dzmag = dyd[sel].abs() * (1 + zs.abs()) * 1.1                  # |dz| and the error of act'(z)
            ge = w0 * s1[s]
            s1n = (ge * dzmag.sum(0)).view(groups, cg).sum(1).repeat_interleave(cg) / n
            s2n = (ge * (dzmag * xhat.abs()).sum(0)).view(groups, cg).sum(1).repeat_interleave(cg) / n
            cy = (w0 * inv_c * mean_c).abs() + h.detach().abs()
            cond["y"][sel] = s1[s].abs() * cy + td.detach()[s].abs()
            cond["dx"][sel] = inv_c * ((ge * dzmag).abs() + s1n + xhat.abs() * s2n)
            bsum = (dzmag * xhat).square().sum(0).sqrt() + inv_c * mean_c.abs() * dzmag.sum(0)
            asum = dzmag.square().sum(0).sqrt()
            sq["dw"] += (s1[s].abs() * bsum).square()
            sq["db"] += (s1[s].abs() * asum).square()
            cond["ds"][s] = w0.abs() * bsum + b0.abs() * asum
            cond["dt"][s] = asum
            if act == "relu":
                near = zs.abs() < 1e-5 * (1 + cond["y"][sel])
                amb[sel] = near
                flip = torch.where(near, dyd[sel].abs(), torch.zeros_like(zs)) * 2e5    # 1e-5 * cond: twice it
                fx = (flip * xhat.abs()).sum(0)
                sq["dw"] += (s1[s].abs() * fx).square()
                sq["db"] += (s1[s].abs() * flip.sum(0)).square()
                cond["ds"][s] += w0.abs() * fx + b0.abs() * flip.sum(0)
                cond["dt"][s] += flip.sum(0)
    y.backward(dyd)
    cond["dw"], cond["db"] = sq["dw"].sqrt(), sq["db"].sqrt()
    grads = [xd.grad if xd.grad is not None else zero, wd.grad, bd.grad, sd.grad, td.grad]
    return [y.detach()] + grads, cond, amb


def _check(got, ref, cond, amb, dtype, pdt, tag):
    y, dx, dw, db, ds, dt = got
    ry, rdx, rdw, rdb, rds, rdt = ref
    assert int(amb.sum()) < 1e-4 * amb.numel() + 10, f"{int(amb.sum())} elements at the kink {tag}"
    dx = torch.where(amb, rdx.to(dx.dtype), dx)
    if dtype == torch.float32:
        _close_f32(y, ry, f"y {tag}", cond["y"])
        _close_f32(dx, rdx, f"dx {tag}", cond["dx"])
    else:
        _close_low(y, ry, dtype, f"y {tag}", cond["y"])
        _close_low(dx, rdx, dtype, f"dx {tag}", cond["dx"])
    if dw is not None:
        close = _close_f32 if pdt == torch.float32 else (lambda g, r, what, cnd: _close_low(g, r, pdt, what, cnd))
        close(dw, rdw, f"dweight {tag}", cond["dw"])
        close(db, rdb, f"dbias {tag}", cond["db"])
    if ds is not None:
        assert ds.dtype == torch.float32
        _close_f32(ds, rds, f"dscale {tag}", cond["ds"])
    if dt is not None:
        assert dt.dtype == torch.float32
        _close_f32(dt, rdt, f"dshift {tag}", cond["dt"])


@pytest.mark.parametrize("batch", BATCHES, ids=lambda t: f"B{t[0]}")
@pytest.mark.parametrize("c", [12, 64, 256])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_against_float64(dname, c, batch, cuda_dev):
    """every act with every modulation (neither / scale / shift / both), G cycling over {1, 8, C}, parameters in
    fp32 and in the feature dtype"""
    dtype = DTYPES[dname]
    b, rows, empty = batch
    x, dy, inds = _inputs(rows, c, b, empty, dtype, cuda_dev, seed=rows + c)
    gs = _groups(c)
    k = 0
    for act in ACTS:
        for which in MODS:
            groups = gs[k % len(gs)]
            pdt = dtype if k % 2 and dtype != torch.float32 else torch.float32
            w, bias = _params(c, pdt, cuda_dev, seed=k)
            scale, shift = _mod(b, c, which, cuda_dev, seed=k)
            got = _run(x, dy, inds, b, groups, w, bias, scale, shift, act)
            ref, cond, amb = _reference(x, dy, inds, b, groups, w, bias, scale, shift, act)
            tag = f"{dname} C={c} G={groups} B={b} act={act} {which} params {pdt}"
            assert got[0].dtype == dtype and got[1].dtype == dtype and got[2].dtype == pdt
            assert (got[4] is None) == (scale is None) and (got[5] is None) == (shift is None)
            _check(got, ref, cond, amb, dtype, pdt, tag)
            if empty is not None:
                for t in got[4:]:
                    assert t is None or bool((t[empty] == 0).all()), f"empty sample's dscale / dshift {tag}"
            k += 1
    # without affine parameters, SiLU and both modulations
    scale, shift = _mod(b, c, "both", cuda_dev, seed=1)
    got = _run(x, dy, inds, b, 1, None, None, scale, shift, "silu")
    ref, cond, amb = _reference(x, dy, inds, b, 1, None, None, scale, shift, "silu")
    assert got[2] is None and got[3] is None
    _check(got, ref, cond, amb, dtype, torch.float32, f"{dname} C={c} B={b} no affine")


def test_low_precision_scale_and_shift_are_computed_in_fp32(cuda_dev):
    """a bf16 / fp16 scale and shift give the results of their fp32 values, with gradients in their own dtype"""
    x, dy, inds = _inputs(3000, 64, 3, None, torch.float16, cuda_dev, seed=4)
    w, bias = _params(64, torch.float32, cuda_dev, seed=4)
    scale, shift = _mod(3, 64, "both", cuda_dev, seed=4)
    s16, t16 = scale.bfloat16(), shift.half()
    want = _run(x, dy, inds, 3, 8, w, bias, s16.float(), t16.float(), "silu")
    got = _run(x, dy, inds, 3, 8, w, bias, s16, t16, "silu")
    assert got[4].dtype == torch.bfloat16 and got[5].dtype == torch.float16
    for a, r in zip(got[:4], want[:4]):
        assert torch.equal(_bits(a), _bits(r))
    assert torch.equal(got[4], want[4].bfloat16()) and torch.equal(got[5], want[5].half())


def _torch_chain(x, dy, inds, b, groups, w, bias, scale, shift, num_valid=None):
    """what a user writes without the fused call: MaskedGroupNorm, then the gather by batch id, (1 + s), + t and
    F.silu, with autograd"""
    xr, sr, tr = x.clone().requires_grad_(True), scale.clone().requires_grad_(True), shift.clone().requires_grad_(True)
    gn = masked_group_norm(xr, w, bias, inds, b, num_valid, groups, EPS)
    ids = inds[:, 0].long()
    y = F.silu(gn * (1 + sr[ids]) + tr[ids])
    y.backward(dy)
    return y.detach(), xr.grad, sr.grad, tr.grad


@pytest.mark.parametrize("c", [12, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_padding_dropped_rows_and_repeat_are_bit_identical(dname, c, cuda_dev):
    """junk rows (NaN / Inf features and dy) with out-of-range batch ids among the kept rows, padding beyond
    num_valid and a num_valid past the end: every output, dscale and dshift included, has the bits of the call on
    the kept rows alone, for each act"""
    dtype = DTYPES[dname]
    b, rows, groups = 3, 3000, 4
    x, dy, inds = _inputs(rows, c, b, None, dtype, cuda_dev, seed=c + 1)
    w, bias = _params(c, torch.float32, cuda_dev, seed=4)
    scale, shift = _mod(b, c, "both", cuda_dev, seed=2)
    g = torch.Generator().manual_seed(9)
    n_drop = 700
    bad_ids = torch.tensor([b, b + 5, -1, -7, 1 << 30], dtype=torch.int32)[torch.randint(0, 5, (n_drop,), generator=g)]
    fd, id_ = _junk_rows(n_drop, c, dtype, cuda_dev, bad_ids.to(cuda_dev))
    ddy, _ = _junk_rows(n_drop, c, dtype, cuda_dev, bad_ids.to(cuda_dev))
    m = rows + n_drop
    pos = torch.randperm(m, generator=g)[:rows].sort().values.to(cuda_dev)
    kept = torch.zeros(m, dtype=torch.bool, device=cuda_dev)
    kept[pos] = True
    mixed_x = torch.empty((m, c), dtype=dtype, device=cuda_dev)
    mixed_dy = torch.empty_like(mixed_x)
    mixed_i = torch.empty((m, 4), dtype=torch.int32, device=cuda_dev)
    mixed_x[pos], mixed_dy[pos], mixed_i[pos] = x, dy, inds
    mixed_x[~kept], mixed_dy[~kept], mixed_i[~kept] = fd, ddy, id_
    names = ("y", "dx", "dweight", "dbias", "dscale", "dshift")
    for act in ACTS:
        base = _run(x, dy, inds, b, groups, w, bias, scale, shift, act)
        again = _run(x, dy, inds, b, groups, w, bias, scale, shift, act)
        for a, r, name in zip(again, base, names):
            assert torch.equal(_bits(a), _bits(r)), f"repeat {name} {act}"
        for total in (m, m + 1, m + 777):
            pad = total - m
            jx, ji = _junk_rows(pad, c, dtype, cuda_dev, torch.randint(-2, b + 2, (pad,), generator=g).to(cuda_dev))
            jdy, _ = _junk_rows(pad, c, dtype, cuda_dev, ji[:, 0])
            px, pdy, pi = torch.cat([mixed_x, jx]), torch.cat([mixed_dy, jdy]), torch.cat([mixed_i, ji])
            for nv_val in ((m, m + 10**6) if pad == 0 else (m,)):
                nv = torch.full((1,), nv_val, dtype=torch.int32, device=cuda_dev)
                got = _run(px, pdy, pi, b, groups, w, bias, scale, shift, act, nv)
                tag = f"{dname} C={c} act={act} rows={total} num_valid={nv_val}"
                assert torch.equal(_bits(got[0][pos]), _bits(base[0])), f"y {tag}"
                assert torch.equal(_bits(got[1][pos]), _bits(base[1])), f"dx {tag}"
                for a, r, name in zip(got[2:], base[2:], names[2:]):
                    assert torch.equal(_bits(a), _bits(r)), f"{name} {tag}"
                dropped = torch.ones(total, dtype=torch.bool, device=cuda_dev)
                dropped[pos] = False
                for t, name in ((got[0], "y"), (got[1], "dx")):
                    z = t[dropped]
                    assert bool((z == 0).all()) and not bool(z.signbit().any()), f"{name} dropped rows {tag}"


def test_padding_never_reaches_the_last_sample(cuda_dev):
    """pad_to's rows carry batch id -1: the torch formulation gathers shift[-1] = shift[B - 1] for them, so they
    leave the norm as silu(shift[B - 1]) instead of 0 and their dy lands in dshift[B - 1]; the fused call keeps 0
    there and the unpadded bits of every gradient"""
    b, rows, c, groups, pad = 3, 2000, 64, 8, 300
    x, dy, inds = _inputs(rows, c, b, None, torch.float32, cuda_dev, seed=12)
    w, bias = _params(c, torch.float32, cuda_dev, seed=12)
    scale, shift = _mod(b, c, "both", cuda_dev, seed=12)
    padded = spconv.SparseConvTensor(x, inds, [50, 50, 50], b).pad_to(rows + pad)
    pdy = torch.cat([dy, torch.randn((pad, c), device=cuda_dev)])
    want = _run(x, dy, inds, b, groups, w, bias, scale, shift, "silu")
    got = _run(padded.features, pdy, padded.indices, b, groups, w, bias, scale, shift, "silu", padded.num_valid)
    for a, r in zip(got[2:], want[2:]):
        assert torch.equal(_bits(a), _bits(r))
    assert bool((got[0][rows:] == 0).all()) and bool((got[1][rows:] == 0).all())
    chain = _torch_chain(padded.features, pdy, padded.indices, b, groups, w, bias, scale, shift, padded.num_valid)
    chain_ref = _torch_chain(x, dy, inds, b, groups, w, bias, scale, shift)
    assert torch.equal(chain[0][rows:], F.silu(shift[b - 1]).expand(pad, c))
    err_last = float((chain[3][b - 1] - chain_ref[3][b - 1]).abs().max())
    err_rest = float((chain[3][:b - 1] - chain_ref[3][:b - 1]).abs().max())
    assert err_last > 1e-2 > err_rest * 100, (err_last, err_rest)
    # the fused call and the torch formulation agree on the unpadded tensor
    _close_f32(want[0], chain_ref[0], "y against the torch formulation", torch.full_like(want[0], 10.0))
    _close_f32(want[4], chain_ref[2], "dscale against the torch formulation", torch.full_like(want[4], 100.0))
    _close_f32(want[5], chain_ref[3], "dshift against the torch formulation", torch.full_like(want[5], 100.0))


def test_backward_reads_bias_only_where_it_is_an_operand(cuda_dev):
    """the plain backward never reads bias, nor the modulated one without an activation and without dscale: a
    NaN bias gives the bits of a NULL one there; with SiLU or dscale it is read"""
    x, dy, inds = _inputs(3000, 64, 3, None, torch.float32, cuda_dev, seed=21)
    w, bias = _params(64, torch.float32, cuda_dev, seed=21)
    scale, shift = _mod(3, 64, "both", cuda_dev, seed=21)
    nan = torch.full_like(bias, float("nan"))
    lib = _cabi.load()
    stream = torch.cuda.current_stream().cuda_stream

    def bwd(bias_bwd, act, want_dscale, mod):
        rows, c = x.shape
        _, mean, invstd, order, offsets, cstart = ops.masked_group_norm_forward(x, inds, 3, None, 8, w, bias, EPS,
                                                                                scale if mod else None,
                                                                                shift if mod else None, act)
        dx, dw, db = torch.empty_like(x), torch.empty_like(w), torch.empty_like(w)
        ds = torch.zeros((3, c), device=cuda_dev)
        m = _cabi.MaskedGroupNormMod()
        m.norm = ops._gn_desc(x, inds, 3, 8, None, ops._DTYPE_CODE[w.dtype])
        d = m.norm
        d.dy, d.dx, d.weight, d.bias, d.dweight, d.dbias = (dy.data_ptr(), dx.data_ptr(), w.data_ptr(),
                                                            bias_bwd.data_ptr(), dw.data_ptr(), db.data_ptr())
        d.mean, d.invstd, d.order, d.offsets, d.cstart = (mean.data_ptr(), invstd.data_ptr(), order.data_ptr(),
                                                          offsets.data_ptr(), cstart.data_ptr())
        ws = torch.empty(lib.spx_masked_group_norm_workspace_size(rows, 3, c), dtype=torch.uint8, device=cuda_dev)
        if mod:
            m.scale, m.shift, m.act = scale.data_ptr(), shift.data_ptr(), ops.GROUP_NORM_ACTS[act]
            m.dscale = ds.data_ptr() if want_dscale else None
            _cabi.check(lib.spx_masked_group_norm_mod_bwd(ctypes.byref(m), ws.data_ptr(), ws.numel(), stream), "bwd")
        else:
            _cabi.check(lib.spx_masked_group_norm_bwd(ctypes.byref(d), ws.data_ptr(), ws.numel(), stream), "bwd")
        return dx, dw, db, ds

    for mod in (False, True):
        want = bwd(bias, None, False, mod)
        got = bwd(nan, None, False, mod)
        for a, r in zip(got, want):
            assert torch.equal(_bits(a), _bits(r)), f"modulated={mod}"
    assert bool(bwd(nan, None, True, True)[3].isnan().any())       # dscale reads bias
    assert bool(bwd(nan, "silu", False, True)[0].isnan().any())     # z reads bias


def test_function_keeps_its_plain_call(cuda_dev):
    """MaskedGroupNormFunction.apply with the eight arguments it took before scale, shift and act"""
    from spconv_b200.pytorch.functional import MaskedGroupNormFunction
    x, dy, inds = _inputs(2000, 64, 3, None, torch.float16, cuda_dev, seed=5)
    w, bias = _params(64, torch.float32, cuda_dev, seed=5)
    want = _run(x, dy, inds, 3, 8, w, bias, None, None, None)
    xr, wr, br = (t.clone().requires_grad_(True) for t in (x, w, bias))
    y = MaskedGroupNormFunction.apply(xr, wr, br, inds, 3, None, 8, EPS)
    y.backward(dy)
    for a, r in zip((y.detach(), xr.grad, wr.grad, br.grad), want[:4]):
        assert torch.equal(_bits(a), _bits(r))


def test_neutral_modulation_equals_the_plain_call(cuda_dev):
    for dtype in DTYPES.values():
        for c, groups in ((12, 3), (64, 8), (256, 256)):
            x, dy, inds = _inputs(4000, c, 3, 1, dtype, cuda_dev, seed=c)
            w, bias = _params(c, torch.float32, cuda_dev, seed=c)
            zero = torch.zeros((3, c), device=cuda_dev)
            plain = _run(x, dy, inds, 3, groups, w, bias, None, None, None)
            neutral = _run(x, dy, inds, 3, groups, w, bias, zero, zero, None)
            for a, r, name in zip(neutral[:4], plain[:4], ("y", "dx", "dweight", "dbias")):
                assert torch.equal(a, r), f"{name} {dtype} C={c}"
            # and the plain entry points through the modulated descriptor give the plain bits
            for a, r in zip(_call(x, dy, inds, 3, groups, w, bias, None, None, 0, torch.empty_like(x),
                                  torch.empty_like(x))[:4], plain[:4]):
                assert torch.equal(_bits(a), _bits(r))


def _call(x, dy, inds, b, groups, w, bias, scale, shift, act, y_out, dx_out):
    """the modulated C entry points with caller-chosen outputs (so y and dx can sit at any address)"""
    rows, c = x.shape
    mean = torch.empty((b, groups), dtype=torch.float32, device=x.device)
    invstd = torch.empty_like(mean)
    order = torch.empty((rows,), dtype=torch.int32, device=x.device)
    offsets = torch.empty((b + 1,), dtype=torch.int32, device=x.device)
    cstart = torch.empty_like(offsets)
    dw, db = torch.empty_like(w), torch.empty_like(w)
    ds = torch.empty((b, c), dtype=torch.float32, device=x.device)
    dt = torch.empty_like(ds)
    m = _cabi.MaskedGroupNormMod()
    m.norm = ops._gn_desc(x, inds, b, groups, None, ops._DTYPE_CODE[w.dtype])
    d = m.norm
    d.eps, d.y, d.dy, d.dx, d.weight, d.bias = EPS, y_out.data_ptr(), dy.data_ptr(), dx_out.data_ptr(), \
        w.data_ptr(), bias.data_ptr()
    d.dweight, d.dbias = dw.data_ptr(), db.data_ptr()
    d.mean, d.invstd, d.order, d.offsets, d.cstart = (mean.data_ptr(), invstd.data_ptr(), order.data_ptr(),
                                                      offsets.data_ptr(), cstart.data_ptr())
    m.scale, m.shift, m.act = ops._ptr(scale), ops._ptr(shift), act
    m.dscale, m.dshift = ds.data_ptr(), dt.data_ptr()
    lib = _cabi.load()
    ws = torch.empty(lib.spx_masked_group_norm_workspace_size(rows, b, c), dtype=torch.uint8, device=x.device)
    stream = torch.cuda.current_stream().cuda_stream
    _cabi.check(lib.spx_masked_group_norm_mod_fwd(ctypes.byref(m), ws.data_ptr(), ws.numel(), stream), "fwd")
    _cabi.check(lib.spx_masked_group_norm_mod_bwd(ctypes.byref(m), ws.data_ptr(), ws.numel(), stream), "bwd")
    return y_out, dx_out, dw, db, ds, dt


@pytest.mark.parametrize("c", [12, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_misaligned_operands_give_the_same_bits(dname, c, cuda_dev):
    """x, dy, y and dx at odd element offsets, one at a time and all together, with scale, shift and each act: the
    same bits as the aligned call, dscale and dshift included"""
    dtype = DTYPES[dname]
    b, rows, groups = 3, 2000, 4
    x, dy, inds = _inputs(rows, c, b, None, dtype, cuda_dev, seed=11 + c)
    w, bias = _params(c, dtype, cuda_dev, seed=2)
    scale, shift = _mod(b, c, "both", cuda_dev, seed=3)
    names = ("y", "dx", "dweight", "dbias", "dscale", "dshift")
    for act in (_cabi.SPX_GN_ACT_NONE, _cabi.SPX_GN_ACT_RELU, _cabi.SPX_GN_ACT_SILU):
        want = _call(x, dy, inds, b, groups, w, bias, scale, shift, act, torch.empty_like(x), torch.empty_like(x))
        for off in (1, 3):
            for moved in ("x", "dy", "y", "dx", "all"):
                mv = {k: (moved in (k, "all")) for k in ("x", "dy", "y", "dx")}
                got = _call(_at_offset(x, off) if mv["x"] else x, _at_offset(dy, off) if mv["dy"] else dy, inds, b,
                            groups, w, bias, scale, shift, act,
                            _at_offset(torch.empty_like(x), off) if mv["y"] else torch.empty_like(x),
                            _at_offset(torch.empty_like(x), off) if mv["dx"] else torch.empty_like(x))
                for a, r, what in zip(got, want, names):
                    assert torch.equal(_bits(a.contiguous()), _bits(r)), \
                        f"{dname} C={c} act={act} {moved}+{off}: {what}"


def test_launch_counts(cuda_dev):
    """the modulated backward is at most 4 launches with fp32 scale / shift, and the forward launches what the
    plain forward does"""
    x, dy, inds = _inputs(5000, 64, 3, None, torch.float16, cuda_dev, seed=1)
    w, bias = _params(64, torch.float32, cuda_dev, seed=1)
    scale, shift = _mod(3, 64, "both", cuda_dev, seed=1)

    def count(fn):
        torch.cuda.synchronize()
        ops.launch_count(reset=True)
        out = fn()
        torch.cuda.synchronize()
        return ops.launch_count(reset=True), out

    leaves = [t.clone().requires_grad_(True) for t in (x, w, bias, scale, shift)]
    n_plain, _ = count(lambda: masked_group_norm(x, w, bias, inds, 3, None, 8, EPS))
    for act in ACTS:
        n_fwd, y = count(lambda: masked_group_norm(*leaves[:3], inds, 3, None, 8, EPS, leaves[3], leaves[4], act))
        assert n_fwd == n_plain, (act, n_fwd, n_plain)
        n_bwd, _ = count(lambda: y.backward(dy))
        assert n_bwd <= 4, (act, n_bwd)


class _CondNet(nn.Module):
    """SubMConv3d -> GroupNorm + SiLU -> SubMConv3d -> GroupNorm with scale / shift from a per-sample embedding MLP
    + SiLU -> SubMConv3d, plus the first block's output -> MaskedGlobalAvgPool"""

    def __init__(self, c=16, emb=8):
        super().__init__()
        torch.manual_seed(3)
        self.conv0 = spconv.SubMConv3d(4, c, 3, indice_key="s1", bias=False)
        self.norm0 = MaskedGroupNorm(4, c, act="silu")
        self.conv1 = spconv.SubMConv3d(c, c, 3, indice_key="s1", bias=False)
        self.norm1 = MaskedGroupNorm(4, c, act="silu")
        self.conv2 = spconv.SubMConv3d(c, c, 3, indice_key="s1", bias=False)
        self.mlp = nn.Sequential(nn.Linear(emb, 32), nn.SiLU(), nn.Linear(32, 2 * c))
        self.pool = MaskedGlobalAvgPool()
        with torch.no_grad():
            for m in (self.norm0, self.norm1):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.5, 0.5)

    def forward(self, x, emb):
        skip = self.norm0(self.conv0(x))
        scale, shift = self.mlp(emb).chunk(2, dim=1)
        h = self.conv2(self.norm1(self.conv1(skip), scale, shift))
        return self.pool(h.replace_feature(h.features + skip.features))


def test_conditioned_net_trains_padded_and_as_one_graph(cuda_dev):
    shape, b = [24, 48, 48], 3
    rng = np.random.default_rng(8)
    clouds = []
    for per in ([3000, 2500, 2800], [2000, 2900, 1000], [2600, 0, 2400]):
        f, i = random_cloud(rng, shape, per, 4)
        perm = rng.permutation(i.shape[0])
        clouds.append((torch.from_numpy(f[perm]).to(cuda_dev), torch.from_numpy(i[perm]).to(cuda_dev)))
    n_pad = 8_600
    net = _CondNet().to(cuda_dev)
    params = list(net.parameters())
    emb = torch.randn((b, 8), device=cuda_dev)
    target = torch.randn((b, 16), device=cuda_dev)

    def step(f, i, nv=None):
        for p in params:
            p.grad = None
        x = spconv.SparseConvTensor(f, i, shape, b)
        x.num_valid = nv
        pooled = net(x, emb)
        loss = (pooled - target).square().sum()
        loss.backward()
        return loss.detach(), [p.grad for p in params], pooled.detach()

    want = []
    for f, i in clouds:                              # eager, exact shapes
        loss, grads, pooled = step(f, i)
        want.append((loss.clone(), [g.clone() for g in grads], pooled.clone()))
    assert bool((want[2][2][1] == 0).all())          # the empty sample pools to 0
    mlp_names = [n for n, _ in net.named_parameters() if n.startswith("mlp.")]
    assert mlp_names and all(bool(g.abs().sum() > 0) for (n, _), g in zip(net.named_parameters(), want[0][1])
                             if n.startswith("mlp."))

    padded = [spconv.SparseConvTensor(f, i, shape, b).pad_to(n_pad) for f, i in clouds]
    args = [(p.features, p.indices, p.num_valid) for p in padded]

    def same(got, ref, what):
        loss, grads, pooled = got
        assert torch.equal(_bits(pooled), _bits(ref[2])), f"{what}: pooled features"
        assert torch.equal(_bits(loss), _bits(ref[0])), f"{what}: loss"
        for (name, _), g, r in zip(net.named_parameters(), grads, ref[1]):
            assert torch.equal(_bits(g), _bits(r)), (what, name)

    step(*args[0])                                   # warm-up: allocator pools
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager = [step(*a) for a in args]             # eager padded: no synchronising call
        eager = [(l.clone(), [g.clone() for g in gs], p.clone()) for l, gs, p in eager]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for k in range(3):
        same(eager[k], want[k], f"eager padded cloud {k} against unpadded")

    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 2, 1):
        same(graphed(*args[k]), eager[k], f"replay of cloud {k}")
