"""MaskedGroupNorm on the GPU: per-sample GroupNorm / InstanceNorm against the per-sample loop over F.group_norm in
float64 (and in fp32 on the GPU), bit-identical results under padding, dropped rows, misaligned operands and
repeats, the empty-sample, no-row and one-row rules, the backward's launch count, and a small net that trains
padded and replays as one CUDA graph."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from tests.util import random_cloud

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedGlobalAvgPool, MaskedGroupNorm, ops
from spconv_b200.pytorch.functional import masked_group_norm

pytestmark = pytest.mark.gpu

DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}
MANT = {torch.float16: 10, torch.bfloat16: 7}
EPS = 1e-5
# (batch_size, rows, empty sample or None)
BATCHES = [(1, 700, None), (3, 5000, 1), (8, 6000, 5)]


def _groups(c):
    """G in {1, 8, 32, C}, where G divides C"""
    return sorted({g for g in (1, 8, 32, c) if c % g == 0})


def _batch_ids(b, rows, empty, seed):
    """interleaved batch ids in [0, b), sample `empty` without rows"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, b, (rows,), generator=g, dtype=torch.int32)
    if empty is not None:
        ids[ids == empty] = (empty + 1) % b
    return ids


def _inputs(rows, c, b, empty, dtype, dev, seed):
    g = torch.Generator().manual_seed(seed)
    ids = _batch_ids(b, rows, empty, seed)
    shift = torch.rand((b, c), generator=g) * 4 - 2           # per-sample, per-channel offsets and scales
    scale = torch.rand((b, c), generator=g) * 2 + 0.25
    x = (torch.randn((rows, c), generator=g) * scale[ids.long()] + shift[ids.long()]).to(dtype)
    dy = torch.randn((rows, c), generator=g).to(dtype)
    inds = torch.zeros((rows, 4), dtype=torch.int32)
    inds[:, 0] = ids
    inds[:, 1:] = torch.randint(0, 50, (rows, 3), generator=g, dtype=torch.int32)
    return x.to(dev), dy.to(dev), inds.to(dev)


def _params(c, dtype, dev, seed, affine=True):
    if not affine:
        return None, None
    g = torch.Generator().manual_seed(seed + 1)
    return ((torch.rand(c, generator=g) + 0.5).to(dtype).to(dev), (torch.rand(c, generator=g) - 0.5).to(dtype).to(dev))


def _run(x, dy, inds, b, groups, w, bias, num_valid=None):
    xr = x.clone().requires_grad_(True)
    wr = None if w is None else w.clone().requires_grad_(True)
    br = None if bias is None else bias.clone().requires_grad_(True)
    y = masked_group_norm(xr, wr, br, inds, b, num_valid, groups, EPS)
    y.backward(dy)
    return y.detach(), xr.grad, None if wr is None else wr.grad, None if br is None else br.grad


def _reference(x, dy, inds, b, groups, w, bias):
    """the per-sample loop over F.group_norm in float64 on the (dtype-rounded) inputs, and per result the size of
    the terms that cancel in it"""
    xd, dyd = x.double(), dy.double()
    rows, c = x.shape
    cg = c // groups
    wd = w.double() if w is not None else torch.ones(c, dtype=torch.float64, device=x.device)
    bd = bias.double() if bias is not None else torch.zeros(c, dtype=torch.float64, device=x.device)
    wr, br = wd.clone().requires_grad_(True), bd.clone().requires_grad_(True)
    y = torch.zeros_like(xd)
    dx = torch.zeros_like(xd)
    cond = {k: torch.zeros_like(xd) for k in ("y", "dx")}
    dw_sq = torch.zeros(c, dtype=torch.float64, device=x.device)
    ids = inds[:, 0].long()
    for s in range(b):
        sel = (ids == s).nonzero().squeeze(1)
        if sel.numel() == 0:
            continue
        xs = xd[sel].clone().requires_grad_(True)
        ys = F.group_norm(xs.T[None], groups, wr, br, EPS)[0].T
        ys.backward(dyd[sel])
        y[sel] = ys.detach()
        dx[sel] = xs.grad
        n = sel.numel() * cg
        xg = xd[sel].view(-1, groups, cg)
        mean = xg.mean((0, 2))
        invstd = 1.0 / torch.sqrt(xg.var((0, 2), unbiased=False) + EPS)
        mean_c, inv_c = mean.repeat_interleave(cg), invstd.repeat_interleave(cg)
        xhat = (xd[sel] - mean_c) * inv_c
        s1 = (wd * dyd[sel].sum(0)).view(groups, cg).sum(1).repeat_interleave(cg)
        s2 = (wd * (dyd[sel] * xhat).sum(0)).view(groups, cg).sum(1).repeat_interleave(cg)
        cond["y"][sel] = (wd * inv_c * mean_c).abs().expand(sel.numel(), c)
        cond["dx"][sel] = inv_c * ((wd * dyd[sel]).abs() + (s1 / n).abs() + (xhat * s2 / n).abs())
        dw_sq += (dyd[sel] * xhat).square().sum(0) + (inv_c * mean_c.abs() * dyd[sel].sum(0).abs()).square()
    cond["dw"] = dw_sq.sqrt()
    cond["db"] = dyd.square().sum(0).sqrt()
    return y, dx, wr.grad, br.grad, cond


def _close_f32(got, ref, what, cond=None):
    """|got - ref| <= 1e-5 * max(1, |ref|, cond), as for MaskedBatchNorm1d: cond is the size of the terms that
    cancel (of the order of |ref| or 1 on well-conditioned data)"""
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    lim = torch.clamp(ref.abs(), min=1.0)
    if cond is not None:
        lim = torch.maximum(lim, cond)
    lim = 1e-5 * lim
    assert bool((err <= lim).all()), f"{what}: max error {float((err - lim).max()):.3e} over the limit"


def _close_low(got, ref, dtype, what, cond):
    """within one ulp of the dtype at the reference, plus 1e-5 * max(|ref|, cond) over the tensor"""
    ref = ref.double()
    _, e = torch.frexp(ref.abs().clamp(min=2.0 ** -14 if dtype == torch.float16 else 2.0 ** -126))
    ulp = torch.ldexp(torch.ones_like(ref), (e - 1 - MANT[dtype]).to(torch.int32))
    err = (got.double() - ref).abs()
    lim = ulp + 1e-5 * max(float(ref.abs().max()), float(cond.max()))
    assert bool((err <= lim).all()), f"{what}: max error {float((err - lim).max()):.3e} over the limit"


@pytest.mark.parametrize("batch", BATCHES, ids=lambda t: f"B{t[0]}")
@pytest.mark.parametrize("c", [12, 64, 256])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_against_float64(dname, c, batch, cuda_dev):
    dtype = DTYPES[dname]
    b, rows, empty = batch
    x, dy, inds = _inputs(rows, c, b, empty, dtype, cuda_dev, seed=rows + c)
    for gi, groups in enumerate(_groups(c)):
        for pdt in ((torch.float32, dtype) if dtype != torch.float32 else (torch.float32,)):
            w, bias = _params(c, pdt, cuda_dev, seed=gi)
            y, dx, dw, db = _run(x, dy, inds, b, groups, w, bias)
            ry, rdx, rdw, rdb, cond = _reference(x, dy, inds, b, groups, w, bias)
            tag = f"{dname} C={c} G={groups} B={b} params {pdt}"
            assert y.dtype == dtype and dx.dtype == dtype and dw.dtype == pdt and db.dtype == pdt
            if dtype == torch.float32:
                _close_f32(y, ry, f"y {tag}", cond["y"])
                _close_f32(dx, rdx, f"dx {tag}", cond["dx"])
            else:
                _close_low(y, ry, dtype, f"y {tag}", cond["y"])
                _close_low(dx, rdx, dtype, f"dx {tag}", cond["dx"])
            if pdt == torch.float32:
                _close_f32(dw, rdw, f"dweight {tag}", cond["dw"])
                _close_f32(db, rdb, f"dbias {tag}", cond["db"])
            else:
                _close_low(dw, rdw, pdt, f"dweight {tag}", cond["dw"])
                _close_low(db, rdb, pdt, f"dbias {tag}", cond["db"])
    # without affine parameters: weight 1, bias 0, no parameter gradients
    y, dx, dw, db = _run(x, dy, inds, b, 1, None, None)
    ry, rdx, _, _, cond = _reference(x, dy, inds, b, 1, None, None)
    assert dw is None and db is None
    if dtype == torch.float32:
        _close_f32(y, ry, "y no affine", cond["y"])
        _close_f32(dx, rdx, "dx no affine", cond["dx"])


@pytest.mark.parametrize("batch", BATCHES[1:], ids=lambda t: f"B{t[0]}")
@pytest.mark.parametrize("c", [12, 64, 256])
def test_fp32_against_torch_group_norm(c, batch, cuda_dev):
    """the module against torch's own F.group_norm per sample on the GPU, in fp32"""
    b, rows, empty = batch
    x, dy, inds = _inputs(rows, c, b, empty, torch.float32, cuda_dev, seed=3 * rows + c)
    for groups in _groups(c):
        ref = nn.GroupNorm(groups, c, EPS).to(cuda_dev)
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5)
            ref.bias.uniform_(-0.5, 0.5)
        mod = MaskedGroupNorm(groups, c, EPS).to(cuda_dev)
        mod.load_state_dict(ref.state_dict())
        xm = x.clone().requires_grad_(True)
        y = mod(spconv.SparseConvTensor(xm, inds, [50, 50, 50], b)).features
        y.backward(dy)
        xr = x.clone().requires_grad_(True)
        yr = torch.zeros_like(x)
        for s in range(b):
            sel = (inds[:, 0] == s).nonzero().squeeze(1)
            if sel.numel():
                yr = yr.index_put((sel,), ref(xr[sel].T[None])[0].T)
        yr.backward(dy)
        cond = _reference(x, dy, inds, b, groups, ref.weight.detach(), ref.bias.detach())[4]
        tag = f"C={c} G={groups} B={b}"
        _close_f32(y, yr, f"y {tag}", cond["y"])
        _close_f32(xm.grad, xr.grad, f"dx {tag}", cond["dx"])
        _close_f32(mod.weight.grad, ref.weight.grad, f"dweight {tag}", cond["dw"])
        _close_f32(mod.bias.grad, ref.bias.grad, f"dbias {tag}", cond["db"])


def _junk_rows(n, c, dtype, dev, ids):
    """n rows of NaN / +Inf / huge features with the given batch ids"""
    vals = torch.tensor([float("nan"), float("inf"), -3e4 if dtype == torch.float16 else -3e38], dtype=dtype)
    f = vals.repeat(n * c // 3 + 3)[:n * c].view(n, c).to(dev)
    inds = torch.full((n, 4), 7, dtype=torch.int32, device=dev)
    inds[:, 0] = ids
    return f, inds


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


@pytest.mark.parametrize("c", [12, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_padding_dropped_rows_and_repeat_are_bit_identical(dname, c, cuda_dev):
    dtype = DTYPES[dname]
    b, rows = 3, 3000
    x, dy, inds = _inputs(rows, c, b, None, dtype, cuda_dev, seed=c + 1)
    w, bias = _params(c, dtype, cuda_dev, seed=4)
    groups = 4
    base = _run(x, dy, inds, b, groups, w, bias)
    assert torch.equal(_bits(base[0]), _bits(_run(x, dy, inds, b, groups, w, bias)[0]))     # repeat
    g = torch.Generator().manual_seed(9)
    # valid rows with batch ids >= B or < 0 inserted among the kept ones
    n_drop = 700
    bad_ids = torch.tensor([b, b + 5, -1, -7, 1 << 30], dtype=torch.int32)[torch.randint(0, 5, (n_drop,), generator=g)]
    fd, id_ = _junk_rows(n_drop, c, dtype, cuda_dev, bad_ids.to(cuda_dev))
    ddy, _ = _junk_rows(n_drop, c, dtype, cuda_dev, bad_ids.to(cuda_dev))
    perm = torch.randperm(rows + n_drop, generator=g).to(cuda_dev)
    # keep the kept rows in their order: place them at the sorted positions of a random subset
    pos = perm[:rows].sort().values
    mixed_x = torch.empty((rows + n_drop, c), dtype=dtype, device=cuda_dev)
    mixed_dy = torch.empty_like(mixed_x)
    mixed_i = torch.empty((rows + n_drop, 4), dtype=torch.int32, device=cuda_dev)
    is_kept = torch.zeros(rows + n_drop, dtype=torch.bool, device=cuda_dev)
    is_kept[pos] = True
    mixed_x[pos], mixed_dy[pos], mixed_i[pos] = x, dy, inds
    mixed_x[~is_kept], mixed_dy[~is_kept], mixed_i[~is_kept] = fd, ddy, id_
    m = rows + n_drop
    for total in (m, m + 1, m + 777):
        pad = total - m
        jx, ji = _junk_rows(pad, c, dtype, cuda_dev, torch.randint(-2, b + 2, (pad,), generator=g).to(cuda_dev))
        jdy, _ = _junk_rows(pad, c, dtype, cuda_dev, ji[:, 0])
        px, pdy, pi = torch.cat([mixed_x, jx]), torch.cat([mixed_dy, jdy]), torch.cat([mixed_i, ji])
        for nv_val in ((m, m + 10**6) if pad == 0 else (m,)):      # num_valid beyond rows is clamped
            nv = torch.full((1,), nv_val, dtype=torch.int32, device=cuda_dev)
            y, dx, dw, db = _run(px, pdy, pi, b, groups, w, bias, nv)
            tag = f"{dname} C={c} rows={total} num_valid={nv_val}"
            assert torch.equal(_bits(y[pos]), _bits(base[0])), f"y {tag}"
            assert torch.equal(_bits(dx[pos]), _bits(base[1])), f"dx {tag}"
            assert torch.equal(_bits(dw), _bits(base[2])) and torch.equal(_bits(db), _bits(base[3])), f"dw/db {tag}"
            dropped = torch.ones(total, dtype=torch.bool, device=cuda_dev)
            dropped[pos] = False
            for t, name in ((y, "y"), (dx, "dx")):
                z = t[dropped]
                assert bool((z == 0).all()) and not bool(z.signbit().any()), f"{name} dropped rows {tag}"


@pytest.mark.parametrize("dname", list(DTYPES))
def test_edge_cases(dname, cuda_dev):
    dtype = DTYPES[dname]
    c = 16
    x, dy, inds = _inputs(40, c, 4, None, dtype, cuda_dev, seed=5)
    w, bias = _params(c, dtype, cuda_dev, seed=6)
    # M = 0: y = 0 and every gradient 0
    nv = torch.zeros((1,), dtype=torch.int32, device=cuda_dev)
    y, dx, dw, db = _run(x, dy, inds, 4, 4, w, bias, nv)
    for t in (y, dx, dw, db):
        assert bool((t == 0).all())
    # empty samples (0 and 3): the others equal the call on their rows alone, bit for bit
    ids = inds[:, 0].clone()
    ids[ids == 0], ids[ids == 3] = 1, 2
    i2 = inds.clone()
    i2[:, 0] = ids
    got = _run(x, dy, i2, 4, 4, w, bias)
    i3 = i2.clone()
    i3[:, 0] -= 1
    want = _run(x, dy, i3, 2, 4, w, bias)
    for a, b_ in zip(got, want):
        assert torch.equal(_bits(a), _bits(b_))
    ry, rdx, rdw, rdb, cond = _reference(x, dy, i2, 4, 4, w, bias)
    if dtype == torch.float32:
        _close_f32(got[0], ry, "y, empty samples", cond["y"])
        _close_f32(got[1], rdx, "dx, empty samples", cond["dx"])
    # one row with Cg = 1 (InstanceNorm): x_hat = 0, y = bias, dx = 0, dbias = dy, dweight = 0
    one = inds[:1].clone()
    one[0, 0] = 2
    y, dx, dw, db = _run(x[:1], dy[:1], one, 3, c, w, bias)
    assert torch.equal(_bits(y[0]), _bits(bias)) and bool((dx == 0).all())
    assert torch.equal(db, dy[0]) and bool((dw == 0).all())
    # torch's own kernel agrees up to its rounding of x - mean (F.group_norm refuses one value per group in Python
    # before reaching it)
    yr = torch.group_norm(x[:1].double().T[None], c, w.double(), bias.double(), EPS)[0].T
    assert float((yr[0] - bias.double()).abs().max()) < 1e-9


def _call(x, dy, inds, b, groups, w, bias, y_out=None, dx_out=None):
    """the C entry points with caller-chosen outputs (so y and dx can sit at any address)"""
    from spconv_b200 import _cabi
    rows, c = x.shape
    code = ops._DTYPE_CODE[w.dtype]
    mean = torch.empty((b, groups), dtype=torch.float32, device=x.device)
    invstd = torch.empty_like(mean)
    order = torch.empty((rows,), dtype=torch.int32, device=x.device)
    offsets = torch.empty((b + 1,), dtype=torch.int32, device=x.device)
    cstart = torch.empty_like(offsets)
    d = ops._gn_desc(x, inds, b, groups, None, code)
    d.eps, d.y, d.dy, d.dx, d.weight, d.bias = EPS, y_out.data_ptr(), dy.data_ptr(), dx_out.data_ptr(), \
        w.data_ptr(), bias.data_ptr()
    dw = torch.empty_like(w)
    db = torch.empty_like(w)
    d.dweight, d.dbias = dw.data_ptr(), db.data_ptr()
    d.mean, d.invstd, d.order, d.offsets, d.cstart = (mean.data_ptr(), invstd.data_ptr(), order.data_ptr(),
                                                      offsets.data_ptr(), cstart.data_ptr())
    lib = _cabi.load()
    ws = torch.empty(lib.spx_masked_group_norm_workspace_size(rows, b, c), dtype=torch.uint8, device=x.device)
    stream = torch.cuda.current_stream().cuda_stream
    import ctypes
    _cabi.check(lib.spx_masked_group_norm_fwd(ctypes.byref(d), ws.data_ptr(), ws.numel(), stream), "fwd")
    _cabi.check(lib.spx_masked_group_norm_bwd(ctypes.byref(d), ws.data_ptr(), ws.numel(), stream), "bwd")
    return y_out, dx_out, dw, db


def _at_offset(t, off):
    """a contiguous copy of t starting `off` elements into a fresh buffer"""
    buf = torch.zeros(t.numel() + off + 8, dtype=t.dtype, device=t.device)
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("c", [12, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_misaligned_operands_give_the_same_bits(dname, c, cuda_dev):
    """x, dy, y and dx at odd element offsets, one at a time and all together: the same bits as the aligned call
    (16-byte vector path for C = 64, element path for C = 12 in 16-bit types), through the C entry points and
    through autograd"""
    dtype = DTYPES[dname]
    b, rows, groups = 3, 2000, 4
    x, dy, inds = _inputs(rows, c, b, None, dtype, cuda_dev, seed=11 + c)
    w, bias = _params(c, dtype, cuda_dev, seed=2)
    want = _call(x, dy, inds, b, groups, w, bias, torch.empty_like(x), torch.empty_like(x))
    for off in (1, 3):
        for moved in ("x", "dy", "y", "dx", "all"):
            ops_ = {k: (moved in (k, "all")) for k in ("x", "dy", "y", "dx")}
            got = _call(_at_offset(x, off) if ops_["x"] else x, _at_offset(dy, off) if ops_["dy"] else dy, inds, b,
                        groups, w, bias, _at_offset(torch.empty_like(x), off) if ops_["y"] else torch.empty_like(x),
                        _at_offset(torch.empty_like(x), off) if ops_["dx"] else torch.empty_like(x))
            for a, r, what in zip(got, want, ("y", "dx", "dweight", "dbias")):
                assert torch.equal(_bits(a.contiguous()), _bits(r)), f"{dname} C={c} {moved}+{off}: {what}"
    # autograd: x and dy at an odd offset (a slice of a torch.cat)
    ref = _run(x, dy, inds, b, groups, w, bias)
    got = _run(_at_offset(x, 1), _at_offset(dy, 1), inds, b, groups, w, bias)
    for a, r in zip(got, ref):
        assert torch.equal(_bits(a), _bits(r))


def test_backward_launches_at_most_four_kernels(cuda_dev):
    x, dy, inds = _inputs(5000, 64, 3, None, torch.float16, cuda_dev, seed=1)
    w, bias = _params(64, torch.float32, cuda_dev, seed=1)
    xr = x.clone().requires_grad_(True)
    wr, br = w.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    y = masked_group_norm(xr, wr, br, inds, 3, None, 8, EPS)
    torch.cuda.synchronize()
    ops.launch_count(reset=True)
    y.backward(dy)
    torch.cuda.synchronize()
    assert ops.launch_count() <= 4


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.body = spconv.SparseSequential(
            spconv.SubMConv3d(4, 16, 3, indice_key="s1", bias=False), MaskedGroupNorm(4, 16), nn.ReLU(),
            spconv.SparseConv3d(16, 32, 3, stride=2, padding=1, bias=False, indice_key="d1"),
            MaskedGroupNorm(8, 32),
            spconv.SparseInverseConv3d(32, 16, 3, indice_key="d1", bias=False), MaskedGroupNorm(16, 16))
        self.pool = MaskedGlobalAvgPool()

    def forward(self, x):
        return self.pool(self.body(x))


def test_small_net_trains_padded_and_as_one_graph(cuda_dev):
    shape, b = [24, 48, 48], 3
    rng = np.random.default_rng(6)
    clouds = []
    for per in ([3000, 2500, 2800], [2000, 2900, 1000], [2600, 0, 2400]):
        f, i = random_cloud(rng, shape, per, 4)
        perm = rng.permutation(i.shape[0])
        clouds.append((torch.from_numpy(f[perm]).to(cuda_dev), torch.from_numpy(i[perm]).to(cuda_dev)))
    n_pad = 8_600
    net = _Net().to(cuda_dev)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, MaskedGroupNorm):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.5, 0.5)
    params = list(net.parameters())
    target = torch.randn((b, 16), device=cuda_dev)

    def step(f, i, nv=None):
        for p in params:
            p.grad = None
        x = spconv.SparseConvTensor(f, i, shape, b)
        x.num_valid = nv
        pooled = net(x)
        loss = (pooled - target).square().sum()
        loss.backward()
        return loss.detach(), [p.grad for p in params], pooled.detach()

    want = []
    for f, i in clouds:                              # eager, exact shapes
        loss, grads, pooled = step(f, i)
        want.append((loss.clone(), [g.clone() for g in grads], pooled.clone()))
    assert bool((want[2][2][1] == 0).all())          # the empty sample pools to 0

    net.eval()
    spconv.set_output_bounds(net.body, spconv.SparseConvTensor(*clouds[0], shape, b), margin=1.25)
    net.train()
    padded = [spconv.SparseConvTensor(f, i, shape, b).pad_to(n_pad) for f, i in clouds]
    args = [(p.features, p.indices, p.num_valid) for p in padded]

    def same(got, ref, what):
        loss, grads, pooled = got
        assert torch.equal(_bits(pooled), _bits(ref[2])), f"{what}: pooled features"
        assert torch.equal(_bits(loss), _bits(ref[0])), f"{what}: loss"
        for (name, _), g, r in zip(net.named_parameters(), grads, ref[1]):
            assert torch.equal(_bits(g), _bits(r)), (what, name)

    step(*args[0])                                   # warm-up: allocator pools, status words
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager = [step(*a) for a in args]             # eager bounded: no synchronising call
        eager = [(l.clone(), [g.clone() for g in gs], p.clone()) for l, gs, p in eager]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for k in range(3):
        same(eager[k], want[k], f"eager padded cloud {k} against unpadded")

    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 2, 1):
        same(graphed(*args[k]), eager[k], f"replay of cloud {k}")
    spconv.check_bounds(net.body)
