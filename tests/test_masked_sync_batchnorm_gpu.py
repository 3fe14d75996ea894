"""MaskedSyncBatchNorm1d on the GPU.

Simulated ranks are streams of one GPU whose exchange buffers all live on it (``PeerGroup.local_ring``), driven
like the data-parallel tests: every rank's call is launched before any host synchronisation, because each
rank's exchange waits for the others on the device.

  * one rank (the peer route at world 1 and the route without a group) equals MaskedBatchNorm1d bit for bit;
  * 2, 3, 4 and 8 ranks: y, dx and the statistics against float64 BatchNorm over the valid rows of all ranks,
    dweight / dbias against each rank's own float64 sums, the statistics and running stats bit-identical on
    every rank, and every result unchanged by padding and by a second run;
  * a rank without rows, and totals of zero and one row;
  * operands at misaligned addresses give the aligned call's bits;
  * a training step SubM -> BN -> ReLU -> bounded SparseConv3d -> BN -> SubM, captured per rank and replayed by
    all ranks together, against a float64 twin and against the eager step bit for bit;
  * with two GPUs, two processes: the peer route and the NCCL route give the same bits.
"""
import contextlib
import copy
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

from tests import net_ref
from tests.conv_ref import SparseConvRef
from tests.test_masked_batchnorm_gpu import CONFIGS, DTYPES, _close_f32, _close_low, _inputs, _module
from tests.util import random_cloud

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedSyncBatchNorm1d, ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _no_group():
    yield
    ops.set_peer_group(None)


@contextlib.contextmanager
def _ring(world, capacity_bytes=1 << 20):
    from spconv_b200.pytorch.dist import PeerGroup
    ring = PeerGroup.local_ring(world, capacity_bytes=capacity_bytes)
    try:
        yield ring
        errors = [pg.error() for pg in ring]
        assert errors == [0] * world, f"an exchange timed out: error words {errors}"
    finally:
        for pg in ring:
            pg.close()


def _round(ring, streams, fn):
    """fn(rank) on every rank's stream with its group installed, without a host synchronisation between ranks.
    Every kernel fn launches must have run once in this process before: the first launch of a kernel loads its
    module, which waits for the device, and so for a rank's exchange that waits for ranks not launched yet."""
    torch.cuda.synchronize()
    out = []
    for r, pg in enumerate(ring):
        ops.set_peer_group(pg)
        with torch.cuda.stream(streams[r]):
            out.append(fn(r))
    ops.set_peer_group(None)
    torch.cuda.synchronize()
    return out


def _load(fn):
    """fn() once on a one-rank group, so that every kernel it launches is loaded (see _round)"""
    with _ring(1) as one:
        _round(one, [torch.cuda.current_stream()], lambda r: fn())


def _bufs(bn):
    return (bn.weight, bn.bias, bn.running_mean if bn.track_running_stats else None,
            bn.running_var if bn.track_running_stats else None,
            bn.num_batches_tracked if bn.track_running_stats else None)


def _plain(bn, x, dy, nv):
    """MaskedBatchNorm1d's ops: y, mean, invstd, dx, dweight, dbias"""
    w, b, rm, rv, nbt = _bufs(bn)
    if nbt is not None:
        nbt.add_(1)
    y, mean, invstd = ops.masked_batch_norm_forward(x, nv, w, b, rm, rv, nbt, bn.momentum, bn.eps)
    dx, dw, db = ops.masked_batch_norm_backward(x, dy, nv, w, mean, invstd, w is not None, b is not None)
    return [y, mean, invstd, dx, dw, db]


def _sync_fwd(bn, x, nv):
    w, b, rm, rv, nbt = _bufs(bn)
    if nbt is not None:
        nbt.add_(1)
    t = ops.sync_bn_transport()
    return ops.masked_sync_batch_norm_forward(x, nv, w, b, rm, rv, nbt, bn.momentum, bn.eps, t) + (t,)


def _sync_bwd(bn, x, dy, nv, fwd):
    y, mean, invstd, t = fwd
    dx, dw, db = ops.masked_sync_batch_norm_backward(x, dy, nv, bn.weight, mean, invstd, t, bn.weight is not None,
                                                     bn.bias is not None)
    return [y, mean, invstd, dx, dw, db]


def _same(a, b, what):
    for i, (u, v) in enumerate(zip(a, b)):
        if u is None or v is None:
            assert u is None and v is None, (what, i)
            continue
        assert u.dtype == v.dtype and u.shape == v.shape, (what, i)
        assert torch.equal(u.reshape(-1).view(torch.uint8), v.reshape(-1).view(torch.uint8)), (what, i)


def _padded(x, rows, value=float("nan")):
    if rows == x.shape[0]:
        return x                                           # keeps the caller's address
    return torch.cat([x, torch.full((rows - x.shape[0], x.shape[1]), value, dtype=x.dtype, device=x.device)])


# ------------------------------------------------------------------ one rank
@pytest.mark.parametrize("c", [12, 64, 128])
@pytest.mark.parametrize("pname", ["fp32", "same"])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_world_of_one_equals_masked_batchnorm_bit_for_bit(dname, pname, c, cuda_dev):
    dtype = DTYPES[dname]
    pdt = torch.float32 if pname == "fp32" else dtype
    for m, rows in ((1500, 2100), (2, 2), (1, 600), (0, 8)):
        x, dy = _inputs(max(m, 1), c, dtype, cuda_dev, seed=m + c)
        x, dy = _padded(x[:m], rows), _padded(dy[:m], rows, 1.0)
        nv = torch.tensor([m], dtype=torch.int32, device=cuda_dev)
        for ci, cfg in enumerate(CONFIGS):
            base = _module(c, cfg, dtype, cuda_dev, seed=ci).to(pdt)
            ref_bn = copy.deepcopy(base)
            want = _plain(ref_bn, x, dy, nv)
            tag = f"{dname} {pname} C={c} M={m} {cfg}"
            bn = copy.deepcopy(base)
            _same(_sync_bwd(bn, x, dy, nv, _sync_fwd(bn, x, nv)), want, f"no group {tag}")
            _same(list(bn.buffers()), list(ref_bn.buffers()), f"no group buffers {tag}")
            with _ring(1) as ring:
                bn = copy.deepcopy(base)
                got = _round(ring, [torch.cuda.current_stream()],
                             lambda r: _sync_bwd(bn, x, dy, nv, _sync_fwd(bn, x, nv)))[0]
            _same(got, want, f"peer {tag}")
            _same(list(bn.buffers()), list(ref_bn.buffers()), f"peer buffers {tag}")


def test_module_world_of_one_equals_masked_batchnorm(cuda_dev):
    x, dy = _inputs(3000, 64, torch.float16, cuda_dev, seed=5)
    inds = torch.zeros((3000, 4), dtype=torch.int32, device=cuda_dev)
    plain = spconv.MaskedBatchNorm1d(64, momentum=None).to(cuda_dev)
    sync = MaskedSyncBatchNorm1d(64, momentum=None).to(cuda_dev)
    sync.load_state_dict(plain.state_dict())
    outs = []
    for bn in (plain, sync):
        xr = x.clone().requires_grad_(True)
        t = spconv.SparseConvTensor(xr, inds, [4, 4, 4], 1).pad_to(3500)
        y = bn(t).features
        y.backward(_padded(dy, 3500, 0.0))
        outs.append([y, xr.grad, bn.weight.grad, bn.bias.grad, *bn.buffers()])
    _same(outs[1], outs[0], "module")


# ------------------------------------------------------------------ several ranks
def _reference(xs, dys, bn, nbt_after):
    """float64 BatchNorm over the valid rows of every rank: per-rank y and dx, the global mean / var, running
    stats, per-rank dweight / dbias, and per-rank bounds of the terms that cancel (test_masked_batchnorm_gpu)"""
    xd = torch.cat(xs).double()
    dyd = torch.cat(dys).double()
    m = xd.shape[0]
    mean, var = xd.mean(0), xd.var(0, unbiased=False)
    invstd = 1.0 / torch.sqrt(var + bn.eps)
    xhat = (xd - mean) * invstd
    w = bn.weight.double() if bn.affine else torch.ones_like(mean)
    b = bn.bias.double() if bn.affine else torch.zeros_like(mean)
    db, dw = dyd.sum(0), (dyd * xhat).sum(0)
    y = xhat * w + b
    dx = w * invstd * (dyd - db / m - xhat * dw / m)
    a = (w * invstd).abs()
    cond_y = (a * mean.abs()).expand_as(y)
    cond_dx = a * (dyd.abs() + (db / m).abs() + (xhat * dw / m).abs())
    run = None
    if bn.track_running_stats and m > 1:
        f = 1.0 / nbt_after if bn.momentum is None else bn.momentum
        run = ((1 - f) * bn.running_mean.double() + f * mean, (1 - f) * bn.running_var.double() + f * var * m / (m - 1))
    per, o = [], 0
    for xr, dr in zip(xs, dys):
        n = xr.shape[0]
        s = slice(o, o + n)
        dyr, xh = dyd[s], xhat[s]
        per.append({"y": y[s], "dx": dx[s], "cy": cond_y[s], "cdx": cond_dx[s], "db": dyr.sum(0),
                    "dw": (dyr * xh).sum(0), "cdb": dyr.square().sum(0).sqrt(),
                    "cdw": (dyr * xh).square().sum(0).sqrt() + invstd * mean.abs() * dyr.abs().sum(0)})
        o += n
    return mean, invstd, run, per


def _ranks(world, c, dtype, dev, seed, counts=None):
    rng = np.random.default_rng(seed)
    counts = counts or [int(v) for v in rng.integers(1, 1400, world)]
    xs, dys = [], []
    for r, m in enumerate(counts):
        x, dy = _inputs(max(m, 1), c, dtype, dev, seed=seed * 31 + r)
        xs.append(x[:m])
        dys.append(dy[:m])
    return counts, xs, dys


def _valid(res, n):
    """y, mean, invstd, dx, dweight, dbias with y and dx cut to the valid rows"""
    return [res[0][:n], res[1], res[2], res[3][:n], res[4], res[5]]


def _sync_round(ring, streams, bns, xs, dys, pads):
    """forward of every rank, then backward of every rank; rank r's features padded by pads[r] rows"""
    world = len(ring)
    xp = [_padded(xs[r], xs[r].shape[0] + pads[r]) for r in range(world)]
    dp = [_padded(dys[r], dys[r].shape[0] + pads[r], 3.0) for r in range(world)]
    nv = [torch.tensor([xs[r].shape[0]], dtype=torch.int32, device=xs[r].device) for r in range(world)]
    _load(lambda: [_sync_bwd(b, xp[r], dp[r], nv[r], _sync_fwd(b, xp[r], nv[r]))
                   for r, b in enumerate(copy.deepcopy(bns))])
    fwd = _round(ring, streams, lambda r: _sync_fwd(bns[r], xp[r], nv[r]))
    res = _round(ring, streams, lambda r: _sync_bwd(bns[r], xp[r], dp[r], nv[r], fwd[r]))
    for r, out in enumerate(res):
        n = xs[r].shape[0]
        assert not out[0][n:].any() and not out[3][n:].any(), f"rank {r}: padding rows of y / dx are not 0"
    return res


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("c", [12, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_ranks_against_float64(dname, c, world, cuda_dev):
    dtype = DTYPES[dname]
    counts, xs, dys = _ranks(world, c, dtype, cuda_dev, seed=world * 10 + c)
    if world >= 4:
        counts[1] = 0                                       # a rank without rows joins every exchange
        xs[1], dys[1] = xs[1][:0], dys[1][:0]
    streams = [torch.cuda.Stream() for _ in range(world)]
    for ci, cfg in enumerate(CONFIGS):
        base = _module(c, cfg, dtype, cuda_dev, seed=ci)
        nbt_after = int(base.num_batches_tracked) + 1 if base.track_running_stats else None
        mean, invstd, run, per = _reference(xs, dys, base, nbt_after)
        with _ring(world) as ring:
            bns = [copy.deepcopy(base) for _ in range(world)]
            res = _sync_round(ring, streams, bns, xs, dys, [0] * world)
            bns2 = [copy.deepcopy(base) for _ in range(world)]
            res2 = _sync_round(ring, streams, bns2, xs, dys, [7 + 300 * r for r in range(world)])
        tag = f"{dname} C={c} world={world} {cfg}"
        for r in range(world):
            _same(_valid(res2[r], counts[r]), _valid(res[r], counts[r]), f"padding {tag} rank {r}")
            _same(list(bns2[r].buffers()), list(bns[r].buffers()), f"padding buffers {tag} rank {r}")
            _same(res[r][1:3], res[0][1:3], f"statistics {tag} rank {r}")
            _same(list(bns[r].buffers()), list(bns[0].buffers()), f"running stats {tag} rank {r}")
        _close_f32(res[0][1], mean, f"mean {tag}")
        _close_f32(res[0][2], invstd, f"invstd {tag}", invstd.abs())
        if run is not None:
            _close_f32(bns[0].running_mean, run[0], f"running_mean {tag}")
            _close_f32(bns[0].running_var, run[1], f"running_var {tag}")
        for r in range(world):
            y, _, _, dx, dw, db = res[r]
            n = counts[r]
            p = per[r]
            if dtype == torch.float32:
                _close_f32(y[:n], p["y"], f"y {tag} rank {r}", p["cy"])
                _close_f32(dx[:n], p["dx"], f"dx {tag} rank {r}", p["cdx"])
            elif n:
                _close_low(y[:n], p["y"], dtype, f"y {tag} rank {r}", p["cy"])
                _close_low(dx[:n], p["dx"], dtype, f"dx {tag} rank {r}", p["cdx"])
            if base.affine:
                _close_f32(dw, p["dw"], f"dweight {tag} rank {r}", p["cdw"])
                _close_f32(db, p["db"], f"dbias {tag} rank {r}", p["cdb"])
                if n == 0:
                    assert not dw.any() and not db.any()


def test_repeat_runs_are_bit_identical(cuda_dev):
    world, c = 4, 64
    _, xs, dys = _ranks(world, c, torch.float16, cuda_dev, seed=3)
    streams = [torch.cuda.Stream() for _ in range(world)]
    base = _module(c, CONFIGS[0], torch.float16, cuda_dev, seed=0)
    with _ring(world) as ring:
        runs = []
        for _ in range(2):
            bns = [copy.deepcopy(base) for _ in range(world)]
            runs.append((_sync_round(ring, streams, bns, xs, dys, [5] * world), bns))
    for r in range(world):
        _same(runs[1][0][r], runs[0][0][r], f"repeat rank {r}")
        _same(list(runs[1][1][r].buffers()), list(runs[0][1][r].buffers()), f"repeat buffers rank {r}")


@pytest.mark.parametrize("counts", [[0, 0, 0], [0, 1, 0], [0, 0, 2]])
def test_totals_of_zero_one_and_two_rows(counts, cuda_dev):
    """M = 0: y = 0, dx = 0, dweight = dbias = 0, running stats unchanged; M = 1: y = bias, dx = 0, dbias = dy,
    dweight = 0, running stats unchanged (MaskedBatchNorm1d's rules); M = 2 updates them"""
    world, c = len(counts), 16
    _, xs, dys = _ranks(world, c, torch.float32, cuda_dev, seed=11, counts=counts)
    base = _module(c, CONFIGS[0], torch.float32, cuda_dev, seed=0)
    streams = [torch.cuda.Stream() for _ in range(world)]
    with _ring(world) as ring:
        bns = [copy.deepcopy(base) for _ in range(world)]
        res = _sync_round(ring, streams, bns, xs, dys, [4] * world)
    one = copy.deepcopy(base)
    total = sum(counts)
    x = torch.cat(xs)
    dy = torch.cat(dys)
    want = _plain(one, _padded(x, total + 4), _padded(dy, total + 4, 3.0),
                  torch.tensor([total], dtype=torch.int32, device=cuda_dev))
    _same(res[0][1:3], want[1:3], "statistics equal one rank holding every row")
    for r in range(world):
        _same(list(bns[r].buffers()), list(one.buffers()), f"running stats rank {r}")
        n = counts[r]
        if total < 2:
            assert not res[r][3].any()
        if total == 1 and n == 1:
            assert torch.equal(res[r][0][0], base.bias) and torch.equal(res[r][5], dys[r][0])
        if n == 0:
            assert not res[r][4].any() and not res[r][5].any()
    if total < 2:
        assert torch.equal(one.running_mean, base.running_mean) and torch.equal(one.running_var, base.running_var)


def test_misaligned_operands_give_the_same_bits(cuda_dev):
    """x and dy at every 2-byte offset below 16 bytes give the aligned call's bits (fp16, one and two ranks)"""
    c, world = 64, 2
    _, xs, dys = _ranks(world, c, torch.float16, cuda_dev, seed=21)
    base = _module(c, CONFIGS[0], torch.float16, cuda_dev, seed=0)
    streams = [torch.cuda.Stream() for _ in range(world)]

    def shifted(t, k):
        buf = torch.empty(t.numel() + 8, dtype=t.dtype, device=t.device)
        v = buf[k:k + t.numel()].view_as(t)
        v.copy_(t)
        return v

    with _ring(world) as ring:
        want = _sync_round(ring, streams, [copy.deepcopy(base) for _ in range(world)], xs, dys, [0] * world)
        for k in range(1, 8):
            got = _sync_round(ring, streams, [copy.deepcopy(base) for _ in range(world)],
                              [shifted(x, k) for x in xs], [shifted(d, k) for d in dys], [0] * world)
            for r in range(world):
                _same(got[r], want[r], f"offset {2 * k} bytes rank {r}")


# ------------------------------------------------------------------ a captured training step
SHAPE = [24, 24, 24]


def _net(c, dev):
    torch.manual_seed(0)
    net = spconv.SparseSequential(
        spconv.SubMConv3d(c, c, 3, bias=False), MaskedSyncBatchNorm1d(c, momentum=0.2), nn.ReLU(),
        spconv.SparseConv3d(c, c, 3, 2, 1, bias=False), MaskedSyncBatchNorm1d(c), spconv.SubMConv3d(c, c, 3, bias=False))
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, MaskedSyncBatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.5, 0.5)
    return net.to(dev).train()


def _twin_step(net, clouds, xs, dys):
    """float64 twin of the step over all ranks: per-rank outputs, per-rank conv dW averaged over the ranks, and
    per-rank BN dweight / dbias"""
    world = len(clouds)
    leaves = [[p.detach().double().cpu().requires_grad_(True) for p in net.parameters()] for _ in range(world)]
    convs = [net[0], net[3], net[5]]
    twins = []
    for inds in clouds:
        refs = []
        cur = inds
        for m in convs:
            ref = SparseConvRef(cur, 1, SHAPE if m is not convs[2] else refs[1].out_shape, m.kernel_size, m.stride,
                                m.padding, m.dilation, m.output_padding, "subm" if m.subm else "conv")
            refs.append(ref)
            cur = ref.out_inds
        twins.append([net_ref.ConvTwin(r) for r in refs])

    def bn(zs, which, eps):
        z = torch.cat(zs)
        mean, var = z.mean(0), z.var(0, unbiased=False)
        return [(zr - mean) / torch.sqrt(var + eps) * leaves[r][which] + leaves[r][which + 1]
                for r, zr in enumerate(zs)]

    # parameters in order: w0, bn1.weight, bn1.bias, w3, bn4.weight, bn4.bias, w5
    h = [twins[r][0](xs[r].double().cpu(), leaves[r][0]) for r in range(world)]
    h = [net_ref.relu(v) for v in bn(h, 1, net[1].eps)]
    h = [twins[r][1](h[r], leaves[r][3]) for r in range(world)]
    h = bn(h, 4, net[4].eps)
    ys = [twins[r][2](h[r], leaves[r][6]) for r in range(world)]
    loss = sum((y * d.double().cpu()).sum() for y, d in zip(ys, dys))
    grads = torch.autograd.grad(loss, [p for ls in leaves for p in ls])
    per = [grads[i * 7:(i + 1) * 7] for i in range(world)]
    out = []
    for r in range(world):
        g = list(per[r])
        for i in (0, 3, 6):                                   # conv weights: the group's mean
            g[i] = sum(per[q][i] for q in range(world)) / world
        out.append((ys[r].detach(), g, twins[r][1].out_inds))
    return out


def _close(got, ref, what):
    ref = ref.to(got.device)
    err = float((got.double() - ref).abs().max())
    lim = 2e-4 * max(float(ref.abs().max()), 1e-3)
    assert err <= lim, f"{what}: max error {err:.3e} over {lim:.3e}"


@pytest.mark.parametrize("world", [2, 8])
def test_graph_replay_of_a_training_step(world, cuda_dev):
    """Every rank captures forward + backward of SubM -> MaskedSyncBatchNorm1d -> ReLU -> SparseConv3d stride 2
    (output bound) -> MaskedSyncBatchNorm1d -> SubM on padded inputs, with its group installed, so BN and conv
    exchanges interleave on one group.  All ranks' graphs replay together on fresh inputs: every replay matches
    the float64 twin and the eager step on the same inputs bit for bit."""
    c, rows, replays = 16, 1024, 10
    clouds = [random_cloud(np.random.default_rng(900 + r), SHAPE, [500 + 37 * r], 1)[1] for r in range(world)]
    net = _net(c, cuda_dev)
    down = [SparseConvRef(inds, 1, SHAPE, [3] * 3, [2] * 3, [1] * 3, [1] * 3, [0] * 3, "conv").n_out
            for inds in clouds]
    bound = 128 * math.ceil(max(down) * 1.25 / 128)
    net[3].num_out_act_bound = bound
    nets = [copy.deepcopy(net) for _ in range(world)]
    xs = [torch.zeros((rows, c), device=cuda_dev) for _ in range(world)]
    dys = [torch.zeros((bound, c), device=cuda_dev) for _ in range(world)]
    bases = [spconv.SparseConvTensor(xs[r][:len(inds)].clone(), torch.from_numpy(inds).to(cuda_dev), SHAPE, 1)
             .pad_to(rows) for r, inds in enumerate(clouds)]
    gen = torch.Generator(device=cuda_dev).manual_seed(world)

    def step(r):
        y = nets[r](bases[r].replace_feature(xs[r]))
        params = list(nets[r].parameters())
        grads = torch.autograd.grad(y.features, params, dys[r])
        return (y.features,) + tuple(grads)

    def refill():
        for r, inds in enumerate(clouds):
            xs[r][:len(inds)] = torch.randn((len(inds), c), generator=gen, device=cuda_dev)
            dys[r][:down[r]] = torch.randn((down[r], c), generator=gen, device=cuda_dev)

    def snapshot():
        return [[p.detach().clone() for p in nets[r].buffers()] for r in range(world)]

    def restore(state):
        for r in range(world):
            for b, s in zip(nets[r].buffers(), state[r]):
                b.copy_(s)

    def check(results, what):
        ref = _twin_step(net, clouds, [xs[r][:len(clouds[r])] for r in range(world)],
                         [dys[r][:down[r]] for r in range(world)])
        for r in range(world):
            y, grads = results[r][0], results[r][1:]
            _close(y[:down[r]], ref[r][0], f"{what} rank {r} output")
            for i, (g, rg) in enumerate(zip(grads, ref[r][1])):
                _close(g, rg.reshape(g.shape), f"{what} rank {r} gradient {i}")
            for i in (0, 3, 6):
                assert torch.equal(grads[i], results[0][1 + i]), f"{what}: conv dW {i} differs between ranks"
        for r in range(world):
            _same(list(nets[r].buffers()), list(nets[0].buffers()), f"{what}: running stats of rank {r}")

    streams = [torch.cuda.Stream() for _ in range(world)]
    refill()
    copies = [copy.deepcopy(n) for n in nets]
    _load(lambda: [copies[r](bases[r].replace_feature(xs[r])).features.backward(dys[r]) for r in range(world)])
    with _ring(world) as ring:
        check(_round(ring, streams, step), "eager warm-up")
        graphs, static = [], []
        for r in range(world):
            ops.set_peer_group(ring[r])
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=streams[r]):
                static.append(step(r))
            graphs.append(g)
        ops.set_peer_group(None)
        for it in range(replays):
            refill()
            state = snapshot()
            torch.cuda.synchronize()
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    graphs[r].replay()
            torch.cuda.synchronize()
            replayed = [[t.clone() for t in s] for s in static]
            after = snapshot()
            check(replayed, f"replay {it}")
            restore(state)
            eager = _round(ring, streams, step)
            for r in range(world):
                _same(replayed[r], eager[r], f"replay {it} rank {r} against the eager step")
                _same(after[r], [b for b in nets[r].buffers()], f"replay {it} rank {r} running stats")
        del graphs, static


# ------------------------------------------------------------------ two processes
@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_peer_and_nccl_routes_agree_across_processes(cuda_dev):
    port = 29900 + os.getpid() % 400
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sync_bn_check.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "sync_bn_check OK" in res.stdout
