"""MaskedBatchNorm1d on the GPU: training-mode statistics, gradients and running stats against BatchNorm in
float64 on the valid rows (and against nn.BatchNorm1d for fp32), bit-identical results under any padding and
across runs, the one-row and no-row rules, the eval path and BN folding, and a SECOND-style encoder with
BatchNorm that trains padded without a host synchronisation and replays as one CUDA graph."""
import copy

import numpy as np
import pytest
import torch
from torch import nn

from bench_utils import make_encoder6
from tests.util import rel_l2, surface_cloud

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedBatchNorm1d
from spconv_b200.pytorch.functional import masked_batch_norm

pytestmark = pytest.mark.gpu

DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}
MANT = {torch.float16: 10, torch.bfloat16: 7}
# (affine, momentum, track_running_stats)
CONFIGS = [(True, 0.1, True), (False, None, True), (True, None, True), (True, 0.1, False), (False, 0.1, False)]
EPS = 1e-5


def _np(t):
    return t.detach().cpu().numpy()


def _inputs(m, c, dtype, dev, seed):
    g = torch.Generator().manual_seed(seed)
    shift = torch.rand((1, c), generator=g) * 4 - 2           # per-channel offsets and scales
    scale = torch.rand((1, c), generator=g) * 2 + 0.25
    x = (torch.randn((m, c), generator=g) * scale + shift).to(dtype).to(dev)
    dy = torch.randn((m, c), generator=g).to(dtype).to(dev)
    return x, dy


def _module(c, cfg, dtype, dev, seed):
    affine, momentum, track = cfg
    bn = MaskedBatchNorm1d(c, EPS, momentum, affine, track).to(dev)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        if affine:
            bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
            bn.bias.copy_(torch.rand(c, generator=g) - 0.5)
        if track:
            bn.running_mean.copy_(torch.randn(c, generator=g))
            bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
            bn.num_batches_tracked.fill_(4)
    return bn


def _run(bn, x, dy, num_valid=None):
    """forward + backward of the module on features x (rows beyond num_valid are padding)"""
    xr = x.clone().requires_grad_(True)
    for p in bn.parameters():
        p.grad = None
    y = masked_batch_norm(xr, bn.weight, bn.bias, bn.running_mean if bn.track_running_stats else None,
                          bn.running_var if bn.track_running_stats else None,
                          bn.num_batches_tracked if bn.track_running_stats else None, num_valid, bn.momentum, bn.eps)
    y.backward(dy)
    return (y.detach(), xr.grad, None if bn.weight is None else bn.weight.grad,
            None if bn.bias is None else bn.bias.grad)


def _reference(x, dy, bn, nbt_after):
    """float64 BatchNorm on the (dtype-rounded) valid rows, the running stats it leads to, and per result the
    size of the terms that cancel in it (see _close_f32)"""
    xd, dyd = x.double(), dy.double()
    m = xd.shape[0]
    mean = xd.mean(0)
    var = xd.var(0, unbiased=False)
    invstd = 1.0 / torch.sqrt(var + bn.eps)
    xhat = (xd - mean) * invstd
    w = bn.weight.double() if bn.affine else torch.ones_like(mean)
    b = bn.bias.double() if bn.affine else torch.zeros_like(mean)
    y = xhat * w + b
    db = dyd.sum(0)
    dw = (dyd * xhat).sum(0)
    dx = w * invstd * (dyd - db / m - xhat * dw / m)
    run = None
    if bn.track_running_stats:
        f = 1.0 / nbt_after if bn.momentum is None else bn.momentum
        run = ((1 - f) * bn.running_mean.double() + f * mean,
               (1 - f) * bn.running_var.double() + f * var * m / (m - 1))
    a = (w * invstd).abs()
    cond = {"y": (a * mean.abs()).expand_as(y),
            "dx": a * (dyd.abs() + (db / m).abs() + (xhat * dw / m).abs()),
            "dw": (dyd * xhat).square().sum(0).sqrt() + invstd * mean.abs() * db.abs(),   # x_hat shares mean's rounding
            "db": dyd.square().sum(0).sqrt()}
    return y, dx, dw, db, run, cond


def _close_f32(got, ref, what, cond=None):
    """|got - ref| <= 1e-5 * max(1, |ref|, cond).  fp32 cannot do better than its rounding of the terms that
    cancel: x - mean when the variance is tiny against the mean (two almost equal values), dy - mean(dy) - ...
    for dx, the partial sums of 100 k terms whose total is small.  `cond` is the size of those terms (the
    random-walk size sqrt(sum t^2) for sums); on well-conditioned data it is of the order of |ref| or 1."""
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


@pytest.mark.parametrize("m", [2, 127, 129, 100_000])
@pytest.mark.parametrize("c", [12, 16, 64, 128, 256])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_against_float64(dname, c, m, cuda_dev):
    dtype = DTYPES[dname]
    x, dy = _inputs(m, c, dtype, cuda_dev, seed=m * 7 + c)
    for ci, cfg in enumerate(CONFIGS):
        bn = _module(c, cfg, dtype, cuda_dev, seed=ci)
        before = copy.deepcopy(bn)
        nbt_after = int(bn.num_batches_tracked) + 1 if bn.track_running_stats else None
        if bn.track_running_stats:
            bn.num_batches_tracked.add_(1)                     # what the module's forward does first
        y, dx, dw, db = _run(bn, x, dy)
        ry, rdx, rdw, rdb, run, cond = _reference(x, dy, before, nbt_after)
        tag = f"{dname} C={c} M={m} {cfg}"
        assert y.dtype == dtype and dx.dtype == dtype
        if dtype == torch.float32:
            _close_f32(y, ry, f"y {tag}", cond["y"])
            _close_f32(dx, rdx, f"dx {tag}", cond["dx"])
        else:
            _close_low(y, ry, dtype, f"y {tag}", cond["y"])
            _close_low(dx, rdx, dtype, f"dx {tag}", cond["dx"])
        if bn.affine:
            _close_f32(dw, rdw, f"dweight {tag}", cond["dw"])
            _close_f32(db, rdb, f"dbias {tag}", cond["db"])
        else:
            assert dw is None and db is None
        if run is not None:
            _close_f32(bn.running_mean, run[0], f"running_mean {tag}")
            _close_f32(bn.running_var, run[1], f"running_var {tag}")
            assert int(bn.num_batches_tracked) == nbt_after
        else:
            assert bn.running_mean is None and bn.num_batches_tracked is None


@pytest.mark.parametrize("m", [2, 129, 100_000])
@pytest.mark.parametrize("c", [12, 64, 256])
def test_fp32_against_torch_batchnorm(c, m, cuda_dev):
    x, dy = _inputs(m, c, torch.float32, cuda_dev, seed=3 * m + c)
    inds = torch.zeros((m, 4), dtype=torch.int32, device=cuda_dev)     # BatchNorm does not look at them
    for ci, cfg in enumerate(CONFIGS):
        bn = _module(c, cfg, torch.float32, cuda_dev, seed=ci)
        ref = nn.BatchNorm1d(c, EPS, cfg[1], cfg[0], cfg[2]).to(cuda_dev)
        ref.load_state_dict(bn.state_dict())
        xr = x.clone().requires_grad_(True)
        yr = ref(xr)
        yr.backward(dy)
        xm = x.clone().requires_grad_(True)
        y = bn(spconv.SparseConvTensor(xm, inds, [4, 4, 4], 1)).features
        y.backward(dy)
        tag = f"C={c} M={m} {cfg}"
        cond = _reference(x, dy, ref, 1)[5]          # the size of the terms both sides round
        _close_f32(y, yr, f"y {tag}", cond["y"])
        _close_f32(xm.grad, xr.grad, f"dx {tag}", cond["dx"])
        for a, b, what in ((bn.weight, ref.weight, "weight"), (bn.bias, ref.bias, "bias")):
            if a is not None:
                _close_f32(a.grad, b.grad, f"d{what} {tag}", cond[f"d{what[0]}"])
        if cfg[2]:
            _close_f32(bn.running_mean, ref.running_mean, f"running_mean {tag}")
            _close_f32(bn.running_var, ref.running_var, f"running_var {tag}")
            assert int(bn.num_batches_tracked) == int(ref.num_batches_tracked)


def _padded(x, rows, fill):
    """x with rows appended up to `rows`, holding NaN / +Inf / -Inf in turn"""
    m, c = x.shape
    pad = torch.tensor([float("nan"), float("inf"), float("-inf")], dtype=x.dtype,
                       device=x.device).repeat((rows - m) * c // 3 + 3)[:(rows - m) * c].view(rows - m, c)
    return torch.cat([x, pad if fill else torch.zeros_like(pad)], 0)


@pytest.mark.parametrize("m", [1, 127, 1000, 20_000])
@pytest.mark.parametrize("c", [12, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_padding_and_repeat_are_bit_identical(dname, c, m, cuda_dev):
    dtype = DTYPES[dname]
    x, dy = _inputs(m, c, dtype, cuda_dev, seed=m + c)
    for ci, cfg in enumerate(CONFIGS[:3]):
        base = _module(c, cfg, dtype, cuda_dev, seed=ci)
        results = []
        for rows in (m, m, m, m + 1, m + 3 * 128):
            bn = copy.deepcopy(base)
            nv = torch.full((1,), m, dtype=torch.int32, device=cuda_dev) if len(results) else None
            y, dx, dw, db = _run(bn, _padded(x, rows, True), _padded(dy, rows, True), nv)
            assert bool((y[m:] == 0).all()) and bool((dx[m:] == 0).all()), f"padding rows {rows}"
            assert not bool(y[m:].signbit().any()) and not bool(dx[m:].signbit().any())
            results.append([y[:m], dx[:m], dw, db, bn.running_mean, bn.running_var])
        for rows, res in zip(("num_valid", "repeat", "m+1", "m+384"), results[1:]):
            for i, (a, b) in enumerate(zip(res, results[0])):
                assert (a is None and b is None) or torch.equal(a, b), f"{dname} C={c} M={m} {cfg} {rows} item {i}"


@pytest.mark.parametrize("dname", list(DTYPES))
def test_one_and_no_valid_rows(dname, cuda_dev):
    dtype = DTYPES[dname]
    c = 16
    x, dy = _inputs(5, c, dtype, cuda_dev, seed=9)
    for cfg in CONFIGS[:3]:
        # one valid row: x_hat = 0, y = bias, dx = 0, dbias = dy, dweight = 0, running stats unchanged
        bn = _module(c, cfg, dtype, cuda_dev, seed=2)
        before = copy.deepcopy(bn)
        nv = torch.ones((1,), dtype=torch.int32, device=cuda_dev)
        y, dx, dw, db = _run(bn, _padded(x[:1], 5, True), _padded(dy[:1], 5, True), nv)
        beta = bn.bias.to(dtype) if bn.affine else torch.zeros(c, dtype=dtype, device=cuda_dev)
        assert torch.equal(y[0], beta) and bool((y[1:] == 0).all())
        assert bool((dx == 0).all())
        if bn.affine:
            assert torch.equal(db, dy[0].float()) and bool((dw == 0).all())
        assert torch.equal(bn.running_mean, before.running_mean)
        assert torch.equal(bn.running_var, before.running_var)
        # no valid row: everything 0, running stats unchanged
        nv.zero_()
        y, dx, dw, db = _run(bn, _padded(x[:1], 5, True)[1:], _padded(dy[:1], 5, True)[1:], nv)
        assert bool((y == 0).all()) and bool((dx == 0).all())
        if bn.affine:
            assert bool((dw == 0).all()) and bool((db == 0).all())
        assert torch.equal(bn.running_mean, before.running_mean)
        assert torch.equal(bn.running_var, before.running_var)
    # through the module: a zero-row tensor passes through, num_valid is kept, num_batches_tracked counts calls
    bn = MaskedBatchNorm1d(c).to(cuda_dev)
    inds = torch.zeros((5, 4), dtype=torch.int32, device=cuda_dev)
    t = spconv.SparseConvTensor(x[:2].clone(), inds[:2], [4, 4, 4], 1).pad_to(5)
    out = bn(t)
    assert out.num_valid is t.num_valid and int(bn.num_batches_tracked) == 1
    empty = spconv.SparseConvTensor(x[:0], inds[:0], [4, 4, 4], 1)
    assert bn(empty) is empty and int(bn.num_batches_tracked) == 1


def _sparse_net(dev, masked):
    torch.manual_seed(11)
    Bn = MaskedBatchNorm1d if masked else nn.BatchNorm1d
    net = spconv.SparseSequential(
        spconv.SubMConv3d(16, 32, 3, indice_key="s1", bias=False), Bn(32), nn.ReLU(),
        spconv.SparseConv3d(32, 64, 3, stride=2, padding=1, bias=False), Bn(64), nn.ReLU(),
        spconv.SubMConv3d(64, 64, 3, indice_key="s2"), spconv.SparseBatchNorm(64))
    g = torch.Generator().manual_seed(5)
    for mod in net.modules():
        if isinstance(mod, nn.BatchNorm1d):
            with torch.no_grad():
                mod.running_mean.copy_(torch.randn(mod.num_features, generator=g))
                mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
                mod.weight.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(mod.num_features, generator=g) * 0.1)
    return net.to(dev)


def test_eval_mode_and_fusion_match_the_unconverted_net(cuda_dev):
    rng = np.random.default_rng(3)
    shape = [20, 80, 80]
    inds = torch.from_numpy(surface_cloud(rng, shape, 6000)).to(cuda_dev)
    feats = torch.randn((inds.shape[0], 16), device=cuda_dev)
    plain = _sparse_net(cuda_dev, masked=False).eval()
    conv = MaskedBatchNorm1d.convert_masked_batchnorm(copy.deepcopy(plain)).eval()
    assert sum(isinstance(m, MaskedBatchNorm1d) for m in conv.modules()) == 3
    with torch.no_grad():
        x = spconv.SparseConvTensor(feats, inds, shape, 1)
        want = plain(x).features
        assert torch.equal(conv(x).features, want)
        fp, fc = spconv.fuse_bn_act_sequential(plain), spconv.fuse_bn_act_sequential(conv)
        for fused in (fp, fc):                       # both BatchNorm1d after a conv folded; SparseBatchNorm stays
            assert sum(isinstance(m, nn.modules.batchnorm._BatchNorm) for m in fused.modules()) == 1
        assert torch.equal(fc(x).features, fp(x).features)


def _encoder(dev):
    torch.manual_seed(4)
    layers = []
    for conv in make_encoder6(spconv, bias=False):
        layers += [conv, nn.BatchNorm1d(conv.out_channels), nn.ReLU()]
    net = spconv.SparseSequential(*layers)
    return MaskedBatchNorm1d.convert_masked_batchnorm(net).to(dev).half()


def _bn_state(net):
    return {k: v.clone() for k, v in net.state_dict().items() if "running" in k or "num_batches" in k}


def _restore(net, state):
    with torch.no_grad():
        for k, v in net.state_dict().items():
            if k in state:
                v.copy_(state[k])


def test_encoder_with_batchnorm_trains_padded_and_as_one_graph(cuda_dev):
    shape = [41, 400, 352]
    rng = np.random.default_rng(8)
    counts = [20000, 17000, 18500]
    clouds = [torch.from_numpy(surface_cloud(rng, shape, c)).to(cuda_dev) for c in counts]
    g = torch.Generator().manual_seed(6)
    feats = [torch.randn((c.shape[0], 16), generator=g).to(cuda_dev).half() for c in clouds]
    n_pad = 20096
    net = _encoder(cuda_dev)
    assert sum(isinstance(m, MaskedBatchNorm1d) for m in net.modules()) == 6
    bns = [m for m in net.modules() if isinstance(m, MaskedBatchNorm1d)]
    params = list(net.parameters())
    state0 = _bn_state(net)

    def step(f, i, nv=None):
        for p in params:
            p.grad = None
        x = spconv.SparseConvTensor(f, i, shape, 1)
        x.num_valid = nv
        y = net(x)
        valid = y.valid_mask().unsqueeze(1)
        loss = torch.where(valid, y.features.float(), 0.0).square().sum()
        loss.backward()
        return loss.detach(), [p.grad for p in params], y.features.detach()

    want = []
    for f, i in zip(feats, clouds):                  # eager, exact shapes, from the same BatchNorm state
        _restore(net, state0)
        loss, grads, y = step(f, i)
        want.append((loss.clone(), [t.detach().clone() for t in grads], y.clone(),
                     [(b.running_mean.clone(), b.running_var.clone()) for b in bns]))
    loss = grads = y = None

    net.eval()                                       # counting outputs needs no batch statistics
    spconv.set_output_bounds(net, spconv.SparseConvTensor(feats[0], clouds[0], shape, 1), margin=1.25)
    net.train()
    padded = [spconv.SparseConvTensor(f, i, shape, 1).pad_to(n_pad) for f, i in zip(feats, clouds)]
    args = [(p.features, p.indices, p.num_valid) for p in padded]

    def same(got, ref, what, exact_fwd=True):
        loss, grads, y = got
        m = ref[2].shape[0]
        if exact_fwd:
            assert torch.equal(y[:m], ref[2]), f"{what}: features"
            for b, (rm, rv) in zip(bns, ref[3]):
                assert torch.equal(b.running_mean, rm) and torch.equal(b.running_var, rv), f"{what}: running stats"
        assert bool((y[m:] == 0).all()), f"{what}: padding rows"
        assert abs(float(loss.detach()) - float(ref[0])) <= 1e-4 * abs(float(ref[0])), what
        for (name, _), a, b in zip(net.named_parameters(), grads, ref[1]):
            assert rel_l2(_np(a.float()), _np(b.float())) < 2e-3, (what, name)

    _restore(net, state0)
    step(*args[0])                                   # warm-up: allocator pools, status words
    torch.cuda.synchronize()
    _restore(net, state0)
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = step(*args[1])                         # eager bounded: no synchronising call
    finally:
        torch.cuda.set_sync_debug_mode("default")
    same(got, want[1], "eager bounded")
    got = None

    graphed = spconv.graph_capture(step, *args[0])  # its warm-up and capture run the step four times
    for k in (0, 1, 2, 1):
        _restore(net, state0)
        same(graphed(*args[k]), want[k], f"replay of cloud {k}")
    spconv.check_bounds(net)
