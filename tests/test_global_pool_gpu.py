"""MaskedGlobalMaxPool / MaskedGlobalAvgPool on the GPU: max bit for bit against numpy's argmax (NaN, +-0, ties,
empty samples, dropped batch ids), the mean against float64, both gradients, bit-identical results under any
padding and across runs, agreement with the default global pools, and a small classification net that trains
padded without a host synchronisation and replays as one CUDA graph."""
import numpy as np
import pytest
import torch
from torch import nn

from tests.util import random_cloud, rel_l2

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedBatchNorm1d, MaskedGlobalAvgPool, MaskedGlobalMaxPool, ops
from spconv_b200.pytorch.functional import masked_global_pool

pytestmark = pytest.mark.gpu

DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}
BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
MANT = {torch.float16: 10, torch.bfloat16: 7}
# (rows, batch size): empty input, one row, small and large clouds
SHAPES = [(0, 3), (1, 1), (700, 17), (5000, 64), (40_000, 3)]
LARGE = (300_000, 17)


def _batch_ids(rows, b, rng):
    """interleaved samples; sample 1 empty when b > 2; ~5 % dropped rows with batch ids -1, b and 2^30"""
    bid = rng.integers(0, b, rows)
    if b > 2:
        bid[bid == 1] = 0
    drop = rng.random(rows) < 0.05
    bid[drop] = rng.choice(np.array([-1, b, 1 << 30]), int(drop.sum()))
    return bid


def _indices(bid, rng, dev):
    coords = rng.integers(0, 50, (bid.shape[0], 3))
    return torch.from_numpy(np.concatenate([bid[:, None], coords], 1).astype(np.int32)).to(dev)


def _max_features(rows, c, dtype, rng, dev):
    """few distinct values (many ties), +-0, and NaN in about 1 % of the entries"""
    v = rng.integers(-6, 6, (rows, c)).astype(np.float32) * 0.75
    v[rng.random((rows, c)) < 0.05] = 0.0
    v[rng.random((rows, c)) < 0.05] = -0.0
    v[rng.random((rows, c)) < 0.01] = np.nan
    return torch.from_numpy(v).to(dtype).to(dev)


def _ref_argmax(x, bid, b):
    """argmax [b, C] int64: first row of the sample attaining the maximum, NaN counting as the maximum; -1 if empty"""
    xs = x.float().cpu().numpy()
    c = xs.shape[1]
    arg = np.full((b, c), -1, np.int64)
    for s in range(b):
        rows = np.nonzero(bid == s)[0]
        if rows.size:
            arg[s] = rows[np.argmax(xs[rows], axis=0)]
    return arg


def _bits(t):
    return t.view(BITS[t.dtype])


def _check_max(x, inds, bid, b, dy, num_valid=None):
    xr = x.clone().requires_grad_(True)
    out = masked_global_pool(xr, inds, b, num_valid, False)
    out.backward(dy)
    m, c = bid.shape[0], x.shape[1]
    arg = torch.from_numpy(_ref_argmax(x[:m], bid, b))
    ref = torch.zeros((b, c), dtype=x.dtype)
    din = torch.zeros((x.shape[0], c), dtype=x.dtype)
    bb, cc = torch.nonzero(arg >= 0, as_tuple=True)
    ref[bb, cc] = x.cpu()[arg[bb, cc], cc]
    din[arg[bb, cc], cc] = dy.cpu()[bb, cc]
    assert torch.equal(_bits(out.detach().cpu()), _bits(ref)), "max output"
    assert torch.equal(_bits(xr.grad.cpu()), _bits(din)), "max gradient"
    return out.detach(), xr.grad


@pytest.mark.parametrize("c", [1, 3, 8, 64, 136, 256])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_max_matches_numpy_argmax_bit_for_bit(dname, c, cuda_dev):
    dtype = DTYPES[dname]
    shapes = SHAPES + ([LARGE] if c in (8, 136) else [])
    for rows, b in shapes:
        rng = np.random.default_rng(rows * 31 + b * 7 + c)
        bid = _batch_ids(rows, b, rng)
        x = _max_features(rows, c, dtype, rng, cuda_dev)
        dy = torch.from_numpy(rng.standard_normal((b, c)).astype(np.float32)).to(dtype).to(cuda_dev)
        inds = _indices(bid, rng, cuda_dev)
        out, _ = _check_max(x, inds, bid, b, dy)
        assert out.shape == (b, c) and out.dtype == dtype
        _, argmax = ops.masked_global_pool_fwd(x, inds, b, None, False)
        assert np.array_equal(argmax.cpu().numpy(), _ref_argmax(x, bid, b)), f"argmax rows={rows} b={b}"


def _round_ulp(ref, dtype):
    """ref (float64) rounded to dtype, and one ulp of dtype there"""
    r = ref.to(dtype).double()
    _, e = torch.frexp(r.abs().clamp(min=2.0 ** -14 if dtype == torch.float16 else 2.0 ** -126))
    return r, torch.ldexp(torch.ones_like(r), (e - 1 - MANT[dtype]).to(torch.int32))


@pytest.mark.parametrize("c", [1, 3, 8, 64, 136, 256])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_mean_against_float64_and_its_gradient(dname, c, cuda_dev):
    dtype = DTYPES[dname]
    shapes = SHAPES + ([LARGE] if c in (8, 136) else [])
    for rows, b in shapes:
        rng = np.random.default_rng(rows * 13 + b * 5 + c)
        bid = _batch_ids(rows, b, rng)
        inds = _indices(bid, rng, cuda_dev)
        x = torch.from_numpy(rng.uniform(0.5, 1.5, (rows, c)).astype(np.float32)).to(dtype).to(cuda_dev)
        dy = torch.from_numpy(rng.standard_normal((b, c)).astype(np.float32)).to(dtype).to(cuda_dev)
        xr = x.clone().requires_grad_(True)
        out = masked_global_pool(xr, inds, b, None, True)
        out.backward(dy)
        _, count = ops.masked_global_pool_fwd(x, inds, b, None, True)
        want_count = np.array([(bid == s).sum() for s in range(b)])
        assert np.array_equal(count.cpu().numpy(), want_count), "count"
        xd = x.double().cpu()
        ref = torch.zeros((b, c), dtype=torch.float64)
        for s in range(b):
            if want_count[s]:
                ref[s] = xd[torch.from_numpy(bid == s)].mean(0)
        got = out.detach().cpu().double()
        tag = f"{dname} C={c} rows={rows} b={b}"
        if dtype == torch.float32:
            assert bool(((got - ref).abs() <= 1e-6 * ref.abs().clamp(min=1.0)).all()), tag
        else:
            r, ulp = _round_ulp(ref, dtype)
            assert bool(((got - r).abs() <= ulp).all()), tag
        assert bool((got[torch.from_numpy(want_count == 0)] == 0).all()), tag
        # din = dy[b] / count[b] in fp32, rounded once; 0 on dropped rows
        cnt = torch.from_numpy(np.maximum(want_count, 1)).float()
        per = (dy.cpu().float() / cnt[:, None]).to(dtype)
        din = torch.zeros((rows, c), dtype=dtype)
        keep = torch.from_numpy((bid >= 0) & (bid < b))
        din[keep] = per[torch.from_numpy(bid[keep.numpy()])]
        assert torch.equal(_bits(xr.grad.cpu()), _bits(din)), f"gradient {tag}"


def _pad(x, inds, extra, b):
    """append `extra` padding rows: NaN / +Inf / -Inf features and in-range batch ids"""
    if extra == 0:
        return x, inds
    fill = torch.tensor([float("nan"), float("inf"), float("-inf")], dtype=x.dtype, device=x.device)
    pf = fill.repeat(extra * x.shape[1] // 3 + 3)[:extra * x.shape[1]].view(extra, x.shape[1])
    pi = torch.zeros((extra, inds.shape[1]), dtype=torch.int32, device=inds.device)
    pi[:, 0] = torch.arange(extra, device=inds.device, dtype=torch.int32) % b
    return torch.cat([x, pf]), torch.cat([inds, pi])


@pytest.mark.parametrize("m", [1, 700, 20_000])
@pytest.mark.parametrize("c", [3, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_padding_and_repeat_are_bit_identical(dname, c, m, cuda_dev):
    dtype = DTYPES[dname]
    b = 5
    rng = np.random.default_rng(m + c)
    bid = _batch_ids(m, b, rng)
    inds = _indices(bid, rng, cuda_dev)
    x = _max_features(m, c, dtype, rng, cuda_dev)
    dy = torch.from_numpy(rng.standard_normal((b, c)).astype(np.float32)).to(dtype).to(cuda_dev)
    for is_mean in (False, True):
        if is_mean:
            x = torch.nan_to_num(x, nan=0.5)
        results = []
        for extra in (0, 0, 1, 5000):
            xp, ip = _pad(x, inds, extra, b)
            nv = torch.full((1,), m, dtype=torch.int32, device=cuda_dev) if results else None
            xr = xp.clone().requires_grad_(True)
            out = masked_global_pool(xr, ip, b, nv, is_mean)
            out.backward(dy)
            assert bool((xr.grad[m:] == 0).all()) and not bool(xr.grad[m:].signbit().any()), f"padding {extra}"
            results.append((_bits(out.detach()), _bits(xr.grad[:m])))
        for k, (o, g) in enumerate(results[1:]):
            assert torch.equal(o, results[0][0]) and torch.equal(g, results[0][1]), \
                f"{dname} C={c} M={m} mean={is_mean} run {k + 1}"


@pytest.mark.parametrize("c", [3, 64])
@pytest.mark.parametrize("dname", list(DTYPES))
def test_agrees_with_the_default_global_pools(dname, c, cuda_dev):
    dtype = DTYPES[dname]
    b, per = 4, [900, 1300, 40, 2000]
    rng = np.random.default_rng(c)
    feats, inds = random_cloud(rng, [30, 30, 30], per, c)
    perm = rng.permutation(inds.shape[0])                  # interleave the samples
    inds = torch.from_numpy(inds[perm]).to(cuda_dev)
    ties = torch.from_numpy(np.round(feats[perm] * 4) / 4).to(dtype).to(cuda_dev)
    x = spconv.SparseConvTensor(ties, inds, [30, 30, 30], b)
    assert torch.equal(_bits(MaskedGlobalMaxPool()(x)), _bits(spconv.SparseGlobalMaxPool()(x)))
    got, want = MaskedGlobalAvgPool()(x).float(), spconv.SparseGlobalAvgPool()(x).float()
    tol = 1e-5 if dtype == torch.float32 else 2.0 ** -MANT[dtype] * 2
    assert bool(((got - want).abs() <= tol * want.abs().clamp(min=1.0)).all())
    # tie-free data (uniform fp32): the max gradient is the default module's autograd gradient
    if dtype != torch.float32:
        return
    tie_free = torch.from_numpy(feats[perm]).to(cuda_dev)
    dy = torch.randn((b, c), device=cuda_dev)
    grads = []
    for mod in (MaskedGlobalMaxPool(), spconv.SparseGlobalMaxPool()):
        xr = tie_free.clone().requires_grad_(True)
        mod(spconv.SparseConvTensor(xr, inds, [30, 30, 30], b)).backward(dy)
        grads.append(xr.grad)
    assert torch.equal(_bits(grads[0]), _bits(grads[1]))


class _Classifier(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(2)
        self.body = spconv.SparseSequential(
            spconv.SubMConv3d(4, 16, 3, indice_key="s1", bias=False), MaskedBatchNorm1d(16), nn.ReLU(),
            spconv.SparseConv3d(16, 32, 3, stride=2, padding=1, bias=False), MaskedBatchNorm1d(32), nn.ReLU(),
            spconv.SubMConv3d(32, 32, 3, indice_key="s2"))
        self.max_pool = MaskedGlobalMaxPool()
        self.avg_pool = MaskedGlobalAvgPool()
        self.head = nn.Linear(64, 5)

    def forward(self, x):
        y = self.body(x)
        return torch.cat([self.max_pool(y), self.avg_pool(y)], 1)


def test_classifier_trains_padded_and_as_one_graph(cuda_dev):
    shape, b = [24, 48, 48], 4
    rng = np.random.default_rng(4)
    clouds = []
    for per in ([3000, 2500, 2800, 2000], [2000, 2900, 1000, 2600], [2600, 0, 2400, 2700]):
        f, i = random_cloud(rng, shape, per, 4)
        perm = rng.permutation(i.shape[0])
        clouds.append((torch.from_numpy(f[perm]).to(cuda_dev).half(), torch.from_numpy(i[perm]).to(cuda_dev)))
    n_pad = 10_400
    net = _Classifier().to(cuda_dev)
    net.body.half()
    params = list(net.parameters())
    labels = torch.tensor([0, 3, 1, 4], device=cuda_dev)
    bn_state = {k: v.clone() for k, v in net.state_dict().items() if "running" in k or "num_batches" in k}

    def restore():
        with torch.no_grad():
            for k, v in net.state_dict().items():
                if k in bn_state:
                    v.copy_(bn_state[k])

    def step(f, i, nv=None):
        for p in params:
            p.grad = None
        x = spconv.SparseConvTensor(f, i, shape, b)
        x.num_valid = nv
        pooled = net(x)
        loss = nn.functional.cross_entropy(net.head(pooled.float()), labels)
        loss.backward()
        return loss.detach(), [p.grad for p in params], pooled.detach()

    want = []
    for f, i in clouds:                              # eager, exact shapes
        restore()
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
        assert abs(float(loss) - float(ref[0])) <= 1e-4 * abs(float(ref[0])), what
        for (name, _), g, r in zip(net.named_parameters(), grads, ref[1]):
            assert rel_l2(g.float().cpu().numpy(), r.float().cpu().numpy()) < 2e-3, (what, name)

    restore()
    step(*args[0])                                   # warm-up: allocator pools, status words
    torch.cuda.synchronize()
    restore()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = step(*args[1])                         # eager bounded: no synchronising call
    finally:
        torch.cuda.set_sync_debug_mode("default")
    same(got, want[1], "eager bounded")
    got = None

    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 2, 1):
        restore()
        same(graphed(*args[k]), want[k], f"replay of cloud {k}")
    spconv.check_bounds(net.body)
