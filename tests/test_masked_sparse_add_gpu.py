"""masked_sparse_add / masked_remove_duplicate and the masked table modules on the GPU: bit for bit against the numpy
oracle (tests/sparse_add_oracle.py) fed the valid rows, bit-identical to sparse_add / remove_duplicate of the valid
rows under any padding (including paddings that invert the ranking by row count), deterministic truncation, and a
two-branch net joined by MaskedAddTableMisaligned that trains padded with no synchronising call and replays as one
CUDA graph."""
import numpy as np
import pytest
import torch
from torch import nn

from tests import sparse_add_oracle as sao
from tests.test_sparse_add_gpu import CASES, _bits, _exact, _operands, _pool
from tests.util import random_cloud, rel_l2

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import functional as Fsp

pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
DEV = torch.device("cuda")


def _padded(rng, inds, feats, extra, dtype, batch, shape):
    """operand with `extra` junk rows appended: coordinates copied from the operand (or fresh in-range ones), so
    they would merge with valid rows if read, and NaN / huge features, so a read shows in every sum"""
    n, ncol = len(inds), len(shape) + 1
    if extra:
        src = inds if n else _pool(rng, batch, shape, 8)
        junk_i = src[rng.integers(0, len(src), extra)]
        junk_f = np.where(rng.random((extra, feats.shape[1])) < 0.5, np.nan, 3e4).astype(np.float32)
    else:
        junk_i, junk_f = np.zeros((0, ncol), np.int32), np.zeros((0, feats.shape[1]), np.float32)
    f = torch.from_numpy(np.concatenate([feats, junk_f], 0)).to(dtype).to(DEV).requires_grad_()
    t = spconv.SparseConvTensor(f, torch.from_numpy(np.concatenate([inds, junk_i], 0).astype(np.int32)).to(DEV),
                                shape, batch)
    t.num_valid = torch.tensor([n], dtype=torch.int32, device=DEV)
    return t


def _unpadded(inds, feats, dtype, batch, shape):
    f = torch.from_numpy(feats).to(dtype).to(DEV).requires_grad_()
    return spconv.SparseConvTensor(f, torch.from_numpy(inds).to(DEV), shape, batch)


def _check_padding_rows(res, m):
    assert bool((res.indices[m:] == -1).all()), "indices of rows [M, bound)"
    assert not res.features[m:].any(), "features of rows [M, bound)"


def _run_masked(rng, inds, feats, extras, dtype, batch, shape, bound=None):
    """masked_sparse_add of the padded operands (extras[t] None: unpadded) -> (result, operands, M)"""
    tens = [_unpadded(i, f, dtype, batch, shape) if e is None else _padded(rng, i, f, e, dtype, batch, shape)
            for i, f, e in zip(inds, feats, extras)]
    res = Fsp.masked_sparse_add(*tens, num_out_act_bound=bound)
    return res, tens, int(res.num_valid)


def _extras(rng, sizes):
    """random paddings; the smallest operand gets the most, so the padded row counts rank the operands differently
    from the valid ones whenever their sizes differ; one operand in three stays unpadded"""
    order = np.argsort(sizes, kind="stable")
    out = [None] * len(sizes)
    for rank, t in enumerate(order):
        if rank % 3 != 2:
            out[t] = int(rng.integers(0, 40)) + (max(sizes) - sizes[t]) + 17 * (len(sizes) - rank)
    return out


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", list(CASES))
def test_masked_sparse_add_bit_exact_against_the_oracle(case, dt):
    batch, shape, sizes, overlap, dups, oob, c = CASES[case]
    dtype = DTYPES[dt]
    rng = np.random.default_rng(sum(map(ord, case)) + 7)
    inds = _operands(rng, batch, shape, sizes, overlap, dups, oob)
    feats = [_exact(dtype, rng.standard_normal((len(i), c))) for i in inds]
    o_inds, o_sum, dst, visit = sao.sparse_add(inds, feats, batch, shape)
    m_ref = o_inds.shape[0]
    res, tens, m = _run_masked(rng, inds, feats, _extras(rng, [len(i) for i in inds]), dtype, batch, shape)
    bound = sum(t.features.shape[0] for t in tens)
    assert m == m_ref and res.features.shape == (bound, c) and res.indices.shape[0] == bound
    assert res.features.dtype == dtype and res.indice_dict == {}
    assert torch.equal(res.indices[:m].cpu(), torch.from_numpy(o_inds)), "output coordinates / row order"
    assert torch.equal(_bits(res.features[:m]), _bits(torch.from_numpy(o_sum).to(dtype))), "features"
    _check_padding_rows(res, m)
    dout = np.concatenate([_exact(dtype, rng.standard_normal((m, c))), np.full((bound - m, c), np.nan, np.float32)], 0)
    res.features.backward(torch.from_numpy(dout).to(dtype).to(DEV))
    want_g = sao.gradients(dout[:m], dst, [len(inds[i]) for i in visit])
    for k, i in enumerate(visit):
        g = tens[i].features.grad
        n = len(inds[i])
        assert torch.equal(_bits(g[:n]), _bits(torch.from_numpy(want_g[k]).to(dtype))), f"grad {i}"
        assert not g[n:].any(), f"padding gradient {i}"


@pytest.mark.parametrize("dt", list(DTYPES))
def test_empty_operands_and_zero_valid_counts(dt):
    dtype = DTYPES[dt]
    rng = np.random.default_rng(3)
    shape, batch, c = [8, 8, 8], 2, 16
    e = np.zeros((0, 4), np.int32)
    # nothing at all: M = 0, no exception, a 0-row result
    res, _, m = _run_masked(rng, [e, e], [np.zeros((0, c), np.float32)] * 2, [None, None], dtype, batch, shape)
    assert m == 0 and res.features.shape == (0, c)
    # only padding rows, or only out-of-range rows: M = 0 over a padded result, zero gradients
    bad = np.array([[2, 0, 0, 0], [0, 8, 1, 1], [-1, 1, 1, 1]], np.int32)
    feats = [np.ones((3, c), np.float32), np.zeros((0, c), np.float32)]
    res, tens, m = _run_masked(rng, [bad, e], feats, [None, 5], dtype, batch, shape)
    assert m == 0 and res.features.shape == (8, c)
    _check_padding_rows(res, 0)
    res.features.sum().backward()
    assert not tens[0].features.grad.any() and not tens[1].features.grad.any()
    # an operand with valid rows next to one whose num_valid is 0
    good = _pool(rng, batch, shape, 20)
    f = _exact(dtype, rng.standard_normal((20, c)))
    res, tens, m = _run_masked(rng, [e, good], [np.zeros((0, c), np.float32), f], [30, 4], dtype, batch, shape)
    ref = Fsp.sparse_add(_unpadded(e, np.zeros((0, c), np.float32), dtype, batch, shape),
                         _unpadded(good, f, dtype, batch, shape))
    assert m == 20 and torch.equal(res.indices[:m], ref.indices)
    assert torch.equal(_bits(res.features[:m]), _bits(ref.features))


@pytest.mark.parametrize("dt", list(DTYPES))
def test_padding_invariance(dt):
    """paddings that invert the ranking by row count: the result equals sparse_add of the valid rows bit for bit,
    and two runs are bit-identical"""
    dtype = DTYPES[dt]
    rng = np.random.default_rng(11)
    batch, shape, c = 2, [30, 40, 50], 32
    inds = _operands(rng, batch, shape, [300, 500, 400, 120], 0.5, 20, 6)
    feats = [_exact(dtype, rng.standard_normal((len(i), c))) for i in inds]
    ref_t = [_unpadded(i, f, dtype, batch, shape) for i, f in zip(inds, feats)]
    ref = Fsp.sparse_add(*ref_t)
    m_ref = ref.features.shape[0]
    dout = _exact(dtype, rng.standard_normal((m_ref, c)))
    ref.features.backward(torch.from_numpy(dout).to(dtype).to(DEV))
    for extras in ([700, 0, 60, None], [None, 1, 200, 900], [0, 0, 0, 0], [5, None, None, 3]):
        runs = []
        for _ in range(2):
            res, tens, m = _run_masked(rng, inds, feats, extras, dtype, batch, shape)
            assert m == m_ref
            assert torch.equal(res.indices[:m], ref.indices) and torch.equal(_bits(res.features[:m]), _bits(ref.features))
            _check_padding_rows(res, m)
            g = torch.full(res.features.shape, float("nan"), dtype=dtype, device=DEV)
            g[:m] = torch.from_numpy(dout).to(dtype)
            res.features.backward(g)
            for t, r in zip(tens, ref_t):
                n = r.features.shape[0]
                assert torch.equal(_bits(t.features.grad[:n]), _bits(r.features.grad)), extras
                assert not t.features.grad[n:].any()
            runs.append((res.indices.clone(), _bits(res.features), [_bits(t.features.grad) for t in tens]))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
        assert all(torch.equal(a, b) for a, b in zip(runs[0][2], runs[1][2]))


def test_truncation():
    rng = np.random.default_rng(17)
    dtype, batch, shape, c = torch.float16, 2, [40, 40, 40], 24
    inds = _operands(rng, batch, shape, [3000, 2000, 2500], 0.3, 50, 10)
    feats = [_exact(dtype, rng.standard_normal((len(i), c))) for i in inds]
    full, _, m = _run_masked(rng, inds, feats, [100, None, 40], dtype, batch, shape)
    bound = int(m * 0.7)
    res, tens, mt = _run_masked(rng, inds, feats, [100, None, 40], dtype, batch, shape, bound=bound)
    assert mt == bound and res.features.shape[0] == bound
    assert torch.equal(res.indices, full.indices[:bound])
    assert torch.equal(_bits(res.features), _bits(full.features[:bound]))
    (word,) = res.bound_status.values()
    assert int(word) & 1 and not int(word) & 2
    with pytest.raises(RuntimeError, match="more outputs than num_out_act_bound"):
        spconv.check_bounds(res)
    # rows of the dropped outputs get a zero gradient: the untruncated backward with dout 0 beyond the bound
    dout = torch.from_numpy(_exact(dtype, rng.standard_normal((bound, c)))).to(dtype).to(DEV)
    res.features.backward(dout)
    ref_t = [_unpadded(i, f, dtype, batch, shape) for i, f in zip(inds, feats)]
    ref = Fsp.sparse_add(*ref_t)
    g = torch.zeros_like(ref.features)
    g[:bound] = dout
    ref.features.backward(g)
    for t, r in zip(tens, ref_t):
        n = r.features.shape[0]
        assert torch.equal(_bits(t.features.grad[:n]), _bits(r.features.grad))
        assert not t.features.grad[n:].any()
    # a larger bound is clamped to the total row count; the default never truncates
    big = Fsp.masked_sparse_add(*tens, num_out_act_bound=10 ** 8)
    assert big.features.shape[0] == sum(t.features.shape[0] for t in tens) and int(big.num_valid) == m
    spconv.check_bounds(big)


@pytest.mark.parametrize("dt", list(DTYPES))
def test_masked_remove_duplicate(dt):
    dtype = DTYPES[dt]
    rng = np.random.default_rng(23)
    batch, shape, c = 2, [12, 14, 16], 8
    inds = _operands(rng, batch, shape, [400], 0.0, 120, 9)[0]
    f = _exact(dtype, rng.standard_normal((len(inds), c)))
    x = _unpadded(inds, f, dtype, batch, shape)
    ref = Fsp.remove_duplicate(x)
    m_ref = ref.features.shape[0]
    dout = torch.from_numpy(_exact(dtype, rng.standard_normal((m_ref, c)))).to(dtype).to(DEV)
    ref.features.backward(dout)
    for extra in (None, 0, 37, 1000):
        p = _unpadded(inds, f, dtype, batch, shape) if extra is None else _padded(rng, inds, f, extra, dtype, batch, shape)
        r = Fsp.masked_remove_duplicate(p)
        m = int(r.num_valid)
        assert m == m_ref and r.features.shape[0] == p.features.shape[0]
        assert torch.equal(r.indices[:m], ref.indices) and torch.equal(_bits(r.features[:m]), _bits(ref.features))
        _check_padding_rows(r, m)
        g = torch.full(r.features.shape, float("nan"), dtype=dtype, device=DEV)
        g[:m] = dout
        r.features.backward(g)
        assert torch.equal(_bits(p.features.grad[:len(inds)]), _bits(x.features.grad))
        assert not p.features.grad[len(inds):].any()
    # truncation through the module: the first `bound` kept rows, status bit 0
    mod = spconv.MaskedRemoveDuplicate(num_out_act_bound=m_ref - 10)
    r = mod(_padded(rng, inds, f, 50, dtype, batch, shape))
    assert int(r.num_valid) == m_ref - 10 and torch.equal(r.indices, ref.indices[:m_ref - 10])
    with pytest.raises(RuntimeError, match="more outputs than num_out_act_bound"):
        spconv.check_bounds(mod)


def test_masked_aligned_tables_on_padded_branches():
    rng = np.random.default_rng(29)
    shape, c = [16, 16, 16], 8
    f, i = random_cloud(rng, shape, [500, 400], c)
    x = spconv.SparseConvTensor(torch.from_numpy(f).to(DEV), torch.from_numpy(i).to(DEV), shape, 2).pad_to(1024)
    a = spconv.SubMConv3d(c, c, 3, indice_key="s").to(DEV)(x)
    b = spconv.SubMConv3d(c, c, 3, indice_key="s").to(DEV)(x)
    assert a.num_valid is x.num_valid and b.num_valid is x.num_valid
    s = spconv.MaskedAddTable()([a, b])
    assert torch.equal(s.features, a.features + b.features) and s.num_valid is x.num_valid
    j = spconv.MaskedJoinTable()([a, b])
    assert torch.equal(j.features, torch.cat([a.features, b.features], 1)) and j.num_valid is x.num_valid
    other = b.replace_feature(b.features)
    other.num_valid = x.num_valid.clone()
    for mod in (spconv.MaskedAddTable(), spconv.MaskedJoinTable()):
        with pytest.raises(ValueError, match="same num_valid tensor object"):
            mod([a, other])


class _TwoBranch(nn.Module):
    """a SubM branch and a strided conv -> transposed conv branch (other coordinates), merged, pooled, classified"""

    def __init__(self):
        super().__init__()
        torch.manual_seed(3)
        self.subm = spconv.SubMConv3d(4, 16, 3, indice_key="s1", bias=False)
        self.down = spconv.SparseConv3d(4, 16, 2, stride=2, bias=False)
        self.up = spconv.SparseConvTranspose3d(16, 16, 2, stride=2, bias=False)
        self.merge = spconv.MaskedAddTableMisaligned()
        self.pool = spconv.MaskedGlobalAvgPool()
        self.head = nn.Linear(16, 5)

    def forward(self, x):
        return self.pool(self.merge([self.subm(x), self.up(self.down(x))]))


def test_two_branch_net_trains_padded_and_as_one_graph():
    from spconv_b200.pytorch.tables import AddTableMisaligned
    shape, b = [24, 48, 48], 4
    rng = np.random.default_rng(4)
    clouds = []
    for per in ([3000, 2500, 2800, 2000], [2000, 2900, 1000, 2600], [2600, 0, 2400, 2700]):
        f, i = random_cloud(rng, shape, per, 4)
        perm = rng.permutation(i.shape[0])
        clouds.append((torch.from_numpy(f[perm]).to(DEV).half(), torch.from_numpy(i[perm]).to(DEV)))
    n_pad = 10_400
    net = _TwoBranch().to(DEV)
    for mod in (net.subm, net.down, net.up):
        mod.half()
    params = list(net.parameters())
    labels = torch.tensor([0, 3, 1, 4], device=DEV)

    def step(f, i, nv=None):
        for p in params:
            p.grad = None
        x = spconv.SparseConvTensor(f, i, shape, b)
        x.num_valid = nv
        pooled = net(x)
        loss = nn.functional.cross_entropy(net.head(pooled.float()), labels)
        loss.backward()
        return loss.detach(), [p.grad for p in params], pooled.detach()

    masked = net.merge
    net.merge = AddTableMisaligned()                 # the reference: unpadded eager with the default sparse_add
    want = []
    for f, i in clouds:
        loss, grads, pooled = step(f, i)
        want.append((loss.clone(), [g.clone() for g in grads], pooled.clone()))
    net.merge = masked

    bounds = spconv.set_output_bounds(net, spconv.SparseConvTensor(*clouds[0], shape, b), margin=1.25)
    assert set(bounds) == {"down", "up", "merge"}
    padded = [spconv.SparseConvTensor(f, i, shape, b).pad_to(n_pad) for f, i in clouds]
    args = [(p.features, p.indices, p.num_valid) for p in padded]

    def same(got, ref, what):
        loss, grads, pooled = got
        assert torch.equal(_bits(pooled), _bits(ref[2])), f"{what}: pooled features"
        assert abs(float(loss) - float(ref[0])) <= 1e-4 * abs(float(ref[0])), what
        for (name, _), g, r in zip(net.named_parameters(), grads, ref[1]):
            assert rel_l2(g.float().cpu().numpy(), r.float().cpu().numpy()) < 2e-3, (what, name)

    step(*args[0])                                   # warm-up: allocator pools, status words
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = step(*args[1])                         # eager, padded: no synchronising call
    finally:
        torch.cuda.set_sync_debug_mode("default")
    same(got, want[1], "eager padded")
    got = None

    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 2, 1):
        same(graphed(*args[k]), want[k], f"replay of cloud {k}")
    spconv.check_bounds(net)
