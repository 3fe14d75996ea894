"""sparse_add / sparse_add_hash_based and the table modules on the GPU, bit for bit against the numpy oracle
(tests/sparse_add_oracle.py): output coordinates and their row order, features, and every operand's
gradient, for fp32, fp16 and bf16."""
import numpy as np
import pytest
import torch

from tests import sparse_add_oracle as sao

pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


def _pool(rng, batch, shape, n):
    """n distinct coordinates (b, *spatial), shuffled"""
    total = batch * int(np.prod(shape, dtype=np.float64))
    if total <= 10_000_000:
        keys = rng.choice(total, n, replace=False)
    else:
        keys = np.unique(rng.integers(0, total, int(n * 1.3) + 16, dtype=np.int64))
        keys = keys[rng.permutation(len(keys))][:n]
    assert len(keys) == n
    return np.stack(np.unravel_index(keys, (batch, *shape)), 1).astype(np.int32)


def _operands(rng, batch, shape, sizes, overlap, dups=0, oob=0):
    """operand 0 takes fresh coordinates; operand t > 0 shares round(overlap * size) of them with operand 0 and
    takes the rest fresh.  `dups` repeated rows go into operand 0, `oob` out-of-range rows into the last one."""
    pool = _pool(rng, batch, shape, sum(sizes) + 1)
    base, used = pool[:sizes[0]], sizes[0]
    ops = [base]
    for s in sizes[1:]:
        shared = min(int(round(overlap * s)), len(base))
        take = np.concatenate([base[rng.permutation(len(base))[:shared]], pool[used:used + s - shared]], 0)
        used += s - shared
        ops.append(take[rng.permutation(len(take))])
    if dups and len(ops[0]):
        d = np.concatenate([ops[0], ops[0][rng.integers(0, len(ops[0]), dups)]], 0)
        ops[0] = d[rng.permutation(len(d))]
    if oob:
        bad = _pool(rng, batch, shape, oob)
        for r in range(oob):
            a = r % (len(shape) + 1)
            bad[r, a] = (batch if a == 0 else shape[a - 1]) if r % 2 == 0 else -1
        last = np.concatenate([ops[-1], bad], 0)
        ops[-1] = last[rng.permutation(len(last))]
    return [o.astype(np.int32).reshape(-1, len(shape) + 1) for o in ops]


# id: (batch, shape, sizes, overlap, duplicates, out-of-range rows, channels)
CASES = {
    "T1-dup-C16": (2, [20, 20, 20], [300], 0.0, 40, 0, 16),
    "T2-disjoint-C64": (2, [30, 30, 30], [400, 300], 0.0, 0, 0, 64),
    "T2-half-C3": (3, [30, 30, 30], [400, 300], 0.5, 0, 0, 3),
    "T2-aligned-tie-C16": (2, [30, 30, 30], [300, 300], 1.0, 0, 0, 16),
    "T3-2d-largest-second-C129": (3, [50, 60], [200, 250, 150], 0.5, 10, 5, 129),
    "T5-4d-empty-tie-C1": (2, [6, 7, 8, 9], [100, 50, 0, 120, 120], 0.5, 0, 5, 1),
    "T2-int64-keys-C64": (2, [2048, 2048, 600], [500, 400], 0.5, 5, 3, 64),
    "T2-100k-C64": (2, [41, 1600, 1408], [100_000, 100_000], 0.5, 0, 0, 64),
}


def _exact(dtype, a):
    """float32 values that are exact in `dtype`"""
    return torch.from_numpy(a.astype(np.float32)).to(dtype).float().numpy()


def _randn(rng, *shape, dtype=torch.float32, requires_grad=False):
    """device tensor from the numpy generator (the CUDA generator's state belongs to other tests)"""
    t = torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).to(dtype).cuda()
    return t.requires_grad_() if requires_grad else t


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _run(inds, batch, shape, c, dtype, seed, fsp_fn=None):
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import functional as Fsp, ops
    rng = np.random.default_rng(seed)
    feats = [_exact(dtype, rng.standard_normal((len(i), c))) for i in inds]
    o_inds, o_sum, dst, visit = sao.sparse_add(inds, feats, batch, shape)
    m = o_inds.shape[0]
    want = torch.from_numpy(o_sum).to(dtype)
    dout = _exact(dtype, rng.standard_normal((m, c)))
    rows_v = [len(inds[i]) for i in visit]
    want_g = sao.gradients(dout, dst, rows_v)

    dev = torch.device("cuda")
    tens = [spconv.SparseConvTensor(torch.from_numpy(f).to(dtype).to(dev).requires_grad_(), torch.from_numpy(i).to(dev),
                                    shape, batch) for f, i in zip(feats, inds)]
    res = (fsp_fn or Fsp.sparse_add)(*tens)
    assert torch.equal(res.indices.cpu(), torch.from_numpy(o_inds)), "output coordinates / row order"
    assert res.features.dtype == dtype
    assert torch.equal(_bits(res.features), _bits(want)), "features"
    res.features.backward(torch.from_numpy(dout).to(dtype).to(dev))
    for k, i in enumerate(visit):
        assert torch.equal(_bits(tens[i].features.grad), _bits(torch.from_numpy(want_g[k]).to(dtype))), f"grad {i}"

    # the same through the op layer into NaN-filled buffers: every output element must be written
    out_inds, d_dst = ops.sparse_add_union([tens[i].indices for i in visit], batch, shape)
    assert torch.equal(d_dst.cpu(), torch.from_numpy(dst))
    order, offsets = ops.sparse_add_group(d_dst, m)
    out = torch.full((m, c), float("nan"), dtype=dtype, device=dev)
    ops.sparse_add_forward([tens[i].features.detach() for i in visit], order, offsets, m, out=out)
    assert torch.equal(_bits(out), _bits(want))
    outs = [torch.full((r, c), float("nan"), dtype=dtype, device=dev) for r in rows_v]
    ops.sparse_add_gather(d_dst, torch.from_numpy(dout).to(dtype).to(dev), rows_v, outs=outs)
    for k in range(len(visit)):
        assert torch.equal(_bits(outs[k]), _bits(torch.from_numpy(want_g[k]).to(dtype)))
    # grouping: ascending visit order within each output, the first row of a group created the output
    o_cpu, off = order.cpu().numpy(), offsets.cpu().numpy()
    assert off[0] == 0 and off[m] == int((dst >= 0).sum()) and np.all(np.diff(off) >= 1)
    for o in range(0, m, max(1, m // 97)):
        seg = o_cpu[off[o]:off[o + 1]]
        assert np.all(np.diff(seg) > 0) and np.all(dst[seg] == o) and np.all(dst[:seg[0]] != o)
    return res, tens


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("case", list(CASES))
def test_sparse_add_bit_exact_against_the_oracle(case, dt):
    batch, shape, sizes, overlap, dups, oob, c = CASES[case]
    rng = np.random.default_rng(sum(map(ord, case)))
    inds = _operands(rng, batch, shape, sizes, overlap, dups, oob)
    _run(inds, batch, shape, c, DTYPES[dt], seed=len(case))


@pytest.mark.parametrize("dt", list(DTYPES))
def test_empty_results(dt):
    """all operands empty, or every row out of range: a 0-row tensor, zero gradients, no exception"""
    from spconv_b200.pytorch import functional as Fsp
    e = np.zeros((0, 4), np.int32)
    res, _ = _run([e, e], 2, [8, 8, 8], 16, DTYPES[dt], seed=1)
    assert res.features.shape == (0, 16)
    bad = np.array([[2, 0, 0, 0], [0, 8, 1, 1], [-1, 1, 1, 1]], np.int32)
    res, tens = _run([bad, bad[:2]], 2, [8, 8, 8], 16, DTYPES[dt], seed=2, fsp_fn=Fsp.sparse_add_hash_based)
    assert res.features.shape == (0, 16) and res.indice_dict == {}
    assert not tens[0].features.grad.any()


def test_usage_example_keeps_the_3x3x3_rulebook():
    """USAGE.md: sparse_add(r133, r313, r333) returns r333's coordinates row for row and its indice_dict, so a
    SparseInverseConv3d on r333's key inverts it; sparse_add(r133, r313) drops the indice_dict"""
    import spconv_b200.pytorch as spconv
    from oracle import oracle
    from spconv_b200.pytorch import functional as Fsp
    rng = np.random.default_rng(5)
    dev = torch.device("cuda")
    shape, c = [16, 24, 24], 16
    inds = _pool(rng, 2, shape, 1500)
    x = spconv.SparseConvTensor(torch.from_numpy(_exact(torch.float16, rng.standard_normal((1500, c)))).half().to(dev),
                                torch.from_numpy(inds).to(dev), shape, 2)
    c133 = spconv.SparseConv3d(c, c, (1, 3, 3), 1, (0, 1, 1), bias=False).to(dev).half()
    c313 = spconv.SparseConv3d(c, c, (3, 1, 3), 1, (1, 0, 1), bias=False).to(dev).half()
    c333 = spconv.SparseConv3d(c, c, 3, 1, 1, bias=False, indice_key="k333").to(dev).half()
    inv = spconv.SparseInverseConv3d(c, c, 3, indice_key="k333", bias=False).to(dev).half()
    with torch.no_grad():
        for conv in (c133, c313, c333, inv):
            conv.weight.copy_(_randn(rng, *conv.weight.shape) * 0.1)
    r133, r313, r333 = c133(x), c313(x), c333(x)
    assert r333.features.shape[0] > max(r133.features.shape[0], r313.features.shape[0])
    for r in (r133, r313, r333):
        r.features.retain_grad()
    s = Fsp.sparse_add(r133, r313, r333)
    assert torch.equal(s.indices, r333.indices)
    assert s.indice_dict is r333.indice_dict and "k333" in s.indice_dict
    assert Fsp.sparse_add(r133, r313).indice_dict == {}

    feats = [r.features.detach().float().cpu().numpy() for r in (r133, r313, r333)]
    o_inds, o_sum, dst, visit = sao.sparse_add([r.indices.cpu().numpy() for r in (r133, r313, r333)], feats, 2, shape)
    assert visit[0] == 2
    np.testing.assert_array_equal(o_inds, r333.indices.cpu().numpy())
    y = inv(s)
    assert torch.equal(y.indices, x.indices)
    g = torch.from_numpy(_exact(torch.float16, rng.standard_normal((1500, c)))).half().to(dev)
    y.features.backward(g)
    # oracle: the inverse of the 3x3x3 rulebook, fed with the oracle's sum
    rb_inds, pairs, num = oracle.get_indice_pairs(inds, 2, shape, [3] * 3, [1] * 3, [1] * 3, [1] * 3, [0] * 3)
    np.testing.assert_array_equal(rb_inds, o_inds)
    w = inv.weight.detach().float().cpu().numpy()
    s16 = torch.from_numpy(o_sum).half().float().numpy()
    y_ref = oracle.indice_conv(s16, w, pairs, num, 1500, inverse=True)
    scale = np.abs(y_ref).max()
    assert np.abs(y.features.detach().float().cpu().numpy() - y_ref).max() <= 2e-2 * scale
    din_ref, _ = oracle.indice_conv_backward(s16, w, g.float().cpu().numpy(), pairs, num, inverse=True)
    grads = sao.gradients(din_ref, dst, [feats[i].shape[0] for i in visit])
    for k, i in enumerate(visit):
        got = (r133, r313, r333)[i].features.grad.float().cpu().numpy()
        assert np.abs(got - grads[k]).max() <= 2e-2 * np.abs(din_ref).max(), i


def _st(inds, feats, shape, batch=2):
    import spconv_b200.pytorch as spconv
    return spconv.SparseConvTensor(feats, inds, shape, batch)


def test_table_modules():
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch.identity import Identity
    from spconv_b200.pytorch.spatial import RemoveDuplicate
    from spconv_b200.pytorch.tables import AddTableMisaligned
    from spconv_b200.pytorch import functional as Fsp
    rng = np.random.default_rng(11)
    dev = torch.device("cuda")
    shape = [10, 12, 14]
    inds = torch.from_numpy(_pool(rng, 2, shape, 200)).to(dev)
    a = _st(inds, _randn(rng, 200, 8), shape)
    b = _st(inds, _randn(rng, 200, 8), shape)
    s = spconv.AddTable()([a, b])
    assert torch.equal(s.features, a.features + b.features) and s.indices is inds
    j = spconv.JoinTable()([a, b])
    assert torch.equal(j.features, torch.cat([a.features, b.features], 1))
    short = _st(inds[:150], _randn(rng, 150, 8), shape)
    with pytest.raises(AssertionError, match="use AddTableMisaligned instead"):
        spconv.AddTable()([a, short])
    with pytest.raises(AssertionError, match="you can't use JoinTable in two sptensor with different indices."):
        spconv.JoinTable()([a, short])
    # ConcatTable inside a SparseSequential, followed by AddTable
    seq = spconv.SparseSequential(spconv.ConcatTable().add(Identity()).add(spconv.SparseReLU()), spconv.AddTable())
    out = seq(a)
    assert torch.equal(out.features, a.features + torch.relu(a.features))
    assert spconv.ConcatTable().add(Identity()).input_spatial_size([3, 4]) == [3, 4]
    ident = spconv.Identity()
    assert ident(a) is a and ident.input_spatial_size([5]) == [5]
    # AddTableMisaligned == sparse_add_hash_based
    m = AddTableMisaligned()([a, short])
    ref = Fsp.sparse_add_hash_based(a, short)
    assert torch.equal(m.indices, ref.indices) and torch.equal(m.features, ref.features)
    assert m.indice_dict is a.indice_dict         # short's rows are a subset: a's coordinates, row for row
    # RemoveDuplicate: the first row of every coordinate, first-touch order, gradient to the kept rows only
    dup_rows = torch.tensor([5, 0, 7, 5, 199, 7], device=dev)
    d_inds = torch.cat([inds[:10], inds[dup_rows]], 0)
    d_inds[3, 1] = shape[0]                                   # out of range: dropped
    f = _randn(rng, 16, 8, requires_grad=True)
    r = RemoveDuplicate()(_st(d_inds, f, shape))
    keep = [0, 1, 2, 4, 5, 6, 7, 8, 9, 14]
    assert torch.equal(r.indices, d_inds[keep]) and torch.equal(r.features, f[keep])
    r.features.sum().backward()
    want = torch.zeros(16, 8, device=dev)
    want[keep] = 1
    assert torch.equal(f.grad, want)


def test_repeatable_partial_grad_and_mixed_dtypes():
    from spconv_b200.pytorch import functional as Fsp
    rng = np.random.default_rng(21)
    dev = torch.device("cuda")
    shape = [40, 40, 40]
    inds = [torch.from_numpy(i).to(dev) for i in _operands(rng, 2, shape, [20000, 30000, 5000], 0.5, 300, 10)]
    fa = _randn(rng, len(inds[0]), 32, dtype=torch.float16, requires_grad=True)
    fb = _randn(rng, len(inds[1]), 32, dtype=torch.float16)
    fc = _randn(rng, len(inds[2]), 32, dtype=torch.float16, requires_grad=True)
    t = [_st(i, f, shape) for i, f in zip(inds, (fa, fb, fc))]
    r1, r2 = Fsp.sparse_add(*t), Fsp.sparse_add(*t)
    assert torch.equal(r1.indices, r2.indices) and torch.equal(_bits(r1.features), _bits(r2.features))
    g = _randn(rng, *r1.features.shape, dtype=torch.float16)
    r1.features.backward(g)
    ga = fa.grad.clone()
    fa.grad = None
    r2.features.backward(g)
    assert torch.equal(_bits(fa.grad), _bits(ga)) and fb.grad is None and fc.grad is not None
    # fp16 + bf16 -> fp32, fp32 + fp16 -> fp32: promoted like `+`, gradients come back in each operand's dtype
    fb32 = fb.float().requires_grad_()
    tb = _st(inds[1], fb32, shape)
    tc = _st(inds[2], fc.detach().bfloat16().requires_grad_(), shape)
    mixed = Fsp.sparse_add(t[0], tb, tc)
    assert mixed.features.dtype == torch.float32
    ref = Fsp.sparse_add(_st(inds[0], fa.detach().float(), shape), tb, _st(inds[2], tc.features.detach().float(), shape))
    assert torch.equal(mixed.features, ref.features)
    mixed.features.sum().backward()
    assert tc.features.grad.dtype == torch.bfloat16 and fb32.grad.dtype == torch.float32


def test_operand_limit():
    from spconv_b200.pytorch import functional as Fsp
    dev = torch.device("cuda")
    shape = [8, 8, 8]
    ts = [_st(torch.tensor([[0, i % 8, i // 8, 1]], dtype=torch.int32, device=dev), torch.ones(1, 4, device=dev), shape)
          for i in range(65)]
    r = Fsp.sparse_add(*ts[:64])
    assert r.features.shape == (64, 4)
    with pytest.raises(ValueError, match="at most 64 operands"):
        Fsp.sparse_add(*ts)


def test_indice_dict_is_kept_only_when_the_rows_match():
    """the largest operand's indice_dict survives exactly when the output coordinates are its coordinates row for
    row -- not merely when the output has as many rows as it"""
    from spconv_b200.pytorch import functional as Fsp
    dev = torch.device("cuda")
    shape = [8, 8, 8]
    p = torch.tensor([[0, 1, 1, 1], [0, 2, 2, 2], [1, 3, 3, 3], [1, 4, 4, 4]], dtype=torch.int32, device=dev)

    def t(rows, tag):
        x = _st(p[rows] if rows else p[:0], torch.ones(len(rows), 4, device=dev), shape)
        x.indice_dict = {tag: tag}
        return x

    oob = _st(torch.cat([p[:2], torch.tensor([[0, 8, 0, 0]], dtype=torch.int32, device=dev)]), torch.ones(3, 4, device=dev),
              shape)
    oob.indice_dict = {"oob": 1}
    cases = [
        ((t([0, 0, 1], "a"), t([2], "b")), {}),              # 3 outputs = 3 rows of a, but a holds a duplicate
        ((oob, t([2], "b")), {}),                             # 3 outputs, one row of the largest out of range
        ((t([0, 1, 2], "a"), t([2, 0, 1], "b")), "a"),        # aligned, tie: the first operand's rulebook
        ((t([1], "a"), t([0, 1, 2], "b")), "b"),              # largest second, the other a subset
        ((t([0, 1], "a"), t([2, 3], "b")), {}),               # disjoint
        ((t([], "a"), t([], "b")), "a"),                      # nothing at all: the first operand
    ]
    for ops_, want in cases:
        for fn in (Fsp.sparse_add, Fsp.sparse_add_hash_based):
            r = fn(*ops_)
            assert r.indice_dict == ({want: want} if isinstance(want, str) else want), (want, r.indice_dict)
