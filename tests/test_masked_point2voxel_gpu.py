"""MaskedPointToVoxel on the GPU: every sample's slice bit for bit against PointToVoxel run on that sample alone and
against the numpy oracle (tests/point2voxel_oracle.py), the offset rule (clamp, then prefix maximum), padding
invariance, repeatability, truncation with its status bit, no synchronising call, and a step from raw points to the
loss (SubM + bounded strided conv + MaskedBatchNorm1d + MaskedGlobalAvgPool) that replays as one CUDA graph."""
import numpy as np
import pytest
import torch
from torch import nn

from tests import point2voxel_oracle as p2v
from tests.util import rel_l2

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedBatchNorm1d

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
KITTI = ([0.4, 0.4, 0.5], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0])          # grid 8 x 200 x 176 (zyx)


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _cloud(rng, n, vs, cr, nf, spread=1.0, junk=0.02):
    """n points over the range (a random sub-box of relative size `spread`), 5 % beyond it, `junk` NaN / inf rows"""
    nd = len(vs)
    lo, hi = np.array(cr[:nd], np.float64), np.array(cr[nd:], np.float64)
    span = (hi - lo) * spread
    corner = lo + rng.random(nd) * (hi - lo - span)
    xyz = corner - 0.05 * span + rng.random((n, nd)) * span * 1.1
    pts = np.concatenate([xyz, rng.random((n, nf - nd)) * 4 - 2], 1).astype(np.float32)
    bad = rng.random(n) < junk
    pts[bad, rng.integers(0, nd, int(bad.sum()))] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32),
                                                                int(bad.sum()))
    return pts


def _eff(off, p):
    return np.maximum.accumulate(np.clip(np.asarray(off, np.int64), 0, p))


def _reference(pts, off, vs, cr, max_voxels, max_points, bound, empty_mean=False, oracle=True):
    """per sample: PointToVoxel on the sample's rows alone, its batch column and row offset applied, truncated at
    the bound; checked against the numpy oracle on the way.  -> (voxels, indices, num, ids, counts, kept)"""
    nf, nd = pts.shape[1], len(vs)
    gen = spconv.PointToVoxel(vs, cr, nf, max_voxels, max_points, device=DEV)
    eff = _eff(off, len(pts))
    ids = np.full(len(pts), -1, np.int64)
    vox, ind, num, counts = [], [], [], []
    base = 0
    for b in range(len(off) - 1):
        lo, hi = int(eff[b]), int(eff[b + 1])
        v, i, n, pid = (t.cpu().numpy() for t in gen.generate_voxel_with_id(torch.from_numpy(pts[lo:hi]).to(DEV),
                                                                            empty_mean=empty_mean))
        if oracle:
            ov, oi, on, oid = p2v.point2voxel(pts[lo:hi], vs, cr, max_voxels, max_points, empty_mean=False)
            assert np.array_equal(oi, i) and np.array_equal(on, n) and np.array_equal(oid, pid), f"oracle, sample {b}"
            if not empty_mean:
                assert np.array_equal(ov.view(np.int32), v.view(np.int32)), f"oracle voxels, sample {b}"
        c, ok = p2v.cells(pts[lo:hi], vs, cr)
        counts.append(len(np.unique(c[ok], axis=0)))                   # voxels before the per-sample cap
        k = max(0, min(len(v), bound - base))
        vox.append(v[:k])
        ind.append(np.concatenate([np.full((k, 1), b, np.int32), i[:k]], 1))
        num.append(n[:k])
        ids[lo:hi] = np.where((pid >= 0) & (pid < k), pid + base, -1)
        base += k
    return (np.concatenate(vox, 0) if vox else np.zeros((0, max_points, nf), np.float32),
            np.concatenate(ind, 0).reshape(-1, nd + 1), np.concatenate(num, 0), ids, counts, base)


def _check(out, ref, bound, what=""):
    voxels, indices, num, ids, nv = (t.cpu() for t in out)
    rv, ri, rn, rid, _, m = ref
    assert int(nv[0]) == m, f"{what}: num_valid {int(nv[0])} != {m}"
    assert voxels.shape[0] == bound and indices.shape[0] == bound and num.shape[0] == bound
    assert torch.equal(_bits(voxels[:m]), _bits(torch.from_numpy(rv))), f"{what}: voxels"
    assert torch.equal(indices[:m], torch.from_numpy(ri)), f"{what}: indices"
    assert torch.equal(num[:m], torch.from_numpy(rn)), f"{what}: num_per_voxel"
    assert torch.equal(ids, torch.from_numpy(rid)), f"{what}: pc_voxel_id"
    assert bool((indices[m:] == -1).all()) and not voxels[m:].any() and not num[m:].any(), f"{what}: padding rows"


def _offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)


def _run(gen, pts, off, empty_mean=False):
    return gen(torch.from_numpy(pts).to(DEV), None if off is None else torch.from_numpy(np.asarray(off, np.int32)).to(DEV),
               empty_mean=empty_mean)


@pytest.mark.parametrize("batch", [1, 3, 8])
def test_kitti_batches_bit_exact(batch):
    vs, cr = KITTI
    rng = np.random.default_rng(batch)
    sizes = rng.integers(20_000, 120_001, batch)
    spreads = [0.12 if b % 2 else 1.0 for b in range(batch)]          # dense samples stay under the cap
    pts = np.concatenate([_cloud(rng, int(n), vs, cr, 4, s) for n, s in zip(sizes, spreads)], 0)
    off = _offsets(sizes)
    max_voxels = 12_000
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, max_voxels, 5, batch, device=DEV)
    ref = _reference(pts, off, vs, cr, max_voxels, 5, gen.max_num_voxels_total)
    _check(_run(gen, pts, off), ref, gen.max_num_voxels_total, f"B={batch}")
    if batch > 1:
        counts = ref[4]
        assert any(c > max_voxels for c in counts) and any(c < max_voxels for c in counts), counts
    spconv.check_bounds(gen)                                           # the default bound never truncates


@pytest.mark.parametrize("max_points", [1, 35])
def test_points_per_voxel_caps_and_empty_mean(max_points):
    vs, cr = KITTI
    rng = np.random.default_rng(20 + max_points)
    sizes = [30_000, 0, 25_000]
    pts = np.concatenate([_cloud(rng, n, vs, cr, 4, 0.1) for n in sizes], 0)
    pts[:, 3] = np.round(pts[:, 3] * 8) / 8                            # exact sums for the oracle's mean
    off = _offsets(sizes)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, 6_000, max_points, 3, device=DEV)
    for empty_mean in (False, True):
        ref = _reference(pts, off, vs, cr, 6_000, max_points, gen.max_num_voxels_total, empty_mean, oracle=True)
        _check(_run(gen, pts, off, empty_mean), ref, gen.max_num_voxels_total, f"empty_mean={empty_mean}")


@pytest.mark.parametrize("nd,vs,cr", [
    (2, [0.25, 0.5], [-4.0, -8.0, 4.0, 8.0]),
    (4, [1.0, 0.5, 0.5, 2.0], [0.0, 0.0, 0.0, 0.0, 8.0, 6.0, 4.0, 16.0]),
    (3, [0.01, 0.01, 0.01], [0.0, 0.0, 0.0, 20.0, 20.0, 10.0]),        # 4e9 cells x B: 64-bit keys
])
def test_other_grids_and_64_bit_keys(nd, vs, cr):
    rng = np.random.default_rng(nd)
    sizes = [9_000, 14_000, 0, 7_000]
    pts = np.concatenate([_cloud(rng, n, vs, cr, nd + 2, s) for n, s in zip(sizes, (1.0, 0.3, 1.0, 0.05))], 0)
    off = _offsets(sizes)
    gen = spconv.MaskedPointToVoxel(vs, cr, nd + 2, 3_000, 3, 4, device=DEV)
    for empty_mean in (False, True):
        ref = _reference(pts, off, vs, cr, 3_000, 3, gen.max_num_voxels_total, empty_mean, oracle=not empty_mean)
        _check(_run(gen, pts, off, empty_mean), ref, gen.max_num_voxels_total, f"nd={nd}")


def test_edges_of_the_offsets():
    vs, cr = KITTI
    rng = np.random.default_rng(5)
    pts = _cloud(rng, 6_000, vs, cr, 4)
    p = len(pts)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, 1_500, 5, 4, device=DEV)
    bound = gen.max_num_voxels_total
    cases = {
        "empty samples": [0, 0, 2_000, 2_000, 6_000],
        "off[B] = 0": [0, 0, 0, 0, 0],
        "decreasing and out of range": [700, -5, 4_000, 1_000, 1 << 30],
        "all beyond P": [p + 1, p + 2, p + 3, p + 4, p + 5],
        "negative": [-9, -8, -7, -1, -100],
        "partial tail": [100, 1_000, 2_500, 3_000, 4_000],
    }
    for name, off in cases.items():
        ref = _reference(pts, off, vs, cr, 1_500, 5, bound)
        _check(_run(gen, pts, off), ref, bound, name)
    far = pts.copy()
    far[:, :3] += 1000.0                                               # every point out of range
    _check(_run(gen, far, [0, 1_000, 3_000, 5_000, p]), _reference(far, [0, 1_000, 3_000, 5_000, p], vs, cr, 1_500, 5,
                                                                  bound), bound, "all out of range")
    one = spconv.MaskedPointToVoxel(vs, cr, 4, 1_500, 5, 1, device=DEV)
    _check(_run(one, pts, None), _reference(pts, [0, p], vs, cr, 1_500, 5, 1_500), 1_500, "point_offsets=None")
    out = _run(one, pts[:0], None)                                     # no points at all
    _check(out, _reference(pts[:0], [0, 0], vs, cr, 1_500, 5, 1_500), 1_500, "P = 0")


def test_padding_invariance():
    vs, cr = KITTI
    rng = np.random.default_rng(6)
    sizes = [40_000, 25_000, 33_000]
    valid = np.concatenate([_cloud(rng, n, vs, cr, 4, s) for n, s in zip(sizes, (1.0, 0.1, 0.4))], 0)
    off = _offsets(sizes)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, 16_000, 5, 3, device=DEV)
    base = [t.clone() for t in _run(gen, valid, off)]
    m = int(base[4])
    for pad in (1, 777, 50_000):
        junk = _cloud(rng, pad, vs, cr, 4, 0.05, junk=0.3)             # in-range points (and NaNs) that would merge
        got = _run(gen, np.concatenate([valid, junk], 0), off)
        assert int(got[4]) == m
        for a, b, name in zip(got[:3], base[:3], ("voxels", "indices", "num_per_voxel")):
            assert torch.equal(_bits(a), _bits(b)), f"pad {pad}: {name}"
        assert torch.equal(got[3][:len(valid)], base[3]) and bool((got[3][len(valid):] == -1).all()), f"pad {pad}"


def test_repeated_calls_leave_no_stale_rows():
    vs, cr = KITTI
    rng = np.random.default_rng(7)
    big = np.concatenate([_cloud(rng, 50_000, vs, cr, 4) for _ in range(4)], 0)
    small = _cloud(rng, 9_000, vs, cr, 4, 0.3)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, 30_000, 5, 4, device=DEV)
    _run(gen, big, _offsets([50_000] * 4), empty_mean=True)
    off = [0, 4_000, 4_000, 9_000, 9_000]
    got = [t.clone() for t in _run(gen, small, off)]
    fresh = spconv.MaskedPointToVoxel(vs, cr, 4, 30_000, 5, 4, device=DEV)
    want = _run(fresh, small, off)
    for a, b in zip(got, want):
        assert torch.equal(_bits(a), _bits(b))
    _check(got, _reference(small, off, vs, cr, 30_000, 5, gen.max_num_voxels_total), gen.max_num_voxels_total)


def test_truncation_keeps_the_prefix_and_sets_the_status_bit():
    vs, cr = KITTI
    rng = np.random.default_rng(8)
    sizes = [20_000, 30_000, 10_000]
    pts = np.concatenate([_cloud(rng, n, vs, cr, 4) for n in sizes], 0)
    off = _offsets(sizes)
    full = spconv.MaskedPointToVoxel(vs, cr, 4, 12_000, 5, 3, device=DEV)
    want = [t.clone() for t in _run(full, pts, off)]
    m_full = int(want[4])
    bound = 17_000
    assert m_full > bound
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, 12_000, 5, 3, max_num_voxels_total=bound, device=DEV)
    got = _run(gen, pts, off)
    assert int(got[4]) == bound
    for a, b in zip(got[:3], want[:3]):
        assert torch.equal(_bits(a), _bits(b[:bound]))
    assert torch.equal(got[3], torch.where(want[3] < bound, want[3], -1))
    _check(got, _reference(pts, off, vs, cr, 12_000, 5, bound, oracle=False), bound, "truncated")
    assert int(gen._bound_status) & 1
    with pytest.raises(RuntimeError, match="MaskedPointToVoxel.*more outputs than"):
        spconv.check_bounds(gen)
    spconv.check_bounds(gen)                                           # cleared by the read
    spconv.check_bounds(full)


def test_no_synchronising_call():
    vs, cr = KITTI
    rng = np.random.default_rng(9)
    pts = torch.from_numpy(_cloud(rng, 30_000, vs, cr, 4)).to(DEV)
    off = torch.tensor([0, 10_000, 10_000, 30_000], dtype=torch.int32, device=DEV)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, 8_000, 5, 3, device=DEV)
    gen(pts, off)
    feats = torch.randn(gen.max_num_voxels_total, 7, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for em in (False, True):
            ids = gen(pts, off, empty_mean=em)[3]
        per_point = spconv.gather_features_by_pc_voxel_id(feats, ids, invalid_value=-3.0)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    valid = ids >= 0
    assert torch.equal(per_point[valid], feats[ids[valid]]) and bool((per_point[~valid] == -3.0).all())


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(11)
        self.body = spconv.SparseSequential(
            spconv.SubMConv3d(4, 16, 3, indice_key="s1", bias=False), MaskedBatchNorm1d(16), nn.ReLU(),
            spconv.SparseConv3d(16, 32, 3, stride=2, padding=1, bias=False), MaskedBatchNorm1d(32), nn.ReLU())
        self.pool = spconv.MaskedGlobalAvgPool()
        self.head = nn.Linear(32, 5)

    def forward(self, x):
        return self.pool(self.body(x))


def test_points_to_loss_captures_as_one_graph():
    vs, cr = KITTI
    batch, max_voxels, p_pad = 3, 16_000, 150_000
    rng = np.random.default_rng(10)
    batches = []
    for sizes in ([40_000, 30_000, 45_000], [20_000, 50_000, 35_000], [48_000, 0, 42_000]):
        pts = np.concatenate([_cloud(rng, n, vs, cr, 4, s) for n, s in zip(sizes, (1.0, 0.3, 0.6))], 0)
        batches.append((pts, _offsets(sizes)))
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, max_voxels, 5, batch, device=DEV)
    shape = gen.grid_size
    net = _Net().to(DEV)
    net.body.half()
    params = list(net.parameters())
    labels = torch.tensor([0, 3, 1], device=DEV)

    def mean_features(voxels, num):
        return (voxels.sum(1) / num.clamp(min=1)[:, None].to(voxels.dtype)).half()

    def train(x):
        for p in params:
            p.grad = None
        pooled = net(x)
        loss = nn.functional.cross_entropy(net.head(pooled.float()), labels)
        loss.backward()
        return loss.detach(), [p.grad for p in params], pooled.detach()

    def step(points, offsets):
        voxels, indices, num, ids, nv = gen(points, offsets)
        x = spconv.SparseConvTensor(mean_features(voxels, num), indices, shape, batch)
        x.num_valid = nv
        return (voxels, indices, num, ids, nv) + train(x)

    # the reference: per-sample PointToVoxel, concatenated on the host, unpadded and eager
    single = spconv.PointToVoxel(vs, cr, 4, max_voxels, 5, device=DEV)
    want, examples = [], []
    for pts, off in batches:
        vox, ind, num, ids = [], [], [], []
        base = 0
        for b in range(batch):
            v, i, n, pid = single.generate_voxel_with_id(torch.from_numpy(pts[off[b]:off[b + 1]]).to(DEV))
            vox.append(v)
            ind.append(torch.cat([torch.full((len(i), 1), b, dtype=torch.int32, device=DEV), i], 1))
            num.append(n)
            ids.append(torch.where(pid >= 0, pid + base, -1))
            base += len(v)
        vox, ind, num = torch.cat(vox), torch.cat(ind), torch.cat(num)
        x = spconv.SparseConvTensor(mean_features(vox, num), ind, shape, batch)
        examples.append(x)
        loss, grads, pooled = train(x)
        want.append((vox, ind, num, torch.cat(ids), loss.clone(), [g.clone() for g in grads], pooled.clone()))
    spconv.set_output_bounds(net, examples[0], margin=1.5)
    args = []
    for pts, off in batches:
        padded = np.concatenate([pts, _cloud(rng, p_pad - len(pts), vs, cr, 4, 0.2, junk=0.2)], 0)
        args.append((torch.from_numpy(padded).to(DEV), torch.from_numpy(off).to(DEV)))

    def same(got, ref, what):
        voxels, indices, num, ids, nv, loss, grads, pooled = got
        m = ref[0].shape[0]
        assert int(nv) == m, what
        assert torch.equal(_bits(voxels[:m]), _bits(ref[0])) and torch.equal(indices[:m], ref[1]), what
        assert torch.equal(num[:m], ref[2]) and torch.equal(ids[:ref[3].shape[0]], ref[3]), what
        assert torch.equal(pooled.view(torch.int16), ref[6].view(torch.int16)), f"{what}: pooled features"
        assert abs(float(loss) - float(ref[4])) <= 1e-4 * abs(float(ref[4])), what
        for (name, _), g, r in zip(net.named_parameters(), grads, ref[5]):
            assert rel_l2(g.float().cpu().numpy(), r.float().cpu().numpy()) < 2e-3, (what, name)

    step(*args[0])                                                     # warm-up: allocator pools, status words
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = step(*args[1])                                           # eager, padded: no synchronising call
    finally:
        torch.cuda.set_sync_debug_mode("default")
    same(got, want[1], "eager padded")
    got = None

    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 2):
        same(graphed(*args[k]), want[k], f"replay of batch {k}")
    spconv.check_bounds(net)
    spconv.check_bounds(gen)
