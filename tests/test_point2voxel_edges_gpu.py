"""``PointToVoxel`` (``csrc/pointops.cu``) at its edges, bit for bit against the numpy restatement
``tests/point2voxel_oracle.py`` and, for finite 3-D clouds, against the reference's own CPU generator
(``oracle/_ref``): voxel order, indices, counts, kept points and per-point voxel ids.

Before each call the generator's ``indices`` and ``num_per_voxel`` buffers are filled with a sentinel,
so a voxel row the kernels never write shows."""
import numpy as np
import pytest
import torch

from tests import point2voxel_oracle as p2v
from tests.util import assert_equals_reference

pytestmark = pytest.mark.gpu

VS, CR = [0.4, 0.4, 0.5], [0, -40, -3, 70.4, 40, 1]          # 8 x 200 x 176 grid (zyx)
SENTINEL = -7


def _run(gen, pts, dev, empty_mean=False):
    gen.indices.fill_(SENTINEL)
    gen.num_per_voxel.fill_(SENTINEL)
    vox, ind, num, ids = gen.generate_voxel_with_id(torch.from_numpy(pts).to(dev), empty_mean=empty_mean)
    return vox.cpu().numpy(), ind.cpu().numpy(), num.cpu().numpy(), ids.cpu().numpy()


def _check(pts, vs, cr, max_voxels, max_points, dev, oracle=None, key=None, empty_mean=False, gen=None):
    from spconv_b200.pytorch.utils import PointToVoxel
    pts = np.ascontiguousarray(pts, dtype=np.float32)
    if gen is None:
        gen = PointToVoxel(vs, cr, pts.shape[1], max_voxels, max_points, dev)
    got = _run(gen, pts, dev, empty_mean)
    want = p2v.point2voxel(pts, vs, cr, max_voxels, max_points, empty_mean)
    for g, w, name in zip(got, want, ("voxels", "indices", "num_per_voxel", "pc_voxel_id")):
        assert g.shape == w.shape, (name, g.shape, w.shape)
        bad = np.argwhere(g.view(np.int32) != w.view(np.int32)) if g.dtype == np.float32 else np.argwhere(g != w)
        assert bad.size == 0, f"{name}: {len(bad)} differ, first at {bad[0].tolist()}"
    if oracle is not None:
        assert_equals_reference(key, got, lambda: oracle.point2voxel_ref(pts, vs, cr, max_voxels, max_points), oracle)
    return gen, got


def _cloud(seed, n, nf=4, span=([-1, -41, -4], [71, 41, 2])):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(span[0], span[1], size=(n, 3))
    return np.concatenate([xyz, rng.uniform(0, 1, size=(n, nf - 3))], axis=1).astype(np.float32)


def test_non_finite_and_extreme_coordinates(cuda_dev):
    """A NaN or infinite coordinate drops the point: it gets id -1 and makes no voxel (an all-NaN point
    used to become a voxel at the grid corner).  +-1e30 is out of range; -0.0 is in cell 0."""
    pts = _cloud(1, 4000)
    rng = np.random.default_rng(2)
    special = [np.nan, np.inf, -np.inf, 1e30, -1e30]
    for axis in range(3):
        for v in special:
            rows = rng.choice(len(pts), 40, replace=False)
            pts[rows, axis] = v
    pts[rng.choice(len(pts), 50, replace=False), :3] = np.nan
    pts[rng.choice(len(pts), 30, replace=False), :] = np.nan
    pts[rng.choice(len(pts), 30, replace=False), 0] = -0.0
    pts[:5, :3] = np.nan                                     # the very first points are NaN
    pts[5] = [-0.0, -0.0, -0.0, 0.5]                         # x = -0 is cell 0; y, z = -0 are inside the range
    _, (vox, ind, num, ids) = _check(pts, VS, CR, 20000, 5, cuda_dev)
    bad = ~np.isfinite(pts[:, :3]).all(axis=1)
    assert (ids[bad] == -1).all() and ids[5] >= 0
    assert np.isfinite(vox).all()


def test_non_finite_points_in_a_2d_grid(cuda_dev):
    rng = np.random.default_rng(3)
    pts = rng.uniform(-1, 11, size=(3000, 3)).astype(np.float32)
    pts[::17, 0] = np.nan
    pts[::19, 1] = -np.inf
    pts[::23, :2] = np.nan
    _check(pts, [0.5, 0.25], [0, 0, 10, 10], 5000, 3, cuda_dev)


@pytest.mark.parametrize("vs,cr", [(VS, CR), ([0.05, 0.05, 0.1], [-10, -10, -2, 10, 10, 2]), ([1, 1, 1], [0, 0, 0, 7, 5, 3])])
def test_voxel_boundaries(vs, cr, oracle, cuda_dev):
    """p one fp32 ulp either side of every voxel boundary on every axis, p == lo (cell 0), p == hi (out)"""
    pts = p2v.boundary_cloud(vs, cr, seed=4, extra_features=1)
    _check(pts, vs, cr, 200000, 4, cuda_dev, oracle, f"p2v-boundary-{vs}-{cr}")


@pytest.mark.parametrize("nd,vs,cr", [
    (2, [0.3, 0.2], [-3, -2, 3, 2]),
    (4, [0.5, 0.5, 0.5, 1.0], [0, 0, 0, 0, 8, 6, 4, 5]),
])
def test_2d_and_4d_grids(nd, vs, cr, cuda_dev):
    pts = p2v.boundary_cloud(vs, cr, seed=nd, extra_features=2, uniform=20000)
    _check(pts, vs, cr, 100000, 3, cuda_dev)
    _check(pts, vs, cr, 50, 2, cuda_dev)


def test_largest_32_bit_key(cuda_dev):
    """grid 2 x 32768 x 32767 (volume just below 2^31 - 1): 32-bit keys up to the far corner"""
    vs, cr = [1, 1, 1], [0, 0, 0, 32767, 32768, 2]
    rng = np.random.default_rng(5)
    far = np.array([32766.5, 32767.5, 1.5], np.float32)
    pts = np.concatenate([rng.uniform(0, 1, size=(200, 3)) * np.array([32767, 32768, 2]),
                          np.tile(far, (5, 1)), [[32766.999, 32767.999, 1.999], [0, 0, 0], [32767, 0, 0]],
                          rng.uniform(32700, 32768, size=(200, 3)) * np.array([1, 1, 2 / 32768])]).astype(np.float32)
    pts = pts[rng.permutation(len(pts))]
    pts = np.concatenate([pts, np.zeros((len(pts), 1), np.float32)], axis=1)
    _, (_, ind, _, _) = _check(pts, vs, cr, 1000, 3, cuda_dev)
    assert [1, 32767, 32766] in ind.tolist()


def test_64_bit_keys(cuda_dev):
    """0.01 m voxels over 200 x 200 x 20 m: the grid volume needs 64-bit keys.  Pairs of voxels whose keys
    differ by exactly 2^32 must stay apart."""
    vs, cr = [0.01, 0.01, 0.01], [-100, -100, -10, 100, 100, 10]
    _, lo, grid = p2v.grid_size(vs, cr)
    assert np.prod(grid.astype(np.float64)) >= 2 ** 31 - 1
    rng = np.random.default_rng(6)
    keys = rng.integers(0, int(np.prod(grid)) - 2 ** 33, size=300)
    keys = np.concatenate([keys, keys + 2 ** 32, keys + 2 ** 33])
    c = np.stack([keys // (grid[1] * grid[2]), keys // grid[2] % grid[1], keys % grid[2]], 1)       # zyx
    xyz = (lo + (c + 0.5) * np.float32(0.01))[:, ::-1]
    pts = np.concatenate([xyz, rng.uniform(-100, 100, size=(5000, 3)) * np.array([1, 1, 0.1])])
    pts = pts[rng.permutation(len(pts))].astype(np.float32)
    pts = np.concatenate([pts, np.ones((len(pts), 1), np.float32)], axis=1)
    _check(pts, vs, cr, 100000, 2, cuda_dev)


@pytest.mark.parametrize("max_voxels,max_points", [(1, 5), (300, 5), (20000, 1), (20000, 64)])
def test_caps(max_voxels, max_points, oracle, cuda_dev):
    """max_voxels = 1; max_voxels below the distinct voxel count (the dropped voxels' points get -1);
    max_points = 1; max_points above any voxel's count"""
    pts = _cloud(7, 6000, span=([0, -10, -3], [20, 10, 1]))
    _, (_, _, num, ids) = _check(pts, VS, CR, max_voxels, max_points, cuda_dev, oracle,
                                 f"p2v-caps-{max_voxels}-{max_points}")
    if max_voxels <= 300:
        assert len(num) == max_voxels
    if max_points == 64:
        assert num.max() < 64


def test_degenerate_clouds(oracle, cuda_dev):
    from spconv_b200.pytorch.utils import PointToVoxel
    # 100 k points in one voxel
    rng = np.random.default_rng(8)
    one = np.concatenate([rng.uniform([0.01, 0.01, 0.01], [0.39, 0.39, 0.49], size=(100000, 3)),
                          rng.uniform(0, 1, size=(100000, 1))], axis=1).astype(np.float32)
    _, (_, ind, num, ids) = _check(one, VS, CR, 10, 5, cuda_dev, oracle, "p2v-one-voxel")
    assert num.tolist() == [5] and (ids == 0).all()
    # every point out of range: M = 0
    out = _cloud(9, 1000, span=([80, 50, 5], [90, 60, 6]))
    _, (vox, ind, num, ids) = _check(out, VS, CR, 10, 5, cuda_dev)
    assert vox.shape[0] == 0 and (ids == -1).all()
    # N = 0 and N = 1
    gen = PointToVoxel(VS, CR, 4, 10, 5, cuda_dev)
    vox, ind, num, ids = _run(gen, np.zeros((0, 4), np.float32), cuda_dev)
    assert vox.shape == (0, 5, 4) and ind.shape == (0, 3) and num.shape == (0,) and ids.shape == (0,)
    _check(np.array([[3.0, 2.0, 0.0, 0.5]], np.float32), VS, CR, 10, 5, cuda_dev, oracle, "p2v-one-point", gen=gen)
    # duplicate points
    dup = np.repeat(_cloud(10, 300), 4, axis=0)[np.random.default_rng(0).permutation(1200)]
    _check(dup, VS, CR, 1000, 3, cuda_dev, oracle, "p2v-duplicates")


@pytest.mark.parametrize("nf", [3, 9])
def test_feature_counts(nf, oracle, cuda_dev):
    pts = _cloud(11, 5000, nf=nf)
    _check(pts, VS, CR, 20000, 4, cuda_dev, oracle, f"p2v-features-{nf}")


def test_empty_mean_exact(cuda_dev):
    """features on a 2^-6 grid: the kernel's fp32 sums are exact, so the unused slots must equal
    fp32(sum) / fp32(num) bit for bit"""
    rng = np.random.default_rng(12)
    pts = (rng.integers(0, 8 * 64, size=(20000, 5)) * 2.0 ** -6).astype(np.float32)
    pts[:, 3:] -= 4
    _, (vox, _, num, _) = _check(pts, [0.5, 0.5, 0.5], [0, 0, 0, 4, 4, 4], 1000, 7, cuda_dev, empty_mean=True)
    assert ((num > 1) & (num < 7)).any() and (num == 7).any()


def test_repeat_calls_match_a_fresh_generator(cuda_dev):
    from spconv_b200.pytorch.utils import PointToVoxel
    big, small = _cloud(13, 30000), _cloud(14, 3000)
    small[::9, 1] = np.nan
    gen = PointToVoxel(VS, CR, 4, 20000, 5, cuda_dev)
    first = _run(gen, big, cuda_dev)
    again = _run(gen, big, cuda_dev)
    after = _run(gen, small, cuda_dev)
    fresh_big = _run(PointToVoxel(VS, CR, 4, 20000, 5, cuda_dev), big, cuda_dev)
    fresh_small = _run(PointToVoxel(VS, CR, 4, 20000, 5, cuda_dev), small, cuda_dev)
    for a, b, c in zip(first, again, fresh_big):
        assert np.array_equal(a, b) and np.array_equal(a, c)
    for a, b in zip(after, fresh_small):
        assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f")
    want = p2v.point2voxel(small, VS, CR, 20000, 5)
    for a, b in zip(after, want):
        assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f")
