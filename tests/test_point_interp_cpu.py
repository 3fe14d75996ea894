"""VoxelPointInterpolator, the parts that need no GPU: the numpy oracle against float64 and against a restatement of
torchsparse's calc_ti_weights / spdevoxelize, grid_positions on hand-computed cases, the workspace size, argument
validation of the C entry points before any launch, the refusal of CPU tensors and other dtypes, and the export."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import VoxelPointInterpolator, grid_positions, ops
from tests import point_interp_oracle as pi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def _tensor(rng, shape, batch, fill=0.5):
    """indices [rows, 1 + ndim] of a random occupancy (zyx), shuffled"""
    cells = np.argwhere(rng.random((batch, *shape)) < fill).astype(np.int32)
    return cells[rng.permutation(cells.shape[0])]


def _points(rng, shape, batch, p):
    pos = (rng.random((p, len(shape))) * (np.array(shape) + 1) - 1).astype(np.float32)
    return pos, rng.integers(0, batch, p).astype(np.int32)


@pytest.mark.parametrize("mode", ["trilinear", "nearest"])
@pytest.mark.parametrize("ndim", [1, 2, 3, 4])
def test_oracle_against_float64(ndim, mode):
    rng = np.random.default_rng(ndim)
    shape = [9, 7, 6, 5][:ndim]
    inds = _tensor(rng, shape, 2)
    pos, bid = _points(rng, shape, 2, 3_000)
    x = rng.standard_normal((inds.shape[0], 5)).astype(np.float32)
    dy = rng.standard_normal((3_000, 5)).astype(np.float32)
    for normalize in (True, False):
        i32, w32 = pi.plan(inds, shape, 2, None, pos, bid, mode, normalize)
        i64, w64 = pi.plan_f64(inds, shape, 2, None, pos, bid, mode, normalize)
        assert np.array_equal(i32, i64) and w32.dtype == np.float32
        assert np.allclose(w32, w64, rtol=2e-6, atol=1e-7)
        assert np.allclose(pi.forward(x, i32, w32), pi.forward_f64(x, i64, w64), rtol=1e-5, atol=1e-5)
        assert np.allclose(pi.backward(dy, i32, w32, inds.shape[0]), pi.backward_f64(dy, i64, w64, inds.shape[0]),
                           rtol=1e-5, atol=1e-4)
        found = i32 >= 0
        if normalize:                                     # the found weights sum to S / (S + 1e-8), ~1 unless S ~ 0
            raw = pi.plan_f64(inds, shape, 2, None, pos, bid, mode, False)[1].sum(1)
            assert np.allclose(w64.sum(1), raw / (raw + 1e-8), rtol=1e-12, atol=1e-12)
            assert (w64.sum(1)[raw > 1e-3] > 1 - 1e-5).all()
        elif mode == "trilinear":
            assert np.all(w32 >= 0) and np.all(w32 <= 1)
    assert (i32 >= 0).any() and (i32 < 0).any()


def test_oracle_weights_rule():
    """one 2-D point by hand: f = (0.25, 0.5), every corner present, then one missing"""
    inds = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 0], [0, 1, 1], [0, 1, 1]], np.int32)   # row 4 duplicates row 3
    pos = np.array([[0.25, 0.5]], np.float32)
    idx, w = pi.plan(inds, [2, 2], 1, None, pos, [0], "trilinear", False)
    assert idx.tolist() == [[0, 2, 1, 3]]                 # bit 0 = axis 0, lowest row of a duplicate
    assert w.tolist() == [[0.375, 0.125, 0.375, 0.125]]
    idx, w = pi.plan(inds[1:], [2, 2], 1, None, pos, [0], "trilinear", True)
    assert idx.tolist() == [[-1, 1, 0, 2]]
    assert np.allclose(w, [[0, 0.2, 0.6, 0.2]], rtol=1e-6)
    idx, w = pi.plan(inds, [2, 2], 1, None, pos, [0], "nearest", True)
    assert idx.tolist() == [[1]] and w.tolist() == [[1.0]]  # (0 + (0.25 >= .5), 0 + (0.5 >= .5)) = (0, 1)
    idx, _ = pi.plan(inds, [2, 2], 1, 2, pos, [0], "trilinear", True)     # num_valid = 2: rows 0 and 1 only
    assert idx.tolist() == [[0, -1, 1, -1]]
    for bad in ([np.nan, 0.5], [np.inf, 0.5], [-1.01, 0.5], [2.0, 0.5], [0.5, 1e30]):
        idx, w = pi.plan(inds, [2, 2], 1, None, np.array([bad], np.float32), [0], "trilinear", True)
        assert (idx == -1).all() and (w == 0).all(), bad
    idx, _ = pi.plan(inds, [2, 2], 1, None, pos, [1], "trilinear", True)
    assert (idx == -1).all()
    idx, w = pi.plan(inds, [2, 2], 1, None, np.array([[-0.5, 1.5]], np.float32), [0], "trilinear", False)
    assert idx.tolist() == [[-1, 1, -1, -1]] and w.tolist() == [[0, 0.25, 0, 0]]     # only corner (0, 1) exists


def _ts_devoxelize(q_xyz, s, batch, rows_xyz, feats):
    """numpy restatement of torchsparse's calc_ti_weights + spdevoxelize (float64): q_xyz are the points in
    stride-1 voxel units, rows_xyz [rows, 4] (b, x, y, z) the tensor's coordinates multiplied by the stride s"""
    pf = np.floor(q_xyz / s) * s
    pc = pf + s
    table = {tuple(int(v) for v in r): i for i, r in reversed(list(enumerate(rows_xyz)))}
    ws, idx = [], []
    for cx in (0, 1):
        for cy in (0, 1):
            for cz in (0, 1):
                c = np.stack([pc[:, 0] if cx else pf[:, 0], pc[:, 1] if cy else pf[:, 1],
                              pc[:, 2] if cz else pf[:, 2]], 1)
                w = np.ones(q_xyz.shape[0])
                for a, bit in enumerate((cx, cy, cz)):
                    w *= (q_xyz[:, a] - pf[:, a]) if bit else (pc[:, a] - q_xyz[:, a])
                ws.append(w / s ** 3)
                idx.append([table.get((int(b), *[int(v) for v in cc]), -1) for b, cc in zip(batch, c)])
    w, idx = np.stack(ws, 1), np.array(idx).T
    w[idx == -1] = 0
    w /= w.sum(1, keepdims=True) + 1e-8
    return (w[:, :, None] * np.where(idx[:, :, None] >= 0, feats[np.maximum(idx, 0)], 0)).sum(1)


@pytest.mark.parametrize("stride", [1, 2, 4])
def test_oracle_against_torchsparse_devoxelize(stride):
    rng = np.random.default_rng(10 + stride)
    vsize, lo = [0.5, 0.25, 0.125], [0.0, -4.0, -1.0]
    grid_xyz = np.array([24, 20, 16])
    shape_xyz = -(-grid_xyz // stride)
    inds = _tensor(rng, list(shape_xyz[::-1]), 2, 0.6)                 # (b, z, y, x) at the stride
    feats = rng.standard_normal((inds.shape[0], 4))
    n = 2_000
    q = rng.random((n, 3)) * grid_xyz
    pts = (q * np.array(vsize) + np.array(lo)).astype(np.float32)
    q = (pts.astype(np.float64) - np.array(lo)) / np.array(vsize)
    bid = rng.integers(0, 2, n).astype(np.int32)
    cr = lo + list(grid_xyz * np.array(vsize) + np.array(lo))
    pos = grid_positions(torch.from_numpy(pts), vsize, cr, stride=stride, center=-0.5).numpy()
    idx, w = pi.plan(inds, list(shape_xyz[::-1]), 2, None, pos, bid, "trilinear", True)
    got = pi.forward(feats.astype(np.float32), idx, w)
    rows_xyz = np.concatenate([inds[:, :1], inds[:, 1:][:, ::-1] * stride], 1)
    want = _ts_devoxelize(q, stride, bid, rows_xyz, feats.astype(np.float32).astype(np.float64))
    assert np.allclose(got, want, rtol=1e-4, atol=2e-5), np.abs(got - want).max()
    assert (idx >= 0).sum() > n


def test_grid_positions_conventions():
    vsize, cr = [0.5, 0.25, 0.125], [0.0, -8.0, -2.0, 8.0, 8.0, 2.0]
    pts = torch.tensor([[1.75, -7.375, -1.5, 9.0]])              # (p - lo) / vsize = (3.5, 2.5, 4.0); 4th column unused
    assert grid_positions(pts, vsize, cr).tolist() == [[3.5, 2.0, 3.0]]                      # zyx
    assert grid_positions(pts, vsize, cr, stride=2).tolist() == [[1.75, 1.0, 1.5]]            # k3 s2 p1 chains
    assert grid_positions(pts, vsize, cr, stride=2, center=0.5).tolist() == [[1.5, 0.75, 1.25]]   # k = s = 2
    assert grid_positions(pts, vsize, cr, stride=2, center=-0.5).tolist() == [[2.0, 1.25, 1.75]]  # torchsparse
    assert grid_positions(pts, vsize, cr, stride=[1, 2, 4], center=[0, 0.5, 1.5]).tolist() == [[0.5, 0.75, 3.0]]
    # a voxel's centre lands on its index; at stride 2, output o of k3 s2 p1 sits at input voxel 2o and output o of
    # k = s = 2 at the middle of input voxels 2o and 2o + 1
    centre = torch.tensor([[0.0 + 5.5 * 0.5, -8.0 + 6.5 * 0.25, -2.0 + 4.5 * 0.125]])
    assert grid_positions(centre, vsize, cr).tolist() == [[4.0, 6.0, 5.0]]
    assert grid_positions(centre, vsize, cr, stride=2).tolist() == [[2.0, 3.0, 2.5]]
    mid = torch.tensor([[0.0 + 5.0 * 0.5, -8.0 + 7.0 * 0.25, -2.0 + 5.0 * 0.125]])      # between voxels 4 and 5 / 6, 7
    assert grid_positions(mid, vsize, cr, stride=2, center=0.5).tolist() == [[2.0, 3.0, 2.0]]
    assert grid_positions(pts, vsize, cr).dtype == torch.float32
    with pytest.raises(ValueError, match="coors_range"):
        grid_positions(pts, vsize, cr[:4])
    with pytest.raises(ValueError, match="center needs 3"):
        grid_positions(pts, vsize, cr, center=[0, 0])
    with pytest.raises(ValueError, match="points must be"):
        grid_positions(pts[:, :2], vsize, cr)


def _workspace(lib, ndim, shape, batch, rows, p, mode):
    k = 1 if mode == 1 else 1 << ndim
    cap = 1024
    while cap < rows * 4:
        cap <<= 1
    i64 = batch * float(np.prod(np.array(shape, np.float64))) >= 2147483647.0
    a = lambda v: (v + 255) // 256 * 256  # noqa: E731
    off = cap * 8
    if i64:
        off = a(off) + cap * 4
    off = a(off) + lib.spx_sparse_add_group_workspace_size(p * k)
    return a(off) + 256


def _args(ndim=3, shape=(4, 4, 4, 4), batch=2, rows=10, p=10, mode=0):
    from spconv_b200 import _cabi
    a = _cabi.PointInterp()
    a.ndim, a.batch_size, a.rows, a.num_points, a.mode = ndim, batch, rows, p, mode
    for i, v in enumerate(shape[:4]):
        a.spatial_shape[i] = v
    return a


def test_workspace_size(lib):
    import ctypes
    fn = lambda **kw: lib.spx_point_interp_plan_workspace_size(ctypes.byref(_args(**kw)))  # noqa: E731
    for ndim, shape, batch in ((3, [41, 1600, 1408], 4), (2, [512, 512], 2), (1, [100], 1), (4, [8, 8, 8, 8], 3),
                               (3, [2048, 2048, 2048], 2)):
        prev = 0
        for rows in (0, 1, 1000, 300_000):
            for p in (0, 7, 200_000):
                for mode in (0, 1):
                    got = fn(ndim=ndim, shape=shape, batch=batch, rows=rows, p=p, mode=mode)
                    assert got == _workspace(lib, ndim, shape, batch, rows, p, mode), (ndim, rows, p, mode)
            assert got >= prev
            prev = got
    assert lib.spx_point_interp_plan_workspace_size(None) == 0
    assert fn(ndim=0) == 0 and fn(ndim=5) == 0 and fn(batch=0) == 0 and fn(rows=-1) == 0 and fn(p=-1) == 0
    assert fn(mode=2) == 0 and fn(p=1 << 28) == 0 and fn(p=1 << 28, mode=1) > 0


def test_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def args(nd=3, sh=(4, 4, 4), b=2, ind=P, rows=10, nv=None, pos=P, bid=P, n=10, mode=0, norm=1, idx=P, w=P,",
        "         order=P, off=P, c=16, dt=1, x=P, y=P, dy=P, dx=P):",
        "    a = _cabi.PointInterp(ndim=nd, batch_size=b, mode=mode, normalize=norm, channels=c, dtype=dt, rows=rows,",
        "                          num_points=n, indices=ind, num_valid=nv, pos=pos, batch_ids=bid, index=idx, weight=w,",
        "                          order=order, offsets=off, x=x, y=y, dy=dy, dx=dx)",
        "    for i, v in enumerate(sh):",
        "        a.spatial_shape[i] = v",
        "    return ctypes.byref(a)",
        "def plan(ws=P, wsb=1 << 40, **kw):",
        "    return lib.spx_point_interp_plan(args(**kw), ws, wsb, None)",
        "def fwd(**kw):",
        "    return lib.spx_point_interp_fwd(args(**kw), None)",
        "def bwd(**kw):",
        "    return lib.spx_point_interp_bwd(args(**kw), None)",
        "def expect(rc, text):",
        "    assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "for f in (lib.spx_point_interp_fwd, lib.spx_point_interp_bwd):",
        "    expect(f(None, None), 'argument block is NULL')",
        "expect(lib.spx_point_interp_plan(None, P, 1 << 40, None), 'argument block is NULL')",
        "expect(plan(nd=0), 'ndim must be')",
        "expect(plan(nd=5), 'ndim must be')",
        "expect(plan(sh=(4, 0, 4)), 'spatial_shape[1] must be positive')",
        "expect(plan(b=0), 'batch_size must be')",
        "expect(plan(norm=2), 'normalize must be')",
        "for k in ('off', 'ws', 'ind', 'pos', 'bid', 'idx', 'w', 'order'):",
        "    expect(plan(**{k: None}), 'NULL pointer')",
        "expect(plan(wsb=64), 'workspace too small')",
        "expect(plan(n=1 << 28), 'too many')",
        "for f in (plan, fwd, bwd):",
        "    expect(f(nd=0), 'ndim must be')",
        "    expect(f(mode=2), 'mode must be')",
        "    expect(f(mode=-1), 'mode must be')",
        "    expect(f(rows=-1), 'bad row count')",
        "    expect(f(rows=(1 << 31) - 1), 'bad row count')",
        "    expect(f(n=-1), 'bad point count')",
        "    expect(f(n=(1 << 31) - 1), 'bad point count')",
        "for f in (fwd, bwd):",
        "    expect(f(n=1 << 28), 'bad point count')",
        "    expect(f(c=0), 'channels must be')",
        "    expect(f(dt=3), 'unsupported dtype')",
        "    expect(f(dt=7), 'unsupported dtype')",
        "    expect(f(n=1 << 26, nd=4, c=1 << 16), 'too many')",
        "for k in ('x', 'idx', 'w', 'y'):",
        "    expect(fwd(**{k: None}), 'NULL pointer')",
        "for k in ('dy', 'w', 'order', 'off', 'dx'):",
        "    expect(bwd(**{k: None}), 'NULL pointer')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def test_refuses_cpu_tensors_and_other_dtypes():
    inds = torch.zeros(4, 4, dtype=torch.int32)
    x = spconv.SparseConvTensor(torch.zeros(4, 8), inds, [4, 4, 4], 1)
    pos, bid = torch.zeros(3, 3), torch.zeros(3, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="indices must be a CUDA tensor"):
        VoxelPointInterpolator(x, pos, bid)
    with pytest.raises(ValueError, match="mode must be 'trilinear' or 'nearest'"):
        VoxelPointInterpolator(x, pos, bid, mode="bilinear")
    with pytest.raises(RuntimeError, match="pos must be a CUDA tensor"):
        ops.point_interp_plan(_Fake(), [4, 4, 4], 1, None, pos, bid)
    index, weight = torch.zeros(3, 8, dtype=torch.int32), torch.zeros(3, 8)
    order, offsets = torch.zeros(24, dtype=torch.int32), torch.zeros(5, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="features must be a CUDA tensor"):
        ops.point_interp_fwd(torch.zeros(4, 8), index, weight)
    with pytest.raises(RuntimeError, match="grad_output must be a CUDA tensor"):
        ops.point_interp_bwd(torch.zeros(3, 8), weight, order, offsets)
    for dt in (torch.int8, torch.float64, torch.int32):
        with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
            ops.point_interp_fwd(torch.zeros(4, 8, dtype=dt), index, weight)
        with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
            ops.point_interp_bwd(torch.zeros(3, 8, dtype=dt), weight, order, offsets)


class _Fake:
    """stands in for a CUDA tensor where the check must fail on another argument first"""
    is_cuda = True


def test_exported_and_documented():
    assert spconv.VoxelPointInterpolator is VoxelPointInterpolator
    assert spconv.grid_positions is grid_positions
    doc = VoxelPointInterpolator.__doc__
    for word in ("MaskedPointToVoxel", "PointVoxelScatter", "scatter.mean", "searchsorted", "grid_positions",
                 "num_valid", "stride=2", "normalize", "nearest", ".index", ".weight"):
        assert word in doc, word
    gdoc = grid_positions.__doc__
    for word in ("k3 s2 p1", "(s - 1) / 2", "-0.5", "torchsparse", "zyx"):
        assert word in gdoc, word
    assert callable(spconv.functional.point_interp)
