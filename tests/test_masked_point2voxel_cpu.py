"""MaskedPointToVoxel, the parts that need no GPU: argument validation of spx_point2voxel_bounded before any launch,
the workspace sizes, the refusal of CPU tensors and bad arguments, and the exports."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

import spconv_b200.pytorch as spconv
from spconv_b200 import _cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KITTI = ([0.4, 0.4, 0.5], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0])


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import build
    build.build()
    return _cabi.load()


def test_workspace_sizes(lib):
    size = lib.spx_point2voxel_bounded_workspace_size
    assert size(-1, 1, 10) == 0 and size(10, 0, 10) == 0 and size(10, _cabi.SPX_P2V_MAX_BATCH + 1, 10) == 0
    assert size(10, 1, 0) == 0 and size(1 << 31, 1, 10) == 0 and size(10, 1, 1 << 31) == 0
    assert size(0, 1, 1) > 0
    prev = 0
    for n in (1, 1000, 100_000, 1 << 20):
        cur = size(n, 8, 4 * n)
        assert cur > prev and cur >= n * (8 + 4 + 4 + 4) + 2 * n * 8      # keys, first, rows, order; the table
        prev = cur
    assert size(100_000, 8, 1000) < size(100_000, 8, 100_000)            # the row starts follow the bound


def test_entry_point_validates_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def arr(t, vals):",
        "    return (t * len(vals))(*vals)",
        "VS, GRID, RNG = arr(ctypes.c_float, [0.5, 0.4, 0.4]), arr(ctypes.c_int, [8, 200, 176]), "
        "arr(ctypes.c_float, [-3.0, -40.0, 0.0, 1.0, 40.0, 70.4])",
        "def run(pts=P, n=100, nf=4, nd=3, vs=VS, grid=GRID, rng=RNG, off=P, b=2, mv=10, bound=20, mp=5, vox=P, "
        "ind=P, num=P, ids=P, nv=P, st=P, ws=P, wsb=1 << 40):",
        "    return lib.spx_point2voxel_bounded(pts, n, nf, nd, 1, vs, grid, rng, off, b, mv, bound, mp, 0, vox, ind,",
        "                                       num, ids, nv, st, ws, wsb, None)",
        "def expect(rc, text):",
        "    assert rc != 0 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "expect(run(n=-1), 'points, must be in')",
        "expect(run(n=1 << 31), 'points, must be in')",
        "expect(run(b=0), 'batch_size 0 not in')",
        f"expect(run(b={_cabi.SPX_P2V_MAX_BATCH + 1}), 'not in [1, {_cabi.SPX_P2V_MAX_BATCH}]')",
        "expect(run(off=None), 'point_offsets may be NULL only with batch_size 1')",
        "expect(run(bound=0), 'bound 0 not in')",
        "expect(run(bound=1 << 31), 'not in [1, 2^31 - 2]')",
        "expect(run(mv=0), 'max_voxels must be positive')",
        "expect(run(mp=0), 'max_points_per_voxel must be positive')",
        "expect(run(nd=0), 'ndim must be in [1, 4]')",
        "expect(run(nd=5), 'ndim must be in [1, 4]')",
        "expect(run(vs=None), 'NULL geometry')",
        "expect(run(grid=None), 'NULL geometry')",
        "expect(run(rng=None), 'NULL geometry')",
        "expect(run(vs=arr(ctypes.c_float, [0.5, 0.0, 0.4])), 'bad voxel size / grid on axis 1')",
        "expect(run(grid=arr(ctypes.c_int, [8, -1, 176])), 'bad voxel size / grid on axis 1')",
        "expect(run(nf=2), 'fewer than the 3 coordinates')",
        "expect(run(grid=arr(ctypes.c_int, [1 << 30, 1 << 30, 1 << 10])), 'below 2^62')",
        "expect(run(b=4, grid=arr(ctypes.c_int, [1 << 30, 1 << 30, 2])), 'below 2^62')",
        "for k in ('vox', 'ind', 'num', 'nv', 'st', 'ws', 'pts', 'ids'):",
        "    expect(run(**{k: None}), 'NULL pointer')",
        "expect(run(wsb=64), 'workspace too small')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def test_refuses_cpu_tensors_and_bad_arguments():
    with pytest.raises(RuntimeError, match="CUDA only"):
        spconv.MaskedPointToVoxel(*KITTI, 4, 100, 5, 2, device="cpu")
    bad = [dict(max_num_voxels=0), dict(max_num_points_per_voxel=0), dict(batch_size=0),
           dict(batch_size=_cabi.SPX_P2V_MAX_BATCH + 1), dict(max_num_voxels_total=0),
           dict(max_num_voxels_total=1 << 31)]
    for kw in bad:
        args = dict(num_point_features=4, max_num_voxels=100, max_num_points_per_voxel=5, batch_size=2)
        args.update(kw)
        with pytest.raises(ValueError, match="MaskedPointToVoxel"):
            spconv.MaskedPointToVoxel(*KITTI, device="cuda", **args)
    # a call with CPU tensors is refused before anything touches the device
    gen = object.__new__(spconv.MaskedPointToVoxel)
    gen.num_point_features, gen.batch_size = 4, 2
    with pytest.raises(RuntimeError, match="must be CUDA tensors"):
        gen(torch.zeros(10, 4))
    with pytest.raises(RuntimeError, match="must be CUDA tensors"):
        gen(torch.zeros(10, 4), torch.zeros(3, dtype=torch.int32))


def test_names_are_exported():
    from spconv_b200.pytorch import utils
    assert spconv.MaskedPointToVoxel is utils.MaskedPointToVoxel
    assert spconv.PointToVoxel is utils.PointToVoxel
    assert "spx_point2voxel_bounded" in _cabi.SIGNATURES and "spx_point2voxel_bounded_workspace_size" in _cabi.SIGNATURES
    with open(os.path.join(ROOT, "include", "spconv_b200.h")) as f:
        header = f.read()
    assert f"#define SPX_P2V_MAX_BATCH {_cabi.SPX_P2V_MAX_BATCH}" in header
