"""PointVoxelScatter, the parts that need no GPU: the numpy oracle against float64 and against torch's CPU
scatter_reduce, the workspace size, argument validation of the C entry points before any launch, the refusal of
CPU tensors and other dtypes, and the export."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import PointVoxelScatter, ops
from tests import point_scatter_oracle as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def _case(seed, p=3_000, rows=400, c=6):
    rng = np.random.default_rng(seed)
    ids = rng.integers(-2, rows + 3, p)
    ids[rng.random(p) < 0.05] = 1 << 30
    ids[: p // 10] = 7                                   # one long row
    ids[(ids >= 100) & (ids < 120)] = -1                 # empty rows
    x =rng.standard_normal((p, c)).astype(np.float32)
    return x, ids, rows


def _scatter(x, ids, rows, reduce):
    """torch CPU scatter_reduce over rows + 1 (dropped points go to the spare last row)"""
    r = torch.from_numpy(np.where(ps.rows_of(ids, rows) >= 0, ids, rows))
    xt = torch.from_numpy(x).double()
    out = torch.zeros(rows + 1, x.shape[1], dtype=torch.float64)
    return out.scatter_reduce_(0, r[:, None].expand_as(xt), xt, reduce, include_self=False)[:rows].numpy()


def test_oracle_sum_and_mean_against_float64():
    x, ids, rows = _case(1)
    s64 = _scatter(x, ids, rows, "sum")
    s = ps.segment_sum(x, ids, rows)
    assert s.dtype == np.float32
    assert np.allclose(s, s64, rtol=1e-5, atol=1e-4)
    count = ps.group(ids, rows)[3]
    m64 = np.where(count[:, None] > 0, s64 / np.maximum(count, 1)[:, None], 0)
    assert np.allclose(ps.segment_mean(x, ids, rows), m64, rtol=1e-5, atol=1e-5)
    xi = np.round(x * 64).astype(np.float32)              # small integers: every fp32 sum is exact
    assert np.array_equal(ps.segment_sum(xi, ids, rows), _scatter(xi, ids, rows, "sum").astype(np.float32))
    assert count[7] >= 300 and (count == 0).any()


def test_oracle_sum_is_sequential_fp32():
    x = np.array([[1e8], [1.0], [-1e8], [1.0]], np.float32)
    ids = np.array([0, 0, 0, 0])
    assert ps.segment_sum(x, ids, 1)[0, 0] == np.float32(1.0)      # ((1e8 + 1) - 1e8) + 1 in float32
    assert ps.segment_sum(np.array([[-0.0]], np.float32), [0], 1).view(np.int32)[0, 0] == 0   # +0 + -0 = +0


def test_oracle_max_against_scatter_reduce():
    x, ids, rows = _case(2)
    arg = ps.segment_argmax(x, ids, rows)
    got = ps.take_argmax(x, arg)
    want = _scatter(x, ids, rows, "amax")
    count = ps.group(ids, rows)[3]
    assert np.array_equal(got[count > 0], want[count > 0].astype(np.float32))
    assert (arg[count == 0] == -1).all() and (got[count == 0] == 0).all()
    r = ps.rows_of(ids, rows)
    assert (r[arg[count > 0]] == np.nonzero(count > 0)[0][:, None]).all()    # the winner lies in its row


def test_oracle_max_rule():
    nan = np.float32(np.nan)
    x = np.array([[1.0, -0.0, 2.0], [nan, 0.0, 2.0], [5.0, 0.0, nan], [nan, -1.0, 3.0]], np.float32)
    ids = np.array([0, 0, 0, 0])
    arg = ps.segment_argmax(x, ids, 1)
    assert arg.tolist() == [[1, 0, 2]]                    # first NaN; -0 ties +0 (first wins); NaN over 3
    out = ps.take_argmax(x, arg)
    assert out.view(np.int32)[0, 1] == np.float32(-0.0).view(np.int32)
    dy = np.array([[4.0, 5.0, 6.0]], np.float32)
    assert ps.max_grad(dy, arg, ids, 1, 4).tolist() == [[0, 5, 0], [4, 0, 0], [0, 0, 6], [0, 0, 0]]
    assert ps.mean_grad(dy, [0, -1, 0, 3], 1).tolist() == [[2, 2.5, 3], [0, 0, 0], [2, 2.5, 3], [0, 0, 0]]
    assert ps.sum_grad(dy, [0, -1, 0, 3], 1).tolist() == [[4, 5, 6], [0, 0, 0], [4, 5, 6], [0, 0, 0]]


def test_workspace_size(lib):
    fn = lib.spx_point_scatter_group_workspace_size
    assert fn(-1) == 0
    prev = 0
    for n in (0, 1, 1000, 300_000):
        cur = fn(n)
        assert cur >= prev and cur >= n * 4 and cur == lib.spx_sparse_add_group_workspace_size(n)
        prev = cur


def test_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def grp(ids=P, ib=8, n=10, rows=4, r32=P, order=P, off=P, ws=P, wsb=1 << 40):",
        "    return lib.spx_point_scatter_group(ids, ib, n, rows, r32, order, off, ws, wsb, None)",
        "def fwd(mode=0, x=P, n=10, c=16, dt=1, order=P, off=P, rows=4, out=P, am=P):",
        "    return lib.spx_point_scatter_fwd(mode, x, n, c, dt, order, off, rows, out, am, None)",
        "def bwd(mode=0, dy=P, r32=P, n=10, rows=4, c=16, dt=1, am=P, cnt=P, dx=P):",
        "    return lib.spx_point_scatter_bwd(mode, dy, r32, n, rows, c, dt, am, cnt, dx, None)",
        "def expect(rc, text):",
        "    assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "expect(grp(ib=2), 'int32 or int64')",
        "expect(grp(n=-1), 'bad point count')",
        "expect(grp(n=(1 << 31) - 1), 'bad point count')",
        "expect(grp(rows=-1), 'bad row count')",
        "expect(grp(rows=1 << 31), 'bad row count')",
        "for k in ('ids', 'r32', 'order', 'off', 'ws'):",
        "    expect(grp(**{k: None}), 'NULL pointer')",
        "expect(grp(wsb=64), 'workspace too small')",
        "for f in (fwd, bwd):",
        "    expect(f(mode=3), 'mode must be')",
        "    expect(f(mode=-1), 'mode must be')",
        "    expect(f(n=-1), 'bad point count')",
        "    expect(f(n=1 << 31), 'bad point count')",
        "    expect(f(rows=-1), 'bad row count')",
        "    expect(f(rows=(1 << 31) - 1), 'bad row count')",
        "    expect(f(c=0), 'channels must be')",
        "    expect(f(dt=3), 'unsupported dtype')",
        "    expect(f(dt=7), 'unsupported dtype')",
        "    expect(f(n=1 << 30, c=1 << 12), 'too many')",
        "    expect(f(am=None), 'NULL pointer')",
        "for k in ('x', 'order', 'off', 'out'):",
        "    expect(fwd(**{k: None}), 'NULL pointer')",
        "for k in ('dy', 'r32', 'dx'):",
        "    expect(bwd(**{k: None}), 'NULL pointer')",
        "expect(bwd(mode=1, cnt=None), 'NULL pointer')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def test_refuses_cpu_tensors_and_other_dtypes():
    ids = torch.tensor([0, 1, -1, 1])
    with pytest.raises(RuntimeError, match="pc_voxel_id must be a CUDA tensor"):
        PointVoxelScatter(ids, 2)
    with pytest.raises(RuntimeError, match="pc_voxel_id must be a CUDA tensor"):
        PointVoxelScatter(ids.int(), 2)
    with pytest.raises(ValueError, match="num_rows"):
        PointVoxelScatter(ids, -1)
    order, offsets = torch.zeros(4, dtype=torch.int32), torch.zeros(3, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        ops.point_scatter_fwd(torch.zeros(4, 8), order, offsets, "max")
    for dt in (torch.int8, torch.float64, torch.int32):
        with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
            ops.point_scatter_fwd(torch.zeros(4, 8, dtype=dt), order, offsets, "mean")
        with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
            ops.point_scatter_bwd(torch.zeros(2, 8, dtype=dt), order, None, "sum")


def test_exported_and_documented():
    assert spconv.PointVoxelScatter is PointVoxelScatter
    for name in ("max", "mean", "sum"):
        assert callable(getattr(PointVoxelScatter, name))
    doc = PointVoxelScatter.__doc__
    assert "MaskedPointToVoxel" in doc and "num_valid" in doc and ".max(" in doc
    assert "PointVoxelScatter" in spconv.MaskedPointToVoxel.__doc__
