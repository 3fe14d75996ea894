"""MaskedGlobalMaxPool / MaskedGlobalAvgPool, the parts that need no GPU: argument validation of the C entry points
before any launch, the workspace size, and the modules' refusal of CPU and int8 tensors."""
import os
import subprocess
import sys

import pytest
import torch

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedGlobalAvgPool, MaskedGlobalMaxPool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def test_workspace_size(lib):
    fn = lib.spx_global_pool_workspace_size
    assert fn(-1, 2, 16) == 0 and fn(10, 0, 16) == 0 and fn(10, 2, 0) == 0
    assert fn(0, 4, 16) >= 4 * 16 * 8                      # one partial per (sample, channel) at least
    prev = 0
    for rows in (1, 512, 513, 100_000):
        cur = fn(rows, 8, 64)
        assert cur >= prev and cur >= ((rows + 511) // 512 + 8) * 64 * 8 + 2 * rows * 4
        prev = cur


def test_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def fwd(mode=0, x=P, co=P, rows=10, ri=4, b=2, c=16, dt=1, nv=None, out=P, am=P, cnt=P, ws=P, wsb=1 << 40):",
        "    return lib.spx_global_pool_fwd(mode, x, co, rows, ri, b, c, dt, nv, out, am, cnt, ws, wsb, None)",
        "def bwd(mode=0, dy=P, co=P, rows=10, ri=4, b=2, c=16, dt=1, nv=None, am=P, cnt=P, din=P):",
        "    return lib.spx_global_pool_bwd(mode, dy, co, rows, ri, b, c, dt, nv, am, cnt, din, None)",
        "def expect(rc, text):",
        "    assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "for f in (fwd, bwd):",
        "    expect(f(mode=2), 'mode must be')",
        "    expect(f(mode=-1), 'mode must be')",
        "    expect(f(rows=-1), 'bad row count')",
        "    expect(f(rows=1 << 31), 'bad row count')",
        "    expect(f(ri=0), 'batch index')",
        "    expect(f(b=0), 'batch_size must be')",
        "    expect(f(b=(1 << 20) + 1), 'batch_size must be')",
        "    expect(f(c=0), 'channels must be')",
        "    expect(f(c=65537), 'channels must be')",
        "    expect(f(dt=3), 'unsupported dtype')",
        "    expect(f(dt=7), 'unsupported dtype')",
        "    expect(f(co=None), 'NULL pointer')",
        "    expect(f(am=None), 'NULL pointer')",
        "    expect(f(mode=1, cnt=None), 'NULL pointer')",
        "expect(fwd(x=None), 'NULL pointer')",
        "expect(fwd(out=None), 'NULL pointer')",
        "expect(fwd(ws=None), 'NULL pointer')",
        "expect(fwd(wsb=64), 'workspace too small')",
        "expect(bwd(dy=None), 'NULL pointer')",
        "expect(bwd(din=None), 'NULL pointer')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def _tensor(dtype=torch.float32):
    inds = torch.tensor([[0, 1, 1, 1], [1, 2, 2, 2], [0, 3, 3, 3]], dtype=torch.int32)
    feats = torch.arange(3 * 8, dtype=torch.float32).view(3, 8).to(dtype)
    return spconv.SparseConvTensor(feats, inds, [4, 4, 4], 2)


@pytest.mark.parametrize("cls", [MaskedGlobalMaxPool, MaskedGlobalAvgPool])
def test_modules_refuse_cpu_and_int8_tensors(cls):
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        cls()(_tensor())
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        cls()(_tensor().pad_to(5))
    for dt in (torch.int8, torch.float64):
        with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
            cls()(_tensor(dt))
    q = torch.quantize_per_tensor(torch.zeros(3, 8), 0.1, 0, torch.qint8)
    with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
        cls()(_tensor().replace_feature(q))


def test_modules_are_exported_and_leave_the_default_pools_alone():
    assert spconv.MaskedGlobalMaxPool is MaskedGlobalMaxPool and spconv.MaskedGlobalAvgPool is MaskedGlobalAvgPool
    assert not MaskedGlobalMaxPool().is_mean and MaskedGlobalAvgPool().is_mean
    assert MaskedGlobalMaxPool(name="gp").name == "gp"
    p = _tensor().pad_to(5)
    for mod in (spconv.SparseGlobalMaxPool(), spconv.SparseGlobalAvgPool()):
        with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
            mod(p)
