"""MaskedGroupNorm, the parts that need no GPU: the C descriptor's layout, workspace sizes, argument validation of
the C entry points and of the Python wrappers before any launch, state_dict compatibility with nn.GroupNorm,
from_groupnorm, the export, and the refusal of CPU tensors."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch
from torch import nn

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedGroupNorm, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def test_descriptor_layout_matches_the_header(tmp_path):
    """spx_masked_group_norm has the same size and field offsets in ctypes as in C"""
    from spconv_b200 import _cabi
    cls = _cabi.MaskedGroupNorm
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "spconv_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(spx_masked_group_norm));']
    lines += [f'  printf("{f} %zu\\n", offsetof(spx_masked_group_norm, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                   check=True).stdout.split("\n") if ln.strip())
    assert int(out.pop("size")) == ctypes.sizeof(cls)
    assert {f: int(v) for f, v in out.items()} == {f: getattr(cls, f).offset for f, _ in cls._fields_}


def test_every_pointer_of_the_descriptor_is_covered():
    """every pointer field is misaligned by test_masked_group_norm_gpu.py::test_misaligned_operands_give_the_same_bits
    or explained here"""
    from spconv_b200 import _cabi
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "spconv_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct spx_masked_group_norm \{(.*?)\} spx_masked_group_norm;", text, re.S).group(1)
    ptrs = set()
    for decl in body.split(";"):
        if "*" in decl:
            ptrs |= {p.strip().lstrip("*").strip() for p in decl.split("*", 1)[1].split(",")}
    assert ptrs == {f for f, t in _cabi.MaskedGroupNorm._fields_ if t is ctypes.c_void_p}
    swept = {"x", "y", "dy", "dx"}
    explained = {
        "coords": "one int32 per row read with __ldg", "num_valid": "one int32 read with __ldg",
        "weight": "a per-channel vector read element by element", "bias": "a per-channel vector read element by element",
        "dweight": "written element by element", "dbias": "written element by element",
        "mean": "fp32 statistics read and written element by element",
        "invstd": "fp32 statistics read and written element by element",
        "order": "int32 read and written element by element", "offsets": "int32 read and written element by element",
        "cstart": "int32 read and written element by element",
    }
    assert ptrs == swept | set(explained)


def test_workspace_sizes(lib):
    fn = lib.spx_masked_group_norm_workspace_size
    assert fn(-1, 1, 16) == 0 and fn(10, 0, 16) == 0 and fn(10, 1, 0) == 0
    assert fn(0, 1, 16) > 0                                # the per-sample statistics
    prev = 0
    for rows in (1, 512, 513, 100_000):
        cur = fn(rows, 4, 64)
        # keys, the chunk partials (one chunk more per sample at most) and two [B, C] float2 tables
        assert cur >= prev and cur >= rows * 4 + ((rows + 511) // 512 + 4) * 64 * 8 + 2 * 4 * 64 * 8
        prev = cur
    assert fn(1000, 8, 64) > fn(1000, 1, 64)


def test_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def call(fwd=True, ws=P, wsb=1 << 30, desc=True, **kw):",
        "    d = _cabi.MaskedGroupNorm()",
        "    d.rows, d.row_ints, d.batch_size, d.channels, d.groups, d.dtype, d.param_dtype, d.eps = \\",
        "        10, 4, 2, 16, 4, 1, 0, 1e-5",
        "    for f in ('coords', 'x', 'y', 'dy', 'dx', 'weight', 'bias', 'dweight', 'dbias', 'mean', 'invstd',",
        "              'order', 'offsets', 'cstart'):",
        "        setattr(d, f, P)",
        "    for k, v in kw.items():",
        "        setattr(d, k, v)",
        "    fn = lib.spx_masked_group_norm_fwd if fwd else lib.spx_masked_group_norm_bwd",
        "    return fn(ctypes.byref(d) if desc else None, ws, wsb, None)",
        "def expect(rc, text):",
        "    assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "for fwd in (True, False):",
        "    expect(call(fwd, desc=False), 'descriptor is NULL')",
        "    expect(call(fwd, rows=-1), 'bad row count')",
        "    expect(call(fwd, row_ints=0), 'batch index')",
        "    expect(call(fwd, batch_size=0), 'batch_size must be')",
        "    expect(call(fwd, batch_size=(1 << 20) + 1), 'batch_size must be')",
        "    expect(call(fwd, channels=0), 'channels must be')",
        "    expect(call(fwd, channels=65537, groups=1), 'channels must be')",
        "    expect(call(fwd, groups=3), 'must divide')",
        "    expect(call(fwd, groups=0), 'must divide')",
        "    expect(call(fwd, dtype=3), 'unsupported dtype')",
        "    expect(call(fwd, param_dtype=2), 'parameter dtype')",
        "    expect(call(fwd, dtype=0, param_dtype=1), 'parameter dtype')",
        "    for f in ('mean', 'invstd', 'offsets', 'cstart', 'x', 'coords', 'order'):",
        "        expect(call(fwd, **{f: None}), 'NULL pointer')",
        "    expect(call(fwd, ws=None), 'NULL pointer')",
        "    expect(call(fwd, wsb=64), 'workspace too small')",
        "expect(call(True, y=None), 'NULL pointer')",
        "expect(call(True, eps=0.0), 'eps must be positive')",
        "expect(call(False, dy=None), 'NULL pointer')",
        "expect(call(False, dx=None), 'NULL pointer')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def _gn(g=4, c=8, affine=True):
    torch.manual_seed(0)
    gn = nn.GroupNorm(g, c, eps=1e-4, affine=affine)
    if affine:
        with torch.no_grad():
            gn.weight.uniform_(0.5, 1.5)
            gn.bias.uniform_(-1, 1)
    return gn


def test_state_dict_loads_both_ways():
    plain = _gn()
    m = MaskedGroupNorm(4, 8, eps=1e-4)
    assert list(m.state_dict()) == list(plain.state_dict()) == ["weight", "bias"]
    assert [n for n, _ in m.named_parameters()] == [n for n, _ in plain.named_parameters()]
    assert not list(m.named_buffers())
    m.load_state_dict(plain.state_dict())
    for k, v in plain.state_dict().items():
        assert torch.equal(m.state_dict()[k], v), k
    with torch.no_grad():
        m.weight.fill_(0.25)
    back = nn.GroupNorm(4, 8)
    back.load_state_dict(m.state_dict())
    assert torch.equal(back.weight, m.weight) and torch.equal(back.bias, m.bias)
    assert list(MaskedGroupNorm(2, 6, affine=False).state_dict()) == list(nn.GroupNorm(2, 6, affine=False).state_dict())
    # nested in a sparse container: the same keys as the plain module there
    seq_p = spconv.SparseSequential(spconv.SubMConv3d(4, 8, 3, indice_key="a"), _gn())
    seq_m = spconv.SparseSequential(spconv.SubMConv3d(4, 8, 3, indice_key="a"), MaskedGroupNorm(4, 8))
    seq_m.load_state_dict(seq_p.state_dict())
    assert list(seq_m.state_dict()) == list(seq_p.state_dict())


def test_from_groupnorm_shares_the_parameters():
    gn = _gn(2, 6).eval()
    m = MaskedGroupNorm.from_groupnorm(gn)
    assert type(m) is MaskedGroupNorm and isinstance(m, nn.GroupNorm) and isinstance(m, spconv.SparseModule)
    assert m.weight is gn.weight and m.bias is gn.bias
    assert (m.num_groups, m.num_channels, m.eps, m.affine) == (2, 6, 1e-4, True)
    assert not m.training
    plain = nn.GroupNorm(3, 6, affine=False)
    m2 = MaskedGroupNorm.from_groupnorm(plain)
    assert m2.weight is None and m2.bias is None and m2.training
    with pytest.raises(ValueError):
        MaskedGroupNorm(4, 6)                              # nn.GroupNorm's own check: G must divide C


def test_exported():
    import spconv_b200.pytorch.modules as modules
    assert spconv.MaskedGroupNorm is modules.MaskedGroupNorm
    assert callable(spconv.functional.masked_group_norm)
    assert callable(ops.masked_group_norm_forward) and callable(ops.masked_group_norm_backward)


def _sparse(rows=6, c=8, b=2):
    feats = torch.randn(rows, c)
    inds = torch.zeros((rows, 4), dtype=torch.int32)
    inds[:, 0] = torch.arange(rows, dtype=torch.int32) % b
    return spconv.SparseConvTensor(feats, inds, [4, 4, 4], b)


def test_cpu_tensors_raise_the_no_cpu_path_error():
    x = _sparse()
    with pytest.raises(RuntimeError, match="no CPU path"):
        MaskedGroupNorm(4, 8)(x)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.masked_group_norm_forward(x.features, x.indices, 2, None, 4, None, None, 1e-5)
    with pytest.raises(ValueError, match="features of shape"):
        MaskedGroupNorm(2, 4)(x)


def test_wrapper_checks_come_before_the_device(monkeypatch):
    """the Python checks that need no device (shape, dtype, limits) name the problem"""
    monkeypatch.setattr(ops, "_require_cuda", lambda t, what: None)
    x = _sparse()
    f, i = x.features, x.indices
    with pytest.raises(RuntimeError, match="must divide"):
        ops.masked_group_norm_forward(f, i, 2, None, 3, None, None, 1e-5)
    with pytest.raises(RuntimeError, match="batch_size must be"):
        ops.masked_group_norm_forward(f, i, 0, None, 4, None, None, 1e-5)
    with pytest.raises(RuntimeError, match="batch_size must be"):
        ops.masked_group_norm_forward(f, i, (1 << 20) + 1, None, 4, None, None, 1e-5)
    with pytest.raises(RuntimeError, match="channels must be"):
        ops.masked_group_norm_forward(torch.zeros((2, 65537)), i[:2], 1, None, 1, None, None, 1e-5)
    with pytest.raises(RuntimeError, match="float32 / float16 / bfloat16"):
        ops.masked_group_norm_forward(f.double(), i, 2, None, 4, None, None, 1e-5)
    with pytest.raises(RuntimeError, match="int32 indices"):
        ops.masked_group_norm_forward(f, i.long(), 2, None, 4, None, None, 1e-5)
    with pytest.raises(RuntimeError, match="num_valid"):
        ops.masked_group_norm_forward(f, i, 2, torch.zeros((1,), dtype=torch.int64), 4, None, None, 1e-5)
    with pytest.raises(RuntimeError, match="parameter dtype"):
        ops.masked_group_norm_forward(f, i, 2, None, 4, torch.ones(8, dtype=torch.float16), None, 1e-5)
    with pytest.raises(RuntimeError, match="eps must be positive"):
        ops.masked_group_norm_forward(f, i, 2, None, 4, None, None, 0.0)
