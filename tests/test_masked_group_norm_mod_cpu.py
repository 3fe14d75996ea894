"""MaskedGroupNorm with per-sample scale / shift and an activation, the parts that need no GPU: the modulated
descriptor's layout, that every new pointer of it is set from the Python call, argument checks of the C entry
points and of the Python wrappers before any launch, the module's state_dict, from_groupnorm and repr, and the
refusal of CPU tensors."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch
from torch import nn

import spconv_b200.pytorch as spconv
from spconv_b200 import _cabi
from spconv_b200.pytorch import MaskedGroupNorm, ops
from spconv_b200.pytorch.functional import masked_group_norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_descriptor_layout_matches_the_header(tmp_path):
    """spx_masked_group_norm_mod has the same size and field offsets in ctypes as in C, and the enum its values"""
    cls = _cabi.MaskedGroupNormMod
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "spconv_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(spx_masked_group_norm_mod));',
             '  printf("none %d\\n", (int)SPX_GN_ACT_NONE);', '  printf("relu %d\\n", (int)SPX_GN_ACT_RELU);',
             '  printf("silu %d\\n", (int)SPX_GN_ACT_SILU);']
    lines += [f'  printf("{f} %zu\\n", offsetof(spx_masked_group_norm_mod, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                   check=True).stdout.split("\n") if ln.strip())
    assert int(out.pop("size")) == ctypes.sizeof(cls)
    assert (int(out.pop("none")), int(out.pop("relu")), int(out.pop("silu"))) == (
        _cabi.SPX_GN_ACT_NONE, _cabi.SPX_GN_ACT_RELU, _cabi.SPX_GN_ACT_SILU)
    assert {f: int(v) for f, v in out.items()} == {f: getattr(cls, f).offset for f, _ in cls._fields_}
    assert cls._fields_[0] == ("norm", _cabi.MaskedGroupNorm) and cls.norm.offset == 0


class _FakeLib:
    """stands in for the library: records the descriptors the wrappers pass, or refuses any call"""

    def __init__(self, refuse=False):
        self.refuse = refuse
        self.calls = []

    def spx_masked_group_norm_workspace_size(self, rows, b, c):
        assert not self.refuse, "a library call before the argument checks"
        return 64

    def _record(self, name):
        def call(desc, ws, wsb, stream):
            assert not self.refuse, f"{name} called before the argument checks"
            m = desc._obj
            self.calls.append((name, {f: getattr(m, f) for f in ("scale", "shift", "act", "dscale", "dshift")},
                               {f: getattr(m.norm, f) for f, _ in _cabi.MaskedGroupNorm._fields_}))
            return 0
        return call

    def __getattr__(self, name):
        if name.startswith("spx_masked_group_norm_mod_"):
            return self._record(name)
        raise AssertionError(f"unexpected library call {name}")


@pytest.fixture
def fake(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(ops, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_lib", lambda: lib)
    return lib


def _sparse(rows=6, c=8, b=2):
    torch.manual_seed(0)
    feats = torch.randn(rows, c)
    inds = torch.zeros((rows, 4), dtype=torch.int32)
    inds[:, 0] = torch.arange(rows, dtype=torch.int32) % b
    return spconv.SparseConvTensor(feats, inds, [4, 4, 4], b)


def test_every_new_pointer_is_set_from_the_python_call(fake):
    """scale, shift (forward and backward), dscale, dshift and the bias the backward recomputes z with reach the
    descriptor; the header's pointer fields of the new struct are exactly those"""
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "spconv_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct spx_masked_group_norm_mod \{(.*?)\} spx_masked_group_norm_mod;", text,
                     re.S).group(1)
    ptrs = set()
    for decl in body.split(";"):
        if "*" in decl:
            ptrs |= {p.strip().lstrip("*").strip() for p in decl.split("*", 1)[1].split(",")}
    assert ptrs == {"scale", "shift", "dscale", "dshift"}
    x = _sparse()
    f, i = x.features, x.indices
    w, bias = torch.rand(8) + 0.5, torch.rand(8)
    scale, shift = torch.randn(2, 8), torch.randn(2, 8)
    y, mean, invstd, order, offsets, cstart = ops.masked_group_norm_forward(f, i, 2, None, 4, w, bias, 1e-5, scale,
                                                                            shift, "silu")
    name, mod, norm = fake.calls[-1]
    assert name == "spx_masked_group_norm_mod_fwd"
    assert mod["scale"] == scale.data_ptr() and mod["shift"] == shift.data_ptr()
    assert mod["act"] == _cabi.SPX_GN_ACT_SILU and mod["dscale"] is None and mod["dshift"] is None
    assert norm["y"] == y.data_ptr() and norm["bias"] == bias.data_ptr() and norm["weight"] == w.data_ptr()
    dy = torch.randn_like(f)
    dx, dw, db, ds, dt = ops.masked_group_norm_backward(f, dy, i, 2, None, 4, w, mean, invstd, order, offsets, cstart,
                                                        True, True, bias, scale, shift, "relu")
    name, mod, norm = fake.calls[-1]
    assert name == "spx_masked_group_norm_mod_bwd"
    assert mod["scale"] == scale.data_ptr() and mod["shift"] == shift.data_ptr()
    assert mod["dscale"] == ds.data_ptr() and mod["dshift"] == dt.data_ptr() and mod["act"] == _cabi.SPX_GN_ACT_RELU
    assert ds.shape == dt.shape == (2, 8) and ds.dtype == dt.dtype == torch.float32
    assert norm["bias"] == bias.data_ptr() and norm["dx"] == dx.data_ptr() and norm["dweight"] == dw.data_ptr()
    # gradients only when asked for: scale without shift, or neither
    _, _, _, ds, dt = ops.masked_group_norm_backward(f, dy, i, 2, None, 4, w, mean, invstd, order, offsets, cstart,
                                                     scale=scale)
    assert ds is not None and dt is None and fake.calls[-1][1]["dshift"] is None
    _, _, _, ds, dt = ops.masked_group_norm_backward(f, dy, i, 2, None, 4, w, mean, invstd, order, offsets, cstart,
                                                     need_shift_grad=True)
    assert ds is None and dt is not None and fake.calls[-1][1]["dshift"] == dt.data_ptr()
    assert fake.calls[-1][1]["scale"] is None and fake.calls[-1][1]["act"] == _cabi.SPX_GN_ACT_NONE
    # a float16 scale reaches the kernels as an fp32 copy
    ops.masked_group_norm_forward(f, i, 2, None, 4, w, bias, 1e-5, scale.half())
    assert fake.calls[-1][1]["scale"] not in (None, scale.data_ptr())


def test_python_checks_come_before_any_launch(monkeypatch):
    lib = _FakeLib(refuse=True)
    monkeypatch.setattr(ops, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_lib", lambda: lib)
    x = _sparse()
    f, i = x.features, x.indices
    fwd = lambda **kw: ops.masked_group_norm_forward(f, i, 2, None, 4, None, None, 1e-5, **kw)  # noqa: E731
    with pytest.raises(RuntimeError, match=r"scale must be \[batch_size, C\] = \[2, 8\]"):
        fwd(scale=torch.zeros(3, 8))
    with pytest.raises(RuntimeError, match=r"shift must be \[batch_size, C\]"):
        fwd(shift=torch.zeros(2, 4))
    with pytest.raises(RuntimeError, match=r"shift must be \[batch_size, C\]"):
        fwd(shift=torch.zeros(16))
    with pytest.raises(RuntimeError, match="features' device"):
        fwd(scale=torch.zeros(2, 8, device="meta"))
    with pytest.raises(RuntimeError, match="floating-point"):
        fwd(scale=torch.zeros(2, 8, dtype=torch.int32))
    for bad in ("gelu", "SiLU", 1, "none"):
        with pytest.raises(RuntimeError, match="act must be None, 'relu' or 'silu'"):
            fwd(act=bad)
    z = torch.zeros(2, 4)
    order, offsets = torch.zeros(6, dtype=torch.int32), torch.zeros(3, dtype=torch.int32)
    bwd = lambda **kw: ops.masked_group_norm_backward(f, f, i, 2, None, 4, None, z, z, order, offsets,  # noqa: E731
                                                      offsets, **kw)
    with pytest.raises(RuntimeError, match="act must be"):
        bwd(act="tanh")
    with pytest.raises(RuntimeError, match=r"scale must be \[batch_size, C\]"):
        bwd(scale=torch.zeros(2, 9))
    with pytest.raises(RuntimeError, match="floating-point"):
        bwd(shift=torch.zeros(2, 8, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="parameters and buffers must be"):
        bwd(bias=torch.zeros(7))
    # through autograd: an integer scale is not cast, it is refused
    with pytest.raises(RuntimeError, match="floating-point"):
        masked_group_norm(f, None, None, i, 2, None, 4, 1e-5, torch.zeros(2, 8, dtype=torch.int32))
    with pytest.raises(ValueError, match="act must be"):
        MaskedGroupNorm(4, 8, act="gelu")


def test_entry_points_validate_before_any_launch():
    """the modulated entry points refuse a NULL descriptor, an unknown act and what the plain ones refuse, with no
    launch; run in a fresh process, the launch counter is process-wide"""
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def call(fwd=True, desc=True, act=0, **kw):",
        "    m = _cabi.MaskedGroupNormMod()",
        "    d = m.norm",
        "    d.rows, d.row_ints, d.batch_size, d.channels, d.groups, d.dtype, d.param_dtype, d.eps = \\",
        "        10, 4, 2, 16, 4, 1, 0, 1e-5",
        "    for f in ('coords', 'x', 'y', 'dy', 'dx', 'weight', 'bias', 'dweight', 'dbias', 'mean', 'invstd',",
        "              'order', 'offsets', 'cstart'):",
        "        setattr(d, f, P)",
        "    for k, v in kw.items():",
        "        setattr(d, k, v)",
        "    m.scale, m.shift, m.dscale, m.dshift, m.act = P, P, P, P, act",
        "    fn = lib.spx_masked_group_norm_mod_fwd if fwd else lib.spx_masked_group_norm_mod_bwd",
        "    return fn(ctypes.byref(m) if desc else None, P, 1 << 30, None)",
        "def expect(rc, text):",
        "    assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "for fwd in (True, False):",
        "    expect(call(fwd, desc=False), 'descriptor is NULL')",
        "    for act in (-1, 3, 1 << 20):",
        "        expect(call(fwd, act=act), 'unknown activation')",
        "    expect(call(fwd, act=2, groups=3), 'must divide')",
        "    expect(call(fwd, act=1, dtype=3), 'unsupported dtype')",
        "    expect(call(fwd, act=2, mean=None), 'NULL pointer')",
        "expect(call(True, act=2, eps=0.0), 'eps must be positive')",
        "expect(call(False, act=1, dx=None), 'NULL pointer')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def test_state_dict_round_trips_with_groupnorm():
    torch.manual_seed(0)
    plain = nn.GroupNorm(4, 8, eps=1e-4)
    with torch.no_grad():
        plain.weight.uniform_(0.5, 1.5)
        plain.bias.uniform_(-1, 1)
    m = MaskedGroupNorm(4, 8, eps=1e-4, act="silu")
    assert list(m.state_dict()) == list(plain.state_dict()) == ["weight", "bias"]
    assert not list(m.named_buffers())
    m.load_state_dict(plain.state_dict())
    assert torch.equal(m.weight, plain.weight) and torch.equal(m.bias, plain.bias)
    with torch.no_grad():
        m.bias.fill_(0.5)
    back = nn.GroupNorm(4, 8)
    back.load_state_dict(m.state_dict())
    assert torch.equal(back.weight, m.weight) and torch.equal(back.bias, m.bias)
    seq_p = spconv.SparseSequential(spconv.SubMConv3d(4, 8, 3, indice_key="a"), nn.GroupNorm(4, 8))
    seq_m = spconv.SparseSequential(spconv.SubMConv3d(4, 8, 3, indice_key="a"), MaskedGroupNorm(4, 8, act="relu"))
    seq_m.load_state_dict(seq_p.state_dict())
    assert list(seq_m.state_dict()) == list(seq_p.state_dict())


def test_from_groupnorm_with_act_shares_the_parameters():
    gn = nn.GroupNorm(2, 6, eps=1e-4).eval()
    m = MaskedGroupNorm.from_groupnorm(gn, act="silu")
    assert type(m) is MaskedGroupNorm and m.act == "silu"
    assert m.weight is gn.weight and m.bias is gn.bias
    assert (m.num_groups, m.num_channels, m.eps, m.affine, m.training) == (2, 6, 1e-4, True, False)
    assert MaskedGroupNorm.from_groupnorm(gn).act is None
    assert repr(m) == "MaskedGroupNorm(2, 6, eps=0.0001, affine=True, act='silu')"
    assert repr(MaskedGroupNorm(2, 6)) == repr(nn.GroupNorm(2, 6)).replace("GroupNorm", "MaskedGroupNorm")
    # the positional arguments of nn.GroupNorm keep their places
    m2 = MaskedGroupNorm(3, 6, 1e-3, False, "cpu", torch.float64, act="relu")
    assert m2.weight is None and m2.act == "relu" and m2.eps == 1e-3


def test_cpu_tensors_raise_the_no_cpu_path_error():
    x = _sparse()
    with pytest.raises(RuntimeError, match="no CPU path"):
        MaskedGroupNorm(4, 8, act="silu")(x, torch.zeros(2, 8), torch.zeros(2, 8))
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.masked_group_norm_forward(x.features, x.indices, 2, None, 4, None, None, 1e-5, torch.zeros(2, 8),
                                      act="relu")
    with pytest.raises(RuntimeError, match="no CPU path"):
        masked_group_norm(x.features, None, None, x.indices, 2, None, 4, 1e-5, torch.zeros(2, 8).half(), None, "silu")
