"""Grouped sparse convolution (1 < groups < channels), the parts that need no GPU: the float64 reference against torch's
grouped dense convs, module construction and the widened groups rule, the int8 / fp8 refusals, the layout of the C
argument block and the argument checks of the C entry points before any launch."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch.fp8 import fp8_refusal
from spconv_b200.pytorch.quantized import QuantizedSparseConv
from tests.conv_ref import SparseConvRef
from tests.grouped_ref import grouped_backward, grouped_forward

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TORCH_CONV = {1: torch.nn.functional.conv1d, 2: torch.nn.functional.conv2d, 3: torch.nn.functional.conv3d}


def _full_grid(shape):
    coords = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"), -1).reshape(-1, len(shape))
    return np.concatenate([np.zeros((len(coords), 1), np.int64), coords], 1)


@pytest.mark.parametrize("nd, kind", [(1, "subm"), (2, "subm"), (3, "subm"), (2, "conv"), (3, "conv")])
def test_reference_is_torch_grouped_conv_on_a_dense_grid(nd, kind):
    """on a fully occupied grid the grouped reference is torch.nn.functional.conv{1,2,3}d(groups=g), forward and
    both gradients"""
    shape = {1: [11], 2: [6, 7], 3: [4, 5, 3]}[nd]
    C, K, g, k = 8, 12, 4, 3
    rng = np.random.default_rng(nd)
    inds = _full_grid(shape)
    stride, pad = ([1] * nd, [1] * nd) if kind == "subm" else ([2] * nd, [1] * nd)
    ref = SparseConvRef(inds, 1, shape, [k] * nd, stride, pad, [1] * nd, kind=kind)
    x = rng.standard_normal((len(inds), C))
    w = rng.standard_normal((K, *([k] * nd), C // g))
    b = rng.standard_normal(K)
    out, mag = grouped_forward(ref, x, w, g, b)
    assert np.all(mag >= np.abs(out) - 1e-12)
    xt = torch.from_numpy(x.T.reshape(1, C, *shape)).requires_grad_(True)
    wt = torch.from_numpy(np.moveaxis(w, -1, 1).copy()).requires_grad_(True)       # KRSC -> [K, C/g, *ksize]
    yt = TORCH_CONV[nd](xt, wt, torch.from_numpy(b), stride=stride, padding=pad, groups=g)
    oc = np.asarray(ref.out_inds)[:, 1:]
    got = yt.detach().numpy()[0][(slice(None), *oc.T)].T
    np.testing.assert_allclose(out, got, rtol=1e-12, atol=1e-12)
    dy = rng.standard_normal(out.shape)
    dyt = np.zeros(yt.shape)
    dyt[0][(slice(None), *oc.T)] = dy.T
    yt.backward(torch.from_numpy(dyt))
    dx, dxm, dw, dwm = grouped_backward(ref, x, w, dy, g)
    np.testing.assert_allclose(dx, xt.grad.numpy().reshape(C, -1).T, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dw, np.moveaxis(wt.grad.numpy(), 1, -1), rtol=1e-12, atol=1e-12)
    assert np.all(dxm >= np.abs(dx) - 1e-12) and np.all(dwm >= np.abs(dw) - 1e-12)


@pytest.mark.parametrize("nd", [1, 2, 3, 4])
@pytest.mark.parametrize("cls", ["SubMConv", "SparseConv", "SparseConvTranspose"])
@pytest.mark.parametrize("C, K, g", [(64, 64, 2), (64, 32, 2), (96, 96, 2), (128, 128, 4), (512, 512, 4)])
def test_module_construction(nd, cls, C, K, g):
    """weight [K, *ksize, C / g], Kaiming fan-in (C / g) * kv, groups in the repr, state-dict round trip"""
    m = getattr(spconv, f"{cls}{nd}d")(C, K, 3, groups=g)
    assert m.groups == g and not m.depthwise
    assert tuple(m.weight.shape) == (K, *([3] * nd), C // g)
    fan_in = C // g * 3 ** nd
    assert float(m.weight.detach().abs().max()) <= math.sqrt(6.0 / ((1 + 5.0) * fan_in)) + 1e-7
    assert float(m.bias.detach().abs().max()) <= 1 / math.sqrt(fan_in) + 1e-7
    assert f"groups={g}" in m.extra_repr()
    fresh = getattr(spconv, f"{cls}{nd}d")(C, K, 3, groups=g)
    fresh.load_state_dict(m.state_dict())
    assert torch.equal(fresh.weight, m.weight) and torch.equal(fresh.bias, m.bias)


def test_inverse_and_depthwise_kinds():
    inv = spconv.SparseInverseConv3d(64, 32, 3, indice_key="d", groups=2)
    assert inv.inverse and tuple(inv.weight.shape) == (32, 3, 3, 3, 32) and not inv.depthwise
    assert spconv.SubMConv3d(32, 32, 3, groups=32).depthwise        # groups == C == K stays depthwise


@pytest.mark.parametrize("C, K, g", [(32, 32, 4), (48, 48, 2), (24, 24, 3), (64, 32, 3), (32, 64, 64), (32, 32, -2),
                                     (16, 32, 2), (33, 33, 3), (64, 64, 0)])
def test_narrow_or_uneven_groups_raise(C, K, g):
    """group widths below 16 or not multiples of 16, groups not dividing both widths, channel multipliers and
    groups <= 0 raise, as before"""
    for ctor in (lambda: spconv.SubMConv3d(C, K, 3, groups=g), lambda: spconv.SparseConv3d(C, K, 3, 2, groups=g)):
        with pytest.raises(AssertionError, match="groups"):
            ctor()


def test_int8_and_fp8_refuse_grouped_layers():
    m = spconv.SubMConv3d(64, 64, 3, groups=2).eval()
    with pytest.raises(NotImplementedError, match="grouped"):
        QuantizedSparseConv.from_float(m, 0.1)
    assert "grouped" in fp8_refusal(m)
    assert fp8_refusal(spconv.SubMConv3d(64, 64, 3)) is None


def test_argument_block_layout_matches_the_header(tmp_path):
    """spx_grouped_gemm has the same size and field offsets in ctypes as in C"""
    from spconv_b200 import _cabi
    cls = _cabi.GroupedGemm
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "spconv_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(spx_grouped_gemm));']
    lines += [f'  printf("{f} %zu\\n", offsetof(spx_grouped_gemm, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                   check=True).stdout.split("\n") if ln.strip())
    assert int(out.pop("size")) == ctypes.sizeof(cls)
    assert {f: int(v) for f, v in out.items()} == {f: getattr(cls, f).offset for f, _ in cls._fields_}


_SCRIPT = r"""
import ctypes, sys
sys.path.insert(0, ROOT)
from spconv_b200 import _cabi
lib = _cabi.load()
lib.spx_launch_count(1)
P = 1 << 20          # a 16-byte aligned stand-in address: no call below may get as far as touching it

def desc(c_in=64, c_out=64, kv=27, dtype=_cabi.SPX_F16, tiles=True):
    d = _cabi.GemmDesc()
    d.dtype, d.f32_mode, d.kv, d.c_in, d.c_out, d.n_in, d.n_out = dtype, _cabi.SPX_F32_EXACT, kv, c_in, c_out, 100, 90
    d.pair, d.pair_stride = P, 100
    if tiles:
        d.tile_table, d.tile_mask = P, P
    return d

def fwd(d, g, **kw):
    a = _cabi.GroupedGemm(features=kw.get("features", P), filters=kw.get("filters", P), out=kw.get("out", P),
                          bias=kw.get("bias"), act=kw.get("act", 0))
    return lib.spx_grouped_gemm_fwd(ctypes.byref(d), g, ctypes.byref(a), None)

def dgrad(d, g, **kw):
    a = _cabi.GroupedGemm(out_bp=kw.get("out_bp", P), filters=kw.get("filters", P), din=kw.get("din", P))
    return lib.spx_grouped_gemm_dgrad(ctypes.byref(d), g, ctypes.byref(a), None)

def wgrad(d, g, **kw):
    a = _cabi.GroupedGemm(features=kw.get("features", P), out_bp=kw.get("out_bp", P), dfilters=kw.get("dfilters", P),
                          workspace=P, workspace_bytes=1 << 30)
    return lib.spx_grouped_gemm_wgrad(ctypes.byref(d), g, ctypes.byref(a), None)

def expect(rc, want, words):
    msg = lib.spx_last_error().decode()
    assert rc == want, (rc, want, msg)
    for w in words:
        assert w in msg, (w, msg)

for call in (fwd, dgrad, wgrad):
    for g in (0, -1, 1):
        expect(call(desc(), g), 2, ["groups"])
    expect(call(desc(), 3), 2, ["divide"])
    expect(call(desc(64, 64), 8), 2, ["multiples of 16"])
    expect(call(desc(96, 64), 4), 2, ["multiples of 16"])
    expect(call(desc(dtype=_cabi.SPX_I8), 2), 2, ["dtype"])
    expect(call(desc(kv=129), 2), 2, ["kernel volume"])
    # an odd address is not aligned to a 16-bit element; the FMA kernels cannot take it either
    expect(call(desc(), 2, **{{fwd: "features", dgrad: "out_bp", wgrad: "features"}[call]: P + 1}), 2, ["aligned"])
expect(fwd(desc(), 2, features=None), 2, ["NULL"])
expect(dgrad(desc(), 2, din=None), 2, ["NULL"])
expect(wgrad(desc(), 2, dfilters=None), 2, ["NULL"])
expect(fwd(desc(), 2, act=99), 2, ["activation"])
assert lib.spx_grouped_gemm_wgrad_push(ctypes.byref(desc()), 2, ctypes.byref(_cabi.GroupedGemm()), None, None) == 2
assert lib.spx_grouped_gemm_wgrad_workspace_size(ctypes.byref(desc()), 1) == 0
# SPX_FORCE_TC=1: what would run on the FMA kernels is refused, before any launch -- 8-byte (not 16-byte) aligned
# operands, fp32, 48-channel groups and calls without tile tables
for call in (fwd, dgrad, wgrad):
    key = {fwd: "features", dgrad: "out_bp", wgrad: "features"}[call]
    expect(call(desc(), 2, **{key: P + 8}), 3, ["SPX_FORCE_TC"])
    expect(call(desc(dtype=_cabi.SPX_F32), 2), 3, ["SPX_FORCE_TC"])
    expect(call(desc(96, 96), 2), 3, ["SPX_FORCE_TC"])
    expect(call(desc(tiles=False), 2), 3, ["SPX_FORCE_TC"])
expect(fwd(desc(512, 512), 2), 3, ["SPX_FORCE_TC"])       # 256-channel 16-bit groups: forward on the FMA kernels
print(lib.spx_launch_count(1))
"""


def test_entry_points_check_every_argument_before_any_launch():
    """in a fresh process with no visible device: the launch counter is process-wide, and a call that slipped past
    its checks fails on the missing device instead of launching"""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", SPX_FORCE_TC="1")
    env.pop("SPX_FORCE_SIMT", None)
    res = subprocess.run([sys.executable, "-c", f"ROOT = {ROOT!r}\n" + _SCRIPT], capture_output=True, text=True,
                         env=env)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout
