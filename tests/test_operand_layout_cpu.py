"""Operand layout, the parts that need no GPU: the C entry points refuse, or keep off the tensor cores, a caller
pointer that is not 16-byte aligned, before any launch; and the Python helper that realigns operands returns
an aligned tensor unchanged and copies any other."""
import os
import subprocess
import sys

import pytest
import torch

from spconv_b200.pytorch import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Runs with no visible device and SPX_FORCE_TC=1.  P is a fake 16-byte aligned address (never dereferenced: a call
# that got past its checks fails on the missing device, it cannot launch); P + 2 / 4 / 8 / 12 are the misaligned
# variants.  Each conv entry point gets a tensor-core-shaped descriptor, so misalignment is the only reason the
# tensor-core kernels cannot take the call: the aligned control must fail some other way (no device).
_SCRIPT = r"""
import ctypes, sys
sys.path.insert(0, ROOT)
from spconv_b200 import _cabi
lib = _cabi.load()
P = 1 << 20
FORCE = "SPX_FORCE_TC=1 but the tensor-core"

def desc(dtype, c):
    d = _cabi.GemmDesc()
    d.dtype, d.f32_mode, d.kv, d.c_in, d.c_out = dtype, _cabi.SPX_F32_TF32, 27, c, c
    d.n_in = d.n_out = 1000
    d.pair, d.pair_stride, d.mask, d.argsort = P, 1000, P, P
    d.tile_table, d.tile_mask = P, P
    return d

def sweep(name, call, want, expect_rc):
    # call(ptrs): each pointer moved off 16 bytes alone gives (expect_rc, want[j]); all aligned, neither refusal
    n = len(want)
    for j in range(n + 1):
        for off in ((0,) if j == n else (2, 4, 8, 12)):
            rc = call([P + 16 * (i + 1) + (off if i == j else 0) for i in range(n)])
            msg = _cabi.last_error()
            if j == n:
                assert rc != 0 and FORCE not in msg and "16-byte aligned" not in msg, (name, "aligned", rc, msg)
            else:
                assert rc == expect_rc and want[j] in msg, (name, j, off, rc, msg)

for dt in (_cabi.SPX_F16, _cabi.SPX_BF16, _cabi.SPX_F32):
    d = desc(dt, 64)
    sweep("fwd", lambda p: lib.spx_implicit_gemm_fwd(ctypes.byref(d), p[0], p[1], p[2], None, 0, 0.0, None),
          [FORCE] * 3, 3)
    sweep("dgrad", lambda p: lib.spx_implicit_gemm_dgrad(ctypes.byref(d), p[0], p[1], p[2], None), [FORCE] * 3, 3)
    dw = desc(dt, 32)            # tf32 weight gradient: c_out <= 64
    sweep("wgrad", lambda p: lib.spx_implicit_gemm_wgrad(ctypes.byref(dw), p[0], p[1], P, P, 1 << 30, None),
          [FORCE] * 2, 3)
d8 = desc(_cabi.SPX_I8, 64)
sweep("int8", lambda p: lib.spx_implicit_gemm_fwd_int8(ctypes.byref(d8), p[0], p[1], p[2], _cabi.SPX_I8, P, None,
                                                        None, 0.0, 0, 0.0, None), [FORCE] * 3, 3)

def named(who, names):
    return [f"{who}: {n} must be 16-byte aligned" for n in names]

sweep("pool_fwd", lambda p: lib.spx_indice_pool_fwd(0, p[0], p[1], P, 100, 27, 100, 64, _cabi.SPX_F16, None, None),
      named("indice_pool_fwd", ["features", "out"]), 2)
for mode in (0, 1):
    sweep("pool_bwd", lambda p: lib.spx_indice_pool_bwd(mode, p[0], p[1], p[2], p[3], P, 100, 27, 100, 64,
                                                        _cabi.SPX_F16, None, None),
          named("indice_pool_bwd", ["features", "out_features", "out_bp", "din"]), 2)
sweep("pool_bwd_avg", lambda p: lib.spx_indice_pool_bwd(2, None, None, p[0], p[1], P, 100, 27, 100, 64,
                                                        _cabi.SPX_F32, P, None),
      named("indice_pool_bwd", ["out_bp", "din"]), 2)

BIG = 1 << 40
for ndim in (1, 2, 3, 4):
    dims = [16] * ndim
    subm = _cabi.make_geometry(ndim, 2, dims, dims, [3] * ndim, [1] * ndim, [1] * ndim, [1] * ndim)
    conv = _cabi.make_geometry(ndim, 2, dims, [8] * ndim, [3] * ndim, [2] * ndim, [1] * ndim, [1] * ndim)
    sweep("subm", lambda p: lib.spx_subm_rulebook(ctypes.byref(subm), p[0], 50, P, P, P, P, BIG, None),
          named("subm_rulebook", ["indices"]), 2)
    sweep("subm_all", lambda p: lib.spx_subm_rulebook_all(ctypes.byref(subm), p[0], 50, P, P, P, P, 1, P, P, P,
                                                          BIG, None), named("subm_rulebook", ["indices"]), 2)
    m = ctypes.c_int64(0)
    sweep("stage1", lambda p: lib.spx_conv_rulebook_stage1(ctypes.byref(conv), p[0], 50, ctypes.byref(m), P, BIG,
                                                           None), named("conv_rulebook_stage1", ["indices"]), 2)
    sweep("stage2", lambda p: lib.spx_conv_rulebook_stage2(ctypes.byref(conv), p[0], 50, 40, P, P, P, P, P, P, BIG,
                                                           None), named("conv_rulebook_stage2", ["indices"]), 2)
    sweep("bounded", lambda p: lib.spx_conv_rulebook_bounded_all(ctypes.byref(conv), p[0], 50, 128, P, P, P, P, P, P,
                                                                 P, 1, P, P, P, P, P, P, P, BIG, None),
          named("conv_rulebook_bounded_all", ["indices"]), 2)
    one = _cabi.make_geometry(ndim, 2, dims, dims, [1] * ndim, [1] * ndim, [0] * ndim, [1] * ndim)
    sweep("union", lambda p: lib.spx_sparse_add_union(ctypes.byref(one), p[0], 50, 50, P, P, P, P, P, BIG, None),
          named("sparse_add_union", ["indices"]), 2)
print(lib.spx_launch_count(1))
"""


def test_misaligned_pointers_are_refused_before_any_launch():
    """in a fresh process with no visible device: the launch counter is process-wide, and a call that slipped past
    its checks fails on the missing device instead of launching"""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", SPX_FORCE_TC="1")
    env.pop("SPX_FORCE_SIMT", None)
    res = subprocess.run([sys.executable, "-c", f"ROOT = {ROOT!r}\n" + _SCRIPT], capture_output=True, text=True,
                         env=env)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def _at(t, nbytes):
    """a contiguous copy of ``t`` starting ``nbytes`` past a 64-byte boundary"""
    raw = torch.empty(t.numel() * t.element_size() + 128, dtype=torch.uint8)
    skip = (-raw.data_ptr()) % 64 + nbytes
    out = raw[skip:skip + t.numel() * t.element_size()].view(t.dtype).view(t.shape)
    out.copy_(t)
    assert out.is_contiguous() and out.data_ptr() % 64 == nbytes
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.int8, torch.int32])
def test_dense_returns_aligned_tensors_unchanged_and_copies_the_rest(dtype):
    base = (torch.arange(48 * 16) % 97 - 40).to(dtype).view(48, 16)
    for nbytes in (0, 16, 48):
        t = _at(base, nbytes)
        assert ops._dense(t) is t
    e = base.element_size()
    for nbytes in range(e, 16, e):
        t = _at(base, nbytes)
        d = ops._dense(t)
        assert d is not t and d.data_ptr() % 16 == 0 and d.is_contiguous() and torch.equal(d, base)
    wide = torch.cat([base, base], 1)
    for view in (wide[:, 3:19], base.t().contiguous().t(), base[:1].expand(48, 16)):
        d = ops._dense(view)
        assert d.is_contiguous() and d.data_ptr() % 16 == 0 and torch.equal(d, view)
