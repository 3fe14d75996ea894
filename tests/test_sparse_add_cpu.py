"""sparse_add without a GPU: the numpy oracle against the reference's own formula (torch.sparse coalesce),
the union as a 1x..x1 regular-conv rulebook, and the host-side checks of the new C entry points."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import oracle
from tests import sparse_add_oracle as sao

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cloud(rng, batch, shape, n, dup=0):
    inds = np.stack([rng.integers(0, batch, n)] + [rng.integers(0, s, n) for s in shape], 1).astype(np.int32)
    if dup:
        inds = np.concatenate([inds, inds[rng.integers(0, n, dup)]], 0)
        inds = inds[rng.permutation(len(inds))]
    return inds


def _linear(inds, batch, shape):
    key = inds[:, 0].astype(np.int64)
    for a, s in enumerate(shape):
        key = key * s + inds[:, a + 1]
    return key


CASES = [  # (operands, batch, spatial shape, rows per operand, duplicates in operand 0)
    (1, 2, [6, 7], 40, 10),
    (2, 2, [5, 6, 7], 60, 0),
    (3, 3, [4, 5, 6, 3], 50, 12),
    (4, 1, [9, 9], 30, 5),
    (4, 2, [3, 4, 2, 5], 25, 0),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"T{c[0]}-{len(c[2])}d")
def test_oracle_matches_torch_sparse_coalesce(case):
    """same coordinate set and per-coordinate sums as the reference's sparse_add formula
    (sum of torch.sparse_coo_tensor, coalesce), after reordering by linear key"""
    t, batch, shape, n, dup = case
    rng = np.random.default_rng(t * 100 + len(shape))
    inds = [_cloud(rng, batch, shape, n + 7 * i, dup if i == 0 else 0) for i in range(t)]
    feats = [rng.integers(-8, 9, (len(x), 5)).astype(np.float64) for x in inds]   # exact in any order
    out_inds, out, dst, visit = sao.sparse_add(inds, feats, batch, shape)
    full = [batch, *shape, 5]
    ref = None
    for x, f in zip(inds, feats):
        s = torch.sparse_coo_tensor(torch.from_numpy(x.T.astype(np.int64)), torch.from_numpy(f), full)
        ref = s if ref is None else ref + s
    ref = ref.coalesce()
    ref_inds = ref.indices().T.numpy().astype(np.int32)
    ref_vals = ref.values().numpy()
    assert out_inds.shape[0] == ref_inds.shape[0]
    mine = np.argsort(_linear(out_inds, batch, shape))
    np.testing.assert_array_equal(out_inds[mine], ref_inds)
    np.testing.assert_array_equal(out[mine].astype(np.float64), ref_vals)
    # visit order: largest operand first, ties to the earliest
    rows = [len(x) for x in inds]
    assert visit[0] == max(range(t), key=lambda i: (rows[i], -i))


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"T{c[0]}-{len(c[2])}d")
def test_union_is_the_1x1_conv_rulebook(case):
    """the visit-order union equals the regular-conv rulebook of a ksize-1, stride-1, padding-0 conv over the
    concatenated coordinates: same out_inds in the same order, same input -> output map"""
    t, batch, shape, n, dup = case
    rng = np.random.default_rng(7 + t)
    inds = [_cloud(rng, batch, shape, n + 3 * i, dup if i == 0 else 0) for i in range(t)]
    visit = sao.visit_order([len(x) for x in inds])
    out_inds, dst = sao.union([inds[i] for i in visit], batch, shape)
    cat = np.concatenate([inds[i] for i in visit], 0)
    nd = len(shape)
    rb_inds, pairs, num = oracle.get_indice_pairs(cat, batch, shape, [1] * nd, [1] * nd, [0] * nd, [1] * nd,
                                                  [0] * nd)
    np.testing.assert_array_equal(out_inds, rb_inds)
    rb_dst = np.full(len(cat), -1, dtype=np.int32)
    rb_dst[pairs[0, 0, :num[0]]] = pairs[1, 0, :num[0]]
    np.testing.assert_array_equal(dst, rb_dst)


def test_oracle_drops_out_of_range_rows_and_sums_in_visit_order():
    inds = [np.array([[0, 1, 1], [0, 1, 1], [2, 0, 0], [0, 3, 0]], np.int32),       # batch 2, y 3: out of range
            np.array([[0, 0, 0], [0, 1, 1], [1, -1, 0]], np.int32)]
    feats = [np.array([[1e8], [1.0], [5.0], [6.0]], np.float32), np.array([[2.0], [-1e8], [7.0]], np.float32)]
    out_inds, out, dst, visit = sao.sparse_add(inds, feats, 2, [3, 2])
    assert visit == [0, 1]
    np.testing.assert_array_equal(out_inds, [[0, 1, 1], [0, 0, 0]])
    np.testing.assert_array_equal(dst, [0, 0, -1, -1, 1, 0, -1])
    want = np.float32(np.float32(np.float32(0) + np.float32(1e8)) + np.float32(1.0)) + np.float32(-1e8)
    assert out[0, 0] == want == 0.0           # visit order: (1e8 + 1) - 1e8 rounds the 1 away
    assert out[1, 0] == 2.0
    grads = sao.gradients(np.array([[3.0], [4.0]], np.float32), dst, [4, 3])
    np.testing.assert_array_equal(grads[0][:, 0], [3, 3, 0, 0])
    np.testing.assert_array_equal(grads[1][:, 0], [4, 3, 0])


def test_oracle_sum_is_a_sequential_float32_loop():
    rng = np.random.default_rng(3)
    dst = rng.integers(-1, 20, 500).astype(np.int32)
    f = (rng.standard_normal((500, 3)) * 10.0 ** rng.integers(-6, 7, (500, 1))).astype(np.float32)
    got = sao.sum_rows([f[:200], f[200:]], dst, 20)
    want = np.zeros((20, 3), np.float32)
    for g in range(500):
        if dst[g] >= 0:
            want[dst[g]] = want[dst[g]] + f[g]
    assert got.tobytes() == want.tobytes()


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def test_sparse_add_entry_points_validate_arguments(lib):
    """invalid arguments are refused before any CUDA call, with a message"""
    from spconv_b200 import _cabi
    ops = _cabi.SparseAddOperands()
    ops.count = 0
    assert lib.spx_sparse_add_fwd(ctypes.byref(ops), 1, 1, 1, 4, _cabi.SPX_F32, 1, None) == 2
    assert "0 operands, must be in [1, 64]" in _cabi.last_error()
    ops.count = 65
    assert lib.spx_sparse_add_gather(1, 1, 1, ctypes.byref(ops), 4, _cabi.SPX_F32, None) == 2
    assert "65 operands" in _cabi.last_error()
    ops.count = 2
    ops.rows[0], ops.rows[1] = 10, 5
    ops.features[0] = 1
    assert lib.spx_sparse_add_fwd(ctypes.byref(ops), 1, 1, 3, 4, _cabi.SPX_F32, 1, None) == 2
    assert "features of operand 1 are NULL" in _cabi.last_error()
    ops.features[1] = 1
    assert lib.spx_sparse_add_fwd(ctypes.byref(ops), 1, 1, 3, 4, _cabi.SPX_I8, 1, None) == 2
    assert "unsupported dtype" in _cabi.last_error()
    assert lib.spx_sparse_add_fwd(ctypes.byref(ops), 1, 1, 3, 0, _cabi.SPX_F16, 1, None) == 2
    assert "channels must be positive" in _cabi.last_error()
    assert lib.spx_sparse_add_fwd(ctypes.byref(ops), 1, 1, 16, 4, _cabi.SPX_F16, 1, None) == 2
    assert "output count 16 not in [0, 15]" in _cabi.last_error()
    assert lib.spx_sparse_add_fwd(ctypes.byref(ops), None, 1, 3, 4, _cabi.SPX_F16, 1, None) == 2
    assert "NULL pointer" in _cabi.last_error()
    ops.rows[1] = -1
    assert lib.spx_sparse_add_gather(1, 1, 1, ctypes.byref(ops), 4, _cabi.SPX_F32, None) == 2
    assert "negative row count" in _cabi.last_error()
    assert lib.spx_sparse_add_group(1, 10, 11, 1, 1, 1, 1 << 20, None) == 2
    assert "output count 11 not in [0, 10]" in _cabi.last_error()
    assert lib.spx_sparse_add_group(1, 10, 4, 1, 1, 1, 16, None) == 2
    assert "workspace too small" in _cabi.last_error()
    assert lib.spx_sparse_add_group(1, 10, 4, 1, None, 1, 1 << 20, None) == 2
    assert "offsets is NULL" in _cabi.last_error()
    assert lib.spx_sparse_add_group_workspace_size(100000) > 100000 * 4 * 5
    assert _cabi.SPX_SPARSE_ADD_MAX_OPERANDS == 64


def test_sparse_add_operands_struct_matches_the_header_layout(tmp_path):
    from spconv_b200 import _cabi
    cls = _cabi.SparseAddOperands
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "spconv_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(spx_sparse_add_operands));']
    for fname, _ in cls._fields_:
        lines.append(f'  printf("{fname} %zu\\n", offsetof(spx_sparse_add_operands, {fname}));')
    lines.append('  printf("max %d\\n", SPX_SPARSE_ADD_MAX_OPERANDS);')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                    check=True).stdout.split("\n") if ln.strip())
    assert int(out.pop("size")) == ctypes.sizeof(cls)
    assert int(out.pop("max")) == _cabi.SPX_SPARSE_ADD_MAX_OPERANDS
    for fname, _ in cls._fields_:
        assert int(out[fname]) == getattr(cls, fname).offset, fname


def test_sparse_add_rejects_cpu_tensors_and_int8():
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import functional as Fsp
    inds = torch.tensor([[0, 1, 1]], dtype=torch.int32)
    a = spconv.SparseConvTensor(torch.ones(1, 4), inds, [3, 3], 1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        Fsp.sparse_add(a, a)
    q = spconv.SparseConvTensor(torch.ones(1, 4, dtype=torch.int8), inds, [3, 3], 1)
    with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
        Fsp.sparse_add_hash_based(a, q)
