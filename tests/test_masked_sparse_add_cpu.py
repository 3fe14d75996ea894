"""masked_sparse_add / masked_remove_duplicate and the masked table modules, the parts that need no GPU: argument
validation of the C entry points before any launch, the workspace sizes, the modules' refusal of CPU and int8
tensors, the exports, the bound selection of set_output_bounds / check_bounds, and the default modules' unchanged
refusal of padded tensors."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

import spconv_b200.pytorch as spconv
from spconv_b200 import _cabi
from spconv_b200.pytorch import functional as Fsp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import build
    build.build()
    return _cabi.load()


def _union_geo(shape=(8, 8, 8), batch=2):
    n = len(shape)
    return _cabi.make_geometry(n, batch, list(shape), list(shape), [1] * n, [1] * n, [0] * n, [1] * n)


def test_workspace_sizes(lib):
    g = _union_geo()
    union = lambda n, b: lib.spx_sparse_add_union_workspace_size(ctypes.byref(g), n, b)  # noqa: E731
    plan = lambda n, b: lib.spx_masked_sparse_add_workspace_size(ctypes.byref(g), n, b)  # noqa: E731
    assert union(100, 0) == 0 and union(100, 101) == 0 and union(0, 0) == 0 and union(-1, 1) == 0
    assert lib.spx_sparse_add_union_workspace_size(None, 100, 10) == 0
    assert plan(100, 101) == 0 and plan(-1, 0) == 0 and plan(10, -1) == 0 and plan(0, 0) > 0
    prev = 0
    for n in (1, 1000, 100_000, 1 << 20):
        cur = plan(n, n)
        assert cur >= prev and cur >= union(n, n) + 4 * n * 4 + 4 * n * 4   # packed coords, src, dst, order
        assert union(n, n) >= 2 * n * 8                                      # a table of >= 2 * bound slots
        prev = cur
    assert union(100_000, 1000) < union(100_000, 100_000)                  # the table is sized from the bound


def test_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def geo(k=1, s=1, out=8, transposed=False):",
        "    return _cabi.make_geometry(3, 2, [8] * 3, [out] * 3, [k] * 3, [s] * 3, [0] * 3, [1] * 3, transposed)",
        "def opnds(rows=(10, 5)):",
        "    o = _cabi.SparseAddOperands()",
        "    o.count = len(rows)",
        "    for t, r in enumerate(rows):",
        "        o.rows[t] = r",
        "    return o",
        "nv = (ctypes.c_void_p * 64)(*([P] * 64))",
        "def plan(g=None, o=None, ind=P, bound=15, out=P, dst=P, order=P, off=P, num=P, st=P, ws=P, wsb=1 << 40):",
        "    g = g or geo()",
        "    return lib.spx_masked_sparse_add_plan(ctypes.byref(g), None if o is False else ctypes.byref(o or opnds()),",
        "                                          nv, ind, bound, out, dst, order, off, num, st, ws, wsb, None)",
        "def union(g=None, n=10, bound=10, ind=P, out=P, dst=P, num=P, st=P, ws=P, wsb=1 << 40):",
        "    g = g or geo()",
        "    return lib.spx_sparse_add_union(ctypes.byref(g), ind, n, bound, out, dst, num, st, ws, wsb, None)",
        "def heads(order=P, off=P, num=P, bound=4, rows=10, h=P, inv=P):",
        "    return lib.spx_masked_sparse_add_heads(order, off, num, bound, rows, h, inv, None)",
        "def expect(rc, text):",
        "    assert rc != 0 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "expect(plan(o=False), 'operands is NULL')",
        "o65 = opnds([1] * 64); o65.count = 65",
        "expect(plan(o=o65), 'operands, must be in [1, 64]')",
        "o0 = _cabi.SparseAddOperands(); o0.count = 0",
        "expect(plan(o=o0), 'operands, must be in [1, 64]')",
        "expect(plan(o=opnds((3, -1))), 'negative row count')",
        "expect(plan(bound=0), 'bound must be')",
        "expect(plan(bound=-1), 'bound must be')",
        "expect(plan(bound=16), 'bound must be')",
        "expect(plan(g=geo(k=3)), 'must be 1x..x1')",
        "expect(plan(g=geo(s=2)), 'must be 1x..x1')",
        "expect(plan(g=geo(out=4)), 'must be 1x..x1')",
        "expect(plan(g=geo(transposed=True)), 'must be 1x..x1')",
        "for k in ('ind', 'out', 'dst', 'order', 'off', 'num', 'st', 'ws'):",
        "    expect(plan(**{k: None}), 'NULL pointer')",
        "expect(plan(wsb=64), 'workspace too small')",
        "expect(union(bound=0), 'bound must be')",
        "expect(union(bound=11), 'bound must be')",
        "expect(union(n=0, bound=1), 'bad row count')",
        "expect(union(g=geo(k=3)), 'must be 1x..x1')",
        "for k in ('ind', 'out', 'dst', 'num', 'st', 'ws'):",
        "    expect(union(**{k: None}), 'NULL pointer')",
        "expect(union(wsb=64), 'workspace too small')",
        "expect(heads(rows=-1), 'bad row count')",
        "expect(heads(bound=11), 'bound')",
        "for k in ('order', 'off', 'num', 'h', 'inv'):",
        "    expect(heads(**{k: None}), 'NULL pointer')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def _tensor(dtype=torch.float32, n=3):
    inds = torch.tensor([[0, 1, 1, 1], [1, 2, 2, 2], [0, 3, 3, 3]], dtype=torch.int32)[:n]
    feats = torch.arange(n * 8, dtype=torch.float32).view(n, 8).to(dtype)
    return spconv.SparseConvTensor(feats, inds, [4, 4, 4], 2)


CALLS = {
    "masked_sparse_add": lambda x: Fsp.masked_sparse_add(x, x),
    "masked_remove_duplicate": lambda x: Fsp.masked_remove_duplicate(x),
    "MaskedAddTableMisaligned": lambda x: spconv.MaskedAddTableMisaligned()([x, x]),
    "MaskedAddTableMisaligned-bounded": lambda x: spconv.MaskedAddTableMisaligned(4)([x, x]),
    "MaskedRemoveDuplicate": lambda x: spconv.MaskedRemoveDuplicate()(x),
}


@pytest.mark.parametrize("call", list(CALLS))
def test_refuse_cpu_and_int8_tensors(call):
    fn = CALLS[call]
    for x in (_tensor(), _tensor().pad_to(5)):
        with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
            fn(x)
    for dt in (torch.int8, torch.float64):
        with pytest.raises(RuntimeError, match="float32, float16 and bfloat16"):
            fn(_tensor(dt))


def test_bad_bound_is_refused():
    with pytest.raises(ValueError, match="num_out_act_bound must be positive"):
        Fsp.masked_sparse_add(_tensor(), num_out_act_bound=0)
    with pytest.raises(ValueError, match="num_out_act_bound must be positive"):
        Fsp.masked_remove_duplicate(_tensor(), num_out_act_bound=-4)


def test_names_are_exported():
    from spconv_b200.pytorch import spatial, tables
    assert spconv.MaskedAddTable is tables.MaskedAddTable and spconv.MaskedJoinTable is tables.MaskedJoinTable
    assert spconv.MaskedAddTableMisaligned is tables.MaskedAddTableMisaligned
    assert spconv.MaskedRemoveDuplicate is spatial.MaskedRemoveDuplicate
    assert callable(spconv.functional.masked_sparse_add) and callable(spconv.functional.masked_remove_duplicate)
    assert spconv.MaskedAddTableMisaligned().num_out_act_bound is None
    assert spconv.MaskedRemoveDuplicate(256, name="rd").num_out_act_bound == 256


def test_masked_tables_on_the_cpu_are_row_wise():
    """MaskedAddTable / MaskedJoinTable are plain torch arithmetic: they run anywhere and keep num_valid"""
    p = _tensor().pad_to(5)
    q = p.replace_feature(p.features * 2)
    s = spconv.MaskedAddTable()([p, q])
    assert torch.equal(s.features, p.features * 3) and s.num_valid is p.num_valid and s.indices is p.indices
    j = spconv.MaskedJoinTable()([p, q])
    assert j.features.shape == (5, 16) and j.num_valid is p.num_valid
    u = _tensor()
    assert spconv.MaskedAddTable()([u, u]).num_valid is None
    other = _tensor().pad_to(5)                                # the same count, but another tensor object
    for mod in (spconv.MaskedAddTable(), spconv.MaskedJoinTable()):
        with pytest.raises(ValueError, match="same num_valid tensor object"):
            mod([p, other])
        with pytest.raises(ValueError, match="same num_valid tensor object"):
            mod([p, u])
    with pytest.raises(AssertionError, match="use MaskedAddTableMisaligned instead"):
        spconv.MaskedAddTable()([u, _tensor(n=2)])


def test_set_output_bounds_and_check_bounds_select_the_masked_modules():
    from spconv_b200.pytorch.bounds import _strided_modules
    net = spconv.SparseSequential(
        spconv.SubMConv3d(4, 4, 3, indice_key="a"), spconv.SparseConv3d(4, 8, 3, stride=2, indice_key="d"),
        spconv.MaskedRemoveDuplicate(), spconv.SparseInverseConv3d(8, 4, 3, indice_key="d"),
        spconv.MaskedAddTable())
    net.add_module("merge", spconv.MaskedAddTableMisaligned(512))
    assert [n for n, _ in _strided_modules(net)] == ["1", "2", "merge"]
    spconv.check_bounds(net)                                   # nothing bounded has run: nothing to read
    word = torch.zeros((1,), dtype=torch.int32)
    net.merge._bound_status = word
    spconv.check_bounds(net)
    word.fill_(1)
    with pytest.raises(RuntimeError, match="'merge': more outputs than num_out_act_bound"):
        spconv.check_bounds(net)
    assert int(word) == 0                                      # a net's words are cleared by the read
    net.merge._bound_status = torch.full((1,), 2, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="'merge': the hash table"):
        spconv.check_bounds(net)


def test_the_default_entry_points_still_refuse_padded_tensors():
    p = _tensor().pad_to(5)
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        Fsp.sparse_add(p, _tensor())
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        Fsp.sparse_add_hash_based(_tensor(), p)
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        Fsp.remove_duplicate(p)
    for mod in (spconv.AddTable(), spconv.JoinTable()):
        with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
            mod([p, p])
