"""Bounded regular-conv rulebook, the parts that need no GPU: argument validation of the new C entry
points, the workspace size, padding helpers of SparseConvTensor, the modules that refuse a padded
tensor, and the truncation rule the GPU test compares against."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.util import random_cloud

from spconv_b200 import _cabi
import spconv_b200.pytorch as spconv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def truncate_rulebook(out_inds, pair_fwd, pair_bwd, bound):
    """What a bounded rulebook holds when the unbounded one has M > bound outputs: the outputs ranked below
    ``bound`` are kept, every pair that pointed at a dropped output is -1, masks follow from the pairs."""
    kv = pair_fwd.shape[0]
    words = (kv + 31) // 32
    pf = pair_fwd[:, :bound].copy()
    pb = np.where(pair_bwd >= bound, -1, pair_bwd)

    def masks(table):
        m = np.zeros((table.shape[1], words), np.uint32)
        for k in range(kv):
            m[:, k // 32] |= (table[k] >= 0).astype(np.uint32) << np.uint32(k % 32)
        return m
    return out_inds[:bound].copy(), pf, pb, masks(pf), masks(pb)


def test_truncation_rule_on_a_hand_made_rulebook():
    # 3 inputs, 2 offsets, 3 outputs; bound 2 drops output 2 and the pairs that point at it
    out_inds = np.array([[0, 1], [0, 2], [0, 3]], np.int32)
    pair_bwd = np.array([[0, 1, 2], [-1, 0, 2]], np.int32)
    pair_fwd = np.array([[0, 1, 2], [1, -1, 2]], np.int32)
    oi, pf, pb, mf, mb = truncate_rulebook(out_inds, pair_fwd, pair_bwd, 2)
    assert oi.tolist() == [[0, 1], [0, 2]]
    assert pf.tolist() == [[0, 1], [1, -1]]
    assert pb.tolist() == [[0, 1, -1], [-1, 0, -1]]
    assert mf[:, 0].tolist() == [3, 1] and mb[:, 0].tolist() == [1, 3, 0]


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import build
    build.build()
    return _cabi.load()


def _geo():
    return _cabi.make_geometry(3, 1, [41, 1600, 1408], [21, 800, 704], [3] * 3, [2] * 3, [1] * 3, [1] * 3)


def test_bounded_workspace_size(lib):
    g = _geo()
    size = lambda n, b: lib.spx_conv_rulebook_bounded_workspace_size(ctypes.byref(g), n, b)  # noqa: E731
    assert size(1000, 0) == 0 and size(1000, -5) == 0 and size(-1, 128) == 0
    assert lib.spx_conv_rulebook_bounded_workspace_size(None, 1000, 128) == 0
    prev = 0
    for b in (128, 1024, 4096, 65536, 1 << 20):
        cur = size(100_000, b)
        assert cur >= prev and cur >= b * 16        # a table of >= 2 * bound 8-byte slots
        prev = cur
    # sized from the bound, not from the worst case of the unbounded path (8 outputs per input)
    assert size(100_000, 65536) < lib.spx_conv_rulebook_all_workspace_size(ctypes.byref(g), 100_000)


def test_bounded_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "g = _cabi.make_geometry(3, 1, [8] * 3, [4] * 3, [3] * 3, [2] * 3, [1] * 3, [1] * 3)",
        "P = 1 << 20",
        "def call(n=10, bound=128, out=P, num=P, ws=P, ws_bytes=1 << 30, tb=P, sb=P):",
        "    return lib.spx_conv_rulebook_bounded_all(ctypes.byref(g), P, n, bound, out, P, P, P, P, P, sb, 1, P, P, tb,"
        " P if tb else None, num, P, ws, ws_bytes, None)",
        "def expect(rc, text):",
        "    assert rc != 0 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "expect(call(bound=0), 'bound must be')",
        "expect(call(bound=-3), 'bound must be')",
        "expect(call(out=None), 'NULL pointer')",
        "expect(call(num=None), 'NULL pointer')",
        "expect(call(ws=None), 'NULL pointer')",
        "expect(call(tb=None), 'all be given')",
        "expect(call(ws_bytes=64), 'workspace too small')",
        "expect(lib.spx_zero_rows_from_count(None, 4, 32, P, None), 'NULL pointer')",
        "expect(lib.spx_zero_rows_from_count(P, 4, 0, P, None), 'bad rows')",
        "expect(lib.spx_zero_rows_from_count(P, 4, 7, P, None), 'bad rows')",
        "assert lib.spx_zero_rows_from_count(P, 0, 32, P, None) == 0",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def _tensor(n=5, c=4):
    rng = np.random.default_rng(0)
    feats, inds = random_cloud(rng, [6, 6, 6], [n], c)
    return spconv.SparseConvTensor(torch.from_numpy(feats), torch.from_numpy(inds), [6, 6, 6], 1)


def test_pad_to_and_valid_mask():
    x = _tensor(5)
    assert x.num_valid is None and x.valid_mask().tolist() == [True] * 5
    p = x.pad_to(8)
    assert p.features.shape == (8, 4) and p.indices.shape == (8, 4)
    assert int(p.num_valid) == 5 and p.num_valid.dtype == torch.int32
    assert p.valid_mask().tolist() == [True] * 5 + [False] * 3
    assert (p.indices[5:] == -1).all() and (p.features[5:] == 0).all()
    assert torch.equal(p.features[:5], x.features) and torch.equal(p.indices[:5], x.indices)
    assert p.indice_dict == {} and x.num_valid is None
    # padding again keeps the count; derived tensors carry it
    q = p.pad_to(16)
    assert q.features.shape[0] == 16 and int(q.num_valid) == 5
    assert p.replace_feature(p.features * 2).num_valid is p.num_valid
    assert p.shadow_copy().num_valid is p.num_valid
    with pytest.raises(ValueError, match="already has"):
        p.pad_to(4)


def test_dense_of_a_padded_tensor_equals_dense_of_its_valid_rows():
    x = _tensor(7)
    p = x.pad_to(12)
    p = p.replace_feature(p.features + 3.0)          # padding rows hold junk after a layer
    want = x.replace_feature(x.features + 3.0).dense()
    assert torch.equal(p.dense(), want)
    assert torch.equal(p.dense(channels_first=False), x.replace_feature(x.features + 3.0).dense(False))


def test_row_reducing_modules_refuse_a_padded_tensor():
    p = _tensor(5).pad_to(8)
    bn = spconv.SparseBatchNorm(4)
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        bn(p)
    bn.eval()
    assert bn(p).features.shape == (8, 4)            # eval-mode BN is row-wise
    seq = spconv.SparseSequential(torch.nn.BatchNorm1d(4))
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        seq(p)
    assert seq.eval()(p).num_valid is p.num_valid
    for mod in (spconv.SparseGlobalMaxPool(), spconv.SparseGlobalAvgPool(), spconv.AddTable()):
        with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
            mod([p, p] if isinstance(mod, spconv.AddTable) else p)
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        spconv.functional.sparse_add(p, p)
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        spconv.functional.remove_duplicate(p)


def test_bound_attributes_and_set_output_bounds_selection():
    from spconv_b200.pytorch.bounds import _strided_modules
    net = spconv.SparseSequential(
        spconv.SubMConv3d(4, 4, 3, indice_key="a"), spconv.SparseConv3d(4, 8, 3, stride=2, indice_key="d"),
        spconv.SparseMaxPool3d(2), spconv.SparseInverseConv3d(8, 4, 3, indice_key="d"),
        spconv.SparseConvTranspose3d(4, 4, 2, stride=2))
    assert [n for n, _ in _strided_modules(net)] == ["1", "2", "4"]
    for _, m in net.named_modules():
        if hasattr(m, "num_out_act_bound"):
            assert m.num_out_act_bound is None
    spconv.check_bounds(net)                         # nothing bounded has run: nothing to read
