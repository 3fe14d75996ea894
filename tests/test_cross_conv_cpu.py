"""Convolution onto given output coordinates, without a GPU: the numpy oracle of the cross rulebook against the
existing rulebooks (target = the SubM output or a strided / transposed conv's own output set) and against the
layer's forward relation, the argument checks of spx_cross_rulebook_all, and the module's refusals, which all
happen on the host before any launch."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests.conv_ref import offset_taps
from tests.cross_rulebook_oracle import cross_tables, forward_relation, usable_rows
from tests.util import random_cloud

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: (shape, ksize, stride, padding, dilation, kind, points per sample)
CASES = {
    "subm_3d": ([12, 14, 16], [3, 3, 3], [1] * 3, [0] * 3, [1] * 3, "subm", [300, 200]),
    "subm_1d_k5": ([90], [5], [1], [0], [2], "subm", [40]),
    "subm_4d": ([5, 6, 7, 8], [3, 1, 3, 3], [1] * 4, [0] * 4, [1] * 4, "subm", [150]),
    "conv_2d": ([30, 40], [3, 3], [2, 2], [1, 1], [1, 1], "conv", [200, 100]),
    "conv_3d_dilated": ([12, 14, 16], [3, 3, 3], [2, 1, 2], [2, 2, 2], [2, 2, 2], "conv", [250]),
    "conv_4d": ([6, 7, 8, 9], [3, 3, 3, 3], [2, 2, 2, 2], [1, 1, 1, 1], [1] * 4, "conv", [120]),
    "transposed_3d": ([6, 7, 8], [2, 3, 2], [2, 2, 2], [0, 1, 0], [1, 1, 1], "transpose", [80, 60]),
    "transposed_1d": ([50], [3], [3], [1], [1], "transpose", [20]),
    "kv125": ([10, 10, 10], [5, 5, 5], [1] * 3, [0] * 3, [1] * 3, "subm", [200]),
}


@pytest.fixture(scope="module")
def orc():
    from oracle import oracle
    oracle.build()
    return oracle


def _geometry(case):
    shape, ksize, stride, padding, dilation, kind, _ = case
    if kind == "subm":
        return shape, [1] * len(shape), [(k // 2) * d for k, d in zip(ksize, dilation)], False
    if kind == "transpose":
        out = [(i - 1) * s - 2 * p + k for i, k, s, p in zip(shape, ksize, stride, padding)]
        return out, stride, padding, True
    out = [(i + 2 * p - d * (k - 1) - 1) // s + 1 for i, k, s, p, d in zip(shape, ksize, stride, padding, dilation)]
    return out, stride, padding, False


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_equals_the_existing_rulebook_on_its_own_output_set(orc, name):
    """target = the SubM input, or the strided / transposed conv's own outids: every table equals
    oracle.implicit_gemm_tables of the reference-order rulebook"""
    case = CASES[name]
    shape, ksize, stride, padding, dilation, kind, per = case
    _, inds = random_cloud(np.random.default_rng(len(name)), shape, per, 1)
    batch = len(per)
    subm = kind == "subm"
    outids, pairs, num = orc.get_indice_pairs(inds, batch, shape, ksize, stride, padding, dilation,
                                              [0] * len(shape), subm, kind == "transpose")
    want = orc.implicit_gemm_tables(pairs, num, inds.shape[0], outids.shape[0], subm)
    out_shape, s, p, tr = _geometry(case)
    got = cross_tables(inds, outids, batch, shape, out_shape, ksize, s, p, dilation, tr)
    for key in ("pair_fwd", "pair_bwd", "mask_fwd", "argsort_fwd", "mask_bwd", "argsort_bwd"):
        assert np.array_equal(got[key], want[key]), (name, key)


@pytest.mark.parametrize("name", ["conv_2d", "transposed_3d", "subm_3d"])
def test_oracle_pairs_follow_the_forward_relation_between_two_clouds(name):
    """two unrelated clouds with duplicates and out-of-range rows on both sides: every pair is the layer's forward
    relation from a usable source row to an active target row, and every such relation is a pair"""
    shape, ksize, stride, padding, dilation, kind, per = CASES[name]
    rng = np.random.default_rng(7)
    out_shape, s, p, tr = _geometry(CASES[name])
    _, src = random_cloud(rng, shape, per, 1)
    _, tgt = random_cloud(rng, out_shape, [max(n // 2, 1) for n in per], 1)
    src = np.concatenate([src, src[:5], np.full((3, src.shape[1]), -1, np.int32)]).astype(np.int32)
    tgt = np.concatenate([tgt, tgt[-4:], tgt[:1] * 0 + 10 ** 6]).astype(np.int32)
    batch = len(per)
    got = cross_tables(src, tgt, batch, shape, out_shape, ksize, s, p, dilation, tr, num_valid_src=src.shape[0] - 1)
    taps = offset_taps(ksize)
    src_ok = usable_rows(src, src.shape[0] - 1, batch, shape)
    assert got["active"][:len(tgt) - 5].sum() == len(tgt) - 5 and not got["active"][-5:].any()
    tkeys = {tuple(tgt[o]): o for o in np.nonzero(got["active"])[0]}
    expect = np.full_like(got["pair_bwd"], -1)
    for i in np.nonzero(src_ok)[0]:
        if any((src[j] == src[i]).all() for j in range(i)):
            continue                                  # a later duplicate of a usable row takes part in no pair
        for k in range(len(taps)):
            o, exact = forward_relation(src[i:i + 1, 1:].astype(np.int64), taps[k], s, p, dilation, tr)
            if exact.all():
                o = tkeys.get((src[i, 0], *o[0].tolist()))
                if o is not None:
                    expect[k, i] = o
    assert np.array_equal(got["pair_bwd"], expect)
    kk, oo = np.nonzero(got["pair_fwd"] >= 0)
    assert np.array_equal(got["pair_bwd"][kk, got["pair_fwd"][kk, oo]], oo)


# ---------------------------------------------------------------------------- C entry point
@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def _call(lib, g, n=10, m=10, src_indices=16, out_indices=32, num_valid=None, out_num_valid=None, pair_fwd=48,
          pair_bwd=64, mask_fwd=80, mask_bwd=96, argsort_fwd=112, argsort_bwd=128, table_fwd=144, tmask_fwd=160,
          table_bwd=176, tmask_bwd=192, workspace=208, ws_bytes=1 << 40):
    """every pointer a fake, 16-byte aligned address: each call must be refused before its first launch"""
    return lib.spx_cross_rulebook_all(ctypes.byref(g), src_indices, n, num_valid, out_indices, m, out_num_valid, pair_fwd,
                                      pair_bwd, mask_fwd, mask_bwd, argsort_fwd, argsort_bwd, 1, table_fwd, tmask_fwd,
                                      table_bwd, tmask_bwd, workspace, ws_bytes, None)


def test_entry_point_is_exported_bound_and_sized(lib):
    from spconv_b200 import _cabi
    for name in ("spx_cross_rulebook_all", "spx_cross_rulebook_all_workspace_size"):
        assert hasattr(lib, name) and name in _cabi.SIGNATURES
    g = _cabi.make_geometry(3, 2, [41, 1600, 1408], [41, 1600, 1408], [3] * 3, [1] * 3, [1] * 3, [1] * 3)
    # two hash tables of 8-byte slots at load factor <= 1/4
    assert lib.spx_cross_rulebook_all_workspace_size(ctypes.byref(g), 100000, 50000) >= (524288 + 262144) * 8
    assert lib.spx_cross_rulebook_all_workspace_size(ctypes.byref(g), -1, 10) == 0
    assert lib.spx_cross_rulebook_all_workspace_size(None, 10, 10) == 0
    g.ndim = 5
    assert lib.spx_cross_rulebook_all_workspace_size(ctypes.byref(g), 10, 10) == 0


def test_entry_point_refuses_bad_arguments_before_any_launch(lib):
    import subprocess
    import sys
    from spconv_b200 import _cabi

    def geo(**kw):
        a = dict(ndim=3, batch=1, ins=[8] * 3, outs=[8] * 3, k=[3] * 3, s=[1] * 3, p=[1] * 3, d=[1] * 3, tr=False)
        a.update(kw)
        return _cabi.make_geometry(a["ndim"], a["batch"], a["ins"], a["outs"], a["k"], a["s"], a["p"], a["d"], a["tr"])

    def refused(rc, text):
        assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())

    g = geo()
    refused(_call(lib, geo(ndim=0)), "ndim")
    bad = geo()
    bad.ndim = 5
    refused(_call(lib, bad), "ndim")
    refused(_call(lib, geo(batch=0)), "batch_size")
    refused(_call(lib, geo(k=[5, 5, 6])), "kernel volume 150")
    refused(_call(lib, geo(s=[1, 0, 1])), "stride")
    refused(_call(lib, geo(outs=[8, 0, 8])), "out_dims")
    refused(_call(lib, geo(p=[1, -1, 1])), "padding must be >= 0")
    refused(_call(lib, geo(ins=[2 ** 30] * 3, outs=[2 ** 30] * 3, s=[2] * 3)), "below 2^31")
    refused(_call(lib, g, n=-1), "bad row counts")
    refused(_call(lib, g, m=2 ** 31), "bad row counts")
    refused(_call(lib, g, workspace=None), "workspace")
    for arg in ("out_indices", "pair_fwd", "mask_fwd", "argsort_fwd", "table_fwd", "tmask_fwd"):
        refused(_call(lib, g, **{arg: None}), "NULL pointer argument (out_indices")
    for arg in ("src_indices", "pair_bwd", "mask_bwd"):
        refused(_call(lib, g, **{arg: None}), "NULL pointer argument (src_indices")
    for arg in ("argsort_bwd", "table_bwd", "tmask_bwd"):
        refused(_call(lib, g, **{arg: None}), "all be NULL (inference)")
    refused(_call(lib, g, src_indices=20), "src_indices must be 16-byte aligned")
    refused(_call(lib, g, out_indices=36), "out_indices must be 16-byte aligned")
    refused(_call(lib, g, ws_bytes=100), "workspace too small")
    # an empty side does not need its pointers
    refused(_call(lib, g, m=0, out_indices=None, pair_fwd=None, ws_bytes=1), "workspace too small")
    refused(_call(lib, g, n=0, src_indices=None, pair_bwd=None, ws_bytes=1), "workspace too small")
    # and none of the refusals launched anything (checked in a fresh process: the counter is process-wide)
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "from tests.test_cross_conv_cpu import _call",
        "lib = _cabi.load()",
        "g = _cabi.make_geometry(3, 1, [8] * 3, [8] * 3, [9, 9, 2], [1] * 3, [1] * 3, [1] * 3)",
        "assert _call(lib, g) == 2",
        "g = _cabi.make_geometry(3, 1, [8] * 3, [8] * 3, [3] * 3, [1] * 3, [1] * 3, [1] * 3)",
        "assert _call(lib, g, src_indices=20) == 2 and _call(lib, g, ws_bytes=100) == 2",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


# ---------------------------------------------------------------------------- module refusals
def _tensor(shape, rows=6, batch=1, channels=4, seed=0):
    import spconv_b200.pytorch as spconv
    _, inds = random_cloud(np.random.default_rng(seed), shape, [rows] * batch, 1)
    return spconv.SparseConvTensor(torch.zeros(inds.shape[0], channels), torch.from_numpy(inds), shape, batch)


def test_module_refusals_happen_on_the_host():
    """CPU tensors: any launch would fail, so every refusal below is raised before the first one"""
    import spconv_b200.pytorch as spconv
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch.core import ImplicitGemmIndiceData
    x = _tensor([8, 8, 8])
    subm = spconv.SubMConv3d(4, 4, 3, indice_key="k")
    down = spconv.SparseConv3d(4, 4, 3, 2, 1)
    with pytest.raises(ValueError, match="batch_size"):
        subm(x, target=_tensor([8, 8, 8], batch=2))
    with pytest.raises(ValueError, match="output shape"):
        subm(x, target=_tensor([8, 8, 9]))
    with pytest.raises(ValueError, match="output shape"):
        down(x, target=_tensor([8, 8, 8]))
    with pytest.raises(ValueError, match="output shape"):
        subm(x, target=_tensor([8, 8]))
    with pytest.raises(TypeError, match="SparseConvTensor"):
        subm(x, target=x.features)
    with pytest.raises(ValueError, match="takes no target"):
        spconv.SparseInverseConv3d(4, 4, 3, indice_key="k")(x, target=x)
    with pytest.raises(NotImplementedError, match="MaskSplitImplicitGemm"):
        spconv.SubMConv3d(4, 4, 3, algo=ConvAlgo.MaskSplitImplicitGemm)(x, target=x)
    x.force_algo = ConvAlgo.MaskSplitImplicitGemm
    with pytest.raises(NotImplementedError, match="MaskSplitImplicitGemm"):
        subm(x, target=x)
    x.force_algo = None
    with pytest.raises(NotImplementedError, match="kernel volume <= 128"):
        spconv.SubMConv3d(4, 4, 7)(x, target=x)
    # a record of a conv onto given coordinates: refused by SubM / strided layers, and by a target layer whose
    # geometry differs
    rec = ImplicitGemmIndiceData(x.indices, x.indices, *([None] * 7), spatial_shape=[8, 8, 8],
                                 out_spatial_shape=[8, 8, 8], ksize=[3] * 3, stride=[1] * 3, padding=[1] * 3,
                                 dilation=[1] * 3, cross=True)
    x.indice_dict = {"k": rec}
    with pytest.raises(ValueError, match="onto given coordinates"):
        subm(x)
    with pytest.raises(ValueError, match="onto given coordinates"):
        spconv.SparseConv3d(4, 4, 3, 2, 1, indice_key="k")(x)
    with pytest.raises(ValueError, match="does not match"):
        spconv.SubMConv3d(4, 4, 3, dilation=2, indice_key="k")(x, target=x)
    with pytest.raises(ValueError, match="does not match"):
        spconv.SubMConv3d(4, 4, 3, indice_key="k")(_tensor([8, 8, 8], rows=7), target=x)
    # same geometry and row counts, but other coordinate tensors (padded tensors all share their row counts)
    with pytest.raises(ValueError, match="does not match"):
        spconv.SubMConv3d(4, 4, 3, indice_key="k")(_tensor([8, 8, 8], seed=1), target=x)
    other = _tensor([8, 8, 8], seed=2)
    other.indice_dict = {"k": rec}
    with pytest.raises(ValueError, match="does not match"):
        spconv.SubMConv3d(4, 4, 3, indice_key="k")(x, target=other)
