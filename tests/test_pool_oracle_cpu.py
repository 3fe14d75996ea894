"""The exact pooling and point -> voxel references of ``tests/pool_oracle.py`` and
``tests/point2voxel_oracle.py`` against the reference's own CPU code (``oracle/_ref``) on finite inputs,
plus the argument checks of ``spx_indice_pool_fwd/bwd`` (no GPU needed for either)."""
import numpy as np
import pytest

from tests import point2voxel_oracle as p2v
from tests import pool_oracle as po
from tests.util import random_cloud


def _need_ref(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref is not built")


def _lib():
    from spconv_b200 import _cabi, build
    build.build(verbose=False)
    return _cabi.load()


@pytest.mark.parametrize("k,s,p", [(3, 2, 1), (2, 2, 0), (3, 1, 1)])
def test_max_pool_helper_equals_reference_cpu_loop(k, s, p, oracle):
    """zero-floor max over pair_fwd == the reference's IndiceMaxPoolCPU::forward over compact pairs"""
    _need_ref(oracle)
    rng = np.random.default_rng(k * 10 + s)
    shape = [14, 15, 16]
    feats, inds = random_cloud(rng, shape, [700, 500], 8)
    feats = po.exact_values(rng, feats.shape).astype(np.float32)
    o, pairs, num = oracle.get_indice_pairs(inds, 2, shape, [k] * 3, [s] * 3, [p] * 3, [1] * 3, [0] * 3, False)
    tabs = oracle.implicit_gemm_tables(pairs, num, inds.shape[0], o.shape[0], False)
    got = po.max_pool(feats, tabs["pair_fwd"], zero_floor=True).astype(np.float32)
    assert np.array_equal(got, oracle.indice_maxpool(feats, pairs, num, o.shape[0]))
    dy = po.exact_values(rng, (o.shape[0], 8)).astype(np.float32)
    ref_y = oracle.indice_maxpool(feats, pairs, num, o.shape[0])
    din = po.max_pool_backward(feats, ref_y, dy, tabs["pair_bwd"]).astype(np.float32)
    assert np.array_equal(din, oracle.indice_maxpool_backward(feats, ref_y, dy, pairs, num))


VS, CR = [0.4, 0.4, 0.5], [0, -40, -3, 70.4, 40, 1]


@pytest.mark.parametrize("case", ["boundary", "uniform", "caps"])
def test_point2voxel_helper_equals_reference_cpu_generator(case, oracle):
    _need_ref(oracle)
    if case == "boundary":
        pts, mv, mp = p2v.boundary_cloud(VS, CR, 1), 100000, 4
    else:
        rng = np.random.default_rng(2)
        pts = rng.uniform([-1, -41, -4, 0], [71, 41, 2, 1], size=(20000, 4)).astype(np.float32)
        pts[::7, 1] = -0.0                                   # -0 lands in the y cell of 0
        pts[::11, 0] = np.float32(1e30)
        pts[::13, 2] = np.float32(-1e30)
        mv, mp = (50000, 5) if case == "uniform" else (700, 2)
    got = p2v.point2voxel(pts, VS, CR, mv, mp)
    want = oracle.point2voxel_ref(pts, VS, CR, mv, mp)
    for g, w, name in zip(got, want, ("voxels", "indices", "num_per_voxel", "pc_voxel_id")):
        assert np.array_equal(g, w), name
    assert (got[3] == -1).any() and got[0].shape[0] > 1


def test_point2voxel_helper_drops_non_finite_points():
    pts = np.array([[np.nan, 0.5, 0.5], [0.5, 0.5, 0.5], [np.nan] * 3, [np.inf, 0.5, 0.5], [0.5, -np.inf, 0.5],
                    [0.5, 0.5, 1.5]], np.float32)
    vox, ind, num, ids = p2v.point2voxel(pts, [1, 1, 1], [0, 0, 0, 2, 2, 2], 10, 2)
    assert ids.tolist() == [-1, 0, -1, -1, -1, 1]
    assert ind.tolist() == [[0, 0, 0], [1, 0, 0]] and num.tolist() == [1, 1]


def test_pool_abi_refuses_bad_arguments():
    """kv above 4096, channel rows that are not whole 16-byte chunks, int8 mean and int8 backward are
    refused with return code 2 before any device work"""
    from spconv_b200 import _cabi
    lib = _lib()
    assert lib.spx_indice_pool_fwd(0, None, None, None, 1, 4097, 1, 4, _cabi.SPX_F32, None, None) == 2
    assert "kernel volume 4097" in _cabi.last_error()
    assert lib.spx_indice_pool_fwd(0, None, None, None, 1, 0, 1, 4, _cabi.SPX_F32, None, None) == 2
    for c, code in ((3, _cabi.SPX_F32), (4, _cabi.SPX_F16), (12, _cabi.SPX_BF16), (8, _cabi.SPX_I8)):
        assert lib.spx_indice_pool_fwd(0, None, None, None, 1, 8, 1, c, code, None, None) == 2
        assert "multiple of 16 bytes" in _cabi.last_error()
    assert lib.spx_indice_pool_fwd(2, None, None, None, 1, 8, 1, 16, _cabi.SPX_I8, None, None) == 2
    assert "unsupported dtype" in _cabi.last_error()
    assert lib.spx_indice_pool_bwd(0, None, None, None, None, None, 1, 8, 1, 16, _cabi.SPX_I8, None, None) == 2
    assert lib.spx_indice_pool_bwd(2, None, None, None, None, None, 1, 4097, 1, 4, _cabi.SPX_F32, None, None) == 2
    assert lib.spx_indice_pool_fwd(3, None, None, None, 1, 8, 1, 4, _cabi.SPX_F32, None, None) == 2
