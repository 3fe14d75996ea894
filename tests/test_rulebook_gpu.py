"""GPU rulebook parity: bit-exact against the oracle (reference CPU order), through the C ABI.

Reference behaviour being pinned: ``SparseConvIndicesCPU`` (spconv/csrc/sparse/indices.py:1640-1778)
for the Native rulebook; SURVEY A.5 for the implicit-GEMM tables.
"""
import numpy as np
import pytest
import torch

from tests.util import check_tile_table, random_cloud, surface_cloud

pytestmark = pytest.mark.gpu

CASES = [
    # (shape, pts per sample, ksize, stride, padding, dilation, subm, transpose)
    ([64, 64, 64], [5000], [3, 3, 3], [1, 1, 1], [1, 1, 1], [1, 1, 1], True, False),     # cfg1
    ([19, 18, 17], [1500, 1500], [3, 3, 3], [1, 1, 1], [0, 0, 0], [2, 2, 2], True, False),
    ([19, 18, 17], [1500, 1500], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], False, False),
    ([19, 18, 17], [1500], [2, 2, 2], [2, 2, 2], [0, 0, 0], [1, 1, 1], False, False),
    ([19, 18, 17], [1500], [3, 3, 3], [1, 1, 1], [0, 0, 0], [2, 2, 2], False, False),
    ([19, 18, 17], [1500], [3, 3, 3], [3, 3, 3], [2, 2, 2], [1, 1, 1], False, False),
    ([19, 18, 17], [700], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], False, True),
    ([40, 50], [900, 800], [3, 3], [1, 1], [1, 1], [1, 1], True, False),                   # 2-D
    ([40, 50], [900], [3, 3], [2, 2], [1, 1], [1, 1], False, False),
    ([9, 10, 11, 12], [2000], [3, 3, 3, 3], [1, 1, 1, 1], [1] * 4, [1] * 4, True, False),  # 4-D, kv=81
    ([30, 30, 30], [3000], [3, 1, 3], [1, 1, 1], [0, 0, 0], [1, 1, 1], True, False),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{'subm' if c[6] else 'conv'}{'T' if c[7] else ''}-{len(c[0])}d-k{c[2][0]}s{c[3][0]}p{c[4][0]}d{c[5][0]}")
def test_native_rulebook_bit_exact(case, oracle, cuda_dev):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    shape, pts, ksize, stride, padding, dilation, subm, transpose = case
    rng = np.random.default_rng(484)
    _, inds = random_cloud(rng, shape, pts, 1)
    bs = len(pts)
    ndim = len(shape)
    ref_out, ref_pairs, ref_num = oracle.get_indice_pairs(inds, bs, shape, ksize, stride, padding,
                                                          dilation, [0] * ndim, subm, transpose)
    out, pairs, num = ops.get_indice_pairs(torch.from_numpy(inds).to(cuda_dev), bs, shape,
                                           ConvAlgo.Native, ksize, stride, padding, dilation,
                                           [0] * ndim, subm, transpose)
    torch.cuda.synchronize()
    assert np.array_equal(num.cpu().numpy(), ref_num), (num.cpu().numpy(), ref_num)
    assert np.array_equal(out.cpu().numpy(), ref_out)
    assert np.array_equal(pairs.cpu().numpy(), ref_pairs)


@pytest.mark.parametrize("case", CASES[:10], ids=lambda c: f"{'subm' if c[6] else 'conv'}{'T' if c[7] else ''}-{len(c[0])}d-k{c[2][0]}s{c[3][0]}p{c[4][0]}d{c[5][0]}")
@pytest.mark.parametrize("do_sort", [True, False])
def test_implicit_gemm_rulebook_bit_exact(case, do_sort, oracle, cuda_dev):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    shape, pts, ksize, stride, padding, dilation, subm, transpose = case
    rng = np.random.default_rng(50051)
    _, inds = random_cloud(rng, shape, pts, 1)
    bs, ndim = len(pts), len(shape)
    ref_out, ref_pairs, ref_num = oracle.get_indice_pairs(inds, bs, shape, ksize, stride, padding,
                                                          dilation, [0] * ndim, subm, transpose)
    tab = oracle.implicit_gemm_tables(ref_pairs, ref_num, inds.shape[0], ref_out.shape[0], subm,
                                      do_sort)
    res = ops.get_indice_pairs_implicit_gemm(torch.from_numpy(inds).to(cuda_dev), bs, shape,
                                             ConvAlgo.MaskImplicitGemm, ksize, stride, padding,
                                             dilation, [0] * ndim, subm, transpose, is_train=True,
                                             do_sort=do_sort)
    torch.cuda.synchronize()
    out_inds, _, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks = res
    assert np.array_equal(out_inds.cpu().numpy(), ref_out)
    assert np.array_equal(pair_fwd.cpu().numpy(), tab["pair_fwd"])
    assert np.array_equal(pair_bwd.cpu().numpy(), tab["pair_bwd"])
    # masks come back SORTED (thrust::sort_by_key sorts keys in place, all.py:935-1000)
    assert np.array_equal(mask_fwd[0].cpu().numpy().view(np.uint32), tab["mask_fwd"])
    assert np.array_equal(sort_fwd[0].cpu().numpy(), tab["argsort_fwd"])
    if not subm:
        assert np.array_equal(mask_bwd[0].cpu().numpy().view(np.uint32), tab["mask_bwd"])
        assert np.array_equal(sort_bwd[0].cpu().numpy(), tab["argsort_bwd"])
    assert masks[0][0] == 0xffffffff


def test_subm_inference_tables(oracle, cuda_dev):
    """is_train=False: SubM returns pair [1, kv, N] only (ops.py:469-479)."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(1)
    _, inds = random_cloud(rng, [20, 20, 20], [2000], 1)
    res = ops.get_indice_pairs_implicit_gemm(torch.from_numpy(inds).to(cuda_dev), 1, [20, 20, 20],
                                             ConvAlgo.MaskImplicitGemm, [3] * 3, [1] * 3, [1] * 3,
                                             [1] * 3, [0] * 3, True, False, is_train=False)
    assert res[3].numel() == 0
    ref_out, ref_pairs, ref_num = oracle.get_indice_pairs(inds, 1, [20] * 3, [3] * 3, [1] * 3,
                                                          [1] * 3, [1] * 3, [0] * 3, True)
    tab = oracle.implicit_gemm_tables(ref_pairs, ref_num, 2000, 2000, True)
    assert np.array_equal(res[2].cpu().numpy(), tab["pair_fwd"])


def test_large_clustered_cloud_properties(oracle, cuda_dev):
    """KITTI-shaped grid at BASELINE size: size-independent properties + oracle equality
    (the C oracle handles 100k voxels in well under a second)."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(50051)
    shape = [41, 1600, 1408]
    inds = surface_cloud(rng, shape, 100_000)
    n = inds.shape[0]
    dev_inds = torch.from_numpy(inds).to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(dev_inds, 1, shape, ConvAlgo.MaskImplicitGemm,
                                             [3] * 3, [1] * 3, [1] * 3, [1] * 3, [0] * 3, True)
    pair_fwd = res[2].cpu().numpy()
    pair_bwd = res[3].cpu().numpy()
    mask = res[4][0].cpu().numpy().view(np.uint32)[:, 0]
    argsort = res[6][0].cpu().numpy()
    kv = 27
    # symmetry of SubM pairs: pair_bwd[k] == pair_fwd[kv-1-k]
    assert np.array_equal(pair_bwd, pair_fwd[::-1])
    # centre is the identity
    assert np.array_equal(pair_fwd[kv // 2], np.arange(n))
    # involution: j = pair_fwd[k][o] >= 0  =>  pair_fwd[kv-1-k][j] == o
    for k in range(kv):
        o = np.nonzero(pair_fwd[k] >= 0)[0]
        assert np.array_equal(pair_fwd[kv - 1 - k][pair_fwd[k][o]], o)
    # masks sorted ascending, argsort a permutation, mask bits == table occupancy
    assert np.all(np.diff(mask.astype(np.int64)) >= 0)
    assert np.array_equal(np.sort(argsort), np.arange(n))
    occ = np.zeros(n, np.uint32)
    for k in range(kv):
        occ |= (pair_fwd[k] >= 0).astype(np.uint32) << np.uint32(k)
    assert np.array_equal(mask, occ[argsort])
    # and the full thing equals the oracle
    ref_out, ref_pairs, ref_num = oracle.get_indice_pairs(inds, 1, shape, [3] * 3, [1] * 3,
                                                          [1] * 3, [1] * 3, [0] * 3, True)
    tab = oracle.implicit_gemm_tables(ref_pairs, ref_num, n, n, True)
    assert np.array_equal(pair_fwd, tab["pair_fwd"])
    assert np.array_equal(argsort, tab["argsort_fwd"])
    # native compact pairs too
    out, pairs, num = ops.get_indice_pairs(dev_inds, 1, shape, ConvAlgo.Native, [3] * 3, [1] * 3,
                                           [1] * 3, [1] * 3, [0] * 3, True)
    assert np.array_equal(num.cpu().numpy(), ref_num)
    assert np.array_equal(pairs.cpu().numpy(), ref_pairs)
    pairs_per_voxel = (2 * int(ref_num.sum()) + n) / n
    assert 3.0 < pairs_per_voxel < 12.0, pairs_per_voxel   # clustered like LiDAR (fixture: 6.28)


def test_strided_large_and_int64_keys(oracle, cuda_dev):
    """nuScenes-like stride-2 rulebook + the int64-key path (volume >= 2^31)."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(7)
    shape = [41, 1440, 1440]
    inds = surface_cloud(rng, shape, 60_000)
    k, s, p, d = [3] * 3, [2] * 3, [1] * 3, [1] * 3
    ref_out, ref_pairs, ref_num = oracle.get_indice_pairs(inds, 1, shape, k, s, p, d, [0] * 3, False)
    out, pairs, num = ops.get_indice_pairs(torch.from_numpy(inds).to(cuda_dev), 1, shape,
                                           ConvAlgo.Native, k, s, p, d, [0] * 3, False)
    assert np.array_equal(out.cpu().numpy(), ref_out)
    assert np.array_equal(num.cpu().numpy(), ref_num)
    assert np.array_equal(pairs.cpu().numpy(), ref_pairs)
    # huge virtual grid -> int64 linear keys (ops.py:188-190)
    big = [2000, 2000, 2000]
    _, inds2 = random_cloud(rng, [50, 50, 50], [4000], 1)
    inds2[:, 1:] += 1900
    ref = oracle.get_indice_pairs(inds2, 1, big, [3] * 3, [1] * 3, [1] * 3, [1] * 3, [0] * 3, True)
    got = ops.get_indice_pairs(torch.from_numpy(inds2).to(cuda_dev), 1, big, ConvAlgo.Native,
                               [3] * 3, [1] * 3, [1] * 3, [1] * 3, [0] * 3, True)
    assert np.array_equal(got[2].cpu().numpy(), ref[2])
    assert np.array_equal(got[1].cpu().numpy(), ref[1])
    ref = oracle.get_indice_pairs(inds2, 1, big, k, s, p, d, [0] * 3, False)
    got = ops.get_indice_pairs(torch.from_numpy(inds2).to(cuda_dev), 1, big, ConvAlgo.Native,
                               k, s, p, d, [0] * 3, False)
    assert np.array_equal(got[0].cpu().numpy(), ref[0])
    assert np.array_equal(got[1].cpu().numpy(), ref[1])


def test_vanished_points_error(cuda_dev):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    # k=2, s=3, p=0 covers input coordinates {0,1,3,4,6,7}: a point at 2 has no output
    inds = torch.tensor([[0, 2, 2, 2]], dtype=torch.int32, device=cuda_dev)
    with pytest.raises(ValueError, match="vanished"):
        ops.get_indice_pairs(inds, 1, [8, 8, 8], ConvAlgo.Native, [2] * 3, [3] * 3, [0] * 3,
                             [1] * 3, [0] * 3, False)
    with pytest.raises(RuntimeError, match="odd ksize"):
        ops.get_indice_pairs(inds, 1, [8, 8, 8], ConvAlgo.Native, [2] * 3, [1] * 3, [0] * 3,
                             [1] * 3, [0] * 3, True)


def test_fused_subm_tile_table_matches_column_path(cuda_dev):
    """A tile table has two sources: spx_subm_rulebook_all builds it for a 3x3x3 SubM from the row-major
    copy of the pair table that the probe kernel keeps in its workspace, spx_build_tile_table from the
    column-major pair table.  Both must give identical blocks and tile masks (== per-tile OR of the
    sorted masks, the reference's mask_output_fwd with mask_width 128,
    spconv/csrc/sparse/convops.py:2180-2189)."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(5)
    shape = [24, 200, 176]
    inds = torch.from_numpy(surface_cloud(rng, shape, 9000 + 77)).to(cuda_dev)
    n = inds.shape[0]
    res = ops.get_indice_pairs_implicit_gemm(inds, 1, shape, ConvAlgo.MaskImplicitGemm, [3] * 3, [1] * 3,
                                             [1] * 3, [1] * 3, [0] * 3, True, False, is_train=True)
    pair_fwd, mask, argsort = res[2], res[4][0], res[6][0]
    cache = getattr(argsort, "_spx_tile_cache", None)
    assert cache is not None, "the fused rulebook call must leave the tile table cached on the argsort"
    assert cache[0] == ops._tile_key(pair_fwd, argsort, n)
    t_rows, m_rows = cache[1], cache[2]
    t_cols, m_cols = ops._tile_tables(pair_fwd, mask, argsort, n, 27, owner=None)
    assert torch.equal(t_rows, t_cols) and torch.equal(m_rows, m_cols)
    # blocks, tile masks, schedule records (every tile once, heaviest first, ties in ascending tile
    # order) and the zeroed scheduler scratch
    check_tile_table(t_rows.cpu().numpy(), m_rows.cpu().numpy(), pair_fwd.cpu().numpy(), mask.cpu().numpy(),
                     argsort.cpu().numpy(), n, 27, 1)


TIMER_CASES = [CASES[0], CASES[7], CASES[2],
               ([9, 10, 11, 12], [2000], [3] * 4, [2] * 4, [1] * 4, [1] * 4, False, False)]   # kv = 81: 3 mask words


@pytest.mark.parametrize("case", TIMER_CASES, ids=lambda c: f"{'subm' if c[6] else 'conv'}-{len(c[0])}d-k{c[2][0]}s{c[3][0]}")
@pytest.mark.parametrize("is_train", [True, False])
def test_timer_does_not_change_rulebook_path(case, is_train, cuda_dev):
    """With a CUDAKernelTimer enabled the MaskImplicitGemm rulebook runs the same fused native calls: the
    9-tuple and the tile tables cached on the argsorts equal those of the call without a timer, and the
    whole rulebook is one gen_*_inds region."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    from spconv_b200.pytorch.core import CUDAKernelTimer
    shape, pts, ksize, stride, padding, dilation, subm, transpose = case
    rng = np.random.default_rng(31)
    _, inds = random_cloud(rng, shape, pts, 1)
    args = (torch.from_numpy(inds).to(cuda_dev), len(pts), shape, ConvAlgo.MaskImplicitGemm, ksize, stride,
            padding, dilation, [0] * len(shape), subm, transpose)
    ref = ops.get_indice_pairs_implicit_gemm(*args, is_train=is_train)
    timer = CUDAKernelTimer(True)
    got = ops.get_indice_pairs_implicit_gemm(*args, is_train=is_train, timer=timer)
    for i in (0, 1, 2, 3):
        assert got[i].dtype == ref[i].dtype and torch.equal(got[i], ref[i]), i
    for i in (4, 5, 6, 7):
        assert len(got[i]) == len(ref[i]), i
        assert all(torch.equal(a, b) for a, b in zip(got[i], ref[i])), i
    assert len(got[8]) == len(ref[8]) and all(np.array_equal(a, b) for a, b in zip(got[8], ref[8]))
    owners = list(zip(got[6] + got[7], ref[6] + ref[7]))
    assert len(owners) == (1 if subm or not is_train else 2)
    for g, r in owners:
        gc, rc = getattr(g, "_spx_tile_cache", None), getattr(r, "_spx_tile_cache", None)
        assert gc is not None and rc is not None, "the rulebook call must leave the tile table cached on the argsort"
        assert torch.equal(gc[1], rc[1]) and torch.equal(gc[2], rc[2])
    assert list(timer.get_all_pair_time()) == ["gen_subm_inds" if subm else "gen_conv_inds"]


ZERO_CASES = [([20, 20, 20], [3] * 3), ([40, 50], [3, 3]), ([9, 10, 11, 12], [3] * 4)]


@pytest.mark.parametrize("case", ZERO_CASES, ids=lambda c: f"{len(c[0])}d-kv{int(np.prod(c[1]))}")
@pytest.mark.parametrize("is_train", [True, False])
def test_zero_row_subm_implicit_gemm_rulebook(case, is_train, cuda_dev):
    """A SubM MaskImplicitGemm rulebook of no voxels is the 9-tuple of empty tables"""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    shape, ksize = case
    ndim, kv = len(shape), int(np.prod(ksize))
    words = (kv + 31) // 32
    inds = torch.empty((0, ndim + 1), dtype=torch.int32, device=cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(inds, 1, shape, ConvAlgo.MaskImplicitGemm, ksize, [1] * ndim,
                                             [1] * ndim, [1] * ndim, [0] * ndim, True, False, is_train=is_train)
    out_inds, num, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks = res
    assert out_inds.shape == (0, ndim + 1) and out_inds.dtype == torch.int32
    assert num.shape == (kv,) and num.dtype == torch.int32 and not num.any()
    assert pair_fwd.shape == (kv, 0) and pair_fwd.dtype == torch.int32
    if is_train:
        assert pair_bwd.shape == (kv, 0) and pair_bwd.dtype == torch.int32
    else:
        assert pair_bwd.shape == (0,) and pair_bwd.dtype == torch.float32
    assert len(mask_fwd) == 1 and mask_fwd[0].shape == (0, words) and mask_fwd[0].dtype == torch.int32
    assert len(sort_fwd) == 1 and sort_fwd[0].shape == (0,) and sort_fwd[0].dtype == torch.int32
    assert mask_bwd == [] and sort_bwd == []
    assert len(masks) == 1 and masks[0].dtype == np.uint32 and masks[0].tolist() == [0xffffffff]
