"""Pooling kernels (``csrc/pool.cu``) against exact references (``tests/pool_oracle.py``).

Inputs lie on a grid every operand dtype holds exactly, so each fp32 sum the kernels form is exact and
every expected value is one stated rounding of an exact value: the outputs are compared bit for bit.
Kernel-level cases call ``spx_indice_pool_fwd/bwd`` directly on NaN-filled outputs, so a row the kernel
never writes fails; module-level cases run the pooling modules against the oracle's rulebook."""
import numpy as np
import pytest
import torch

from tests import pool_oracle as po

pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "i8": torch.int8}


def _lib():
    from spconv_b200 import _cabi
    return _cabi.load()


def _code(dtype):
    from spconv_b200.pytorch import ops
    return ops._DTYPE_CODE[dtype]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _filled(shape, dtype, dev):
    # NaN for floats; int8 rows get 127, a value no int8 case below can produce
    return torch.full(shape, 127 if dtype == torch.int8 else float("nan"), dtype=dtype, device=dev)


def _table_view(table, dev, pad, rng):
    """``table`` on the device as a view whose row stride exceeds its row count; the padding holds
    valid row indices, so a kernel that ignores the stride reads wrong entries"""
    if pad == 0:
        return torch.from_numpy(np.ascontiguousarray(table)).to(dev)
    kv, m = table.shape
    base = np.empty((kv, m + pad), np.int32)
    base[:, :m] = table
    base[:, m:] = rng.integers(0, max(int(table.max()) + 1, 1), size=(kv, pad))
    t = torch.from_numpy(base).to(dev)[:, :m]
    assert t.stride(0) == m + pad
    return t


def _features(rng, n, c, dtype, ties=False):
    """grid values on the device (int8: integers in [-127, 126]) and their float64 copy"""
    if dtype == torch.int8:
        v = rng.integers(-127, 127, size=(n, c)).astype(np.float64)
    elif ties:
        v = rng.choice(np.array([-1.0, -0.5, -0.0, 0.0, 0.25, 1.0]), size=(n, c))
    else:
        v = po.exact_values(rng, (n, c))
    if dtype == torch.int8:
        t = torch.from_numpy(v.astype(np.int8))
    else:
        t = po.to_dtype(v, dtype)
    return t, v


def _fwd(mode, x, table, n_out, count_out=None):
    out = _filled((n_out, x.shape[1]), x.dtype, x.device)
    rc = _lib().spx_indice_pool_fwd(mode, x.data_ptr(), out.data_ptr(), table.data_ptr(), table.stride(0),
                                    table.shape[0], n_out, x.shape[1], _code(x.dtype),
                                    None if count_out is None else count_out.data_ptr(), _stream())
    assert rc == 0, rc
    return out


def _bwd(mode, x, y, dy, table, n_in, count=None):
    din = _filled((n_in, dy.shape[1]), dy.dtype, dy.device)
    rc = _lib().spx_indice_pool_bwd(mode, None if x is None else x.data_ptr(), None if y is None else y.data_ptr(),
                                    dy.data_ptr(), din.data_ptr(), table.data_ptr(), table.stride(0), table.shape[0],
                                    n_in, dy.shape[1], _code(dy.dtype), None if count is None else count.data_ptr(),
                                    _stream())
    assert rc == 0, rc
    return din


def _assert_bits(got, want, what):
    g, w = po.bits(got), po.bits(want)
    bad = np.argwhere(g != w)
    assert bad.size == 0, (f"{what}: {len(bad)} of {g.size} elements differ; first at {bad[0].tolist()}: "
                           f"got {got.cpu()[tuple(bad[0])].item()!r} want {want[tuple(bad[0])].item()!r}")


# kernel level: (dtype, channels, kv, n_in, n_out, table padding)
SHAPES = [
    ("f32", 4, 27, 300, 200, 0),          # one 16-byte chunk per row
    ("f32", 1024, 8, 90, 40, 5),          # 256 chunks per row
    ("f32", 12, 1, 50, 50, 0),
    ("f32", 4, 343, 900, 700, 3),
    ("f16", 8, 27, 500, 333, 7),
    ("f16", 24, 125, 400, 301, 0),
    ("bf16", 8, 343, 800, 600, 0),
    ("bf16", 16, 27, 60, 1, 2),           # a single output row
    ("i8", 16, 27, 400, 300, 1),
    ("i8", 48, 125, 300, 257, 0),
    ("f32", 8, 4096, 5000, 4099, 0),      # the largest kernel volume; rows * chunks = 8198, not a multiple of 256
]


@pytest.mark.parametrize("dt,c,kv,n_in,n_out,pad", SHAPES)
@pytest.mark.parametrize("mode", [0, 1])
def test_max_pool_kernel_bit_exact(mode, dt, c, kv, n_in, n_out, pad, cuda_dev):
    dtype = DTYPES[dt]
    rng = np.random.default_rng(kv * 7 + c + mode)
    fwd, bwd = po.random_tables(rng, kv, n_in, n_out, p_empty=0.5, empty_rows=range(0, n_out, 9))
    x, xv = _features(rng, n_in, c, dtype, ties=(dt != "i8" and kv <= 343))
    if dtype != torch.int8 and dt == "f32":
        x.view(-1)[::37] = float("nan")                  # NaN never wins
        xv = x.double().numpy()
    want = po.max_pool(xv, fwd, zero_floor=(mode == 1), low=po.lowest(dtype))
    want_t = torch.from_numpy(want.astype(np.int8)) if dtype == torch.int8 else po.to_dtype(want, dtype)
    got = _fwd(mode, x.to(cuda_dev), _table_view(fwd, cuda_dev, pad, rng), n_out)
    _assert_bits(got, want_t, f"max mode {mode}")
    empty = (fwd < 0).all(axis=0)
    assert empty.any()
    if mode == 0 and dtype != torch.int8:
        assert (got[torch.from_numpy(empty).to(cuda_dev)] == po.lowest(dtype)).all()
    if dtype == torch.int8 or kv == 4096:
        return                                             # no int8 backward; the 4096 case is forward only
    # backward against the forward result: every tied input (-0 ties +0) receives dout
    dy, dyv = _features(rng, n_out, c, dtype)
    din_want = po.max_pool_backward(xv, want_t.double().numpy(), dyv, bwd)
    din = _bwd(0, x.to(cuda_dev), want_t.to(cuda_dev), dy.to(cuda_dev), _table_view(bwd, cuda_dev, pad, rng), n_in)
    _assert_bits(din, po.to_dtype(din_want, dtype), f"max backward mode {mode}")


@pytest.mark.parametrize("dt,c,kv,n_in,n_out,pad", [s for s in SHAPES if s[0] != "i8" and s[2] <= 343])
def test_avg_pool_kernel_bit_exact(dt, c, kv, n_in, n_out, pad, cuda_dev):
    dtype = DTYPES[dt]
    rng = np.random.default_rng(kv * 5 + c)
    fwd, bwd = po.random_tables(rng, kv, n_in, n_out, p_empty=0.4, empty_rows=range(1, n_out, 11))
    x, xv = _features(rng, n_in, c, dtype)
    s, count = po.avg_pool(xv, fwd)
    mean32 = po.avg_pool_fp32(s, count)
    cnt = torch.full((n_out,), -5, dtype=torch.int32, device=cuda_dev)
    got = _fwd(2, x.to(cuda_dev), _table_view(fwd, cuda_dev, pad, rng), n_out, cnt)
    assert np.array_equal(cnt.cpu().numpy(), count)
    want = torch.from_numpy(mean32).to(dtype)
    _assert_bits(got, want, "mean")
    if dtype != torch.float32:                                  # within one output ulp of the fp64 mean
        exact = s / np.maximum(count, 1)[:, None]
        g = got.double().cpu().numpy()
        ulp = np.abs(torch.from_numpy(exact.astype(np.float32)).to(dtype).double().numpy()) * 2.0 ** -(
            10 if dtype == torch.float16 else 7)
        assert (np.abs(g - exact) <= np.maximum(ulp, 2.0 ** -24)).all()
    dy, dyv = _features(rng, n_out, c, dtype)
    din = _bwd(2, None, None, dy.to(cuda_dev), _table_view(bwd, cuda_dev, pad, rng), n_in, cnt)
    _assert_bits(din, po.to_dtype(po.avg_pool_backward(dyv, bwd, count), dtype), "mean backward")


def test_avg_pool_fp32_divides_like_the_reference(cuda_dev):
    """5 / 3 = 1.6666666269 in fp32; multiplying by the reciprocal gives 1.6666667461.  Sums of grid values
    over 3 neighbours hit the difference for about one row in three."""
    rng = np.random.default_rng(3)
    n_out = 4096
    fwd, _ = po.random_tables(rng, 3, 3 * n_out, n_out, p_empty=0.0)
    x, xv = _features(rng, 3 * n_out, 4, torch.float32)
    x[[0, 4, 8], 0] = torch.tensor([2.0, 2.0, 1.0])
    fwd[:, 0] = [0, 4, 8]                                       # output row 0, channel 0: (2 + 2 + 1) / 3
    xv = x.double().numpy()
    s, count = po.avg_pool(xv, fwd)
    got = _fwd(2, x.to(cuda_dev), torch.from_numpy(fwd).to(cuda_dev), n_out)
    assert got[0, 0].item() == np.float32(5) / np.float32(3)
    _assert_bits(got, torch.from_numpy(po.avg_pool_fp32(s, count)), "mean fp32")


def test_max_pool_kernel_two_million_rows(cuda_dev):
    rng = np.random.default_rng(9)
    n = 2_000_000
    fwd, _ = po.random_tables(rng, 8, n, n, p_empty=0.3)
    x, xv = _features(rng, n, 4, torch.float32)
    got = _fwd(0, x.to(cuda_dev), torch.from_numpy(fwd).to(cuda_dev), n)
    _assert_bits(got, po.to_dtype(po.max_pool(xv, fwd, low=po.lowest(torch.float32)), torch.float32), "max 2M rows")


def test_pool_ops_refuse_partial_chunks(cuda_dev):
    from spconv_b200.pytorch import ops
    t = torch.zeros((1, 4), dtype=torch.int32, device=cuda_dev)
    for c, dtype in ((3, torch.float32), (4, torch.float16), (12, torch.bfloat16)):
        with pytest.raises(RuntimeError, match="multiple of 16 bytes"):
            ops.indice_maxpool_implicit_gemm(torch.zeros((4, c), dtype=dtype, device=cuda_dev), t, 4)
    with pytest.raises(RuntimeError, match="kernel volume 4097"):
        ops.indice_maxpool_implicit_gemm(torch.zeros((4, 4), device=cuda_dev),
                                         torch.zeros((4097, 4), dtype=torch.int32, device=cuda_dev), 4)


# ---------------------------------------------------------------------------- modules
def _module_case(oracle, rng, shape, batch, pts, c, ksize, stride, padding, dilation, subm):
    from tests.util import random_cloud
    _, inds = random_cloud(rng, shape, [pts] * batch, 1)
    nd = len(shape)
    o, pairs, num = oracle.get_indice_pairs(inds, batch, shape, ksize, stride, padding, dilation, [0] * nd, subm)
    tabs = oracle.implicit_gemm_tables(pairs, num, inds.shape[0], o.shape[0], subm)
    return inds, o, tabs


MODULE_CASES = [
    # (ndim, shape, kernel, stride, padding, dilation, subm, dtype, channels)
    (1, [3000], 3, 2, 1, 1, False, "f32", 8),
    (2, [30, 34], 3, 2, 1, 2, False, "f16", 16),
    (3, [18, 20, 22], 3, 2, 1, 1, False, "bf16", 8),
    (3, [18, 20, 22], 2, 2, 0, 1, False, "f32", 4),
    (3, [16, 17, 18], 3, 1, 1, 1, True, "f16", 8),
    (4, [6, 7, 8, 9], 3, 2, 1, 1, False, "f32", 4),
    (3, [24, 24, 24], 7, 2, 3, 1, False, "f32", 4),     # kv = 343: the Native path
]


@pytest.mark.parametrize("nd,shape,k,s,p,d,subm,dt,c", MODULE_CASES)
def test_max_pool_modules(nd, shape, k, s, p, d, subm, dt, c, oracle, cuda_dev):
    import spconv_b200.pytorch as spconv
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch.pool import SparseMaxPool
    dtype = DTYPES[dt]
    rng = np.random.default_rng(nd * 100 + k)
    ks, st, pd, dl = [k] * nd, [s] * nd, [p] * nd, [d] * nd
    inds, o, tabs = _module_case(oracle, rng, shape, 2, 700 if nd < 4 else 500, c, ks, st, pd, dl, subm)
    x, xv = _features(rng, inds.shape[0], c, dtype, ties=True)
    if subm:
        pool = SparseMaxPool(nd, k, 1, p, d, subm=True)
    else:
        pool = getattr(spconv, f"SparseMaxPool{nd}d")(k, s, p, d)
    pool.train(True)
    native = k ** nd > 128
    assert (pool.algo == ConvAlgo.Native) == native
    xf = x.to(cuda_dev).requires_grad_(True)
    y = pool(spconv.SparseConvTensor(xf, torch.from_numpy(inds).to(cuda_dev), shape, 2))
    assert np.array_equal(y.indices.cpu().numpy(), o)
    want = po.max_pool(xv, tabs["pair_fwd"], zero_floor=native, low=po.lowest(dtype))
    want_t = po.to_dtype(want, dtype)
    _assert_bits(y.features, want_t, "module max")
    dy, dyv = _features(rng, o.shape[0], c, dtype)
    y.features.backward(dy.to(cuda_dev))
    din_want = po.max_pool_backward(xv, want_t.double().numpy(), dyv, tabs["pair_bwd"])
    _assert_bits(xf.grad, po.to_dtype(din_want, dtype), "module max backward")


AVG_CASES = [
    (1, [3000], 3, 2, 1, 1, "f32", 8),
    (2, [30, 34], 3, 2, 1, 1, "f32", 4),
    (2, [30, 34], 2, 1, 0, 2, "f16", 8),
    (3, [18, 20, 22], 3, 2, 1, 1, "f32", 4),
    (3, [18, 20, 22], 3, 3, 0, 1, "bf16", 16),
]


@pytest.mark.parametrize("nd,shape,k,s,p,d,dt,c", AVG_CASES)
def test_avg_pool_modules(nd, shape, k, s, p, d, dt, c, oracle, cuda_dev):
    import spconv_b200.pytorch as spconv
    dtype = DTYPES[dt]
    rng = np.random.default_rng(nd * 10 + k + s)
    ks, st, pd, dl = [k] * nd, [s] * nd, [p] * nd, [d] * nd
    inds, o, tabs = _module_case(oracle, rng, shape, 2, 600, c, ks, st, pd, dl, False)
    x, xv = _features(rng, inds.shape[0], c, dtype)
    pool = getattr(spconv, f"SparseAvgPool{nd}d")(k, s, p, d)
    pool.train(True)
    xf = x.to(cuda_dev).requires_grad_(True)
    y = pool(spconv.SparseConvTensor(xf, torch.from_numpy(inds).to(cuda_dev), shape, 2))
    assert np.array_equal(y.indices.cpu().numpy(), o)
    s_, count = po.avg_pool(xv, tabs["pair_fwd"])
    _assert_bits(y.features, torch.from_numpy(po.avg_pool_fp32(s_, count)).to(dtype), "module mean")
    dy, dyv = _features(rng, o.shape[0], c, dtype)
    y.features.backward(dy.to(cuda_dev))
    _assert_bits(xf.grad, po.to_dtype(po.avg_pool_backward(dyv, tabs["pair_bwd"], count), dtype), "module mean bwd")


# ---------------------------------------------------------------------------- global pool rearrange
def _check_rearrange(coords, batch, cuda_dev, oracle=None):
    from spconv_b200.pytorch import ops
    oi, cnt = ops.global_pool_rearrange(torch.from_numpy(coords).to(cuda_dev), batch)
    rows, counts = po.global_pool_rearrange(coords, batch)
    assert np.array_equal(cnt.cpu().numpy(), counts)
    oi = oi.cpu().numpy()
    for b in range(batch):
        assert np.array_equal(oi[b, :counts[b]], rows[b]), b
    if oracle is not None:                     # the reference's own loop (valid batch indices only)
        r_oi, r_cnt = oracle.global_pool_rearrange(coords, batch)
        assert np.array_equal(r_cnt, counts)
        for b in range(batch):
            assert np.array_equal(oi[b, :counts[b]], r_oi[b, :r_cnt[b]])


@pytest.mark.parametrize("row_ints", [2, 4, 5])
def test_global_pool_rearrange_interleaved(row_ints, oracle, cuda_dev):
    rng = np.random.default_rng(row_ints)
    n = 100_003
    coords = rng.integers(0, 50, size=(n, row_ints)).astype(np.int32)
    coords[:, 0] = rng.choice(np.array([0, 1, 3, 4]), size=n, p=[0.1, 0.4, 0.3, 0.2])   # sample 2 is empty
    _check_rearrange(coords, 5, cuda_dev, oracle)


def test_global_pool_rearrange_out_of_range_batch(cuda_dev):
    rng = np.random.default_rng(5)
    coords = rng.integers(0, 9, size=(5000, 4)).astype(np.int32)
    coords[::3, 0] = -1
    coords[1::7, 0] = 3
    coords[2::11, 0] = 1 << 30
    _check_rearrange(coords, 3, cuda_dev)
