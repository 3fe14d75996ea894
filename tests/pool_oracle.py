"""Exact references for the pooling kernels (``csrc/pool.cu``) and the point -> voxel generator
(``csrc/pointops.cu``).

The pooling tests draw their inputs from a grid that fp32, fp16 and bf16 all hold exactly (multiples
of 2^-6 in [-1, 1]).  Every fp32 sum a kernel forms is then exact, and each expected output below is
one stated rounding of an exact value, so the tests can ask for equality bit for bit.
"""
import numpy as np
import torch

GRID_STEP = 2.0 ** -6


def exact_values(rng, shape, lo=-1.0, hi=1.0, step=GRID_STEP):
    """float64 multiples of ``step`` in ``[lo, hi]``; with the defaults fp32, fp16 and bf16 hold each one."""
    k = rng.integers(int(round(lo / step)), int(round(hi / step)) + 1, size=shape)
    return k.astype(np.float64) * step


def to_dtype(a, dtype):
    """Round ``a`` once to ``dtype`` (a CPU torch tensor).  The values must be exact in fp32, so the
    conversion through fp32 that torch makes for fp16 / bf16 is a single rounding."""
    a = np.asarray(a, dtype=np.float64)
    f = a.astype(np.float32)
    assert np.array_equal(f.astype(np.float64), a, equal_nan=True), "value not exact in fp32"
    return torch.from_numpy(f).to(dtype)


def bits(t):
    """Integer view of a tensor's elements, for bit-for-bit comparisons (+0 and -0 differ, NaN == NaN)."""
    t = t.detach().cpu().contiguous()
    return t.view({4: torch.int32, 2: torch.int16, 1: torch.int8}[t.element_size()]).numpy()


def lowest(dtype):
    return float(torch.iinfo(dtype).min if dtype == torch.int8 else torch.finfo(dtype).min)


def max_pool(x, table, zero_floor=False, low=None):
    """``out[o] = max over k of x[table[k, o]]`` (entries < 0 skipped) starting from ``low`` (MODE 0) or 0
    (MODE 1, the Native pool's zero floor).  As in the reference, a candidate replaces the running max
    only when it is greater: NaN never wins and the first of two equal values (e.g. -0 then +0) stays."""
    x = np.asarray(x, dtype=np.float64)
    kv, m = table.shape
    out = np.full((m, x.shape[1]), 0.0 if zero_floor else low, dtype=np.float64)
    for k in range(kv):
        o = np.nonzero(table[k] >= 0)[0]
        cand, cur = x[table[k, o]], out[o]
        out[o] = np.where(cand > cur, cand, cur)
    return out


def max_pool_backward(x, y, dy, table_bwd):
    """``din[i] = sum over k of (x[i] == y[o]) ? dy[o] : 0`` with ``o = table_bwd[k, i]``, in fp64 (exact
    for grid-valued ``dy``): every input tied with its output's max receives the gradient."""
    x, y, dy = (np.asarray(a, dtype=np.float64) for a in (x, y, dy))
    din = np.zeros_like(x)
    for k in range(table_bwd.shape[0]):
        i = np.nonzero(table_bwd[k] >= 0)[0]
        o = table_bwd[k, i]
        din[i] += np.where(x[i] == y[o], dy[o], 0.0)
    return din


def avg_pool(x, table):
    """-> ``(exact sum [M, C] fp64, count [M] int32)`` over the valid entries of ``table[:, o]``."""
    x = np.asarray(x, dtype=np.float64)
    kv, m = table.shape
    s = np.zeros((m, x.shape[1]), dtype=np.float64)
    for k in range(kv):
        o = np.nonzero(table[k] >= 0)[0]
        s[o] += x[table[k, o]]
    return s, (table >= 0).sum(axis=0).astype(np.int32)


def avg_pool_fp32(s, count):
    """The reference's mean in fp32: ``fp32(sum) / fp32(count)``, 0 for rows with no entry."""
    s32 = np.asarray(s, dtype=np.float64).astype(np.float32)
    assert np.array_equal(s32.astype(np.float64), s), "sum not exact in fp32"
    c = np.maximum(count, 1).astype(np.float32)[:, None]
    return np.where(count[:, None] > 0, s32 / c, np.float32(0)).astype(np.float32)


def avg_pool_backward(dy, table_bwd, count):
    """``din[i] = sum over k of dy[o] * count[o]`` (the reference multiplies by the count), in fp64."""
    dy = np.asarray(dy, dtype=np.float64)
    din = np.zeros((table_bwd.shape[1], dy.shape[1]), dtype=np.float64)
    for k in range(table_bwd.shape[0]):
        i = np.nonzero(table_bwd[k] >= 0)[0]
        o = table_bwd[k, i]
        din[i] += dy[o] * count[o][:, None]
    return din


def random_tables(rng, kv, n_in, n_out, p_empty=0.3, empty_rows=()):
    """A forward table ``[kv, n_out]`` and its inverse ``[kv, n_in]``.  Each offset maps distinct outputs
    to distinct inputs (as a rulebook does), a share ``p_empty`` of the entries is -1, and the rows
    ``empty_rows`` have no entry at all."""
    assert n_out <= n_in
    fwd = np.full((kv, n_out), -1, np.int32)
    bwd = np.full((kv, n_in), -1, np.int32)
    for k in range(kv):
        src = rng.permutation(n_in)[:n_out].astype(np.int32)
        keep = rng.random(n_out) >= p_empty
        keep[list(empty_rows)] = False
        o = np.nonzero(keep)[0].astype(np.int32)
        fwd[k, o] = src[o]
        bwd[k, src[o]] = o
    return fwd, bwd


def global_pool_rearrange(coords, batch_size):
    """Rows of each sample in input order -> ``(rows per sample: list of int32 arrays, counts)``.  Rows
    whose batch index is outside ``[0, batch_size)`` belong to no sample."""
    b = np.asarray(coords)[:, 0]
    rows = [np.nonzero(b == s)[0].astype(np.int32) for s in range(batch_size)]
    return rows, np.array([len(r) for r in rows], np.int32)
