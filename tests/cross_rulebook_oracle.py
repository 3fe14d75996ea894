"""Numpy restatement of the rulebook onto given output coordinates (``spx_cross_rulebook_all``).

Source rows ``x`` (grid ``in_dims``) and target rows ``t`` (grid ``out_dims``), ``batch`` samples:
  * a source row is usable when it lies below ``num_valid_x``, its batch is in ``[0, batch)`` and every
    coordinate is inside ``in_dims``; the lowest usable row wins a duplicated coordinate;
  * a target row is active under the same conditions against ``num_valid_t`` and ``out_dims``, and when no lower
    active row has its coordinate;
  * per axis, the forward relation of the layer takes input ``c`` through tap ``r`` to output ``o``: regular
    ``o = (c + p - r d) / s`` when exact, transposed ``o = c s - p + r d``.  The rulebook uses its inverse from
    the output side: regular ``c = o s - p + r d``, transposed ``c = (o + p - r d) / s`` when exact; valid iff
    ``0 <= c < in_dims``.  SubM geometry is stride 1 with ``p = (k // 2) d``;
  * ``pair_fwd[k][o] = i`` for the usable row i at that c, ``pair_bwd[k][i] = o`` for every such pair, masks with
    bit ``k % 32`` of word ``k // 32`` set per entry, argsorts the stable ascending sort of the masks (word 0 most
    significant), as ``oracle.implicit_gemm_tables``.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from tests.conv_ref import linear_keys, offset_taps


def forward_relation(c: np.ndarray, r: np.ndarray, stride, padding, dilation, transposed: bool):
    """(o, exact) of input coordinates ``c [n, ndim]`` through taps ``r [ndim]``; ``exact`` is False where a regular
    conv's division by the stride leaves a remainder."""
    s, p, d = (np.asarray(v, np.int64) for v in (stride, padding, dilation))
    if transposed:
        return c * s - p + r * d, np.ones(c.shape, bool)
    h = c + p - r * d
    return np.floor_divide(h, s), (h % s) == 0


def inverse_relation(o: np.ndarray, r: np.ndarray, stride, padding, dilation, transposed: bool):
    """(c, exact): the input coordinates that outputs ``o [n, ndim]`` read through taps ``r [ndim]``."""
    s, p, d = (np.asarray(v, np.int64) for v in (stride, padding, dilation))
    if transposed:
        h = o + p - r * d
        return np.floor_divide(h, s), (h % s) == 0
    return o * s - p + r * d, np.ones(o.shape, bool)


def usable_rows(indices: np.ndarray, num_valid: Optional[int], batch: int, dims: Sequence[int]) -> np.ndarray:
    """bool [rows]: below num_valid, batch in range, every coordinate inside dims (duplicates not considered)."""
    indices = np.asarray(indices, np.int64)
    rows = indices.shape[0]
    nv = rows if num_valid is None else min(max(int(num_valid), 0), rows)
    ok = (np.arange(rows) < nv) & (indices[:, 0] >= 0) & (indices[:, 0] < batch)
    for a, dim in enumerate(dims):
        ok &= (indices[:, a + 1] >= 0) & (indices[:, a + 1] < dim)
    return ok


def _first_rows(indices, ok, dims):
    """(sorted unique keys, lowest usable row of each) over the usable rows."""
    rows = np.nonzero(ok)[0]
    keys = linear_keys(np.asarray(indices, np.int64)[rows], dims)
    ukeys, first = np.unique(keys, return_index=True)
    return ukeys, rows[first]


def sort_masks(mask: np.ndarray, do_sort: bool = True):
    n, words = mask.shape
    if not do_sort:
        return mask.copy(), np.arange(n, dtype=np.int32)
    order = np.arange(n)
    for w in range(words - 1, -1, -1):
        order = order[np.argsort(mask[order, w], kind="stable")]
    return mask[order].copy(), order.astype(np.int32)


def cross_tables(src, tgt, batch: int, in_dims, out_dims, ksize, stride, padding, dilation, transposed: bool,
                 num_valid_src: Optional[int] = None, num_valid_tgt: Optional[int] = None, do_sort: bool = True):
    src = np.asarray(src, np.int64)
    tgt = np.asarray(tgt, np.int64)
    n, m = src.shape[0], tgt.shape[0]
    kv = int(np.prod(ksize))
    words = (kv + 31) // 32
    skeys, srows = _first_rows(src, usable_rows(src, num_valid_src, batch, in_dims), in_dims)
    tok = usable_rows(tgt, num_valid_tgt, batch, out_dims)
    active = np.zeros(m, bool)
    active[_first_rows(tgt, tok, out_dims)[1]] = True
    pair_fwd = np.full((kv, m), -1, np.int32)
    pair_bwd = np.full((kv, n), -1, np.int32)
    mask_fwd = np.zeros((m, words), np.uint32)
    mask_bwd = np.zeros((n, words), np.uint32)
    o_rows = np.nonzero(active)[0]
    taps = offset_taps(ksize)
    dims = np.asarray(in_dims, np.int64)
    for k in range(kv):
        c, exact = inverse_relation(tgt[o_rows, 1:], taps[k], stride, padding, dilation, transposed)
        valid = np.all(exact & (c >= 0) & (c < dims), axis=1)
        rows = o_rows[valid]
        if not len(rows) or not len(skeys):
            continue
        q = linear_keys(np.concatenate([tgt[rows, :1], c[valid]], 1), in_dims)
        pos = np.minimum(np.searchsorted(skeys, q), len(skeys) - 1)
        hit = skeys[pos] == q
        o, i = rows[hit], srows[pos[hit]]
        pair_fwd[k, o] = i
        pair_bwd[k, i] = o
        bit = np.uint32(1 << (k % 32))
        mask_fwd[o, k // 32] |= bit
        mask_bwd[i, k // 32] |= bit
    mf, af = sort_masks(mask_fwd, do_sort)
    mb, ab = sort_masks(mask_bwd, do_sort)
    return {"pair_fwd": pair_fwd, "pair_bwd": pair_bwd, "mask_fwd_unsorted": mask_fwd, "mask_bwd_unsorted": mask_bwd,
            "mask_fwd": mf, "mask_bwd": mb, "argsort_fwd": af, "argsort_bwd": ab, "active": active}
