"""Numpy restatement of ``functional.sparse_add``: the first-touch union in visit order and the fp32 sum of
every output row's visited rows in visit order.  The reference for tests/test_sparse_add_*.py."""
from typing import List, Sequence, Tuple

import numpy as np


def visit_order(rows: Sequence[int]) -> List[int]:
    """The largest operand first (ties: the earliest), then the others in argument order."""
    largest = 0
    for i, r in enumerate(rows):
        if r > rows[largest]:
            largest = i
    return [largest] + [i for i in range(len(rows)) if i != largest]


def union(indices: Sequence[np.ndarray], batch_size: int, spatial_shape: Sequence[int]
          ) -> Tuple[np.ndarray, np.ndarray]:
    """Operands' coordinates in visit order -> ``(out_inds [M, ndim+1], dst [sum N])``: every distinct in-range
    coordinate once, ranked by the first visited row that carries it; ``dst[g]`` = output row of visited row
    ``g`` or -1 when its batch index or coordinate is out of range."""
    ndim = len(spatial_shape)
    cat = np.concatenate([np.asarray(i, dtype=np.int64).reshape(-1, ndim + 1) for i in indices], 0)
    shape = np.array([batch_size, *spatial_shape], dtype=np.int64)
    valid = np.all((cat >= 0) & (cat < shape), axis=1)
    strides = np.ones(ndim + 1, dtype=np.int64)
    for a in range(ndim - 1, -1, -1):
        strides[a] = strides[a + 1] * shape[a + 1]
    keys = (cat * strides).sum(1)
    dst = np.full(cat.shape[0], -1, dtype=np.int64)
    rank = {}
    out = []
    for g in np.flatnonzero(valid):
        k = int(keys[g])
        r = rank.get(k)
        if r is None:
            r = rank[k] = len(out)
            out.append(cat[g])
        dst[g] = r
    out_inds = np.array(out, dtype=np.int32).reshape(-1, ndim + 1)
    return out_inds, dst.astype(np.int32)


def sum_rows(features: Sequence[np.ndarray], dst: np.ndarray, m: int) -> np.ndarray:
    """``out [M, C]`` float32: per output row, the float32 sum (from 0) of its visited rows in visit order."""
    cat = np.concatenate([np.asarray(f, dtype=np.float32) for f in features], 0)
    acc = np.zeros((m, cat.shape[1]), dtype=np.float32)
    keep = dst >= 0
    np.add.at(acc, dst[keep].astype(np.int64), cat[keep])      # unbuffered: in index order, one row at a time
    return acc


def gradients(dout: np.ndarray, dst: np.ndarray, rows: Sequence[int]) -> List[np.ndarray]:
    """Per visited operand: ``din[i] = dout[dst[g]]`` or 0 for a dropped row."""
    full = np.zeros((dst.shape[0], dout.shape[1]), dtype=dout.dtype)
    keep = dst >= 0
    full[keep] = dout[dst[keep]]
    return np.split(full, np.cumsum(rows)[:-1], 0)


def sparse_add(indices: Sequence[np.ndarray], features: Sequence[np.ndarray], batch_size: int,
               spatial_shape: Sequence[int]):
    """Operands in ARGUMENT order -> ``(out_inds, out_f32, dst, visit)``; ``dst`` is in visit order."""
    visit = visit_order([len(f) for f in features])
    out_inds, dst = union([indices[i] for i in visit], batch_size, spatial_shape)
    out = sum_rows([features[i] for i in visit], dst, out_inds.shape[0])
    return out_inds, out, dst, visit
