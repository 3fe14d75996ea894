"""numpy restatement of PointVoxelScatter (csrc/point_scatter.cu), the reference of its tests.

Point p belongs to row ids[p] when 0 <= ids[p] < rows and is dropped otherwise.  Every reduction visits a row's
points in ascending point index:
  * sum  : a float32 accumulator starting at +0, one addition per point, in that order;
  * mean : that sum / count in float32;
  * max  : the first point that attains the maximum, a NaN counting as the maximum and -0 == +0 (so the first of
           them wins); the output is that point's value.
The sequential sums are vectorised by position within the row: step k adds the k-th point of every row that has
one, so the work is O(P) whatever the row lengths.  Features come in as float32 arrays holding the values exactly
(fp16 / bf16 widen without rounding); rounding the results to the dtype is the caller's.
"""
import numpy as np


def rows_of(ids, rows):
    ids = np.asarray(ids, np.int64)
    return np.where((ids >= 0) & (ids < rows), ids, -1)


def group(ids, rows):
    """-> (row [P] with -1 for dropped points, order: kept points sorted by row then index, offsets [rows+1], count)"""
    r = rows_of(ids, rows)
    keep = np.nonzero(r >= 0)[0]
    order = keep[np.argsort(r[keep], kind="stable")]
    count = np.bincount(r[keep], minlength=rows).astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(count)]).astype(np.int64)
    return r, order, offsets, count


def _by_position(r, order, offsets):
    """the kept points grouped by their position k within the row: a list of point arrays, k = 0, 1, .."""
    if len(order) == 0:
        return []
    pos = np.arange(len(order)) - offsets[r[order]]
    by = np.argsort(pos, kind="stable")
    bounds = np.concatenate([[0], np.cumsum(np.bincount(pos))])
    return [order[by[bounds[k]:bounds[k + 1]]] for k in range(len(bounds) - 1)]


def segment_sum(x, ids, rows):
    """float32 [rows, C]: every row's points added in ascending index to a float32 +0"""
    x = np.asarray(x, np.float32)
    r, order, offsets, count = group(ids, rows)
    acc = np.zeros((rows, x.shape[1]), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for pts in _by_position(r, order, offsets):
            acc[r[pts]] = acc[r[pts]] + x[pts]          # each row at most once per step
    return acc


def segment_mean(x, ids, rows):
    """float32 [rows, C]: segment_sum / count in float32, 0 on an empty row"""
    s = segment_sum(x, ids, rows)
    count = group(ids, rows)[3]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        m = s / np.maximum(count, 1).astype(np.float32)[:, None]
    m[count == 0] = 0
    return m.astype(np.float32)


def segment_argmax(x, ids, rows):
    """int64 [rows, C]: the winning point of every row and channel (-1 on an empty row)"""
    x = np.asarray(x, np.float32)
    r, order, offsets, count = group(ids, rows)
    c = x.shape[1]
    best = np.zeros((rows, c), np.float32)
    arg = np.full((rows, c), -1, np.int64)
    for pts in _by_position(r, order, offsets):
        rr = r[pts]
        v, bv, ba = x[pts], best[rr], arg[rr]
        vn, bn = np.isnan(v), np.isnan(bv)
        with np.errstate(invalid="ignore"):
            beats = (ba < 0) | (vn & ~bn) | (~vn & ~bn & (v > bv))   # later points never win a tie
        best[rr] = np.where(beats, v, bv)
        arg[rr] = np.where(beats, pts[:, None], ba)
    return arg


def take_argmax(x, arg):
    """out[r, c] = x[arg[r, c], c], 0 where arg is -1 (x in any dtype: the values are copied)"""
    x = np.asarray(x)
    out = np.zeros(arg.shape, x.dtype)
    ok = arg >= 0
    out[ok] = x[arg[ok], np.nonzero(ok)[1]]
    return out


def max_grad(dy, arg, ids, rows, n):
    """dx [n, C]: dy[r, c] at the point arg[r, c], 0 elsewhere (dy in any dtype: the values are copied)"""
    dy = np.asarray(dy)
    dx = np.zeros((n, dy.shape[1]), dy.dtype)
    ok = arg >= 0
    rr, cc = np.nonzero(ok)
    dx[arg[ok], cc] = dy[rr, cc]
    return dx


def mean_grad(dy, ids, rows):
    """float32 [P, C]: dy[r] / count[r] in float32 for the points of row r, 0 for dropped points"""
    dy = np.asarray(dy, np.float32)
    r, _, _, count = group(ids, rows)
    dx = np.zeros((len(r), dy.shape[1]), np.float32)
    ok = r >= 0
    dx[ok] = dy[r[ok]] / count[r[ok]].astype(np.float32)[:, None]
    return dx


def sum_grad(dy, ids, rows):
    """dx [P, C]: dy[r] for the points of row r, 0 for dropped points (dy in any dtype)"""
    dy = np.asarray(dy)
    r = rows_of(ids, rows)
    dx = np.zeros((len(r), dy.shape[1]), dy.dtype)
    ok = r >= 0
    dx[ok] = dy[r[ok]]
    return dx
