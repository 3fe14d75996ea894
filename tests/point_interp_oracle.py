"""numpy restatement of VoxelPointInterpolator (csrc/point_interp.cu, DESIGN §2.5k).

`plan` / `forward` / `backward` follow the contract's float32 operation sequence, one IEEE rounding per operation
(numpy float32 arithmetic never contracts to an FMA), so their results equal the kernels' bit for bit.  `*_f64` do
the same in float64 for the accuracy checks."""
import numpy as np


def _keys(b, coords, shape):
    k = np.asarray(b, np.int64).copy()
    for a in range(len(shape)):
        k = k * int(shape[a]) + coords[:, a]
    return k


def usable_rows(indices, shape, batch_size, num_valid=None):
    """(sorted keys, their rows): every usable row's coordinate key (batch outermost, row-major) and the lowest
    usable row with it"""
    indices = np.asarray(indices, np.int64).reshape(-1, len(shape) + 1)
    rows = indices.shape[0]
    m = rows if num_valid is None else min(max(int(num_valid), 0), rows)
    c = indices[:m]
    ok = (c[:, 0] >= 0) & (c[:, 0] < batch_size)
    for a in range(len(shape)):
        ok &= (c[:, a + 1] >= 0) & (c[:, a + 1] < shape[a])
    r = np.nonzero(ok)[0]
    keys = _keys(c[r, 0], c[r, 1:], shape)
    keys, first = np.unique(keys, return_index=True)       # first occurrence in ascending row order
    return keys, r[first]


def corners(ndim, mode):
    return 1 if mode == "nearest" else 1 << ndim


def plan(indices, shape, batch_size, num_valid, pos, batch_ids, mode="trilinear", normalize=True, dtype=np.float32):
    """(index [P, K] int32, weight [P, K] dtype)"""
    f = dtype
    pos = np.asarray(pos, np.float32).astype(f)
    bids = np.asarray(batch_ids, np.int64)
    p, ndim = pos.shape[0], len(shape)
    k = corners(ndim, mode)
    tkeys, trows = usable_rows(indices, shape, batch_size, num_valid)
    with np.errstate(invalid="ignore"):
        keep = (bids >= 0) & (bids < batch_size)
        for a in range(ndim):
            # on the float, before any conversion: NaN fails both comparisons, +-inf one of them
            keep &= (pos[:, a] >= -1) & (pos[:, a].astype(np.float64) < shape[a])
    safe = np.where(keep[:, None], pos, f(0))
    base = np.floor(safe)
    frac = (safe - base).astype(f)
    base = base.astype(np.int64)
    index = np.full((p, k), -1, np.int32)
    w = np.zeros((p, k), f)
    one = f(1)
    for j in range(k):
        wj = None
        coord = np.empty((p, ndim), np.int64)
        for a in range(ndim):
            bit = (frac[:, a] >= f(0.5)).astype(np.int64) if mode == "nearest" else np.full(p, (j >> a) & 1)
            coord[:, a] = base[:, a] + bit
            if mode != "nearest":
                fa = np.where(bit == 1, frac[:, a], (one - frac[:, a]).astype(f)).astype(f)
                wj = fa if wj is None else (wj * fa).astype(f)
        if wj is None:
            wj = np.ones(p, f)
        live = keep.copy()
        for a in range(ndim):
            live &= (coord[:, a] >= 0) & (coord[:, a] < shape[a])
        q = np.nonzero(live)[0]
        key = _keys(bids[q], coord[q], shape)
        at = np.minimum(np.searchsorted(tkeys, key), max(tkeys.size - 1, 0))
        hit = tkeys[at] == key if tkeys.size else np.zeros(q.size, bool)
        index[q[hit], j] = trows[at[hit]]
        w[:, j] = np.where(index[:, j] >= 0, wj, f(0))
    if normalize:
        s = np.zeros(p, f)
        for j in range(k):
            s = np.where(index[:, j] >= 0, (s + w[:, j]).astype(f), s)
        d = (s + f(1e-8)).astype(f)
        for j in range(k):
            w[:, j] = np.where(index[:, j] >= 0, (w[:, j] / d).astype(f), f(0))
    return index, w


def forward(x, index, weight, dtype=np.float32):
    """y [P, C]: the found corners in ascending j, (y + w * x) per step"""
    f = dtype
    x = np.asarray(x).astype(f)
    p, k = index.shape
    y = np.zeros((p, x.shape[1]), f)
    for j in range(k):
        hit = index[:, j] >= 0
        prod = (weight[hit, j].astype(f)[:, None] * x[index[hit, j]]).astype(f)
        y[hit] = (y[hit] + prod).astype(f)
    return y


def backward(dy, index, weight, rows, dtype=np.float32):
    """dx [rows, C]: per row, its entries e = p * K + j in ascending e, (dx + w_e * dy[p]) per step"""
    f = dtype
    dy = np.asarray(dy).astype(f)
    p, k = index.shape
    flat = index.reshape(-1).astype(np.int64)
    wflat = weight.reshape(-1).astype(f)
    dx = np.zeros((rows, dy.shape[1]), f)
    e = np.nonzero(flat >= 0)[0]                          # ascending
    e = e[np.argsort(flat[e], kind="stable")]             # grouped by row, ascending e inside a row
    r = flat[e]
    if e.size == 0:
        return dx
    start = np.r_[0, np.nonzero(np.diff(r))[0] + 1]
    rank = np.arange(e.size) - np.repeat(start, np.diff(np.r_[start, e.size]))
    for t in range(int(rank.max()) + 1):
        sel = rank == t
        prod = (wflat[e[sel]][:, None] * dy[e[sel] // k]).astype(f)
        dx[r[sel]] = (dx[r[sel]] + prod).astype(f)
    return dx


def plan_f64(*args, **kw):
    return plan(*args, **kw, dtype=np.float64)


def forward_f64(x, index, weight):
    return forward(x, index, weight, np.float64)


def backward_f64(dy, index, weight, rows):
    return backward(dy, index, weight, rows, np.float64)
