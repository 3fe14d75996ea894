"""numpy restatement of ``PointToVoxel`` (``csrc/pointops.cu``) for any number of axes.

It follows the reference's CPU generator (``Point2VoxelCPU::point_to_voxel_static``): the cell of a
point on each axis is ``floor((p - lo) / vsize)`` in fp32, voxels are numbered by their first point in
input order, voxels past ``max_voxels`` are dropped (their points get id -1), and a voxel keeps its
first ``max_points`` points.  One rule is explicit here: a point whose cell is not a finite value in
``[0, grid)`` on every axis -- NaN and infinite coordinates included -- gets id -1 and makes no voxel.
"""
import numpy as np


def grid_size(vsize_xyz, coors_range_xyz):
    """zyx-ordered ``(vsize, lo, grid)``; grid = round((hi - lo) / vsize) in fp32."""
    nd = len(vsize_xyz)
    vs = np.array([vsize_xyz[nd - 1 - j] for j in range(nd)], np.float32)
    lo = np.array([coors_range_xyz[nd - 1 - j] for j in range(nd)], np.float32)
    hi = np.array([coors_range_xyz[2 * nd - 1 - j] for j in range(nd)], np.float32)
    return vs, lo, np.round((hi - lo) / vs).astype(np.int64)


def cells(points, vsize_xyz, coors_range_xyz):
    """-> ``(cell [N, nd] int64 in zyx order, in_range [N] bool)``."""
    pts = np.ascontiguousarray(points, dtype=np.float32)
    nd = len(vsize_xyz)
    vs, lo, grid = grid_size(vsize_xyz, coors_range_xyz)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor((pts[:, [nd - 1 - j for j in range(nd)]] - lo) / vs)       # fp32 throughout
        ok = (np.isfinite(f) & (f >= 0) & (f < grid)).all(axis=1)
    c = np.where(ok[:, None], f, 0).astype(np.int64)
    return c, ok


def _cell(p, lo, vs):
    return np.floor((np.float32(p) - lo) / vs)


def boundary_cloud(vsize_xyz, coors_range_xyz, seed=0, extra_features=1, uniform=2000):
    """Points one fp32 ulp either side of every voxel boundary on every axis: for each boundary b the
    smallest fp32 p with ``floor(fp32((p - lo) / vs)) >= b`` and its neighbours, the other axes at random
    cell centres.  Plus p == lo and p == hi on every axis, and ``uniform`` points over the range and 5 %
    beyond it; shuffled, with ``extra_features`` grid-valued features after the coordinates."""
    rng = np.random.default_rng(seed)
    nd = len(vsize_xyz)
    vs, lo, grid = grid_size(vsize_xyz, coors_range_xyz)
    up, down = np.float32(np.inf), np.float32(-np.inf)

    def centre(a):
        return np.float32(lo[a] + (np.float32(rng.integers(0, grid[a])) + np.float32(0.5)) * vs[a])

    rows = []
    for j in range(nd):                                    # internal (zyx) axis j = point column nd-1-j
        for b in range(int(grid[j]) + 1):
            # bisect to adjacent fp32 values a < p with cell(a) < b <= cell(p)
            a = np.float32(lo[j] + np.float32(b - 1) * vs[j])
            p = np.float32(lo[j] + np.float32(b + 1) * vs[j])
            while np.nextafter(a, up, dtype=np.float32) != p:
                m = np.float32((np.float64(a) + np.float64(p)) / 2)
                if m == a or m == p:
                    m = np.nextafter(a, up, dtype=np.float32)
                if _cell(m, lo[j], vs[j]) >= b:
                    p = m
                else:
                    a = m
            for q in (np.nextafter(a, down, dtype=np.float32), a, p, np.nextafter(p, up, dtype=np.float32)):
                row = [centre(a) for a in range(nd)]
                row[j] = q
                rows.append(row[::-1])
        for edge in (lo[j], np.float32(coors_range_xyz[2 * nd - 1 - j])):
            row = [centre(a) for a in range(nd)]
            row[j] = edge
            rows.append(row[::-1])
    lo_xyz, hi_xyz = np.array(coors_range_xyz[:nd], np.float64), np.array(coors_range_xyz[nd:], np.float64)
    span = hi_xyz - lo_xyz
    extra = rng.uniform(lo_xyz - 0.05 * span, hi_xyz + 0.05 * span, size=(uniform, nd))
    xyz = np.concatenate([np.array(rows, np.float32), extra.astype(np.float32)])
    xyz = xyz[rng.permutation(xyz.shape[0])]
    feats = (rng.integers(-64, 65, size=(xyz.shape[0], extra_features)) * 2.0 ** -6).astype(np.float32)
    return np.concatenate([xyz, feats], axis=1)


def point2voxel(points, vsize_xyz, coors_range_xyz, max_voxels, max_points, empty_mean=False):
    """-> ``(voxels [M, max_points, F] f32, indices [M, nd] i32, num_per_voxel [M] i32, pc_voxel_id [N] i64)``.
    ``empty_mean`` fills a voxel's unused slots with ``fp32(sum) / fp32(num)`` of its kept points, the sum
    taken in fp64 (equal to the kernel's fp32 sum when the features lie on an exact grid)."""
    pts = np.ascontiguousarray(points, dtype=np.float32)
    n, nf = pts.shape
    nd = len(vsize_xyz)
    _, _, grid = grid_size(vsize_xyz, coors_range_xyz)
    c, ok = cells(pts, vsize_xyz, coors_range_xyz)
    key = np.zeros(n, np.int64)
    for j in range(nd):
        key = key * grid[j] + c[:, j]
    valid = np.nonzero(ok)[0]
    ids = np.full(n, -1, np.int64)
    uniq, first, inv = np.unique(key[valid], return_index=True, return_inverse=True)
    rank = np.empty(len(uniq), np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(len(uniq))        # first-touch order
    m = min(len(uniq), int(max_voxels))
    vid = rank[inv.reshape(-1)]
    ids[valid] = np.where(vid < m, vid, -1)
    voxels = np.zeros((m, max_points, nf), np.float32)
    indices = np.zeros((m, nd), np.int32)
    num = np.zeros(m, np.int32)
    kept = valid[vid < m]
    kv = ids[kept]
    order = np.argsort(kv, kind="stable")                                 # input order inside a voxel
    sp, sv = kept[order], kv[order]
    start = np.searchsorted(sv, np.arange(m))
    pos = np.arange(len(sv)) - start[sv]
    sel = pos < max_points
    voxels[sv[sel], pos[sel]] = pts[sp[sel]]
    np.add.at(num, sv[sel], 1)
    firsts = valid[first[np.argsort(first, kind="stable")][:m]]
    indices[:] = c[firsts]
    if empty_mean:
        sums = np.zeros((m, nf), np.float64)
        np.add.at(sums, sv[sel], pts[sp[sel]].astype(np.float64))
        for v in np.nonzero((num > 0) & (num < max_points))[0]:
            voxels[v, num[v]:] = sums[v].astype(np.float32) / np.float32(num[v])
    return voxels, indices, num, ids
