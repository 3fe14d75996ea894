"""VoxelPointInterpolator on the GPU: the plan (index, weight), the forward and the backward bit for bit against the
numpy oracle (tests/point_interp_oracle.py) in fp32, fp16 and bf16 over the vector and scalar paths, 1-D to 4-D,
both modes and both normalisations; exact voxel centres, affine fields and the torch formulation; invariance to
padding rows, padding points and repetition; edges (empty inputs, missing corners, non-finite positions, grid faces,
64-bit keys, misaligned operands); launch counts; and an SPVCNN-style step that replays as one CUDA graph."""
import numpy as np
import pytest
import torch
from torch import nn

from tests import point_interp_oracle as pi

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import ops

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
_BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
# (ndim, mode, normalize): the emphasis on 3-D and 2-D
CONFIGS = [(3, "trilinear", True), (3, "trilinear", False), (3, "nearest", True), (2, "trilinear", True),
           (2, "nearest", False), (2, "trilinear", False), (1, "trilinear", True), (4, "trilinear", True),
           (4, "nearest", True)]
SHAPES = {1: [40], 2: [24, 20], 3: [14, 12, 10], 4: [6, 5, 7, 4]}


def _same(got, want, what):
    got, want = got.contiguous().cpu(), want.contiguous().cpu()
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    gb, wb = got.view(_BITS[got.dtype]), want.view(_BITS[want.dtype])
    bad = gb != wb
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"


def _round(a32, dtype):
    return torch.from_numpy(np.ascontiguousarray(a32, np.float32)).to(dtype)


def _tensor(rng, shape, batch, fill=0.5, junk=True):
    """indices [rows, 1 + ndim]: a random occupancy, shuffled, with duplicated coordinates and rows out of range"""
    cells = np.argwhere(rng.random((batch, *shape)) < fill).astype(np.int32)
    cells = cells[rng.permutation(cells.shape[0])]
    if junk and cells.shape[0] > 10:
        extra = cells[rng.integers(0, cells.shape[0], cells.shape[0] // 10)]          # duplicates: later rows
        bad = cells[: max(cells.shape[0] // 20, 1)].copy()
        bad[:, 0] = rng.choice([-1, batch, batch + 3], bad.shape[0])
        oob = cells[: max(cells.shape[0] // 20, 1)].copy()
        oob[:, 1] = rng.choice([-1, shape[0], shape[0] + 2], oob.shape[0])
        cells = np.concatenate([cells, extra, bad, oob], 0)
    return cells


def _points(rng, shape, batch, p, special=True):
    """positions over [-1.5, shape + 0.5) with grid points, f = 0.5, faces, NaN / inf / huge and bad batch ids"""
    nd = len(shape)
    pos = (rng.random((p, nd)) * (np.array(shape) + 2) - 1.5).astype(np.float32)
    bid = rng.integers(0, batch, p).astype(np.int32)
    if special and p >= 100:
        k = p // 10
        pos[:k] = np.round(pos[:k])                               # on grid points
        pos[k:2 * k] = np.floor(pos[k:2 * k]) + np.float32(0.5)   # f = 0.5
        pos[2 * k:2 * k + 5, 0] = np.float32(shape[0] - 1)        # the upper face
        pos[2 * k + 5:2 * k + 10, 0] = np.float32(-1)             # the lower bound
        pos[2 * k + 10, 0] = np.nextafter(np.float32(shape[0]), np.float32(0))
        pos[2 * k + 11:2 * k + 13, 0] = np.nan
        pos[2 * k + 13, -1] = np.inf
        pos[2 * k + 14, -1] = -np.inf
        pos[2 * k + 15, 0] = np.float32(3e9)
        pos[2 * k + 16, 0] = np.float32(-3e9)
        bid[2 * k + 17:2 * k + 20] = [-1, batch, 1 << 30]
    return pos, bid


def _features(rng, rows, c, dtype):
    t = torch.from_numpy(rng.standard_normal((rows, c)).astype(np.float32)).to(dtype)
    return t.to(DEV), t.float().numpy()


def _run(inds, shape, batch, nv, pos, bid, mode, normalize, x, dy):
    """(index, weight, y, dx) of the CUDA op"""
    st = spconv.SparseConvTensor(x, torch.from_numpy(inds).to(DEV), shape, batch)
    if nv is not None:
        st.num_valid = torch.tensor([nv], dtype=torch.int32, device=DEV)
    interp = spconv.VoxelPointInterpolator(st, torch.from_numpy(pos).to(DEV), torch.from_numpy(bid).to(DEV), mode,
                                           normalize)
    xg = x.detach().clone().requires_grad_(True)
    y = interp(xg)
    (dx,) = torch.autograd.grad(y, xg, dy)
    return interp.index, interp.weight, y, dx


def _check(inds, shape, batch, nv, pos, bid, mode, normalize, x, x32, dy, what):
    dtype = x.dtype
    idx, w, y, dx = _run(inds, shape, batch, nv, pos, bid, mode, normalize, x, dy)
    want_i, want_w = pi.plan(inds, shape, batch, nv, pos, bid, mode, normalize)
    assert torch.equal(idx.cpu(), torch.from_numpy(want_i)), f"{what}: index"
    _same(w, torch.from_numpy(want_w), f"{what}: weight")
    _same(y, _round(pi.forward(x32, want_i, want_w), dtype), f"{what}: forward")
    _same(dx, _round(pi.backward(dy.float().cpu().numpy(), want_i, want_w, inds.shape[0]), dtype), f"{what}: backward")
    return idx, w, y, dx


@pytest.mark.parametrize("c", [1, 12, 64, 256])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).replace("torch.", ""))
def test_bit_exact_against_oracle(dtype, c):
    rng = np.random.default_rng(c * 3 + DTYPES.index(dtype))
    for ndim, mode, normalize in CONFIGS:
        shape, batch = SHAPES[ndim], 3
        inds = _tensor(rng, shape, batch)
        pos, bid = _points(rng, shape, batch, 4_000)
        x, x32 = _features(rng, inds.shape[0], c, dtype)
        dy, _ = _features(rng, pos.shape[0], c, dtype)
        nv = None if ndim != 3 else inds.shape[0] - 7
        _check(inds, shape, batch, nv, pos, bid, mode, normalize, x, x32, dy, f"{dtype} C={c} {ndim}-D {mode} "
               f"normalize={normalize}")


def test_voxel_centres_return_the_rows():
    rng = np.random.default_rng(50)
    shape = [30, 28, 12]
    inds = _tensor(rng, shape, 2, junk=False)
    for dtype in DTYPES:
        x, _ = _features(rng, inds.shape[0], 64, dtype)
        pos = inds[:, 1:].astype(np.float32)
        for mode in ("trilinear", "nearest"):
            for normalize in (True, False):
                idx, w, y, _ = _run(inds, shape, 2, None, pos, inds[:, 0].copy(), mode, normalize, x,
                                    torch.zeros_like(x))
                _same(y, x, f"{dtype} {mode} {normalize}")
                assert torch.equal(idx[:, 0].cpu(), torch.arange(inds.shape[0], dtype=torch.int32))


def test_affine_field_is_reproduced():
    rng = np.random.default_rng(51)
    shape = [9, 11, 13]
    inds = np.argwhere(np.ones([1, *shape], bool)).astype(np.int32)
    a = np.array([0.75, -1.25, 0.5]), 2.0
    x = torch.from_numpy((inds[:, 1:] @ a[0] + a[1]).astype(np.float32)[:, None]).to(DEV)
    pos = (rng.random((20_000, 3)) * (np.array(shape) - 1.01)).astype(np.float32)
    for normalize in (True, False):
        _, _, y, _ = _run(inds, shape, 1, None, pos, np.zeros(20_000, np.int32), "trilinear", normalize, x,
                          torch.zeros(20_000, 1, device=DEV))
        want = pos.astype(np.float64) @ a[0] + a[1]
        assert np.allclose(y[:, 0].detach().cpu().numpy(), want, rtol=4e-6, atol=1e-4)


def test_against_torch_formulation_with_autograd():
    rng = np.random.default_rng(52)
    shape = [40, 400, 352]
    inds = np.unique(rng.integers(0, [2, *shape], (60_000, 4)), axis=0).astype(np.int32)
    inds = inds[rng.permutation(inds.shape[0])]
    seeds = inds[rng.integers(0, inds.shape[0], 80_000)]
    pos = (seeds[:, 1:] + rng.random((80_000, 3)) * 1.6 - 0.8).astype(np.float32)
    bid = seeds[:, 0].copy()
    for dtype, tol in ((torch.float32, 1e-5), (torch.float16, 2e-3), (torch.bfloat16, 1.6e-2)):
        x = torch.randn(inds.shape[0], 32, dtype=torch.float64).to(dtype).to(DEV)
        st = spconv.SparseConvTensor(x, torch.from_numpy(inds).to(DEV), shape, 2)
        interp = spconv.VoxelPointInterpolator(st, torch.from_numpy(pos).to(DEV), torch.from_numpy(bid).to(DEV))
        xg = x.clone().requires_grad_(True)
        xt = x.double().clone().requires_grad_(True)
        y = interp(xg)
        idx, w = interp.index.long(), interp.weight.double()
        want = (w[:, :, None] * xt[idx.clamp(min=0)] * (idx >= 0)[:, :, None]).sum(1)
        assert (y.double() - want).abs().max().item() <= tol * max(1.0, want.abs().max().item()), dtype
        dy = torch.randn(80_000, 32, dtype=torch.float64).to(dtype).to(DEV)
        (g,) = torch.autograd.grad(y, xg, dy)
        (gt,) = torch.autograd.grad(want, xt, dy.double())
        assert (g.double() - gt).abs().max().item() <= tol * 8 * max(1.0, gt.abs().max().item()), dtype
        assert (idx >= 0).float().mean().item() > 0.05


def test_padding_invariance_and_repeat():
    rng = np.random.default_rng(53)
    shape, batch, c = [20, 40, 36], 2, 24
    inds = _tensor(rng, shape, batch, 0.3)
    rows = inds.shape[0]
    pos, bid = _points(rng, shape, batch, 30_000)
    p = pos.shape[0]
    x, _ = _features(rng, rows, c, torch.float16)
    dy, _ = _features(rng, p, c, torch.float16)
    base = _run(inds, shape, batch, None, pos, bid, "trilinear", True, x, dy)
    again = _run(inds, shape, batch, None, pos, bid, "trilinear", True, x, dy)
    for a, b, name in zip(base, again, ("index", "weight", "y", "dx")):
        assert torch.equal(a, b), f"run to run: {name}"
    for pad_rows, pad_pts in ((1, 0), (5_000, 1), (0, 20_000), (2_000, 7_000)):
        # rows >= num_valid hold junk: real coordinates (some equal to valid rows') and NaN features
        junk = inds[rng.integers(0, rows, pad_rows)].copy() if pad_rows else inds[:0]
        ip = np.concatenate([inds, junk], 0)
        xp = torch.cat([x, torch.full((pad_rows, c), float("nan"), dtype=x.dtype, device=DEV)], 0)
        jp, jb = _points(rng, shape, batch, pad_pts, special=False)
        jb[: pad_pts // 2] = -1
        jp[pad_pts // 2:] = np.nan
        pp, bp = np.concatenate([pos, jp], 0), np.concatenate([bid, jb], 0)
        dyp = torch.cat([dy, torch.randn(pad_pts, c, device=DEV).half()], 0)
        idx, w, y, dx = _run(ip, shape, batch, rows, pp, bp, "trilinear", True, xp, dyp)
        what = f"pad rows {pad_rows}, points {pad_pts}"
        assert torch.equal(idx[:p], base[0]) and torch.equal(w[:p], base[1]), what
        assert (idx[p:] == -1).all() and not bool(w[p:].any()), what
        _same(y[:p], base[2], what)
        _same(dx[:rows], base[3], what)
        assert not bool(dx[rows:].any()), what
    # pad_to: -1 index rows appended, num_valid set
    st = spconv.SparseConvTensor(x, torch.from_numpy(inds).to(DEV), shape, batch).pad_to(rows + 333)
    interp = spconv.VoxelPointInterpolator(st, torch.from_numpy(pos).to(DEV), torch.from_numpy(bid).to(DEV))
    xg = st.features.clone().requires_grad_(True)
    y = interp(xg)
    (dx,) = torch.autograd.grad(y, xg, dy)
    _same(y, base[2], "pad_to")
    _same(dx[:rows], base[3], "pad_to grad")
    assert not bool(dx[rows:].any())


def test_duplicates_resolve_to_the_lowest_row():
    rng = np.random.default_rng(54)
    shape = [10, 10, 10]
    inds = _tensor(rng, shape, 1, 0.5, junk=False)
    dup = np.concatenate([inds, inds[::-1], inds], 0)            # every coordinate three times
    pos, bid = _points(rng, shape, 1, 5_000, special=False)
    x, _ = _features(rng, dup.shape[0], 8, torch.float32)
    idx, _, _, dx = _run(dup, shape, 1, None, pos, bid, "trilinear", True, x, torch.ones(5_000, 8, device=DEV))
    assert int(idx.max()) < inds.shape[0]
    assert not bool(dx[inds.shape[0]:].any())


def test_edges():
    rng = np.random.default_rng(55)
    shape = [8, 9, 10]
    inds = _tensor(rng, shape, 2)
    for dtype in DTYPES:
        x, x32 = _features(rng, inds.shape[0], 12, dtype)
        pos, bid = _points(rng, shape, 2, 500)
        dy, _ = _features(rng, 500, 12, dtype)
        # P = 0
        idx, w, y, dx = _run(inds, shape, 2, None, pos[:0], bid[:0], "trilinear", True, x, dy[:0])
        assert idx.shape == (0, 8) and y.shape == (0, 12) and not bool(dx.any())
        # rows = 0
        idx, w, y, dx = _run(inds[:0], shape, 2, None, pos, bid, "trilinear", True, x[:0], dy)
        assert (idx == -1).all() and not bool(w.any()) and not bool(y.any()) and dx.shape == (0, 12)
        # num_valid = 0
        _check(inds, shape, 2, 0, pos, bid, "trilinear", True, x, x32, dy, f"{dtype} num_valid = 0")
        # every corner missing: the points sit far from the occupied corner of the grid
        far = np.argwhere(np.ones([1, 2, 2, 2], bool)).astype(np.int32)
        xf, xf32 = _features(rng, far.shape[0], 12, dtype)
        fp = (rng.random((500, 3)) * 4 + 4).astype(np.float32)
        idx, w, y, dx = _check(far, shape, 2, None, fp, bid, "trilinear", True, xf, xf32, dy, "no corner")
        assert (idx == -1).all() and not bool(y.any()) and not bool(dx.any())
        # batch ids out of range, non-finite and huge positions only
        bad = np.array([[np.nan, 1, 1], [1, np.inf, 1], [1, 1, -np.inf], [3e9, 1, 1], [-3e9, 1, 1], [1, 1, 1e38],
                        [-1.0001, 1, 1], [8, 1, 1]], np.float32)
        idx, w, y, dx = _check(inds, shape, 2, None, bad, np.zeros(8, np.int32), "trilinear", True, x, x32, dy[:8],
                               "non-finite")
        assert (idx == -1).all() and not bool(y.any())
        _check(inds, shape, 2, None, pos[:4], np.array([-1, 2, 7, -(1 << 30)], np.int32), "nearest", True, x, x32,
               dy[:4], "batch ids")


def test_64_bit_keys():
    """batch * volume >= 2^31: the table takes 64-bit keys; coordinates near the far corner of the grid"""
    rng = np.random.default_rng(56)
    shape, batch = [1500, 1200, 1100], 2
    hi = np.array(shape) - 30
    cells = np.argwhere(rng.random((batch, 30, 30, 30)) < 0.4).astype(np.int32)
    cells[:, 1:] += hi.astype(np.int32)
    cells = cells[rng.permutation(cells.shape[0])]
    seeds = cells[rng.integers(0, cells.shape[0], 20_000)]
    pos = (seeds[:, 1:] + rng.random((20_000, 3)) * 2 - 1).astype(np.float32)
    for dtype in (torch.float32, torch.bfloat16):
        x, x32 = _features(rng, cells.shape[0], 64, dtype)
        dy, _ = _features(rng, 20_000, 64, dtype)
        for mode in ("trilinear", "nearest"):
            idx, _, _, _ = _check(cells, shape, batch, None, pos, seeds[:, 0].copy(), mode, True, x, x32, dy,
                                  f"64-bit {dtype} {mode}")
            assert (idx >= 0).float().mean().item() > 0.2


def test_misaligned_operands_give_the_same_bits():
    rng = np.random.default_rng(57)
    shape = [12, 30, 30]
    inds = _tensor(rng, shape, 2)
    pos, bid = _points(rng, shape, 2, 6_000)
    for dtype in DTYPES:
        x, _ = _features(rng, inds.shape[0], 64, dtype)
        dy, _ = _features(rng, 6_000, 64, dtype)
        st = spconv.SparseConvTensor(x, torch.from_numpy(inds).to(DEV), shape, 2)
        interp = spconv.VoxelPointInterpolator(st, torch.from_numpy(pos).to(DEV), torch.from_numpy(bid).to(DEV))
        y = ops.point_interp_fwd(x, interp.index, interp.weight)
        dx = ops.point_interp_bwd(dy, interp.weight, interp.order, interp.offsets)
        xb = torch.empty(x.numel() + 1, dtype=dtype, device=DEV)
        xm = xb[1:].view_as(x)
        xm.copy_(x)
        dyb = torch.empty(dy.numel() + 3, dtype=dtype, device=DEV)
        dym = dyb[3:].view_as(dy)
        dym.copy_(dy)
        assert xm.data_ptr() % 16 != 0 and dym.data_ptr() % 16 != 0
        _same(ops.point_interp_fwd(xm, interp.index, interp.weight), y, f"{dtype} misaligned x")
        _same(ops.point_interp_bwd(dym, interp.weight, interp.order, interp.offsets), dx, f"{dtype} misaligned dy")
        _same(interp(xm), y, f"{dtype} misaligned x, module")


def test_launch_counts():
    rng = np.random.default_rng(58)
    shape = [20, 200, 176]
    inds = torch.from_numpy(_tensor(rng, shape, 2, 0.05)).to(DEV)
    pos, bid = _points(rng, shape, 2, 50_000)
    pos, bid = torch.from_numpy(pos).to(DEV), torch.from_numpy(bid).to(DEV)
    x = torch.randn(inds.shape[0], 32, device=DEV).half()
    st = spconv.SparseConvTensor(x, inds, shape, 2)
    for mode, k in (("trilinear", 8), ("nearest", 1)):
        spconv.VoxelPointInterpolator(st, pos, bid, mode)          # warm-up
        torch.cuda.synchronize()
        ops.launch_count(True)
        interp = spconv.VoxelPointInterpolator(st, pos, bid, mode)
        plan = ops.launch_count(True)
        ops.point_scatter_group(torch.zeros(50_000 * k, dtype=torch.int32, device=DEV), inds.shape[0])
        group = ops.launch_count(True) - 1                         # point_scatter_group = one id kernel + grouping
        bits = max(1, int(inds.shape[0]).bit_length())
        assert group == 3 + 2 * -(-bits // 9), (group, bits)
        assert plan == 2 + group, (mode, plan, group)
        xg = x.clone().requires_grad_(True)
        ops.launch_count(True)
        y = interp(xg)
        assert ops.launch_count(True) == 1
        y.backward(torch.ones_like(y))
        assert ops.launch_count(True) == 1


class _Spv(nn.Module):
    """an SPVCNN-style block: a point MLP, voxel features as the mean of the points' features, SubM + a k3 s2 p1
    conv, back to the points at stride 2 (trilinear) and at stride 1 (nearest), then a per-point head"""

    def __init__(self):
        super().__init__()
        torch.manual_seed(21)
        self.pfn = nn.Linear(4, 16)
        self.body = spconv.SparseSequential(
            spconv.SubMConv3d(16, 16, 3, indice_key="s1", bias=False), nn.ReLU(),
            spconv.SparseConv3d(16, 32, 3, stride=2, padding=1, bias=False), nn.ReLU())
        self.point = nn.Linear(16, 32)
        self.head = nn.Linear(32 + 16, 5)

    def forward(self, x):
        return self.body(x)


def _sweep(rng, n, cr):
    lo, hi = np.array(cr[:3]), np.array(cr[3:])
    r = (hi[0] - lo[0]) * rng.random(n) ** 2
    th = (rng.random(n) - 0.5) * np.pi
    y = np.clip(r * np.sin(th), lo[1], hi[1] - 1e-3)
    ground = rng.random(n) < 0.7
    z = np.where(ground, lo[2] + 1.3 + 0.05 * rng.standard_normal(n), lo[2] + 1.3 + 3.0 * rng.random(n))
    return np.stack([lo[0] + r * np.cos(th), y, z, rng.random(n)], 1).astype(np.float32)


def test_spvcnn_step_captures_as_one_graph():
    vs, cr = [0.4, 0.4, 0.5], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0]
    batch, max_voxels, p_pad = 3, 16_000, 150_000
    rng = np.random.default_rng(14)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, max_voxels, 1, batch, device=DEV)
    net = _Spv().to(DEV)
    params = list(net.parameters())
    args = []
    for sizes in ([40_000, 30_000, 45_000], [20_000, 50_000, 35_000], [48_000, 0, 42_000]):
        pts = np.concatenate([_sweep(rng, n, cr) for n in sizes] + [_sweep(rng, p_pad - sum(sizes), cr)], 0)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
        labels = rng.integers(0, 5, p_pad)
        args.append((torch.from_numpy(pts).to(DEV), torch.from_numpy(off).to(DEV), torch.from_numpy(labels).to(DEV)))

    def voxel_input(points, offsets):
        _, indices, _, ids, nv = gen(points.detach(), offsets)
        feats = torch.relu(net.pfn(points))
        x = spconv.SparseConvTensor(spconv.PointVoxelScatter(ids, gen.max_num_voxels_total).mean(feats), indices,
                                    gen.grid_size, batch)
        x.num_valid = nv
        return x, feats, nv

    def step(points, offsets, labels):
        for p in params:
            p.grad = None
        points = points.clone().requires_grad_(True)
        x, feats, nv = voxel_input(points, offsets)
        y = net(x)
        p = torch.arange(points.shape[0], dtype=torch.int32, device=points.device)
        bids = torch.searchsorted(offsets, p, right=True, out_int32=True) - 1
        pos2 = spconv.grid_positions(points[:, :3].detach(), vs, cr, stride=2)
        up = spconv.VoxelPointInterpolator(y, pos2, bids)(y.features)
        pos1 = spconv.grid_positions(points[:, :3].detach(), vs, cr)
        near = spconv.VoxelPointInterpolator(x, pos1, bids, mode="nearest")(x.features)
        logits = net.head(torch.cat([torch.relu(net.point(feats) + up), near], 1))
        keep = ((bids >= 0) & (bids < batch)).float()
        loss = (nn.functional.cross_entropy(logits, labels, reduction="none") * keep).sum() / keep.sum().clamp(min=1)
        loss.backward()
        return loss.detach(), [p.grad for p in params], points.grad, nv

    with torch.no_grad():                    # no autograd graph of the example may outlive it into the capture
        x, _, nv = voxel_input(*args[0][:2])
        m = int(nv)
        ex = spconv.SparseConvTensor(x.features[:m].clone(), x.indices[:m].clone(), gen.grid_size, batch)
    del x
    spconv.set_output_bounds(net, ex, margin=1.5)
    want = []
    for a in args:
        loss, grads, pgrad, nv = step(*a)
        want.append((loss.clone(), [g.clone() for g in grads], pgrad.clone(), int(nv)))
    assert len({w[3] for w in want}) == 3, "three batches of different sizes"
    graphed = spconv.graph_capture(step, *args[0])
    for k in (1, 2, 0):
        loss, grads, pgrad, nv = graphed(*args[k])
        assert int(nv) == want[k][3], k
        assert torch.equal(loss, want[k][0]), (k, float(loss), float(want[k][0]))
        for (name, _), g, w in zip(net.named_parameters(), grads, want[k][1]):
            assert torch.equal(g, w), (k, name)
        assert torch.equal(pgrad, want[k][2]), k
    spconv.check_bounds(net)
    spconv.check_bounds(gen)
