"""PointVoxelScatter on the GPU: max / mean / sum and both gradients bit for bit against the numpy oracle
(tests/point_scatter_oracle.py) in fp32, fp16 and bf16 over the scalar path, the vector path and tails, with empty
rows, dropped ids of every kind, NaN, +-0 and ties; agreement with float64 torch and with scatter_reduce("amax");
invariance to padding and repetition; .count against MaskedPointToVoxel; no synchronising call; and a dynamic-VFE
training step from raw points to the loss that replays as one CUDA graph, bit for bit with the eager step."""
import numpy as np
import pytest
import torch
from torch import nn

from tests import point_scatter_oracle as ps

import spconv_b200.pytorch as spconv

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
CHANNELS = [1, 3, 4, 8, 9, 64, 128, 136]
_BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}


def _same(got, want, what, strict=False):
    """bit equality; a NaN matches any NaN unless `strict` (a sum's NaN payload is the hardware's)"""
    got, want = got.contiguous().cpu(), want.contiguous().cpu()
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if strict:
        assert torch.equal(got.view(_BITS[got.dtype]), want.view(_BITS[want.dtype])), what
        return
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), f"{what}: NaN positions"
    gb, wb = got.view(_BITS[got.dtype]), want.view(_BITS[want.dtype])
    bad = (gb != wb) & ~gn
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"


def _round(a32, dtype):
    """float32 numpy -> dtype, rounded once to nearest even"""
    return torch.from_numpy(np.ascontiguousarray(a32, np.float32)).to(dtype)


def _features(rng, p, c, dtype, special=True):
    """random features in dtype with ties (values on a coarse grid), +-0 and NaNs -> (torch on the device, float32 numpy
    holding the same values exactly)"""
    x = np.round(rng.standard_normal((p, c)) * 4) / 4
    if special and p:
        x[rng.random((p, c)) < 0.05] = 0.0
        x[rng.random((p, c)) < 0.05] = -0.0
        x[rng.random((p, c)) < 0.01] = np.nan
    t = torch.from_numpy(x.astype(np.float32)).to(dtype)
    return t.to(DEV), t.float().numpy()


def _ids(rng, p, rows, as_int64=True):
    """ids over [0, rows) with empty rows, one long row, and dropped ids: -1, -7, rows, rows + 5, 2^30"""
    ids = rng.integers(0, max(rows, 1), p)
    if rows > 8:
        ids[(ids % 7) == 3] = rows // 2                    # holes: rows = 3 mod 7 stay empty, one row gets long
    drop = rng.random(p)
    ids[drop < 0.04] = -1
    ids[(drop >= 0.04) & (drop < 0.05)] = -7
    ids[(drop >= 0.05) & (drop < 0.06)] = rows
    ids[(drop >= 0.06) & (drop < 0.07)] = rows + 5
    ids[(drop >= 0.07) & (drop < 0.08)] = 1 << 30
    return torch.from_numpy(ids.astype(np.int64 if as_int64 else np.int32)).to(DEV)


def _check_all(ids, rows, x, x32, rng, what):
    """every reduction, forward and backward, bit for bit against the oracle"""
    dtype = x.dtype
    ids_np = ids.cpu().numpy().astype(np.int64)
    scatter = spconv.PointVoxelScatter(ids, rows)
    count = ps.group(ids_np, rows)[3]
    assert scatter.count.dtype == torch.int32 and torch.equal(scatter.count.cpu(), torch.from_numpy(count).int())
    c = x.shape[1]
    dy, dy32 = _features(rng, rows, c, dtype, special=False)
    xg = x.clone().requires_grad_(True)

    out = scatter.sum(xg)
    _same(out, _round(ps.segment_sum(x32, ids_np, rows), dtype), f"{what}: sum")
    (gx,) = torch.autograd.grad(out, xg, dy)
    _same(gx, torch.from_numpy(ps.sum_grad(dy.cpu().float().numpy(), ids_np, rows)).to(dtype), f"{what}: sum grad",
          strict=True)

    out = scatter.mean(xg)
    _same(out, _round(ps.segment_mean(x32, ids_np, rows), dtype), f"{what}: mean")
    (gx,) = torch.autograd.grad(out, xg, dy)
    _same(gx, _round(ps.mean_grad(dy32, ids_np, rows), dtype), f"{what}: mean grad", strict=True)

    out = scatter.max(xg)
    arg = torch.from_numpy(ps.segment_argmax(x32, ids_np, rows))
    ok = arg >= 0
    rr, cc = ok.nonzero(as_tuple=True)
    want = torch.zeros((rows, c), dtype=dtype)
    want[rr, cc] = x.cpu()[arg[ok], cc]                     # a copy of the winning point, NaN payloads included
    _same(out, want, f"{what}: max", strict=True)
    (gx,) = torch.autograd.grad(out, xg, dy)
    want = torch.zeros((x.shape[0], c), dtype=dtype)
    want[arg[ok], cc] = dy.cpu()[rr, cc]
    _same(gx, want, f"{what}: max grad", strict=True)
    return scatter


@pytest.mark.parametrize("c", CHANNELS)
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).replace("torch.", ""))
def test_reductions_and_gradients_bit_exact(dtype, c):
    rng = np.random.default_rng(c * 3 + DTYPES.index(dtype))
    p, rows = 6_000, 900
    x, x32 = _features(rng, p, c, dtype)
    for as_int64 in (True, False):
        _check_all(_ids(rng, p, rows, as_int64), rows, x, x32, rng, f"{dtype} C={c} int{64 if as_int64 else 32}")


def test_unaligned_features_take_the_scalar_path():
    rng = np.random.default_rng(40)
    base, _ = _features(rng, 3_000, 65, torch.float16)
    x = base[:, 1:]                                         # 64 channels, rows 130 bytes apart: no 16-byte vectors
    x32 = x.float().cpu().numpy()
    _check_all(_ids(rng, 3_000, 500), 500, x, x32, rng, "unaligned")


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).replace("torch.", ""))
def test_edges(dtype):
    rng = np.random.default_rng(41)
    for c in (1, 8, 9):
        x, x32 = _features(rng, 0, c, dtype)
        _check_all(torch.zeros(0, dtype=torch.int64, device=DEV), 5, x, x32, rng, "P = 0")
        x, x32 = _features(rng, 200, c, dtype)
        _check_all(_ids(rng, 200, 1), 1, x, x32, rng, "rows = 1")
        _check_all(torch.full((200,), -1, dtype=torch.int64, device=DEV), 3, x, x32, rng, "every point dropped")
        sc = spconv.PointVoxelScatter(_ids(rng, 200, 4), 0)       # no rows at all
        assert sc.max(x).shape == (0, c) and sc.count.shape == (0,)
    x, x32 = _features(rng, 5_000, 64, dtype)
    ids = torch.full((5_000,), 2, dtype=torch.int32, device=DEV)
    _check_all(ids, 4, x, x32, rng, "one row of 5000 points")


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).replace("torch.", ""))
def test_300k_points(dtype):
    rng = np.random.default_rng(42)
    x, x32 = _features(rng, 300_000, 64, dtype)
    _check_all(_ids(rng, 300_000, 60_000), 60_000, x, x32, rng, "300k")


def test_mean_and_sum_against_float64_torch():
    rng = np.random.default_rng(43)
    p, rows, c = 50_000, 7_000, 32
    x = torch.randn(p, c, dtype=torch.float64).to(DEV)      # drawn on the CPU, as every input here
    ids = _ids(rng, p, rows)
    sc = spconv.PointVoxelScatter(ids, rows)
    r = torch.where((ids >= 0) & (ids < rows), ids, rows)
    n = torch.bincount(r, minlength=rows + 1)[:rows].double()
    for dtype, tol in ((torch.float32, 1e-5), (torch.float16, 2e-3), (torch.bfloat16, 1.6e-2)):
        xd = x.to(dtype).requires_grad_(True)
        xs = xd.detach().double()
        s64 = torch.zeros(rows + 1, c, dtype=torch.float64, device=DEV).index_add_(0, r, xs)[:rows]
        m64 = s64 / n.clamp(min=1)[:, None]
        for got, want in ((sc.sum(xd), s64), (sc.mean(xd), m64)):
            err = (got.double() - want).abs().max().item()
            assert err <= tol * max(1.0, want.abs().max().item()), (dtype, err)
        dy = torch.randn(rows, c, dtype=torch.float64).to(DEV)
        (g,) = torch.autograd.grad(sc.mean(xd), xd, dy.to(dtype))
        keep = r < rows
        want = torch.zeros(p, c, dtype=torch.float64, device=DEV)
        want[keep] = dy.to(dtype).double()[r[keep]] / n[r[keep]][:, None]
        assert (g.double() - want).abs().max().item() <= tol * 4, dtype
        (g,) = torch.autograd.grad(sc.sum(xd), xd, dy.to(dtype))
        want[keep] = dy.to(dtype).double()[r[keep]]
        assert torch.equal(g.double(), want), dtype


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).replace("torch.", ""))
def test_max_agrees_with_scatter_reduce_amax(dtype):
    """NaN-free data; the gradients are compared where the row's maximum is attained once (scatter_reduce splits it
    between ties, this scatter gives it to the first point)"""
    rng = np.random.default_rng(44)
    p, rows, c = 40_000, 5_000, 16
    x = torch.randn(p, c).to(dtype).to(DEV)
    ids = _ids(rng, p, rows)
    sc = spconv.PointVoxelScatter(ids, rows)
    r = torch.where((ids >= 0) & (ids < rows), ids, rows)
    idx = r[:, None].expand(p, c)
    xg = x.clone().requires_grad_(True)
    xt = x.clone().requires_grad_(True)
    got = sc.max(xg)
    want = torch.zeros(rows + 1, c, dtype=dtype, device=DEV).scatter_reduce(0, idx, xt, "amax", include_self=False)
    assert torch.equal(got, want[:rows])
    hits = torch.zeros(rows + 1, c, dtype=torch.int32, device=DEV).scatter_add_(0, idx, (x == want.detach()[r]).int())
    untied = hits[r] == 1                                   # [p, c]: the point's row attains its maximum once
    assert float(untied[r < rows].float().mean()) > 0.5, "mostly tie-free"
    dy = torch.randn(rows + 1, c).to(dtype).to(DEV)
    (g1,) = torch.autograd.grad(got, xg, dy[:rows])
    (g2,) = torch.autograd.grad(want[:rows], xt, dy[:rows])
    assert torch.equal(g1[untied], g2[untied])
    assert not bool(g1[r == rows].any())


def test_padding_and_repeat_invariance():
    rng = np.random.default_rng(45)
    p, rows, c = 30_000, 4_000, 24
    x, _ = _features(rng, p, c, torch.float16)
    ids = _ids(rng, p, rows)
    dy = torch.randn(rows, c).half().to(DEV)
    base = {}
    sc = spconv.PointVoxelScatter(ids, rows)
    for mode in ("max", "mean", "sum"):
        xg = x.clone().requires_grad_(True)
        out = getattr(sc, mode)(xg)
        base[mode] = (out.detach(), torch.autograd.grad(out, xg, dy)[0])
    for pad_at in ("end", "front", "spread"):
        for pad in (1, 999, 40_000):
            junk, _ = _features(rng, pad, c, torch.float16)
            bad = torch.from_numpy(rng.choice(np.array([-1, rows, rows + 3, 1 << 30]), pad)).to(DEV)
            if pad_at == "end":
                pos = torch.arange(p, device=DEV)
            elif pad_at == "front":
                pos = torch.arange(pad, pad + p, device=DEV)
            else:
                pos = torch.from_numpy(np.sort(rng.choice(p + pad, p, replace=False))).to(DEV)
            xp = torch.empty(p + pad, c, dtype=x.dtype, device=DEV)
            idp = torch.empty(p + pad, dtype=torch.int64, device=DEV)
            mask = torch.ones(p + pad, dtype=torch.bool, device=DEV)
            mask[pos] = False
            xp[pos], idp[pos] = x, ids
            xp[mask], idp[mask] = junk, bad
            sp = spconv.PointVoxelScatter(idp, rows)
            for mode in ("max", "mean", "sum"):
                for _ in range(2):                          # and run to run
                    xg = xp.clone().requires_grad_(True)
                    out = getattr(sp, mode)(xg)
                    (g,) = torch.autograd.grad(out, xg, dy)
                    _same(out, base[mode][0], f"{pad_at} {pad} {mode}", strict=mode == "max")
                    _same(g[pos], base[mode][1], f"{pad_at} {pad} {mode} grad", strict=True)
                    assert not bool(g[mask].any()), f"{pad_at} {pad} {mode}: dropped points get 0"


def test_count_matches_masked_point_to_voxel():
    vs, cr = [0.4, 0.4, 0.5], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0]
    rng = np.random.default_rng(46)
    sizes = [30_000, 0, 20_000]
    pts = np.concatenate([np.stack([rng.random(n) * 30, rng.random(n) * 20 - 10, rng.random(n) * 3 - 2.5,
                                    rng.random(n)], 1) for n in sizes], 0).astype(np.float32)
    pts = np.concatenate([pts, pts[:5_000] + 0.01], 0).astype(np.float32)     # padding beyond off[B]
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32, device=DEV)
    for max_points in (1, 5):
        gen = spconv.MaskedPointToVoxel(vs, cr, 4, 9_000, max_points, 3, device=DEV)
        _, _, num, ids, nv = gen(torch.from_numpy(pts).to(DEV), off)
        sc = spconv.PointVoxelScatter(ids, gen.max_num_voxels_total)
        m = int(nv)
        assert 0 < m < gen.max_num_voxels_total
        assert torch.equal(sc.count.clamp(max=max_points), num), max_points
        assert int(sc.count[:m].min()) >= 1 and not bool(sc.count[m:].any())
        if max_points == 1:
            assert int(sc.count.max()) > 1


def test_no_synchronising_call():
    rng = np.random.default_rng(47)
    x, _ = _features(rng, 20_000, 32, torch.bfloat16)
    ids = _ids(rng, 20_000, 3_000)
    dy = torch.randn(3_000, 32).bfloat16().to(DEV)
    spconv.PointVoxelScatter(ids, 3_000).max(x)            # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for id_t in (ids, ids.int()):
            sc = spconv.PointVoxelScatter(id_t, 3_000)
            xg = x.clone().requires_grad_(True)
            loss = (sc.max(xg) * dy).sum() + (sc.mean(xg) * dy).sum() + (sc.sum(xg) * dy).sum() + sc.count.sum()
            loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert xg.grad is not None and xg.grad.shape == x.shape


class _Vfe(nn.Module):
    """a dynamic VFE (Linear + ReLU per point, then the voxel max, plus the voxel mean of xyz) and a small backbone"""

    def __init__(self):
        super().__init__()
        torch.manual_seed(12)
        self.pfn = nn.Linear(4, 16)
        self.body = spconv.SparseSequential(
            spconv.SubMConv3d(19, 16, 3, indice_key="s1", bias=False), nn.ReLU(),
            spconv.SparseConv3d(16, 32, 3, stride=2, padding=1, bias=False), nn.ReLU())
        self.pool = spconv.MaskedGlobalAvgPool()
        self.head = nn.Linear(32, 5)

    def voxel_features(self, points, ids, rows):
        sc = spconv.PointVoxelScatter(ids, rows)
        per_point = torch.relu(self.pfn(points))
        return torch.cat([sc.max(per_point), sc.mean(points[:, :3])], 1)

    def forward(self, x):
        return self.head(self.pool(self.body(x)))


def _sweep(rng, n, cr):
    """n points in the range box, dense near the sensor (range ~ u^2), 70 % on a ground plane, 4 features"""
    lo, hi = np.array(cr[:3]), np.array(cr[3:])
    r = (hi[0] - lo[0]) * rng.random(n) ** 2
    th = (rng.random(n) - 0.5) * np.pi
    y = np.clip(r * np.sin(th), lo[1], hi[1] - 1e-3)
    ground = rng.random(n) < 0.7
    z = np.where(ground, lo[2] + 1.3 + 0.05 * rng.standard_normal(n), lo[2] + 1.3 + 3.0 * rng.random(n))
    return np.stack([lo[0] + r * np.cos(th), y, z, rng.random(n)], 1).astype(np.float32)


def test_dynamic_vfe_step_captures_as_one_graph():
    vs, cr = [0.4, 0.4, 0.5], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0]
    batch, max_voxels, p_pad = 3, 16_000, 160_000
    rng = np.random.default_rng(13)
    sweep = _sweep
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, max_voxels, 1, batch, device=DEV)
    net = _Vfe().to(DEV)
    params = list(net.parameters())
    labels = torch.tensor([0, 3, 1], device=DEV)
    args = []
    for sizes in ([40_000, 30_000, 45_000], [20_000, 50_000, 35_000], [48_000, 0, 42_000]):
        pts = np.concatenate([sweep(rng, n, cr) for n in sizes] + [sweep(rng, p_pad - sum(sizes), cr)], 0)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
        args.append((torch.from_numpy(pts).to(DEV), torch.from_numpy(off).to(DEV)))

    def step(points, offsets):
        for p in params:
            p.grad = None
        points = points.clone().requires_grad_(True)
        _, indices, _, ids, nv = gen(points.detach(), offsets)
        x = spconv.SparseConvTensor(net.voxel_features(points, ids, gen.max_num_voxels_total), indices,
                                    gen.grid_size, batch)
        x.num_valid = nv
        loss = nn.functional.cross_entropy(net(x), labels)
        loss.backward()
        return loss.detach(), [p.grad for p in params], points.grad, nv

    # eager: bounds from one eager forward, then every batch once
    _, indices, _, ids, nv = gen(args[0][0], args[0][1])
    m = int(nv)
    with torch.no_grad():
        ex = spconv.SparseConvTensor(net.voxel_features(args[0][0], ids, gen.max_num_voxels_total)[:m],
                                     indices[:m].clone(), gen.grid_size, batch)
    spconv.set_output_bounds(net, ex, margin=1.5)
    want = []
    for a in args:
        loss, grads, pgrad, nv = step(*a)
        want.append((loss.clone(), [g.clone() for g in grads], pgrad.clone(), int(nv)))
    assert len({w[3] for w in want}) == 3, "three batches of different sizes"
    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 2):
        loss, grads, pgrad, nv = graphed(*args[k])
        assert int(nv) == want[k][3], k
        assert torch.equal(loss, want[k][0]), (k, float(loss), float(want[k][0]))
        for (name, _), g, w in zip(net.named_parameters(), grads, want[k][1]):
            assert torch.equal(g, w), (k, name)
        assert torch.equal(pgrad, want[k][2]), k
    spconv.check_bounds(net)
    spconv.check_bounds(gen)
