"""Time VoxelPointInterpolator (the plan, the forward, the forward + backward) against what a user writes without it:
the torch formulation ``sum_j w[:, j] * x.index_select(0, index[:, j])`` on the same table (its backward is
index_select's: ``index_add_`` with float atomics), so the torch side does not even pay for the corner lookup.

Workloads: 4 synthetic LiDAR sweeps (the ``sweep`` generator of tools/point2voxel_timing.py) voxelised by
MaskedPointToVoxel, KITTI-like (0.05 x 0.05 x 0.1 m, grid 40 x 1600 x 1408, ~120 k points per cloud) and Waymo-like
(0.1 x 0.1 x 0.15 m, grid 40 x 1504 x 1504, ~180 k points per cloud).  x is the voxel tensor at stride 1, 2 or 4 (the
distinct voxel coordinates divided by the stride, as a chain of k3 s2 p1 convs keeps them up to its dilation), C 32
to 128 in fp16 or bf16; the points are interpolated trilinearly at grid_positions(stride).  Every variant is a
replayed CUDA graph.  The backward is the forward + backward time minus the forward time.  Algorithmic bytes: forward
8 P K (index, weight) + F C e (the found corner rows, F of the P K entries) + P C e (y); backward 8 F (order,
weight) + F C e (dy rows) + 4 rows (offsets) + rows C e (dx), set against the 3.35 TB/s data-sheet bandwidth.  A
number is the median over ``--reps`` alternating windows of ``--steps`` replays, CUDA events closed by a synchronise,
every variant warmed up first.  Prints one JSON line with the card's name and power limit.

    python tools/point_interp_timing.py [--steps 20] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bounded_encoder_timing import card, measure  # noqa: E402
from tools.masked_bn_timing import HBM_GBS, graphed  # noqa: E402
from tools.point2voxel_timing import WAYMO, sweep  # noqa: E402

FINE = ([0.05, 0.05, 0.1], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0])


def strided(indices, num_valid, stride):
    """the distinct coordinates of the valid rows divided by the stride (set-up only: reads the count back)"""
    rows = indices[: int(num_valid)]
    if stride == 1:
        return rows.contiguous()
    c = rows.clone()
    c[:, 1:] = torch.div(c[:, 1:], stride, rounding_mode="floor")
    return torch.unique(c, dim=0).int().contiguous()


def run(spconv, name, vs, cr, per_cloud, max_voxels, stride, c, dtype, steps, reps, dev):
    rng = np.random.default_rng(per_cloud + c + stride)
    clouds = [sweep(rng, int(per_cloud * (0.9 + 0.2 * rng.random())), cr) for _ in range(4)]
    sizes = [len(cl) for cl in clouds]
    points = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(dev)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, max_voxels, 1, 4, device=dev)
    _, indices, _, _, nv = gen(points, offsets)
    inds = strided(indices, nv, stride)
    shape = [-(-g // stride) for g in gen.grid_size]
    rows, p = inds.shape[0], points.shape[0]
    torch.manual_seed(0)
    x = torch.randn((rows, c), device=dev).to(dtype).requires_grad_(True)
    dy = torch.randn((p, c), device=dev).to(dtype)
    ar = torch.arange(p, dtype=torch.int32, device=dev)
    bids = torch.searchsorted(offsets, ar, right=True, out_int32=True) - 1
    pos = spconv.grid_positions(points[:, :3], vs, cr, stride=stride)
    st = spconv.SparseConvTensor(x.detach(), inds, shape, 4)
    interp = spconv.VoxelPointInterpolator(st, pos, bids)
    index, weight = interp.index, interp.weight
    k = index.shape[1]

    def torch_interp():
        y = None
        for j in range(k):
            t = weight[:, j:j + 1] * x.index_select(0, index[:, j].clamp(min=0))
            y = t if y is None else y + t
        return y.to(dtype)

    def ours_plan():
        spconv.VoxelPointInterpolator(st, pos, bids)

    def ours_fwd():
        with torch.no_grad():
            interp(x)

    def ours_fwd_bwd():
        x.grad = None
        interp(x).backward(dy)

    def torch_fwd():
        with torch.no_grad():
            torch_interp()

    def torch_fwd_bwd():
        x.grad = None
        torch_interp().backward(dy)

    variants = {n: (lambda s, g=graphed(fn): g()) for n, fn in (
        ("ours_plan", ours_plan), ("ours_fwd", ours_fwd), ("ours_fwd_bwd", ours_fwd_bwd), ("torch_fwd", torch_fwd),
        ("torch_fwd_bwd", torch_fwd_bwd))}
    ms = measure(variants, steps, reps)
    e = x.element_size()
    found = int((index >= 0).sum())
    fwd_bytes = 8 * p * k + found * c * e + p * c * e
    bwd_bytes = 8 * found + found * c * e + 4 * rows + rows * c * e
    derived = {}
    for impl in ("ours", "torch"):
        f = ms[f"{impl}_fwd"]
        bw = ms[f"{impl}_fwd_bwd"] - f
        derived[impl] = {"fwd_ms": round(f, 4), "bwd_ms": round(bw, 4),
                         "fwd_of_peak": round(fwd_bytes / f / 1e6 / HBM_GBS, 3),
                         "bwd_of_peak": round(bwd_bytes / bw / 1e6 / HBM_GBS, 3) if bw > 0 else None}
    with torch.no_grad():
        err = float((interp(x).double() - torch_interp().double()).abs().max())
    return {"case": name, "stride": stride, "dtype": str(dtype).replace("torch.", ""), "channels": c, "points": sizes,
            "rows": rows, "corner_hits": round(found / (p * k), 3), "max_abs_diff_vs_torch": err, "ms": ms,
            "derived": derived}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("point_interp_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "point_interp": []}
    for name, (vs, cr), per, mv, stride, c, dtype in (
            ("kitti", FINE, 120_000, 120_000, 1, 32, torch.float16),
            ("kitti", FINE, 120_000, 120_000, 2, 64, torch.bfloat16),
            ("kitti", FINE, 120_000, 120_000, 4, 128, torch.float16),
            ("waymo", WAYMO, 180_000, 150_000, 1, 32, torch.bfloat16),
            ("waymo", WAYMO, 180_000, 150_000, 2, 64, torch.float16),
            ("waymo", WAYMO, 180_000, 150_000, 4, 128, torch.bfloat16)):
        out["point_interp"].append(run(spconv, name, vs, cr, per, mv, stride, c, dtype, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
