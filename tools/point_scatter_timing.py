"""Time PointVoxelScatter (the group, then max / mean / sum, forward and forward + backward) against what a user does
without it: ``torch.Tensor.scatter_reduce_(..., include_self=False)`` on the same ids, with dropped ids sent to a
spare row (float atomics for the sum and the mean, and a max gradient split between ties).

Workloads: the ids are the pc_voxel_id of MaskedPointToVoxel over 4 synthetic LiDAR sweeps (the ``sweep`` generator
of tools/point2voxel_timing.py), one row per voxel of the bound:
  * KITTI-like, 0.05 x 0.05 x 0.1 m voxels (grid 40 x 1600 x 1408), ~120 k points per cloud, C = 64, fp32 and fp16;
  * KITTI-like, 0.16 m pillars (grid 1 x 496 x 432), ~120 k points per cloud, C = 64 fp16: long segments near the
    sensor (the longest is printed);
  * Waymo-like, 0.1 x 0.1 x 0.15 m (grid 40 x 1504 x 1504), ~180 k points per cloud, C = 32 fp16.
Each call builds the group and reduces (a user builds it once per step and may reduce several times over it).  The
backward is the forward + backward time minus the forward time.  Algorithmic bytes: forward P C e (features) + 12 P
(ids, row32, order) + rows C e (out), plus rows C 4 for the max's argmax; backward P C e (the gradient written), set
against the 3.35 TB/s data-sheet bandwidth.  A number is the median over ``--reps`` windows of ``--steps`` calls, CUDA
events closed by a synchronise, the variants alternating in one process, every shape warmed up first.  Prints one
JSON line with the card's name and power limit.

    python tools/point_scatter_timing.py [--steps 20] [--reps 5]
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
from tools.point2voxel_timing import KITTI, WAYMO, sweep  # noqa: E402

FINE = ([0.05, 0.05, 0.1], KITTI[1])
PILLAR = ([0.16, 0.16, 4.0], [0.0, -39.68, -3.0, 69.12, 39.68, 1.0])
REDUCE = {"max": "amax", "mean": "mean", "sum": "sum"}


def run(spconv, name, vs, cr, per_cloud, max_voxels, c, dtype, steps, reps, dev):
    rng = np.random.default_rng(per_cloud + c)
    clouds = [sweep(rng, int(per_cloud * (0.9 + 0.2 * rng.random())), cr) for _ in range(4)]
    sizes = [len(cl) for cl in clouds]
    points = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(dev)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, max_voxels, 1, 4, device=dev)
    ids = gen(points, offsets)[3].clone()
    rows = gen.max_num_voxels_total
    p = points.shape[0]
    torch.manual_seed(0)
    x = torch.randn((p, c), device=dev).to(dtype).requires_grad_(True)
    dy = torch.randn((rows, c), device=dev).to(dtype)
    spare = torch.where((ids >= 0) & (ids < rows), ids, rows)[:, None].expand(p, c)
    variants, not_captured = {}, []
    for mode in ("max", "mean", "sum"):
        def ours_fwd(mode=mode):
            with torch.no_grad():
                getattr(spconv.PointVoxelScatter(ids, rows), mode)(x)

        def ours_fwd_bwd(mode=mode):
            x.grad = None
            getattr(spconv.PointVoxelScatter(ids, rows), mode)(x).backward(dy)

        def torch_fwd(mode=mode):
            with torch.no_grad():
                r = torch.where((ids >= 0) & (ids < rows), ids, rows)[:, None].expand(p, c)
                torch.zeros((rows + 1, c), dtype=dtype, device=dev).scatter_reduce_(0, r, x, REDUCE[mode],
                                                                                     include_self=False)

        def torch_fwd_bwd(mode=mode):
            x.grad = None
            r = torch.where((ids >= 0) & (ids < rows), ids, rows)[:, None].expand(p, c)
            out = torch.zeros((rows + 1, c), dtype=dtype, device=dev).scatter_reduce_(0, r, x, REDUCE[mode],
                                                                                       include_self=False)
            out[:rows].backward(dy)

        for impl, fns in (("ours", (ours_fwd, ours_fwd_bwd)), ("torch", (torch_fwd, torch_fwd_bwd))):
            for kind, fn in zip(("fwd", "fwd_bwd"), fns):
                variants[f"{impl}_{mode}_{kind}_eager"] = lambda s, fn=fn: fn()
                try:
                    g = graphed(fn)
                except RuntimeError as err:                # a torch backward that does not capture stays eager
                    if impl == "ours":
                        raise
                    not_captured.append(f"{impl}_{mode}_{kind}: {str(err).splitlines()[0][:120]}")
                    continue
                variants[f"{impl}_{mode}_{kind}_graph"] = lambda s, g=g: g()
    ms = measure(variants, steps, reps)
    e = x.element_size()
    derived = {}
    for mode in ("max", "mean", "sum"):
        fwd_bytes = p * c * e + 12 * p + rows * c * e + (rows * c * 4 if mode == "max" else 0)
        for impl in ("ours", "torch"):
            for how in ("graph", "eager"):
                if f"{impl}_{mode}_fwd_bwd_{how}" not in ms or f"{impl}_{mode}_fwd_{how}" not in ms:
                    continue
                f = ms[f"{impl}_{mode}_fwd_{how}"]
                bw = ms[f"{impl}_{mode}_fwd_bwd_{how}"] - f
                d = {"fwd_ms": round(f, 4), "bwd_ms": round(bw, 4)}
                if impl == "ours":
                    d["fwd_of_peak"] = round(fwd_bytes / f / 1e6 / HBM_GBS, 3)
                    d["bwd_of_peak"] = round(p * c * e / bw / 1e6 / HBM_GBS, 3) if bw > 0 else None
                derived[f"{impl}_{mode}_{how}"] = d
    with torch.no_grad():                                  # the same values as scatter_reduce
        sc = spconv.PointVoxelScatter(ids, rows)
        ref = torch.zeros((rows + 1, c), dtype=dtype, device=dev).scatter_reduce_(0, spare, x, "amax",
                                                                                   include_self=False)[:rows]
        max_equal = bool(torch.equal(sc.max(x), ref))
        ref = torch.zeros((rows + 1, c), dtype=torch.float64, device=dev).scatter_reduce_(
            0, spare, x.double(), "sum", include_self=False)[:rows]
        sum_err = float((sc.sum(x).double() - ref).abs().max())
        count = sc.count
        kept = int((count > 0).sum())
        longest = int(count.max())
    return {"case": name, "dtype": str(dtype).replace("torch.", ""), "channels": c, "points": sizes, "rows": rows,
            "voxels": kept, "longest_segment": longest, "dropped_points": int(p - int(count.sum())),
            "max_equals_scatter_reduce": max_equal, "sum_max_abs_err_vs_fp64": sum_err, "not_captured": not_captured,
            "ms": ms, "derived": derived}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("point_scatter_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "point_scatter": []}
    for name, (vs, cr), per, mv, c, dtype in (
            ("kitti_fine", FINE, 120_000, 120_000, 64, torch.float32),
            ("kitti_fine", FINE, 120_000, 120_000, 64, torch.float16),
            ("kitti_pillar", PILLAR, 120_000, 16_000, 64, torch.float16),
            ("waymo", WAYMO, 180_000, 150_000, 32, torch.float16)):
        out["point_scatter"].append(run(spconv, name, vs, cr, per, mv, c, dtype, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
