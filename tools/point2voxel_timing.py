"""Time MaskedPointToVoxel (one batched call, graph-replayed and eager) against what a user does without it: B eager
PointToVoxel calls, one per cloud, each with its host read-back of the voxel count, plus the host-side
concatenation that prepends the batch column.  Same clouds for both; the tool checks that the batched rows equal the
concatenation bit for bit before timing.

Workloads (5 points per voxel, 4 features x, y, z, intensity):
  * KITTI-like: grid 8 x 200 x 176 (0.4 x 0.4 x 0.5 m), B = 4 and 8, ~120 k points per cloud, max_num_voxels 16 000
    and 40 000;
  * Waymo-like: grid 40 x 1504 x 1504 (0.1 x 0.1 x 0.15 m), B = 4, ~180 k points per cloud, max_num_voxels 150 000.
The clouds are synthetic LiDAR sweeps (density falling with range, most points near a ground plane), from a seed.

Launches are the native launches of one call (spx_launch_count).  Algorithmic bytes of one batched call: the points
read once, pc_voxel_id written, and the voxels, indices and num_per_voxel written for every one of the `bound` rows;
set against the 3.35 TB/s data-sheet bandwidth.  A number is the median over ``--reps`` windows of ``--steps`` calls,
CUDA events closed by a synchronise, the variants alternating in one process, every shape warmed up first.  Prints
one JSON line with the card's name and power limit.

    python tools/point2voxel_timing.py [--steps 30] [--reps 5]
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

KITTI = ([0.4, 0.4, 0.5], [0.0, -40.0, -3.0, 70.4, 40.0, 1.0])
WAYMO = ([0.1, 0.1, 0.15], [-75.2, -75.2, -2.0, 75.2, 75.2, 4.0])


def sweep(rng, n, cr):
    """one synthetic LiDAR sweep over the range box: range ~ r_max * u^2 (dense near the sensor), 70 % of the
    points on a ground plane, the rest on objects up to 3 m; x, y limited to the box (a few points fall outside)"""
    lo, hi = np.array(cr[:3]), np.array(cr[3:])
    centre = np.array([max(lo[0], 0.0), (lo[1] + hi[1]) / 2])
    r = np.max(hi[:2] - centre) * rng.random(n) ** 2
    th = rng.random(n) * 2 * np.pi
    x, y = centre[0] + r * np.cos(th), centre[1] + r * np.sin(th)
    ground = rng.random(n) < 0.7
    z = np.where(ground, lo[2] + 1.3 + 0.05 * rng.standard_normal(n), lo[2] + 1.3 + 3.0 * rng.random(n))
    return np.stack([x, y, z, rng.random(n)], 1).astype(np.float32)


def run(spconv, name, vs, cr, batch, per_cloud, max_voxels, steps, reps, dev):
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(batch * 7 + max_voxels)
    clouds = [sweep(rng, int(per_cloud * (0.9 + 0.2 * rng.random())), cr) for _ in range(batch)]
    sizes = [len(c) for c in clouds]
    points = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)).to(dev)
    gen = spconv.MaskedPointToVoxel(vs, cr, 4, max_voxels, 5, batch, device=dev)
    single = spconv.PointToVoxel(vs, cr, 4, max_voxels, 5, device=dev)
    pieces = [points[int(a):int(b)] for a, b in zip(offsets[:-1].tolist(), offsets[1:].tolist())]

    def batched():
        return gen(points, offsets)

    def per_cloud_calls():
        vox, ind, num = [], [], []
        for b, pc in enumerate(pieces):
            v, i, n = single(pc)
            vox.append(v)
            ind.append(torch.cat([torch.full((len(i), 1), b, dtype=torch.int32, device=dev), i], 1))
            num.append(n)
        return torch.cat(vox), torch.cat(ind), torch.cat(num)

    v, i, n, _, nv = batched()
    rv, ri, rn = per_cloud_calls()
    m = int(nv)
    same = (m == len(rv) and torch.equal(v[:m].view(torch.int32), rv.view(torch.int32)) and torch.equal(i[:m], ri)
            and torch.equal(n[:m], rn))
    g = graphed(batched)
    launches = {}
    for key, fn in (("masked", batched), ("per_cloud", per_cloud_calls)):
        fn()
        torch.cuda.synchronize()
        ops.launch_count(True)
        fn()
        torch.cuda.synchronize()
        launches[key] = ops.launch_count(True)
    ms = measure({"masked_graph": lambda s: g(), "masked_eager": lambda s: batched(),
                  "per_cloud_eager": lambda s: per_cloud_calls()}, steps, reps)
    bound = gen.max_num_voxels_total
    p = points.shape[0]
    nbytes = p * 4 * 4 + p * 8 + bound * (5 * 4 * 4 + 4 * 4 + 4)
    return {"case": name, "batch": batch, "points": sizes, "max_num_voxels": max_voxels, "bound": bound,
            "voxels": m, "masked_equals_per_cloud": bool(same), "launches": launches, "ms": ms, "bytes": nbytes,
            "graph_of_peak": round(nbytes / ms["masked_graph"] / 1e6 / HBM_GBS, 3),
            "speedup_graph_vs_per_cloud": round(ms["per_cloud_eager"] / ms["masked_graph"], 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("point2voxel_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "point2voxel": []}
    for name, (vs, cr), batch, per, mv in (("kitti", KITTI, 4, 120_000, 16_000), ("kitti", KITTI, 4, 120_000, 40_000),
                                           ("kitti", KITTI, 8, 120_000, 16_000), ("kitti", KITTI, 8, 120_000, 40_000),
                                           ("waymo", WAYMO, 4, 180_000, 150_000)):
        out["point2voxel"].append(run(spconv, name, vs, cr, batch, per, mv, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
