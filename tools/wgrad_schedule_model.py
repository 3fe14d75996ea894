"""Stage counts of the weight-gradient kernel's tile schedule, restated in numpy.

tc_wgrad_kernel (spconv_b200/csrc/gemm_tc_wgrad.cu) stacks the atoms of kernel offsets into groups of
one M = 128 accumulator, deals the groups to `passes` CTA columns and runs one pipeline stage per
(tile, active group) of its pass over the tiles of its chunk (a snake over the cost-sorted schedule
records).  This script counts those stages for bench.py's headline cloud (configs[1]: SubMConv3d 3^3,
C = K = 64, fp16, 100 k voxels) under the old and the new schedule:

  * pairing: mirror (offset k with kv-1-k) or natural (k with k+1);
  * passes: groups dealt round-robin (the kernel), or LPT on their active-tile counts (heaviest first
    to the least-loaded pass with fewer than G groups, ties to the lower index).

It prints the stages of every pass, the per-CTA stage spread and the busiest CTA, and the warpgroup-atom
wgmma units issued (one per warpgroup and stage; the new kernel skips a warpgroup whose atom is
inactive).  Counts, not times.

    python tools/wgrad_schedule_model.py [--voxels N] [--seed S] [--sms 132]
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_utils import surface_cloud  # noqa: E402

KITTI = [41, 1600, 1408]
KV, APG, G = 27, 2, 4          # 3^3 offsets; C = 64 fp16: two offsets per group; K = 64: G = 256 / K groups per pass


def tile_masks(inds, shape):
    """offset masks of the 128-row tiles in mask-sorted row order, as the rulebook builds them"""
    d, h, w = shape
    z, y, x = (inds[:, i].astype(np.int64) for i in (1, 2, 3))
    key = lambda zz, yy, xx: (zz * h + yy) * w + xx            # noqa: E731
    ks = np.sort(key(z, y, x))
    n = len(ks)
    mask = np.zeros(n, np.uint32)
    k = 0
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                zz, yy, xx = z + dz, y + dy, x + dx
                ok = (zz >= 0) & (zz < d) & (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
                q = key(zz, yy, xx)
                pos = np.minimum(np.searchsorted(ks, q), n - 1)
                mask |= ((ok & (ks[pos] == q)).astype(np.uint32) << np.uint32(k))
                k += 1
    sm = np.sort(mask, kind="stable")
    tiles = (n + 127) // 128
    pad = np.zeros(tiles * 128, np.uint32)
    pad[:n] = sm
    rows = pad.reshape(tiles, 128)
    act = ((rows[:, :, None] >> np.arange(KV, dtype=np.uint32)) & 1).any(1)       # [tiles, kv]
    return act


def snake(tiles, chunks, c):
    i = np.arange(tiles // chunks + 2)
    r = i * chunks + np.where(i & 1, chunks - 1 - c, c)
    return r[r < tiles]


def lpt(counts, passes):
    bins, load = [[] for _ in range(passes)], [0] * passes
    for g in sorted(range(len(counts)), key=lambda g: (-counts[g], g)):
        b = min((i for i in range(passes) if len(bins[i]) < G), key=lambda i: (load[i], i))
        bins[b].append(g)
        load[b] += counts[g]
    return bins


def model(act, pairing, balance, sms):
    tiles = act.shape[0]
    groups = (KV + APG - 1) // APG
    slots = list(range(groups * APG))
    if pairing == "mirror":
        off = [KV if s >= KV else ((KV - 1 - (s >> 1)) if s & 1 else (s >> 1)) for s in slots]
    else:
        off = [s if s < KV else KV for s in slots]
    half = np.zeros((tiles, groups, APG), bool)                 # [tile, group, warpgroup]: atom active
    for g in range(groups):
        for s in range(APG):
            k = off[g * APG + s]
            if k < KV:
                half[:, g, s] = act[:, k]
    gact = half.any(2)
    passes = (groups + G - 1) // G
    chunks = sms // passes
    bins = ([[g for g in range(groups) if g % passes == p] for p in range(passes)] if balance == "round-robin"
            else lpt(gact.sum(0).tolist(), passes))
    cost = act.sum(1)
    cost[cost == 0] = 1
    rec = np.argsort(-cost, kind="stable")                      # schedule records: decreasing offset count
    rows, worst = [], 0
    for p, gs in enumerate(bins):
        per = [int(gact[rec[snake(tiles, chunks, c)]][:, gs].sum()) for c in range(chunks)]
        worst = max(worst, max(per))
        rows.append((p, gs, int(gact[:, gs].sum()), min(per), float(np.mean(per)), max(per)))
    units_old = 2 * int(gact.sum())                             # both warpgroups multiply every stage
    units_new = int(half.sum())                                 # only warpgroups with an active atom
    return rows, worst, int(gact.sum()), units_old, units_new


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--voxels", type=int, default=100_000)
    ap.add_argument("--seed", type=int, default=50051)
    ap.add_argument("--sms", type=int, default=132)
    a = ap.parse_args()
    act = tile_masks(surface_cloud(np.random.default_rng(a.seed), KITTI, a.voxels), KITTI)
    print(f"cloud: surface_cloud(default_rng({a.seed}), {KITTI}, {a.voxels}): {act.shape[0]} tiles, "
          f"{int(act.sum())} active (tile, offset) pairs")
    for label, pairing, balance in (("mirror pairs, round-robin passes (previous kernel)", "mirror", "round-robin"),
                                    ("natural pairs, round-robin passes (kernel)", "natural", "round-robin"),
                                    ("mirror pairs, LPT passes", "mirror", "lpt"),
                                    ("natural pairs, LPT passes", "natural", "lpt")):
        rows, worst, stages, u_old, u_new = model(act, pairing, balance, a.sms)
        print(f"\n{label}: {stages} stages, busiest CTA {worst} stages; warpgroup-atom wgmma units: "
              f"{u_old} issued by both warpgroups, {u_new} with an active atom")
        for p, gs, st, lo, mean, hi in rows:
            print(f"  pass {p} groups {gs}: {st} stages; per CTA min {lo} mean {mean:.1f} max {hi}")


if __name__ == "__main__":
    main()
