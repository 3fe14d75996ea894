"""Time functional.sparse_add on LiDAR-like clouds (C = 64, fp16) and the reference's formulation.

    python tools/sparse_add_timing.py [--iters 50]

Two cases: two ~100 k-voxel surface clouds that share about half of their voxels, and the USAGE.md case of
three operands whose largest holds the other two's coordinates.  Prints one JSON line per case: CUDA-event
times of the union (1x1 rulebook, including its host read-back), the grouping, the forward sum kernel and
the backward gather kernel; algorithmic bytes of the two feature kernels over their time against the
3.35 TB/s data-sheet bandwidth of the H100 SXM; the whole sparse_add call; and the reference's formulation
(sum of torch.sparse_coo_tensor + coalesce + index conversion) on the same inputs.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_utils import surface_cloud  # noqa: E402

PEAK_BPS = 3.35e12
SHAPE = [41, 1600, 1408]


def _power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def _subset(rng, inds, frac):
    return inds[np.sort(rng.permutation(len(inds))[:int(frac * len(inds))])]


def _cases(rng):
    a = surface_cloud(rng, SHAPE, 100_000)
    other = surface_cloud(rng, SHAPE, 100_000)
    key = lambda x: (x[:, 1].astype(np.int64) * SHAPE[1] + x[:, 2]) * SHAPE[2] + x[:, 3]  # noqa: E731
    fresh = other[~np.isin(key(other), key(a))][:50_000]
    b = np.concatenate([_subset(rng, a, 0.5), fresh], 0)
    b = b[rng.permutation(len(b))]
    yield "two_clouds_half_overlap", [a, b]
    big = surface_cloud(rng, SHAPE, 100_000)
    yield "usage_three_operands", [_subset(rng, big, 0.6), _subset(rng, big, 0.6), big]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import functional as Fsp, ops
    dev = torch.device("cuda")
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit": _power_limit()}), flush=True)
    rng = np.random.default_rng(0)
    c = 64
    for name, clouds in _cases(rng):
        tens = [spconv.SparseConvTensor(torch.randn(len(x), c, device=dev, dtype=torch.float16),
                                        torch.from_numpy(x).to(dev), SHAPE, 1) for x in clouds]
        rows = [t.features.shape[0] for t in tens]
        largest = max(range(len(rows)), key=lambda i: (rows[i], -i))
        visit = [largest] + [i for i in range(len(rows)) if i != largest]
        vi = [tens[i].indices for i in visit]
        vf = [tens[i].features for i in visit]
        out_inds, dst = ops.sparse_add_union(vi, 1, SHAPE)
        m = out_inds.shape[0]
        order, offsets = ops.sparse_add_group(dst, m)
        out = torch.empty((m, c), dtype=torch.float16, device=dev)
        dout = torch.randn(m, c, dtype=torch.float16, device=dev)
        grads = [torch.empty_like(f) for f in vf]
        n = sum(rows)
        kept = int((dst >= 0).sum())
        t_union = _time(lambda: ops.sparse_add_union(vi, 1, SHAPE), args.iters)
        t_group = _time(lambda: ops.sparse_add_group(dst, m), args.iters)
        t_fwd = _time(lambda: ops.sparse_add_forward(vf, order, offsets, m, out=out), args.iters)
        t_bwd = _time(lambda: ops.sparse_add_gather(dst, dout, [len(f) for f in vf], outs=grads), args.iters)
        row = c * 2
        fwd_bytes = kept * row + m * row + 4 * kept + 4 * (m + 1)          # rows read, rows written, order, offsets
        bwd_bytes = 4 * n + kept * row + n * row                           # dst, dout rows read, every grad row written
        t_call = _time(lambda: Fsp.sparse_add(*tens), args.iters)

        def reference():
            full = [1, *SHAPE, c]
            acc = None
            for t in tens:
                s = torch.sparse_coo_tensor(t.indices.T, t.features, full)
                acc = s if acc is None else acc + s
            acc = acc.coalesce()
            return acc.indices().T.contiguous().int(), acc.values()

        t_ref = _time(reference, args.iters)
        print(json.dumps({
            "case": name, "rows": rows, "outputs": m, "channels": c, "dtype": "float16",
            "union_ms": round(t_union, 4), "group_ms": round(t_group, 4),
            "fwd_sum_kernel_ms": round(t_fwd, 4), "bwd_gather_kernel_ms": round(t_bwd, 4),
            "fwd_bytes": fwd_bytes, "fwd_TBps": round(fwd_bytes / (t_fwd * 1e-3) / 1e12, 3),
            "fwd_frac_of_3.35TBps": round(fwd_bytes / (t_fwd * 1e-3) / PEAK_BPS, 3),
            "bwd_bytes": bwd_bytes, "bwd_TBps": round(bwd_bytes / (t_bwd * 1e-3) / 1e12, 3),
            "bwd_frac_of_3.35TBps": round(bwd_bytes / (t_bwd * 1e-3) / PEAK_BPS, 3),
            "sparse_add_call_ms": round(t_call, 4), "reference_torch_sparse_ms": round(t_ref, 4),
        }), flush=True)


if __name__ == "__main__":
    main()
