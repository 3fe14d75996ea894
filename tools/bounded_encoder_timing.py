"""Step time of nets with strided layers: (a) eager with exact shapes (one output-count read-back per strided
layer), (b) eager with output bounds (no read-back, padded rows), (c) the bounded step replayed as one CUDA graph.

Workloads: the six-layer SECOND encoder at 100 k voxels (fp16, forward + backward) and one SparseConv3d
64 -> 128, stride 2, at 300 k voxels (bf16, forward + backward), each on four rotating clouds padded to one size.
The variants alternate inside one process; a number is the median over ``--reps`` windows of ``--steps`` steps,
timed with CUDA events and closed by a synchronise.  Also times the rulebook call alone, bounded against
stage 1 + stage 2.  Prints one JSON line with the card's name and power limit.

    python tools/bounded_encoder_timing.py [--steps 20] [--reps 3] [--margins 1.0,1.25,1.5]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_utils import make_encoder6, surface_cloud  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().split("\n")[0]
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown"}


def window(fn, steps):
    beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    beg.record()
    for s in range(steps):
        fn(s)
    end.record()
    torch.cuda.synchronize()
    return beg.elapsed_time(end) / steps


def measure(variants, steps, reps, warmup=5):
    """variants: {name: fn(step index)}; alternating windows, median ms per step"""
    for fn in variants.values():
        for s in range(warmup):
            fn(s)
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(reps):
        for k, fn in variants.items():
            times[k].append(window(fn, steps))
    return {k: round(statistics.median(v), 4) for k, v in times.items()}


def run_net(spconv, name, make_net, shape, n, c_in, dtype, margins, steps, reps, dev):
    rng = np.random.default_rng(0)
    clouds = [torch.from_numpy(surface_cloud(rng, shape, n - 3000 * j)).to(dev) for j in range(4)]
    feats = [torch.randn((c.shape[0], c_in), device=dev).to(dtype) for c in clouds]
    n_pad = (n + 127) // 128 * 128
    largest = spconv.SparseConvTensor(feats[0], clouds[0], shape, 1)
    torch.manual_seed(0)
    base = make_net().to(dev).to(dtype)

    def make_step(net):
        params = list(net.parameters())

        def step(f, i, nv=None):
            for p in params:
                p.grad = None
            x = spconv.SparseConvTensor(f, i, shape, 1)
            x.num_valid = nv
            y = net(x)
            loss = torch.where(y.valid_mask().unsqueeze(1), y.features.float(), 0.0).square().sum()
            loss.backward()
            return loss
        return step

    eager = make_step(base)
    variants = {"eager_unbounded": lambda s: eager(feats[s % 4], clouds[s % 4])}
    rows_out = {}
    keep = []
    for margin in margins:
        net = copy.deepcopy(base)
        bounds = spconv.set_output_bounds(net, largest, margin=margin)
        rows_out[str(margin)] = bounds
        padded = [spconv.SparseConvTensor(f, i, shape, 1).pad_to(n_pad) for f, i in zip(feats, clouds)]
        args = [(p.features, p.indices, p.num_valid) for p in padded]
        step = make_step(net)
        graphed = spconv.graph_capture(step, *args[0])
        keep.append((net, args, graphed))
        variants[f"eager_bounded_m{margin}"] = lambda s, step=step, args=args: step(*args[s % 4])
        variants[f"graph_bounded_m{margin}"] = lambda s, graphed=graphed, args=args: graphed(*args[s % 4])
    res = measure(variants, steps, reps)
    flagged = []
    for net, _, _ in keep:
        try:
            spconv.check_bounds(net)
        except RuntimeError as e:
            flagged.append(str(e)[:80])
    return {"workload": name, "voxels": n, "padded_rows": n_pad, "ms_per_step": res, "bounds": rows_out,
            "bound_exceeded": flagged}


def run_rulebook(shape, n, steps, reps, dev):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(1)
    inds = torch.from_numpy(surface_cloud(rng, shape, n)).to(dev)

    def call(bound):
        return ops.get_indice_pairs_implicit_gemm(inds, 1, shape, ConvAlgo.MaskImplicitGemm, [3] * 3, [2] * 3, [1] * 3,
                                                  [1] * 3, [0] * 3, False, False, num_out_act_bound=bound)
    m = call(-1)[0].shape[0]
    variants = {"stage1_stage2": lambda s: call(-1)}
    for margin in (1.0, 1.25, 1.5):
        b = (int(m * margin) + 127) // 128 * 128
        variants[f"bounded_m{margin}"] = lambda s, b=b: call(b)
    return {"workload": "rulebook 3x3x3 stride 2", "voxels": n, "outputs": m, "ms_per_call": measure(variants, steps, reps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--margins", default="1.0,1.25,1.5")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bounded_encoder_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    margins = [float(m) for m in a.margins.split(",")]
    kitti = [41, 1600, 1408]
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "results": []}
    out["results"].append(run_net(
        spconv, "second_encoder6_fp16", lambda: spconv.SparseSequential(*make_encoder6(spconv, bias=True, relu=True)),
        kitti, 100_000, 16, torch.float16, margins, a.steps, a.reps, dev))
    out["results"].append(run_net(
        spconv, "sparseconv3d_k3s2_c64_128_bf16", lambda: spconv.SparseSequential(
            spconv.SparseConv3d(64, 128, 3, stride=2, padding=1, bias=False, indice_key="d")),
        [41, 1440, 1440], 300_000, 64, torch.bfloat16, margins, a.steps, a.reps, dev))
    out["results"].append(run_rulebook(kitti, 100_000, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
