"""Time MaskedBatchNorm1d: (1) the BatchNorm alone, forward and forward + backward, against nn.BatchNorm1d (cuDNN) on
the same valid rows, at 100 k x 64 fp16 and 300 k x 128 bf16; (2) a SECOND-style six-layer encoder step with
conv -> BatchNorm -> ReLU at 100 k voxels, fp16: eager with exact shapes and nn.BatchNorm1d, eager bounded with
MaskedBatchNorm1d, and the bounded step replayed as one CUDA graph.

BatchNorm alone is timed twice: eager (a Python call per step, so host time counts) and as CUDA-graph replays
(device time).  The backward is the forward + backward time minus the forward time.  Achieved bandwidth uses the
algorithmic bytes: forward 3 N C e (read x twice, write y), backward 5 N C e (read x and dy twice, write dx).
A number is the median over ``--reps`` windows of ``--steps`` steps, CUDA events closed by a synchronise, the
variants alternating in one process.  Prints one JSON line with the card's name and power limit.

    python tools/masked_bn_timing.py [--steps 50] [--reps 5]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import sys

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_utils import make_encoder6, surface_cloud  # noqa: E402
from tools.bounded_encoder_timing import card, measure  # noqa: E402

HBM_GBS = 3350.0       # H100 SXM data sheet


def graphed(fn):
    """capture fn() (after a warm-up on a side stream) and return a replay callable"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def run_bn_alone(spconv, n, c, dtype, steps, reps, dev):
    torch.manual_seed(0)
    x = (torch.randn((n, c), device=dev) * 1.5 + 0.3).to(dtype).requires_grad_(True)
    dy = torch.randn((n, c), device=dev).to(dtype)
    inds = torch.zeros((n, 4), dtype=torch.int32, device=dev)        # BatchNorm does not look at them
    ours = spconv.MaskedBatchNorm1d(c).to(dev)
    cudnn = nn.BatchNorm1d(c).to(dev)
    fns = {
        "masked": lambda: ours(spconv.SparseConvTensor(x, inds, [4, 4, 4], 1)).features,
        "cudnn": lambda: cudnn(x),
    }
    variants = {}
    for name, f in fns.items():
        def fwd(f=f):
            f()

        def fwd_bwd(f=f):
            x.grad = None
            f().backward(dy)
        variants[f"{name}_fwd_eager"] = lambda s, fn=fwd: fn()
        variants[f"{name}_fwd_bwd_eager"] = lambda s, fn=fwd_bwd: fn()
        g_fwd, g_fb = graphed(fwd), graphed(fwd_bwd)
        variants[f"{name}_fwd_graph"] = lambda s, fn=g_fwd: fn()
        variants[f"{name}_fwd_bwd_graph"] = lambda s, fn=g_fb: fn()
    ms = measure(variants, steps, reps)
    e = x.element_size()
    out = {"rows": n, "channels": c, "dtype": str(dtype).replace("torch.", ""), "ms": ms, "derived": {}}
    for name in fns:
        for mode in ("eager", "graph"):
            f = ms[f"{name}_fwd_{mode}"]
            b = ms[f"{name}_fwd_bwd_{mode}"] - f
            out["derived"][f"{name}_{mode}"] = {
                "fwd_ms": round(f, 4), "bwd_ms": round(b, 4),
                "fwd_gbs": round(3 * n * c * e / f / 1e6, 1), "bwd_gbs": round(5 * n * c * e / b / 1e6, 1) if b > 0 else None,
                "fwd_of_peak": round(3 * n * c * e / f / 1e6 / HBM_GBS, 3),
                "bwd_of_peak": round(5 * n * c * e / b / 1e6 / HBM_GBS, 3) if b > 0 else None}
    # the two agree on the valid rows
    with torch.no_grad():
        a = fns["masked"]().float()
        r = nn.functional.batch_norm(x, None, None, cudnn.weight, cudnn.bias, True, 0.0, cudnn.eps).float()
        out["max_abs_diff_vs_cudnn"] = float((a - r).abs().max())
    return out


def run_encoder(spconv, n, steps, reps, dev, margin):
    shape = [41, 1600, 1408]
    rng = np.random.default_rng(0)
    clouds = [torch.from_numpy(surface_cloud(rng, shape, n - 3000 * j)).to(dev) for j in range(4)]
    feats = [torch.randn((c.shape[0], 16), device=dev).half() for c in clouds]
    n_pad = (n + 127) // 128 * 128
    torch.manual_seed(0)
    layers = []
    for conv in make_encoder6(spconv, bias=False):
        layers += [conv, nn.BatchNorm1d(conv.out_channels), nn.ReLU()]
    plain = spconv.SparseSequential(*layers).to(dev).half()
    masked = spconv.MaskedBatchNorm1d.convert_masked_batchnorm(copy.deepcopy(plain))

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

    eager = make_step(plain)
    bounds = spconv.set_output_bounds(masked, spconv.SparseConvTensor(feats[0], clouds[0], shape, 1), margin=margin)
    padded = [spconv.SparseConvTensor(f, i, shape, 1).pad_to(n_pad) for f, i in zip(feats, clouds)]
    args = [(p.features, p.indices, p.num_valid) for p in padded]
    step = make_step(masked)
    graph = spconv.graph_capture(step, *args[0])
    variants = {
        "eager_exact_batchnorm1d": lambda s: eager(feats[s % 4], clouds[s % 4]),
        "eager_bounded_masked": lambda s: step(*args[s % 4]),
        "graph_bounded_masked": lambda s: graph(*args[s % 4]),
    }
    res = measure(variants, steps, reps)
    spconv.check_bounds(masked)
    return {"workload": "second_encoder6_conv_bn_relu_fp16", "voxels": n, "padded_rows": n_pad, "margin": margin,
            "bounds": bounds, "ms_per_step": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--margin", type=float, default=1.25)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("masked_bn_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "batchnorm": [], "encoder": None}
    out["batchnorm"].append(run_bn_alone(spconv, 100_000, 64, torch.float16, a.steps, a.reps, dev))
    out["batchnorm"].append(run_bn_alone(spconv, 300_000, 128, torch.bfloat16, a.steps, a.reps, dev))
    out["encoder"] = run_encoder(spconv, 100_000, max(a.steps // 2, 10), a.reps, dev, a.margin)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
