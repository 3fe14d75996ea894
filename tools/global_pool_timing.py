"""Time MaskedGlobalMaxPool / MaskedGlobalAvgPool, forward and forward + backward, against the default
SparseGlobalMaxPool / SparseGlobalAvgPool (a host read-back of the sample counts, then a gather and a torch
reduction per sample) at 100 k x 64 fp16 with 8 samples and 300 k x 128 bf16 with 16 samples, samples interleaved.

The new modules are timed eagerly (a Python call per step, so host time counts) and as CUDA-graph replays (device
time); the default modules synchronise, so they only run eagerly.  The backward is the forward + backward time
minus the forward time.  Achieved bandwidth uses the algorithmic bytes: the forward reads the features and the
indices, N C e + N (ndim + 1) 4; the backward writes the features' gradient, N C e.  A number is the median over
``--reps`` windows of ``--steps`` steps, CUDA events closed by a synchronise, the variants alternating in one
process.  Prints one JSON line with the card's name and power limit.

    python tools/global_pool_timing.py [--steps 50] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bounded_encoder_timing import card, measure  # noqa: E402
from tools.masked_bn_timing import HBM_GBS, graphed  # noqa: E402


def run(spconv, n, c, b, dtype, steps, reps, dev):
    torch.manual_seed(0)
    x = torch.randn((n, c), device=dev).to(dtype).requires_grad_(True)
    inds = torch.randint(0, 200, (n, 4), dtype=torch.int32, device=dev)
    inds[:, 0] = torch.randint(0, b, (n,), dtype=torch.int32, device=dev)
    dy = torch.randn((b, c), device=dev).to(dtype)
    t = spconv.SparseConvTensor(x, inds, [200, 200, 200], b)
    mods = {"masked_max": spconv.MaskedGlobalMaxPool(), "masked_avg": spconv.MaskedGlobalAvgPool(),
            "default_max": spconv.SparseGlobalMaxPool(), "default_avg": spconv.SparseGlobalAvgPool()}
    variants = {}
    for name, mod in mods.items():
        def fwd(mod=mod):
            mod(t)

        def fwd_bwd(mod=mod):
            x.grad = None
            mod(t).backward(dy)
        variants[f"{name}_fwd_eager"] = lambda s, fn=fwd: fn()
        variants[f"{name}_fwd_bwd_eager"] = lambda s, fn=fwd_bwd: fn()
        if name.startswith("masked"):
            g_fwd, g_fb = graphed(fwd), graphed(fwd_bwd)
            variants[f"{name}_fwd_graph"] = lambda s, fn=g_fwd: fn()
            variants[f"{name}_fwd_bwd_graph"] = lambda s, fn=g_fb: fn()
    ms = measure(variants, steps, reps)
    e = x.element_size()
    fwd_bytes = n * c * e + n * inds.shape[1] * 4
    bwd_bytes = n * c * e
    out = {"rows": n, "channels": c, "batch": b, "dtype": str(dtype).replace("torch.", ""), "ms": ms, "derived": {}}
    for name in mods:
        for mode in ("eager", "graph"):
            if f"{name}_fwd_{mode}" not in ms:
                continue
            f = ms[f"{name}_fwd_{mode}"]
            bw = ms[f"{name}_fwd_bwd_{mode}"] - f
            out["derived"][f"{name}_{mode}"] = {
                "fwd_ms": round(f, 4), "bwd_ms": round(bw, 4),
                "fwd_gbs": round(fwd_bytes / f / 1e6, 1), "bwd_gbs": round(bwd_bytes / bw / 1e6, 1) if bw > 0 else None,
                "fwd_of_peak": round(fwd_bytes / f / 1e6 / HBM_GBS, 3),
                "bwd_of_peak": round(bwd_bytes / bw / 1e6 / HBM_GBS, 3) if bw > 0 else None}
    with torch.no_grad():                                  # the new and the default modules agree
        out["max_bitwise_equal"] = bool(torch.equal(mods["masked_max"](t), mods["default_max"](t)))
        out["avg_max_abs_diff"] = float((mods["masked_avg"](t).float() - mods["default_avg"](t).float()).abs().max())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("global_pool_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "pool": []}
    out["pool"].append(run(spconv, 100_000, 64, 8, torch.float16, a.steps, a.reps, dev))
    out["pool"].append(run(spconv, 300_000, 128, 16, torch.bfloat16, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
