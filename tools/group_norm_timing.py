"""Time MaskedGroupNorm, forward and backward, as CUDA-graph replays (device time), at 100 k x 64 fp16 (B = 4, G = 32),
300 k x 128 bf16 (B = 8, G = 32) and 100 k x 64 fp16 instance norm (B = 4, G = 64).  Beside it, on the same matrix:
the eager per-sample torch loop (``F.group_norm`` on each sample's rows, forward + backward; it reads the sample
masks back, so it cannot be captured) and MaskedBatchNorm1d replayed, as a bandwidth yardstick.

The backward is the forward + backward time minus the forward time.  Achieved bandwidth uses the algorithmic bytes:
forward 3 N C e (read x twice, write y) plus 16 bytes a row for the grouping (read the batch index, write and read
the key, write the row order), backward 5 N C e (read x and dy twice, write dx).  Launches per call are counted by
the library.  A number is the median over ``--reps`` windows of ``--steps`` steps, CUDA events closed by a
synchronise, the variants alternating in one process.  Prints one JSON line with the card's name and power limit.

    python tools/group_norm_timing.py [--steps 50] [--reps 5]
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


def run(spconv, ops, n, c, b, groups, dtype, steps, reps, dev):
    torch.manual_seed(0)
    ids = torch.randint(0, b, (n,), dtype=torch.int32, device=dev)
    inds = torch.zeros((n, 4), dtype=torch.int32, device=dev)
    inds[:, 0] = ids
    x = (torch.randn((n, c), device=dev) * 1.5 + 0.3).to(dtype).requires_grad_(True)
    dy = torch.randn((n, c), device=dev).to(dtype)
    gn = spconv.MaskedGroupNorm(groups, c).to(dev)
    bn = spconv.MaskedBatchNorm1d(c).to(dev)
    ref = torch.nn.GroupNorm(groups, c).to(dev).to(dtype)        # torch wants the parameters in x's dtype

    def gn_fwd():
        return gn(spconv.SparseConvTensor(x, inds, [4, 4, 4], b)).features

    def bn_fwd():
        return bn(spconv.SparseConvTensor(x, inds, [4, 4, 4], b)).features

    def loop_fwd():
        # what a user writes today: a boolean mask per sample (a read-back in nonzero), one group_norm per sample
        y = torch.zeros_like(x)
        for s in range(b):
            sel = (ids == s).nonzero().squeeze(1)
            y = y.index_put((sel,), ref(x[sel].T[None])[0].T)
        return y

    variants = {}
    for name, f, graph in (("masked_group_norm", gn_fwd, True), ("masked_batch_norm", bn_fwd, True),
                           ("torch_loop", loop_fwd, False)):
        def fwd(f=f):
            f()

        def fwd_bwd(f=f):
            x.grad = None
            f().backward(dy)
        if graph:
            variants[f"{name}_fwd"] = lambda s, fn=graphed(fwd): fn()
            variants[f"{name}_fwd_bwd"] = lambda s, fn=graphed(fwd_bwd): fn()
        else:
            variants[f"{name}_fwd"] = lambda s, fn=fwd: fn()
            variants[f"{name}_fwd_bwd"] = lambda s, fn=fwd_bwd: fn()
    ms = measure(variants, steps, reps)
    e = x.element_size()
    out = {"rows": n, "channels": c, "batch": b, "groups": groups, "dtype": str(dtype).replace("torch.", ""),
           "ms": ms, "derived": {}}
    fwd_bytes = {"masked_group_norm": 3 * n * c * e + 16 * n, "masked_batch_norm": 3 * n * c * e,
                 "torch_loop": 3 * n * c * e}
    for name in ("masked_group_norm", "masked_batch_norm", "torch_loop"):
        f = ms[f"{name}_fwd"]
        bw = ms[f"{name}_fwd_bwd"] - f
        out["derived"][name] = {
            "fwd_ms": round(f, 4), "bwd_ms": round(bw, 4),
            "fwd_of_peak": round(fwd_bytes[name] / f / 1e6 / HBM_GBS, 3),
            "bwd_of_peak": round(5 * n * c * e / bw / 1e6 / HBM_GBS, 3) if bw > 0 else None}
    # launches per call of the library's entry points
    torch.cuda.synchronize()
    ops.launch_count(reset=True)
    y = gn_fwd()
    torch.cuda.synchronize()
    out["launches_fwd"] = ops.launch_count(reset=True)
    x.grad = None
    y.backward(dy)
    torch.cuda.synchronize()
    out["launches_bwd"] = ops.launch_count(reset=True)
    # the two agree
    with torch.no_grad():
        a = gn_fwd().float()
        r = loop_fwd().float()
        out["max_abs_diff_vs_torch_loop"] = float((a - r).abs().max())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("group_norm_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "group_norm": []}
    for n, c, b, g, dt in ((100_000, 64, 4, 32, torch.float16), (300_000, 128, 8, 32, torch.bfloat16),
                           (100_000, 64, 4, 64, torch.float16)):
        out["group_norm"].append(run(spconv, ops, n, c, b, g, dt, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
