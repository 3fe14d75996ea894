"""Time the grouped sparse convolution against what a user has without it, on one shared SubM 3^3 rulebook
(``bench_utils.surface_cloud``, 100 k voxels on a 41 x 1600 x 1408 grid, MaskImplicitGemm), fp16 and bf16:
  * ``grouped``: ``SubMConv3d(C, K, 3, groups=g)``;
  * ``dense``: ``SubMConv3d(C, K, 3)``, g times the FLOPs and weights;
  * ``sliced``: the workaround, g ``SubMConv3d(C / g, K / g, 3)`` layers on feature slices and ``torch.cat``.
(C, K, g) in (64, 64, 2), (128, 128, 4), (256, 256, 8), (256, 256, 16), (512, 512, 4).  Per variant: the module forward
(``fwd``) and forward + backward (``step``), eager, the rulebook built once before timing.  A number is the median
over ``--reps`` windows of ``--steps`` calls, CUDA events closed by a synchronise, the variants alternating in one
process, every shape warmed up first.  Algorithmic bytes of a grouped forward, for comparison with 3.35 TB/s:
N C e (features) + kv N 4 (table) + K kv C / g e (filter) + N K e (output).  Prints one JSON line per shape and one
with the card's name and power limit.

    python tools/grouped_conv_timing.py [--steps 20] [--reps 5]
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

from bench_utils import surface_cloud  # noqa: E402
from tools.bounded_encoder_timing import card, measure  # noqa: E402

SHAPE = [41, 1600, 1408]
CASES = [(64, 64, 2), (128, 128, 4), (256, 256, 8), (256, 256, 16), (512, 512, 4)]


def run(spconv, inds, c, k, g, dtype, steps, reps, dev):
    from spconv_b200.pytorch import ops
    n = inds.shape[0]
    torch.manual_seed(c + g)
    key = "s"
    grouped = spconv.SubMConv3d(c, k, 3, groups=g, indice_key=key, bias=False).to(dev).to(dtype).train()
    dense = spconv.SubMConv3d(c, k, 3, indice_key=key, bias=False).to(dev).to(dtype).train()
    parts = [spconv.SubMConv3d(c // g, k // g, 3, indice_key=key, bias=False).to(dev).to(dtype).train()
             for _ in range(g)]
    x0 = spconv.SparseConvTensor(torch.randn((n, c), device=dev).to(dtype), inds, SHAPE, 1)
    with torch.no_grad():
        x = grouped(x0).replace_feature(x0.features)      # the rulebook, built once and shared by every variant
    feats = x.features.detach().clone().requires_grad_(True)
    xt = x.replace_feature(feats)
    dy = torch.randn((n, k), device=dev).to(dtype)
    cg = c // g

    def sliced(t):
        return torch.cat([m(t.replace_feature(t.features[:, j * cg:(j + 1) * cg])).features
                          for j, m in enumerate(parts)], 1)

    fwd = {
        "grouped": lambda s: grouped(xt).features,
        "dense": lambda s: dense(xt).features,
        "sliced": lambda s: sliced(xt),
    }

    def step(f):
        def go(s):
            f(s).backward(dy)
        return go

    with torch.no_grad():
        t_fwd = measure(fwd, steps, reps)
    t_step = measure({name: step(f) for name, f in fwd.items()}, steps, reps)
    with torch.no_grad():
        grouped(xt)
    fam = ops.last_kernel_family()
    e = torch.tensor([], dtype=dtype).element_size()
    fwd_bytes = n * c * e + 27 * n * 4 + k * 27 * cg * e + n * k * e
    return {"C": c, "K": k, "groups": g, "dtype": str(dtype).replace("torch.", ""), "voxels": n,
            "family": "tensor cores" if fam == 2 else "FMA",
            "fwd_ms": t_fwd, "fwd_bwd_ms": t_step, "grouped_fwd_bytes": fwd_bytes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--voxels", type=int, default=100_000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "grouped_conv_timing needs a CUDA device"
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    inds = torch.from_numpy(surface_cloud(np.random.default_rng(0), SHAPE, args.voxels)).to(dev)
    print(json.dumps(card()), flush=True)
    for dtype in (torch.float16, torch.bfloat16):
        for c, k, g in CASES:
            print(json.dumps(run(spconv, inds, c, k, g, dtype, args.steps, args.reps, dev)), flush=True)


if __name__ == "__main__":
    main()
