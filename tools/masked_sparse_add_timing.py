"""Time functional.masked_sparse_add, forward and forward + backward, eagerly and as CUDA-graph replays, against the
eager functional.sparse_add on the same valid rows, at the two sizes of tools/sparse_add_timing.py (C = 64, fp16):
two ~100 k-voxel clouds that share half their voxels, and the USAGE.md case of 60 k + 60 k + 100 k rows.

Each operand of the masked call is padded by 10 % with junk rows (num_valid = its true row count), as a captured net
would feed it.  The eager calls include the host time of a Python call per step; sparse_add also reads the size of
the union back to the host (a synchronisation) and cannot be captured.  The backward is the forward + backward time
minus the forward time.  Algorithmic bytes of one masked forward: the coordinates read by the pack kernel and the
packed copy written, the union's read of it and its out_inds / dst writes, the remap (order, src, dst), the feature
rows kept read once, the `bound` output rows written; of the backward: dst read, the kept dout rows read and every
operand gradient row written.  They are set against the 3.35 TB/s data-sheet bandwidth.  Launches are the native
launches of one call (spx_launch_count).  A number is the median over ``--reps`` windows of ``--steps`` steps, CUDA
events closed by a synchronise, the variants alternating in one process, every shape warmed up first.  Prints one
JSON line with the card's name and power limit.

    python tools/masked_sparse_add_timing.py [--steps 50] [--reps 5]
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
from tools.sparse_add_timing import SHAPE, _cases  # noqa: E402


def run(spconv, name, clouds, c, steps, reps, dev):
    from spconv_b200.pytorch import functional as Fsp, ops
    torch.manual_seed(0)
    dtype = torch.float16
    feats = [torch.randn((len(x), c), device=dev).to(dtype).requires_grad_(True) for x in clouds]
    plain = [spconv.SparseConvTensor(f, torch.from_numpy(x).to(dev), SHAPE, 1) for f, x in zip(feats, clouds)]
    padded = []
    for t in plain:
        n = t.features.shape[0]
        p = t.pad_to(n + n // 10)
        p = p.replace_feature(p.features.detach().clone().requires_grad_(True))
        padded.append(p)
    ref = Fsp.sparse_add(*plain)
    m = ref.features.shape[0]
    res = Fsp.masked_sparse_add(*padded)
    bound = res.features.shape[0]
    dy_ref = torch.randn((m, c), device=dev).to(dtype)
    dy = torch.zeros((bound, c), device=dev, dtype=dtype)
    dy[:m] = dy_ref
    with torch.no_grad():
        same = bool(torch.equal(res.indices[:m], ref.indices) and torch.equal(res.features[:m], ref.features))
    del res, ref                      # an autograd graph kept alive pins the leaves' gradient nodes to this stream

    def masked_fwd():
        Fsp.masked_sparse_add(*padded)

    def masked_fwd_bwd():
        for p in padded:
            p.features.grad = None
        Fsp.masked_sparse_add(*padded).features.backward(dy)

    def default_fwd():
        Fsp.sparse_add(*plain)

    def default_fwd_bwd():
        for f in feats:
            f.grad = None
        Fsp.sparse_add(*plain).features.backward(dy_ref)

    g_fwd, g_fb = graphed(masked_fwd), graphed(masked_fwd_bwd)
    launches = {}
    for key, fn in (("masked_fwd", masked_fwd), ("masked_fwd_bwd", masked_fwd_bwd), ("default_fwd", default_fwd),
                    ("default_fwd_bwd", default_fwd_bwd)):
        fn()
        torch.cuda.synchronize()
        ops.launch_count(True)
        fn()
        torch.cuda.synchronize()
        launches[key] = ops.launch_count(True)
    variants = {
        "masked_fwd_eager": lambda s: masked_fwd(), "masked_fwd_bwd_eager": lambda s: masked_fwd_bwd(),
        "masked_fwd_graph": lambda s: g_fwd(), "masked_fwd_bwd_graph": lambda s: g_fb(),
        "default_fwd_eager": lambda s: default_fwd(), "default_fwd_bwd_eager": lambda s: default_fwd_bwd(),
    }
    ms = measure(variants, steps, reps)
    rows = sum(p.features.shape[0] for p in padded)
    valid = sum(t.features.shape[0] for t in plain)
    row = c * 2
    ncol = len(SHAPE) + 1
    fwd_bytes = (rows * ncol * 4 * 2 + rows * ncol * 4 + bound * ncol * 4 + rows * 4
                 + rows * 4 * 5 + valid * row + bound * row + (bound + 1) * 4)
    bwd_bytes = rows * 4 + valid * row + rows * row
    out = {"case": name, "valid_rows": [t.features.shape[0] for t in plain],
           "padded_rows": [p.features.shape[0] for p in padded], "outputs": m, "bound": bound, "channels": c,
           "dtype": "float16", "masked_equals_default": same, "launches": launches, "ms": ms,
           "fwd_bytes": fwd_bytes, "bwd_bytes": bwd_bytes, "derived": {}}
    for mode in ("eager", "graph"):
        f = ms[f"masked_fwd_{mode}"]
        bw = ms[f"masked_fwd_bwd_{mode}"] - f
        out["derived"][f"masked_{mode}"] = {
            "fwd_ms": round(f, 4), "bwd_ms": round(bw, 4),
            "fwd_of_peak": round(fwd_bytes / f / 1e6 / HBM_GBS, 3),
            "bwd_of_peak": round(bwd_bytes / bw / 1e6 / HBM_GBS, 3) if bw > 0 else None}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("masked_sparse_add_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "sparse_add": []}
    for name, clouds in _cases(np.random.default_rng(0)):
        out["sparse_add"].append(run(spconv, name, clouds, 64, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
