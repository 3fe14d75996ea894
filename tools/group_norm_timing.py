"""Time MaskedGroupNorm, forward and backward, as CUDA-graph replays (device time), at 100 k x 64 fp16 (B = 4, G = 32),
300 k x 128 bf16 (B = 8, G = 32) and 100 k x 64 fp16 instance norm (B = 4, G = 64).  Beside it, on the same matrix:
the eager per-sample torch loop (``F.group_norm`` on each sample's rows, forward + backward; it reads the sample
masks back, so it cannot be captured) and MaskedBatchNorm1d replayed, as a bandwidth yardstick.  Then the
modulated norm of a diffusion ResBlock, y = silu(GN(x) * (1 + scale[b]) + shift[b]) with scale / shift [B, C]
fp32 leaves, both replayed: the fused call (``MaskedGroupNorm(act="silu")(x, scale, shift)``) and the torch chain
a user writes without it (MaskedGroupNorm, then the gather by batch id, ``1 + s``, ``+ t`` and ``F.silu``, with
autograd; it does not synchronise, so it captures too).

The backward is the forward + backward time minus the forward time.  Achieved bandwidth uses the algorithmic bytes:
forward 3 N C e (read x twice, write y) plus 16 bytes a row for the grouping (read the batch index, write and read
the key, write the row order), backward 5 N C e (read x and dy twice, write dx); the fused modulated call moves the
same bytes (scale and shift are [B, C]).  The torch chain adds, counted from its passes over [N, C], 8 N C e in the
forward (two gathers written, the modulate and the SiLU pass, each reading and writing) and 11 N C e in the backward
(SiLU backward 3, the two products 3 + 3, the two gathers' accumulating backwards reading 1 each).  Launches per
call are counted by the library for the plain call and by torch.profiler for the modulated legs.  A number is the median over
``--reps`` windows of ``--steps`` steps, CUDA events closed by a synchronise, the variants alternating in one
process.  Prints one JSON line with the card's name and power limit.

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

    scale = (torch.rand((b, c), device=dev) - 0.5).requires_grad_(True)
    shift = (torch.rand((b, c), device=dev) - 0.5).requires_grad_(True)
    ada = spconv.MaskedGroupNorm(groups, c, act="silu").to(dev)
    plain = spconv.MaskedGroupNorm(groups, c).to(dev)
    long_ids = ids.long()

    def fused_fwd():
        return ada(spconv.SparseConvTensor(x, inds, [4, 4, 4], b), scale, shift).features

    def chain_fwd():
        h = plain(spconv.SparseConvTensor(x, inds, [4, 4, 4], b)).features
        return torch.nn.functional.silu(h * (1 + scale[long_ids]) + shift[long_ids])

    def loop_fwd():
        # what a user writes today: a boolean mask per sample (a read-back in nonzero), one group_norm per sample
        y = torch.zeros_like(x)
        for s in range(b):
            sel = (ids == s).nonzero().squeeze(1)
            y = y.index_put((sel,), ref(x[sel].T[None])[0].T)
        return y

    variants = {}
    legs = (("masked_group_norm", gn_fwd, True), ("masked_batch_norm", bn_fwd, True),
            ("torch_loop", loop_fwd, False), ("adagn_silu_fused", fused_fwd, True),
            ("adagn_silu_torch_chain", chain_fwd, True))
    for name, f, graph in legs:
        def fwd(f=f):
            f()

        def fwd_bwd(f=f):
            x.grad = scale.grad = shift.grad = None
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
    gn_bytes = (3 * n * c * e + 16 * n, 5 * n * c * e)
    nbytes = {"masked_group_norm": gn_bytes, "masked_batch_norm": (3 * n * c * e, 5 * n * c * e),
              "torch_loop": (3 * n * c * e, 5 * n * c * e), "adagn_silu_fused": gn_bytes,
              "adagn_silu_torch_chain": (gn_bytes[0] + 8 * n * c * e, gn_bytes[1] + 11 * n * c * e)}
    for name, _, _ in legs:
        f = ms[f"{name}_fwd"]
        bw = ms[f"{name}_fwd_bwd"] - f
        out["derived"][name] = {
            "fwd_ms": round(f, 4), "bwd_ms": round(bw, 4), "fwd_bytes": nbytes[name][0], "bwd_bytes": nbytes[name][1],
            "fwd_of_peak": round(nbytes[name][0] / f / 1e6 / HBM_GBS, 3),
            "bwd_of_peak": round(nbytes[name][1] / bw / 1e6 / HBM_GBS, 3) if bw > 0 else None}
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
    # launches of the modulated legs, library and torch kernels alike
    for name, f in (("adagn_silu_fused", fused_fwd), ("adagn_silu_torch_chain", chain_fwd)):
        out["derived"][name]["launches_fwd"], out["derived"][name]["launches_bwd"] = launches(f, x, scale, shift, dy)
    # the two agree
    with torch.no_grad():
        a = gn_fwd().float()
        r = loop_fwd().float()
        out["max_abs_diff_vs_torch_loop"] = float((a - r).abs().max())
        out["adagn_max_abs_diff_fused_vs_chain"] = float((fused_fwd().float() - chain_fwd().float()).abs().max())
    return out


def launches(f, x, scale, shift, dy):
    """kernels run by one forward and by its backward, the library's and torch's, from torch.profiler's device
    activity (copies and memsets not counted)"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    def count(fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        return sum(1 for ev in prof.events() if ev.device_type == DeviceType.CUDA
                   and not ev.name.startswith(("Memcpy", "Memset"))), out

    x.grad = scale.grad = shift.grad = None
    n_fwd, y = count(f)
    n_bwd, _ = count(lambda: y.backward(dy))
    return n_fwd, n_bwd


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
