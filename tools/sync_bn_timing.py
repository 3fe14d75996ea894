"""Time MaskedSyncBatchNorm1d against MaskedBatchNorm1d, forward and forward + backward, replayed as CUDA graphs,
at 100 k x 64 fp16 and 300 k x 128 bf16 rows per rank.

World 1 is one rank with the peer route of a one-rank group and with no group.  Worlds 2 and 4 are simulated
ranks: streams of ONE GPU whose exchange buffers all live on it (``PeerGroup.local_ring``), every rank with its
own rows.  One timed step replays every rank's graph on its own stream, joined to the timing stream; the
MaskedBatchNorm1d baseline replays the same number of rank-local graphs the same way.  The ranks share the SMs
and HBM of one GPU, so these numbers show the cost of the extra kernels and of the exchange protocol, not NVLink.
The backward is the forward + backward time minus the forward time.  A number is the median over ``--reps``
windows of ``--steps`` steps (tools/bounded_encoder_timing.measure).  Launches per call are counted with
``ops.launch_count`` on one eager call of each.  Prints one JSON line with the card's name and power limit.

    python tools/sync_bn_timing.py [--steps 50] [--reps 5]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bounded_encoder_timing import card, measure  # noqa: E402


def capture_ranks(ring, fns):
    """one graph per rank (fns[r] captured with ring[r] installed, ring None: no group); returns a callable that
    replays all of them together, each on its own stream"""
    from spconv_b200.pytorch import ops
    world = len(fns)
    streams = [torch.cuda.Stream() for _ in range(world)]
    for _ in range(2):                                      # warm-up: every rank's eager call before a host wait
        torch.cuda.synchronize()
        for r in range(world):
            ops.set_peer_group(ring[r] if ring else None)
            with torch.cuda.stream(streams[r]):
                fns[r]()
        ops.set_peer_group(None)
        torch.cuda.synchronize()
    graphs = []
    for r in range(world):
        ops.set_peer_group(ring[r] if ring else None)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=streams[r]):
            fns[r]()
        graphs.append(g)
    ops.set_peer_group(None)

    def replay():
        main = torch.cuda.current_stream()
        for r in range(world):
            streams[r].wait_stream(main)
            with torch.cuda.stream(streams[r]):
                graphs[r].replay()
        for s in streams:
            main.wait_stream(s)
    return replay


def launches(ring0, fn):
    from spconv_b200.pytorch import ops
    ops.set_peer_group(ring0)
    torch.cuda.synchronize()
    ops.launch_count(True)
    fn()
    n = ops.launch_count()
    torch.cuda.synchronize()
    ops.set_peer_group(None)
    return n


def run(spconv, n, c, dtype, world, steps, reps, dev):
    from spconv_b200.pytorch.dist import PeerGroup
    torch.manual_seed(world)
    xs = [(torch.randn((n, c), device=dev) * 1.5 + 0.3).to(dtype).requires_grad_(True) for _ in range(world)]
    dys = [torch.randn((n, c), device=dev).to(dtype) for _ in range(world)]
    inds = torch.zeros((n, 4), dtype=torch.int32, device=dev)        # BatchNorm does not look at them
    plain = [spconv.MaskedBatchNorm1d(c).to(dev) for _ in range(world)]
    sync = [spconv.MaskedSyncBatchNorm1d(c).to(dev) for _ in range(world)]

    def fns(mods, backward):
        out = []
        for r in range(world):
            def f(r=r):
                y = mods[r](spconv.SparseConvTensor(xs[r], inds, [4, 4, 4], 1)).features
                if backward:
                    xs[r].grad = None
                    y.backward(dys[r])
            out.append(f)
        return out

    ring = PeerGroup.local_ring(world, capacity_bytes=1 << 20)
    try:
        variants = {}
        for bwd in (False, True):
            tag = "fwd_bwd" if bwd else "fwd"
            variants[f"masked_{tag}"] = capture_ranks(None, fns(plain, bwd))
            variants[f"sync_peer_{tag}"] = capture_ranks(ring, fns(sync, bwd))
            if world == 1:
                variants[f"sync_nogroup_{tag}"] = capture_ranks(None, fns(copy.deepcopy(sync), bwd))
        variants = {k: (lambda s, f=f: f()) for k, f in variants.items()}
        ms = measure(variants, steps, reps)
        counts = {}
        if world == 1:
            counts = {"masked_fwd": launches(None, fns(plain, False)[0]),
                      "masked_fwd_bwd": launches(None, fns(plain, True)[0]),
                      "sync_peer_fwd": launches(ring[0], fns(sync, False)[0]),
                      "sync_peer_fwd_bwd": launches(ring[0], fns(sync, True)[0]),
                      "sync_nogroup_fwd": launches(None, fns(sync, False)[0])}
        assert all(pg.error() == 0 for pg in ring), "an exchange timed out"
    finally:
        for pg in ring:
            pg.close()
    derived = {}
    for name in ("masked", "sync_peer", "sync_nogroup"):
        if f"{name}_fwd" in ms:
            f = ms[f"{name}_fwd"]
            derived[name] = {"fwd_ms": round(f, 4), "bwd_ms": round(ms[f"{name}_fwd_bwd"] - f, 4)}
    return {"rows_per_rank": n, "channels": c, "dtype": str(dtype).replace("torch.", ""), "world": world,
            "ms": ms, "derived": derived, "launches_per_call": counts}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sync_bn_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "results": []}
    for n, c, dt in ((100_000, 64, torch.float16), (300_000, 128, torch.bfloat16)):
        for world in (1, 2, 4):
            out["results"].append(run(spconv, n, c, dt, world, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
