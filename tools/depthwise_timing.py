"""Time the depthwise sparse convolution (groups = in_channels = out_channels) against what a user has without it,
on one shared rulebook:
  * ``dense``: a ``SubMConv3d(C, C)`` on the same ``indice_key`` (the tensor-core conv; kv <= 128 only), C x the
    FLOPs and weights of the layer the user wants;
  * ``torch``: the formulation a user writes today, a gather / multiply / sum over the kv offsets of the same table
    (``where(T[k] >= 0, x.index_select(0, T[k]) * W[:, k], 0)``, kv launches per pass, autograd for the backward,
    timed over ``--steps / 10`` calls per window, 3 windows).
Workloads (``bench_utils.surface_cloud`` on a 41 x 1600 x 1408 grid):
  * 100 k voxels, C = 64 fp16: SubM 3^3 (MaskImplicitGemm), SubM 5^3 (``large_kernel_fast_algo``), SubM 7^3 (Native);
  * 300 k voxels, C = 128 bf16: SubM 3^3.
Per variant: the module forward (``fwd``) and forward + backward, graph-replayed; the backward is the difference.
``ours_op`` times the ops-level forward and backward alone (no module, no bias).  Algorithmic bytes, set against the
3.35 TB/s data-sheet bandwidth:
  forward N C e + kv M 4 + M C e; input gradient M C e + kv N 4 + N C e; weight gradient N C e + M C e + kv M 4 +
  partials (written and read once, ceil(M / 512) kv C 4 bytes each way).
A number is the median over ``--reps`` windows of ``--steps`` calls, CUDA events closed by a synchronise, the
variants alternating in one process, every shape warmed up first.  Prints one JSON line with the card's name and
power limit.

    python tools/depthwise_timing.py [--steps 20] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_utils import surface_cloud  # noqa: E402
from tools.bounded_encoder_timing import card, measure  # noqa: E402
from tools.masked_bn_timing import HBM_GBS, graphed  # noqa: E402

SHAPE = [41, 1600, 1408]
CHUNK = 512


def log(msg):
    """progress on stderr: a full run captures a few hundred graphs"""
    print(f"[depthwise_timing {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def _tables(spconv, x, key, mod):
    """the dense forward table [kv, M] of the cached rulebook, as the depthwise layer walks it"""
    from spconv_b200.pytorch import ops
    d = x.indice_dict[key]
    if mod.algo == spconv.ConvAlgo.Native:
        kv = int(d.indice_pairs.shape[1])
        return ops._native_tables(d.indice_pairs, d.indice_pair_num, x.features.shape[0], d.out_indices.shape[0], kv,
                                  True, False, True, False)[0]
    return d.pair_fwd


def run(spconv, n, c, dtype, k, large, steps, reps, dev):
    from spconv_b200.pytorch import ops
    log(f"subm{k}^3 C={c} {dtype}: {n} voxels")
    rng = np.random.default_rng(n + k)
    inds = torch.from_numpy(surface_cloud(rng, SHAPE, n)).to(dev)
    n_rows = inds.shape[0]
    torch.manual_seed(k)
    key = f"k{k}"
    dw = spconv.SubMConv3d(c, c, k, groups=c, indice_key=key, large_kernel_fast_algo=large).to(dev).to(dtype).train()
    kv = k ** 3
    dense = None
    if kv <= 128:
        dense = spconv.SubMConv3d(c, c, k, indice_key=key, large_kernel_fast_algo=large).to(dev).to(dtype).train()
    x0 = spconv.SparseConvTensor(torch.randn((n_rows, c), device=dev).to(dtype), inds, SHAPE, 1)
    with torch.no_grad():
        x = dw(x0).replace_feature(x0.features)       # builds the rulebook once; every variant below reuses it
    feats = x.features.detach().clone().requires_grad_(True)
    xt = x.replace_feature(feats)
    dy = torch.randn((n_rows, c), device=dev).to(dtype)
    table = _tables(spconv, x, key, dw).contiguous()
    w = dw.weight.detach()

    def torch_forward(f, weight):
        wv = weight.view(c, kv)
        out = torch.zeros((n_rows, c), dtype=dtype, device=dev)
        for j in range(kv):
            t = table[j].long()
            out = out + torch.where((t >= 0)[:, None], f.index_select(0, t.clamp(min=0)) * wv[:, j], 0)
        return out

    variants = {}

    def add(name, fwd, fwd_bwd):
        log(f"subm{k}^3 C={c}: capturing {name}")
        variants[f"{name}_fwd"] = (lambda g: lambda s: g())(graphed(fwd))
        variants[f"{name}_fwd_bwd"] = (lambda g: lambda s: g())(graphed(fwd_bwd))

    def mod_fwd(m):
        def f():
            with torch.no_grad():
                m(xt)
        return f

    def mod_fwd_bwd(m):
        def f():
            feats.grad = None
            m.weight.grad = None
            m(xt).features.backward(dy)
        return f

    add("ours", mod_fwd(dw), mod_fwd_bwd(dw))
    if dense is not None:
        add("dense", mod_fwd(dense), mod_fwd_bwd(dense))
    wt = w.clone().requires_grad_(True)

    def t_fwd():
        with torch.no_grad():
            torch_forward(feats, wt)

    def t_fwd_bwd():
        feats.grad = None
        wt.grad = None
        torch_forward(feats, wt).backward(dy)

    add("torch", t_fwd, t_fwd_bwd)
    fd = feats.detach()
    variants["ours_op_fwd"] = (lambda g: lambda s: g())(graphed(lambda: ops.depthwise_conv(fd, w, table, n_rows)))
    variants["ours_op_bwd"] = (lambda g: lambda s: g())(
        graphed(lambda: ops.depthwise_conv_backward(fd, w, dy, table, None)))
    log(f"subm{k}^3 C={c}: measuring {len(variants)} variants")
    slow = {v: variants.pop(v) for v in list(variants) if v.startswith("torch")}
    ms = measure(variants, steps, reps)
    log(f"subm{k}^3 C={c}: measuring the torch formulation")
    ms.update(measure(slow, max(1, steps // 10), 3, warmup=1))     # kv launches per pass: fewer, longer windows

    e = torch.finfo(dtype).bits // 8
    m_rows = n_rows
    part = -(-m_rows // CHUNK) * kv * c * 4
    b_fwd = n_rows * c * e + kv * m_rows * 4 + m_rows * c * e
    b_dgrad = m_rows * c * e + kv * n_rows * 4 + n_rows * c * e
    b_wgrad = n_rows * c * e + m_rows * c * e + kv * m_rows * 4 + 2 * part
    derived = {}
    for name in ("ours", "dense", "torch"):
        if f"{name}_fwd" not in ms:
            continue
        f = ms[f"{name}_fwd"]
        bw = ms[f"{name}_fwd_bwd"] - f
        d = {"fwd_ms": round(f, 4), "bwd_ms": round(bw, 4)}
        if name == "ours":
            d["fwd_of_peak"] = round(b_fwd / f / 1e6 / HBM_GBS, 3)
            d["bwd_of_peak"] = round((b_dgrad + b_wgrad) / bw / 1e6 / HBM_GBS, 3) if bw > 0 else None
        derived[name] = d
    derived["ours_op"] = {"fwd_ms": ms["ours_op_fwd"], "bwd_ms": ms["ours_op_bwd"],
                          "fwd_of_peak": round(b_fwd / ms["ours_op_fwd"] / 1e6 / HBM_GBS, 3),
                          "bwd_of_peak": round((b_dgrad + b_wgrad) / ms["ours_op_bwd"] / 1e6 / HBM_GBS, 3)}
    with torch.no_grad():                             # the kernel and the torch formulation agree
        ours = ops.depthwise_conv(fd, w, table, n_rows).double()
        ref = torch_forward(fd.double(), w.double()).double()
        err = float(((ours - ref).abs() / (ref.abs() + 1e-3)).max())
    pairs = int((table >= 0).sum())
    return {"case": f"subm{k}^3", "algo": str(dw.algo), "dtype": str(dtype).replace("torch.", ""), "channels": c,
            "voxels": n_rows, "kv": kv, "pairs_per_voxel": round(pairs / n_rows, 2), "bytes": {
                "fwd": b_fwd, "dgrad": b_dgrad, "wgrad": b_wgrad}, "max_rel_err_vs_fp64_torch": err,
            "ms": ms, "derived": derived}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("depthwise_timing needs a CUDA device: there is no CPU path to time")
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    out = {"card": card(), "steps": a.steps, "reps": a.reps, "depthwise": []}
    for n, c, dtype, k, large in ((100_000, 64, torch.float16, 3, False), (100_000, 64, torch.float16, 5, True),
                                  (100_000, 64, torch.float16, 7, False), (300_000, 128, torch.bfloat16, 3, False)):
        out["depthwise"].append(run(spconv, n, c, dtype, k, large, a.steps, a.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
