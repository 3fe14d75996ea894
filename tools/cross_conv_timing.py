"""Time the convolution onto given output coordinates against the SubM convolution it generalises.

Workloads (``bench_utils.surface_cloud`` on the 41 x 1600 x 1408 KITTI grid, 100 k voxels, seed 0; the "next frame"
is a second cloud from seed 1):
  * rulebooks, 3^3, training form (both directions the layer needs):
      ``subm_rulebook``         ``get_indice_pairs_implicit_gemm`` SubM (one hash, mirror-symmetric probe);
      ``cross_rulebook_same``   ``get_indice_pairs_to`` with the cloud as its own target (two hashes, scattered
                                backward table, both mask sorts and tile tables);
      ``cross_rulebook_next``   ``get_indice_pairs_to`` onto the next frame;
  * a C = K = 64 fp16 layer, forward + backward with its rulebook: ``subm_layer`` (SubMConv3d), ``cross_layer_same``
    and ``cross_layer_next`` (the same layer given ``target=``).
Every variant is graph-replayed; a number is the median over ``--reps`` alternating windows of ``--steps`` replays,
CUDA events closed by a synchronise.  Prints one JSON line with the card's name and power limit.

    python tools/cross_conv_timing.py [--steps 50] [--reps 7]
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
from tools.masked_bn_timing import graphed  # noqa: E402

SHAPE = [41, 1600, 1408]
N = 100_000
C = 64


def replay(fn):
    g = graphed(fn)
    return lambda s: g()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import spconv_b200.pytorch as spconv
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    dev = torch.device("cuda:0")
    res = {**card()}
    cloud = torch.from_numpy(surface_cloud(np.random.default_rng(0), SHAPE, N)).to(dev)
    nxt = torch.from_numpy(surface_cloud(np.random.default_rng(1), SHAPE, N)).to(dev)
    res["voxels"] = [int(cloud.shape[0]), int(nxt.shape[0])]
    k3, one = [3] * 3, [1] * 3

    def subm_rb():
        ops.get_indice_pairs_implicit_gemm(cloud, 1, SHAPE, ConvAlgo.MaskImplicitGemm, k3, one, [0] * 3, one, [0] * 3,
                                           True, False, is_train=True)

    def cross_rb(target):
        return lambda: ops.get_indice_pairs_to(cloud, target, 1, SHAPE, SHAPE, k3, one, one, one, False, True)

    rulebooks = {"subm_rulebook": replay(subm_rb), "cross_rulebook_same": replay(cross_rb(cloud)),
                 "cross_rulebook_next": replay(cross_rb(nxt))}
    res["rulebook_ms"] = measure(rulebooks, a.steps, a.reps)
    print(json.dumps({"rulebook_ms": res["rulebook_ms"]}), file=sys.stderr, flush=True)
    del rulebooks

    torch.manual_seed(0)
    conv = spconv.SubMConv3d(C, C, 3, bias=False).to(dev).half().train()
    feats = torch.randn((cloud.shape[0], C), device=dev).half().requires_grad_(True)
    x = spconv.SparseConvTensor(feats, cloud, SHAPE, 1)
    same = spconv.SparseConvTensor(torch.zeros(cloud.shape[0], 1, device=dev), cloud, SHAPE, 1)
    nxt_t = spconv.SparseConvTensor(torch.zeros(nxt.shape[0], 1, device=dev), nxt, SHAPE, 1)
    dy = {n: torch.randn((n, C), device=dev).half() for n in (cloud.shape[0], nxt.shape[0])}

    def layer(target):
        def fn():
            y = conv(x) if target is None else conv(x, target=target)
            y.features.backward(dy[y.features.shape[0]])
        return fn

    layers = {"subm_layer": replay(layer(None)), "cross_layer_same": replay(layer(same)),
              "cross_layer_next": replay(layer(nxt_t))}
    res["layer_fwd_bwd_ms"] = measure(layers, a.steps, a.reps)
    res.update(card())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
