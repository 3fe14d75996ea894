"""Time FP8 (e4m3) sparse convolution inference against fp16 and int8 on the same rulebook.

Workloads (``bench_utils.surface_cloud`` on the 41 x 1600 x 1408 KITTI grid, 100 k voxels, the bench's int8 cloud):
  * SubM 3^3 forward at C = K = 64 and 128, one shared rulebook:
      ``fp16``          the float layer (tensor cores, bias, fp16 out);
      ``int8``          ``spx_implicit_gemm_fwd_int8``, int8 in -> int8 out;
      ``fp8_e4m3``      ``Fp8SparseConv`` e4m3 in -> e4m3 out (static output scale);
      ``fp8_dyn_fp16``  ``Fp8SparseConv`` fp16 in -> dynamic quantise -> e4m3 GEMM -> fp16 out;
      ``quantise``      the dynamic quantise pass alone (amax + cast of the fp16 features).
  * the six-layer SECOND encoder (``bench_utils.make_encoder6``) in inference, fp16 against ``convert_to_fp8``
    (its C = 16 layers are below the tensor cores' 32-channel e4m3 step and run on the FMA kernel), eager: its
    strided layers have no output bounds and size their outputs on the host.
The layer variants are graph-replayed; a number is the median over ``--reps`` alternating windows of ``--steps`` replays,
CUDA events closed by a synchronise.  The relative L2 error of each fp8 output against the fp16 module is printed
too (the tests do not assert it).  Prints one JSON line with the card's name and power limit.

    python tools/fp8_timing.py [--steps 50] [--reps 7]
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

from bench_utils import make_encoder6, surface_cloud  # noqa: E402
from tools.bounded_encoder_timing import card, measure  # noqa: E402
from tools.masked_bn_timing import graphed  # noqa: E402

SHAPE = [41, 1600, 1408]
N = 100_000


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def replay(fn):
    g = graphed(fn)
    return lambda s: g()


def run_layer(spconv, inds, c, steps, reps, dev):
    from spconv_b200.pytorch import fp8, ops, quantized
    torch.manual_seed(c)
    conv = spconv.SubMConv3d(c, c, 3, indice_key="k").to(dev).half().eval()
    x = spconv.SparseConvTensor(torch.randn((inds.shape[0], c), device=dev).half(), inds, SHAPE, 1)
    with torch.no_grad():
        ref = conv(x)
        x = ref.replace_feature(x.features)           # the rulebook is built once and shared by every variant
        out_scale = fp8.calibrate_fp8_output_scale(conv, x)
        q_e4m3 = fp8.Fp8SparseConv.from_float(conv, output_dtype=torch.float8_e4m3fn, output_scale=out_scale)
        q_f16 = fp8.Fp8SparseConv.from_float(conv)
        xq = fp8.quantize_fp8(x)
        i8 = quantized.QuantizedSparseConv.from_float(conv, float(out_scale.item()) * 448 / 127)
        xi = quantized.quantize_tensor(x, float(x.features.float().abs().max()) / 127)
        errs = {"fp8_e4m3": rel_l2(fp8.dequantize_fp8(q_e4m3(xq)).features, ref.features),
                "fp8_dyn_fp16": rel_l2(q_f16(x).features, ref.features),
                "int8": rel_l2(quantized.dequantize_tensor(i8(xi)).features, ref.features)}
    fns = {}
    with torch.no_grad():
        fns["fp16"] = replay(lambda: conv(x))
        fns["int8"] = replay(lambda: i8(xi))
        fns["fp8_e4m3"] = replay(lambda: q_e4m3(xq))
        fns["fp8_dyn_fp16"] = replay(lambda: q_f16(x))
        fns["quantise"] = replay(lambda: ops.fp8_quantize(x.features))
    return {"ms": measure(fns, steps, reps), "rel_l2_vs_fp16": errs}


def _eager(net, x):
    with torch.no_grad():
        return net(x)


def run_encoder(spconv, inds, steps, reps, dev):
    from spconv_b200.pytorch import fp8
    torch.manual_seed(0)
    net = spconv.SparseSequential(*make_encoder6(spconv, bias=True)).to(dev).half().eval()
    q = spconv.SparseSequential(*make_encoder6(spconv, bias=True)).to(dev).half().eval()
    q.load_state_dict(net.state_dict())
    skipped = fp8.convert_to_fp8(q)
    x = spconv.SparseConvTensor(torch.randn((inds.shape[0], 16), device=dev).half(), inds, SHAPE, 1)
    with torch.no_grad():
        err = rel_l2(q(x).features, net(x).features)
    # the strided layers size their output on the host (no output bounds): timed eagerly, as a user runs them
    fns = {"fp16": lambda s: _eager(net, x), "fp8": lambda s: _eager(q, x)}
    return {"ms": measure(fns, steps, reps), "rel_l2_vs_fp16": err, "skipped": skipped}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import spconv_b200.pytorch as spconv
    dev = torch.device("cuda:0")
    res = {**card()}
    inds = torch.from_numpy(surface_cloud(np.random.default_rng(0), SHAPE, N)).to(dev)
    res["voxels"] = int(inds.shape[0])
    for c in (64, 128):
        res[f"subm3_c{c}"] = run_layer(spconv, inds, c, a.steps, a.reps, dev)
        print(json.dumps({f"subm3_c{c}": res[f"subm3_c{c}"]}), file=sys.stderr, flush=True)
    res["second_encoder6"] = run_encoder(spconv, inds, a.steps, a.reps, dev)
    res.update(card())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
