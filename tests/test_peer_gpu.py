"""Weight-gradient exchange fused into the weight-gradient kernel (csrc/peer.cu, include/spconv_b200.h
``spx_peer_group``): protocol tests on ONE GPU -- the "ranks" are streams whose exchange buffers all
live on the same device (``PeerGroup.local_ring``) -- and, when the box has two GPUs, the real thing over
CUDA IPC / NVLink in two processes (``tools/peer_check.py``).

Parity statement: the reference has no distributed code (SURVEY section 5); data-parallel users all-reduce
dW with NCCL after backward.  The fused exchange must therefore equal  scale * sum_r dW_r  where dW_r is
what the single-GPU kernel (already pinned to the oracle in test_conv_gpu.py) returns on rank r's shard:
bit-identical on all ranks, and within one rounding of the fp32 sum of the per-rank results."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.util import random_cloud

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _shard(cuda_dev, seed, C, K, subm, dt, pts=(1200, 900)):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(seed)
    shape = [19, 18, 17]
    feats, inds = random_cloud(rng, shape, list(pts), C)
    st = [1] * 3 if subm else [2] * 3
    res = ops.get_indice_pairs_implicit_gemm(torch.from_numpy(inds).to(cuda_dev), len(pts), shape, ConvAlgo.MaskImplicitGemm,
                                             [3] * 3, st, [1] * 3, [1] * 3, [0] * 3, subm, False, is_train=True)
    m = res[0].shape[0]
    x = torch.from_numpy(feats).to(cuda_dev, dt)
    dout = torch.from_numpy(rng.uniform(-0.2, 0.2, size=(m, K)).astype(np.float32)).to(cuda_dev, dt)
    return x, dout, res


def _weights(cuda_dev, seed, C, K, dt):
    w = np.random.default_rng(seed).uniform(-0.5, 0.5, size=(K, 3, 3, 3, C)).astype(np.float32)
    return torch.from_numpy(w).to(cuda_dev, dt)


def _backward(x, w, dout, res, subm):
    from spconv_b200.pytorch import ops
    return ops.implicit_gemm_backward(x, w, dout, res[2], res[3], res[4], res[5], res[6], res[7], None, res[8], 128, subm)


@pytest.fixture()
def no_peers():
    from spconv_b200.pytorch import ops
    yield
    ops.set_peer_group(None)
    from spconv_b200 import _cabi
    _cabi.check(_cabi.load().spx_debug_configure(-1, 0, 0, None, 0), "debug_configure")


def test_world_of_one_equals_the_plain_weight_gradient(cuda_dev, no_peers):
    from spconv_b200.pytorch import ops
    from spconv_b200.pytorch.dist import PeerGroup
    (pg,) = PeerGroup.local_ring(1, capacity_bytes=1 << 20)
    for it, (C, K, subm, dt) in enumerate([(64, 64, True, torch.float16), (32, 64, False, torch.bfloat16),
                                           (64, 64, True, torch.float16), (48, 24, True, torch.float16),
                                           (16, 16, True, torch.float32), (64, 64, True, torch.float16)]):
        x, dout, res = _shard(cuda_dev, 100 + it, C, K, subm, dt)
        w = _weights(cuda_dev, it, C, K, dt)
        ops.set_peer_group(None)
        din0, dw0 = _backward(x, w, dout, res, subm)
        ops.set_peer_group(pg)
        din1, dw1 = _backward(x, w, dout, res, subm)
        assert torch.equal(dw0, dw1) and torch.equal(din0, din1), (it, C, K)
    assert pg.error() == 0
    pg.close()


@pytest.mark.parametrize("world", [2, 3], ids=["2", "3"])
def test_ranks_on_one_gpu_exchange_through_the_fused_kernel(world, cuda_dev, no_peers):
    """world ranks = world streams: every rank's reduction kernel writes its slices, every finish publishes them
    and pulls them all."""
    from spconv_b200.pytorch import ops
    from spconv_b200.pytorch.dist import PeerGroup
    ring = PeerGroup.local_ring(world, capacity_bytes=1 << 20, average=True)
    streams = [torch.cuda.Stream() for _ in range(world)]
    cases = [(64, 64, True, torch.float16), (64, 128, False, torch.bfloat16), (32, 32, True, torch.float16),
             (48, 24, True, torch.float16), (64, 64, True, torch.float16)]       # K=24: FMA kernel + standalone exchange
    for it, (C, K, subm, dt) in enumerate(cases * 2):                               # 10 exchanges: slots, epochs, sizes
        w = _weights(cuda_dev, it, C, K, dt)
        shards = [_shard(cuda_dev, 1000 + 10 * it + r, C, K, subm, dt, pts=(900 + 150 * r, 700)) for r in range(world)]
        ops.set_peer_group(None)
        local = [_backward(x, w, dout, res, subm)[1] for x, dout, res in shards]
        torch.cuda.synchronize()
        fused = []
        for r in range(world):
            ops.set_peer_group(ring[r])
            with torch.cuda.stream(streams[r]):
                fused.append(_backward(*shards[r][:1], w, *shards[r][1:], subm)[1])
        torch.cuda.synchronize()
        for r in range(1, world):
            assert torch.equal(fused[0], fused[r]), f"replicas differ (exchange {it}, rank {r})"
        want = sum(d.float() for d in local) / world
        got = fused[0].float()
        ulp = 2.0 ** -7 if dt == torch.bfloat16 else 2.0 ** -10
        # one rounding of the fp32 sum vs the mean of `world` separately rounded gradients
        tol = ulp * (sum(d.float().abs() for d in local) / world + want.abs()) + 1e-6
        assert (got - want).abs().le(tol).all(), (it, float((got - want).abs().max()))
    assert all(pg.error() == 0 for pg in ring)
    for pg in ring:
        pg.close()


def test_small_tensor_allreduce_in_place(cuda_dev, no_peers):
    from spconv_b200.pytorch import ops
    from spconv_b200.pytorch.dist import PeerGroup
    world = 4
    ring = PeerGroup.local_ring(world, capacity_bytes=1 << 18, average=False)
    streams = [torch.cuda.Stream() for _ in range(world)]
    rng = np.random.default_rng(3)
    for n in (4, 3, 64, 1001, 40000, 64):
        parts = [torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(cuda_dev) for _ in range(world)]
        want = parts[0].clone()
        for p in parts[1:]:
            want = want + p                                   # rank order, fp32: exact match expected
        work = [p.clone() for p in parts]
        torch.cuda.synchronize()
        for r in range(world):
            ops.set_peer_group(ring[r])
            with torch.cuda.stream(streams[r]):
                ops.peer_allreduce_(work[r])
        torch.cuda.synchronize()
        for r in range(world):
            assert torch.equal(work[r], want), (n, r)
    for pg in ring:
        pg.close()


def test_a_missing_peer_times_out_instead_of_hanging(cuda_dev, no_peers):
    from spconv_b200.pytorch import ops
    from spconv_b200.pytorch.dist import PeerGroup
    ring = PeerGroup.local_ring(2, capacity_bytes=1 << 16, timeout_ms=200)
    t = torch.ones(256, device=cuda_dev)
    ops.set_peer_group(ring[0])
    ops.peer_allreduce_(t)                                    # rank 1 never calls
    assert ring[0].error() == 1
    assert torch.isnan(t).all()
    for pg in ring:
        pg.close()


@pytest.mark.skipif(torch.cuda.is_available() and torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_processes_over_cuda_ipc(cuda_dev):
    """the real transport: one process per GPU, buffers mapped through CUDA IPC handles"""
    port = 29500 + os.getpid() % 400
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tools", "peer_check.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "peer_check OK" in res.stdout
