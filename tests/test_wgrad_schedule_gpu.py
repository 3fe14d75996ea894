"""The weight-gradient kernel's offset groups and passes, checked bit for bit.

tc_wgrad_kernel stacks kernel offsets in natural order into groups, deals the groups to passes, skips
the wgmma of a warpgroup whose atoms of a stage are all inactive and keeps one wgmma group in flight.
These cases push that schedule to its edges: all activity in one group, few tiles, several mask
words, one to sixteen groups per pass, every operand type, one row.  Inputs are on
the exact grid of test_bench_workloads_gpu.py (integers in [-2, 2] / 8), so dW must equal the float64
sum rounded once, whatever the partition, and two runs must agree bit for bit.
"""
import numpy as np
import pytest
import torch

from tests.test_bench_workloads_gpu import Q, _assert_exact, _grid
from tests.test_conv_tc_coverage_gpu import ENV_FAMILY, Conv, _configure, _reference, wgrad_instance
from tests.util import random_cloud

pytestmark = pytest.mark.gpu

TORCH_DT = {"f16": torch.float16, "bf16": torch.bfloat16, "tf32": torch.float32}


@pytest.fixture(autouse=True)
def _restore_forced_family():
    yield
    if torch.cuda.is_available():
        _configure(ENV_FAMILY)


def _lattice(shape, step):
    """voxels on every `step`-th site: with step 2 no voxel has a neighbour, so a 3^3 SubM conv has only
    the centre offset active and all activity sits in one offset group"""
    g = np.stack(np.meshgrid(*[np.arange(0, s, step) for s in shape], indexing="ij"), -1).reshape(-1, len(shape))
    return np.concatenate([np.zeros((len(g), 1), np.int32), g.astype(np.int32)], 1)


def _random(shape, n, seed):
    _, inds = random_cloud(np.random.default_rng(seed), shape, [n], 1)
    return inds


# name: (dtype, voxels, spatial shape, ksize, C, K); SubM convs.  "few_tiles" has 8 tiles, fewer than
# the 33 CTAs a pass would get on 132 SMs.
CASES = {
    "one_group": ("f16", lambda: _lattice([40, 40, 40], 2), [40, 40, 40], 3, 64, 64),
    "few_tiles":("f16", lambda: _random([30, 30, 30], 900, 1), [30, 30, 30], 3, 64, 64),
    "kv125": ("f16", lambda: _random([19, 18, 17], 3000, 2), [19, 18, 17], 5, 32, 16),
    "c_out16": ("f16", lambda: _random([40, 40, 40], 20000, 3), [40, 40, 40], 3, 64, 16),
    "c_out128": ("f16", lambda: _random([40, 40, 40], 20000, 4), [40, 40, 40], 3, 64, 128),
    "c_out256": ("f16", lambda: _random([40, 40, 40], 20000, 5), [40, 40, 40], 1, 256, 256),
    "bf16": ("bf16", lambda: _random([40, 40, 40], 20000, 6), [40, 40, 40], 3, 64, 64),
    "tf32": ("tf32", lambda: _random([40, 40, 40], 20000, 7), [40, 40, 40], 3, 32, 32),
    "one_row": ("f16", lambda: np.array([[0, 5, 6, 7]], np.int32), [12, 12, 12], 3, 64, 64),
}
# wgrad groups per pass of each case's kernel instance: 16 / 2 / 1 at c_out = 16 / 128 / 256
GROUPS_PER_PASS = {"c_out16": 16, "c_out128": 2, "c_out256": 1}


@pytest.mark.parametrize("name", sorted(CASES))
def test_wgrad_partition_exact(name, oracle, cuda_dev):
    dt, make, shape, ks, C, K = CASES[name]
    inds = make()
    conv = Conv(oracle, cuda_dev, inds, 1, shape, ks, 1, 0, 1, True)
    inst = wgrad_instance(dt, conv.kv, C, K)
    assert inst is not None, f"{name}: not a tensor-core weight-gradient shape"
    if name in GROUPS_PER_PASS:
        assert min(256 // K, 16) == GROUPS_PER_PASS[name]
    tdt = TORCH_DT[dt]
    gen = torch.Generator(device=cuda_dev).manual_seed(7)
    x = _grid(gen, (conv.n_in, C), cuda_dev)
    dout = _grid(gen, (conv.n_out, K), cuda_dev)
    w = torch.zeros((K, conv.kv, C), device=cuda_dev)
    xd, dd = x.to(tdt), dout.to(tdt)
    dw = conv.wgrad_call(xd, dd, w.shape, inst)
    again = conv.wgrad_call(xd, dd, w.shape, inst)
    torch.cuda.synchronize()
    r = _reference(x, w, dout, conv.ref_pair, cuda_dev)
    _assert_exact(f"{name} dw", dw.reshape(K, conv.kv, C), r["dw"], r["dw_abs"], Q, tdt)
    assert torch.equal(dw, again), f"{name}: two runs differ"
