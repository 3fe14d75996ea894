"""Rulebook edges, bit-exact against the oracle: the Native 3-tuple and the MaskImplicitGemm 9-tuple, as
test_rulebook_gpu.py compares them.

* Overflow re-run: stage 1 of the regular-conv rulebook sizes its hash table for a quarter of the output
  bound and re-runs at full size when a probe chain overflows.  Isolated points (odd coordinates, 4 apart)
  give every point its own outputs, so M exceeds the optimistic capacity and the re-run always happens.
* Hash collisions: the keys of a grid are bucketed with a numpy copy of ``mix32`` at the capacity the table
  will get, and whole runs of buckets are taken, so probe chains are dozens of slots long.  If the hash
  changes these clouds stop being adversarial, but the tests still check the rulebooks.
* Smaller edges: duplicate coordinates, out-of-range batch rows, coordinates on the grid boundary,
  N = 1, 127, 128, 129, and a batch whose middle sample is empty.
"""
import numpy as np
import pytest
import torch

from tests.util import random_cloud

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ copies of the host-side sizing (hash.cuh, rulebook.cu)
def table_capacity(n_items, factor=4):
    cap = 1024
    while cap < n_items * factor:
        cap <<= 1
    return cap


def conv_max_out(ksize, stride, n, transposed):
    kv = int(np.prod(ksize))
    if transposed:
        return kv * n
    res = n
    for k, s in zip(ksize, stride):
        if k > s:
            res *= (k + s - 1) // s
    return min(res, kv * n)


def optimistic_capacity(max_out):
    return min(table_capacity((max_out + 3) // 4, 2), table_capacity(max_out, 2))


def mix32(x):
    x = np.asarray(x, np.uint64) & np.uint64(0xFFFFFFFF)
    m = np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x85EBCA6B)) & m
    x ^= x >> np.uint64(13)
    x = (x * np.uint64(0xC2B2AE35)) & m
    x ^= x >> np.uint64(16)
    return x


def probe_lengths(keys, cap):
    """slots visited by each insert of a linear-probing table of `cap` slots, keys inserted in order"""
    used = np.zeros(cap, bool)
    out = []
    for h in (mix32(keys) & np.uint64(cap - 1)).astype(np.int64):
        n = 1
        while used[h]:
            h = (h + 1) & (cap - 1)
            n += 1
        used[h] = True
        out.append(n)
    return np.array(out)


def _g(kind, shape, ksize, stride=None, padding=None, dilation=None, batch=1):
    nd = len(shape)
    return {"kind": kind, "shape": shape, "batch": batch, "ksize": ksize, "stride": stride or [1] * nd,
            "padding": padding or [0] * nd, "dilation": dilation or [1] * nd, "output_padding": [0] * nd}


def _with_batch(pts, b=0):
    return np.concatenate([np.full((len(pts), 1), b, np.int64), pts], 1).astype(np.int32)


def _isolated(nd, n, seed, side=16, offset=0):
    """n points with odd coordinates 4 apart (a lattice of side^nd sites)"""
    rng = np.random.default_rng(seed)
    grid = np.stack(np.meshgrid(*[np.arange(side)] * nd, indexing="ij"), -1).reshape(-1, nd)
    pts = 4 * grid[rng.permutation(len(grid))[:n]] + 1 + offset
    return _with_batch(pts)


def _collision_cloud(shape, n_groups, run, cap, seed):
    """whole buckets of `shape`'s keys: n_groups runs of `run` adjacent buckets (at capacity cap), runs spaced
    cap / (2 n_groups) apart and all below 1024, so a 1024-slot table sees the same chains"""
    keys = np.arange(int(np.prod(shape)), dtype=np.int64)
    b = (mix32(keys) & np.uint64(cap - 1)).astype(np.int64)
    starts = [g * (1024 // n_groups) + 7 for g in range(n_groups)]
    chosen = np.isin(b, [s + j for s in starts for j in range(run)])
    sel = keys[chosen]
    sel = sel[np.random.default_rng(seed).permutation(len(sel))]
    return _with_batch(np.stack(np.unravel_index(sel, shape), -1))


HUGE = [2600, 2600, 2600]        # output grid of a stride-2 conv >= 2^31 cells: int64 keys; input grid >= 2^32


def rulebook_cases():
    """name -> (indices, geometry) of every case in this file"""
    c = {}
    # overflow re-run
    c["overflow_3d_k3s2p1"] = (_isolated(3, 1000, 1), _g("conv", [64] * 3, [3] * 3, [2] * 3, [1] * 3))
    c["overflow_2d_k3s2p1"] = (_isolated(2, 1000, 2, side=40), _g("conv", [160, 160], [3] * 2, [2] * 2, [1] * 2))
    c["overflow_3d_k3s2p1_T"] = (_isolated(3, 300, 3), _g("transpose", [64] * 3, [3] * 3, [2] * 3, [1] * 3))
    c["overflow_3d_k3s2p1_i64"] = (_isolated(3, 1000, 4, offset=2400), _g("conv", HUGE, [3] * 3, [2] * 3, [1] * 3))
    # hash collisions (SubM table: table_capacity(N, 4) = 2048 for these N; conv k1: 1024)
    coll = _collision_cloud([32, 32, 48], 5, 3, 2048, 6)
    c["collide_subm_k3"] = (coll, _g("subm", [32, 32, 48], [3] * 3))
    c["collide_subm_k513"] = (coll, _g("subm", [32, 32, 48], [5, 1, 3]))
    c["collide_conv_k1"] = (coll, _g("conv", [32, 32, 48], [1] * 3))
    # duplicates and out-of-range batch rows
    rng = np.random.default_rng(7)
    _, base = random_cloud(rng, [12, 11, 10], [400, 300], 1)
    dup = np.concatenate([base, base[rng.permutation(len(base))[:150]]], 0)
    bad = base[:40].copy()
    bad[:20, 0] = 2
    bad[20:, 0] = -1
    mixed = np.concatenate([dup, bad], 0)[rng.permutation(len(dup) + 40)]
    c["dup_badbatch_conv_k3s2p1"] = (mixed, _g("conv", [12, 11, 10], [3] * 3, [2] * 3, [1] * 3, batch=2))
    c["dup_badbatch_conv_k2s2"] = (mixed, _g("conv", [12, 11, 10], [2] * 3, [2] * 3, batch=2))
    c["badbatch_subm_k3"] = (np.concatenate([base, bad], 0), _g("subm", [12, 11, 10], [3] * 3, batch=2))
    # the grid boundary: every corner and edge cell of a small grid, plus random interior points
    shape = [7, 6, 5]
    grid = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"), -1).reshape(-1, 3)
    edge = grid[np.any((grid == 0) | (grid == np.array(shape) - 1), axis=1)]
    bnd = _with_batch(edge[np.random.default_rng(8).permutation(len(edge))])
    c["boundary_subm_k3"] = (bnd, _g("subm", shape, [3] * 3))
    c["boundary_conv_k3s2p1"] = (bnd, _g("conv", shape, [3] * 3, [2] * 3, [1] * 3))
    c["boundary_conv_k3s2p0"] = (bnd, _g("conv", shape, [3] * 3, [2] * 3))
    c["boundary_conv_k2s3"] = (bnd, _g("conv", shape, [2] * 3, [3] * 3))
    c["boundary_T_k3s2p1"] = (bnd, _g("transpose", shape, [3] * 3, [2] * 3, [1] * 3))
    # row counts around one 128-row tile
    for n in (1, 127, 128, 129):
        _, inds = random_cloud(np.random.default_rng(n), [16, 16, 16], [n], 1)
        c[f"n{n}_subm_k3"] = (inds, _g("subm", [16] * 3, [3] * 3))
        c[f"n{n}_conv_k3s2p1"] = (inds, _g("conv", [16] * 3, [3] * 3, [2] * 3, [1] * 3))
    # a batch of three whose middle sample is empty
    _, a = random_cloud(np.random.default_rng(9), [14, 13, 12], [500, 400], 1)
    a[a[:, 0] == 1, 0] = 2
    c["empty_middle_subm_k3"] = (a, _g("subm", [14, 13, 12], [3] * 3, batch=3))
    c["empty_middle_conv_k3s2p1"] = (a, _g("conv", [14, 13, 12], [3] * 3, [2] * 3, [1] * 3, batch=3))
    return c


CASES = rulebook_cases()


def _compare(inds, g, oracle, dev, implicit=True):
    """implicit=False (duplicate input coordinates): the Native pairs only.  Two copies of a coordinate reach
    the same output through the same offset, the implicit-GEMM tables hold one input per (offset, output),
    and which copy they keep is not specified."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    subm, transpose = g["kind"] == "subm", g["kind"] == "transpose"
    args = (g["shape"], g["ksize"], g["stride"], g["padding"], g["dilation"], g["output_padding"])
    ref_out, ref_pairs, ref_num = oracle.get_indice_pairs(inds, g["batch"], *args, subm, transpose)
    d_inds = torch.from_numpy(inds).to(dev)
    out, pairs, num = ops.get_indice_pairs(d_inds, g["batch"], g["shape"], ConvAlgo.Native, *args[1:], subm,
                                           transpose)
    assert np.array_equal(num.cpu().numpy(), ref_num)
    assert np.array_equal(out.cpu().numpy(), ref_out)
    assert np.array_equal(pairs.cpu().numpy(), ref_pairs)
    if int(np.prod(g["ksize"])) > 128 or not implicit:
        return ref_out
    tab = oracle.implicit_gemm_tables(ref_pairs, ref_num, inds.shape[0], ref_out.shape[0], subm)
    res = ops.get_indice_pairs_implicit_gemm(d_inds, g["batch"], g["shape"], ConvAlgo.MaskImplicitGemm, *args[1:],
                                             subm, transpose, is_train=True)
    out_inds, _, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks = res
    assert np.array_equal(out_inds.cpu().numpy(), ref_out)
    assert np.array_equal(pair_fwd.cpu().numpy(), tab["pair_fwd"])
    assert np.array_equal(pair_bwd.cpu().numpy(), tab["pair_bwd"])
    assert np.array_equal(mask_fwd[0].cpu().numpy().view(np.uint32), tab["mask_fwd"])
    assert np.array_equal(sort_fwd[0].cpu().numpy(), tab["argsort_fwd"])
    if not subm:
        assert np.array_equal(mask_bwd[0].cpu().numpy().view(np.uint32), tab["mask_bwd"])
        assert np.array_equal(sort_bwd[0].cpu().numpy(), tab["argsort_bwd"])
    return ref_out


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("overflow")])
def test_overflow_rerun_rulebook_bit_exact(name, oracle, cuda_dev):
    inds, g = CASES[name]
    ref_out = _compare(inds, g, oracle, cuda_dev)
    m, n = ref_out.shape[0], inds.shape[0]
    kv = int(np.prod(g["ksize"]))
    per_point = kv if g["kind"] == "transpose" else int(np.prod([(k + s - 1) // s for k, s in zip(g["ksize"], g["stride"])]))
    assert m == per_point * n                                    # every point has its own outputs
    assert m > optimistic_capacity(conv_max_out(g["ksize"], g["stride"], n, g["kind"] == "transpose"))
    if name.endswith("i64"):
        assert np.prod([float(s) for s in g["shape"]]) >= 2.0 ** 32
        out_dims = [(s + 2 * p - (k - 1) - 1) // st + 1
                    for s, k, st, p in zip(g["shape"], g["ksize"], g["stride"], g["padding"])]
        assert np.prod([float(s) for s in out_dims]) >= 2.0 ** 31


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("collide")])
def test_hash_collision_chains_bit_exact(name, oracle, cuda_dev):
    inds, g = CASES[name]
    n = inds.shape[0]
    keys = ((inds[:, 0].astype(np.int64) * g["shape"][0] + inds[:, 1]) * g["shape"][1] + inds[:, 2]) * g["shape"][2] \
        + inds[:, 3]
    if g["kind"] == "subm":
        cap = table_capacity(n, 4)
        assert cap == 2048
    else:
        cap = optimistic_capacity(conv_max_out(g["ksize"], g["stride"], n, False))
        assert cap == 1024
    lengths = probe_lengths(keys, cap)
    assert 30 <= lengths.max() < 96, lengths.max()               # long chains, under CONV_MAX_PROBES
    _compare(inds, g, oracle, cuda_dev)


@pytest.mark.parametrize("name", [n for n in CASES if not n.startswith(("overflow", "collide"))])
def test_small_edges_bit_exact(name, oracle, cuda_dev):
    inds, g = CASES[name]
    _compare(inds, g, oracle, cuda_dev, implicit=not name.startswith("dup"))
