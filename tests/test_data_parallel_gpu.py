"""Data-parallel weight gradients on one GPU: the fused exchange and the all-reduce hook.

The "ranks" are streams of one GPU whose exchange buffers all live on it (``PeerGroup.local_ring``).  Within
one exchange nothing synchronises the host between ranks: every rank's finish kernel waits for the others'
publishes, so a host wait in the middle would leave it waiting for a rank that is not launched yet (it
then times out, with NaN and ``error() == 1``).  That is why every case ends with ``error() == 0`` on every
rank.

Exactness.  Features and output gradients are integers in [-2, 2] / 8 (``_grid``), so every product of
the weight gradient is a multiple of Q = 2^-6.  Where the sum of |terms| over all ranks stays below 2^24 Q
(asserted), each rank's fp32 dW and the fp32 sum over the ranks are exact, whatever the summation order, and
the scale 1 / world is a power of two (``average=True`` only at world 1, 2, 4 and 8).  So:
  * tensor cores: the exchange sums the unrounded fp32 partials; the result must be the float64 sum (mean)
    rounded once to the output type, bit for bit, and bit-identical on every rank;
  * FMA kernels: each rank rounds its dW to the output type before the push; the result must be the
    rank-order fp32 sum of those rounded gradients, scaled and rounded once.
The one case with inputs off the grid checks identical bits on every rank and one rounding of the float64
sum, and on the FMA kernels in fp32 the exact rank-order sum.

With SPX_FORCE_SIMT=1 in the environment every case runs on the FMA kernels.
"""
import contextlib
import copy
import ctypes
import math

import numpy as np
import pytest
import torch

from tests.test_bench_workloads_gpu import Q, _assert_exact, _grid
from tests.test_conv_tc_coverage_gpu import (CASES, ENV_FAMILY, GEOMS, KV, U_OUT, Conv, _check, _configure,
                                             _reference, wgrad_instance)
from tests.util import random_cloud

gpu = pytest.mark.gpu
SIMT = ENV_FAMILY == 1
TORCH_DT = {"f16": torch.float16, "bf16": torch.bfloat16, "tf32": torch.float32, "f32": torch.float32}
SHAPE = [19, 18, 17]
CAPACITY = 4 << 20                 # bytes: the largest dW here is 27 x 128 x 128 fp32 values


@pytest.fixture(autouse=True)
def _no_group_no_hook(monkeypatch):
    """fp32 is exact fp32 on the FMA kernels unless a case allows tf32; nothing installed after a case"""
    from spconv_b200.pytorch import ops
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", False)
    yield
    ops.set_peer_group(None)
    ops.set_wgrad_hook(None)
    if torch.cuda.is_available():
        _configure(ENV_FAMILY)


@contextlib.contextmanager
def _ring(world, average, capacity_bytes=CAPACITY):
    """world ranks of one GPU; every exchange must have completed without a timeout on every rank"""
    from spconv_b200.pytorch.dist import PeerGroup
    assert not average or world & (world - 1) == 0, "the mean is exact only for a power-of-two world"
    ring = PeerGroup.local_ring(world, capacity_bytes=capacity_bytes, average=average)
    try:
        yield ring
        errors = [pg.error() for pg in ring]
        assert errors == [0] * world, f"a finish timed out waiting for a peer: error words {errors}"
    finally:
        for pg in ring:
            pg.close()


def _round(ring, streams, fn):
    """fn(rank) on every rank's stream with its group installed, one after the other without a host
    synchronisation between them; synchronised before and after"""
    from spconv_b200.pytorch import ops
    torch.cuda.synchronize()
    out = []
    for r, pg in enumerate(ring):
        ops.set_peer_group(pg)
        with torch.cuda.stream(streams[r]):
            out.append(fn(r))
    ops.set_peer_group(None)
    torch.cuda.synchronize()
    return out


def _family(dt, kv, C, K):
    """kernel family of the weight gradient: 2 tensor cores, 1 FMA kernels"""
    return 1 if SIMT or dt == "f32" or wgrad_instance(dt, kv, C, K) is None else 2


# ------------------------------------------------------------------ one rank's conv
class Shard:
    """One rank's conv layer over its own cloud (inds None: a rank without rows): the rulebook in the form
    `algo` consumes ("igemm" MaskImplicitGemm, "native" ConvAlgo.Native, "split" MaskSplitImplicitGemm),
    its inputs, and the float64 weight gradient with its sum of |terms|."""

    def __init__(self, oracle, dev, inds, subm, algo, dt, C, K, w, gen, shape=SHAPE, ks=(3, 3, 3), stride=2,
                 padding=1, dilation=1, normal=False):
        from spconv_b200.core import ConvAlgo
        from spconv_b200.pytorch import ops
        nd = len(shape)
        self.subm, self.algo, self.dt, self.C, self.K = subm, algo, dt, C, K
        self.kv = kv = int(np.prod(ks))
        tdt = TORCH_DT[dt]
        st, pd = (1, 0) if subm else (stride, padding)
        self.conv = None
        if inds is not None:
            self.conv = Conv(oracle, dev, inds, int(inds[:, 0].max()) + 1, shape, list(ks), st, pd, dilation, subm)
        n_in, n_out = (self.conv.n_in, self.conv.n_out) if self.conv is not None else (0, 0)
        if normal:
            x = torch.randn((n_in, C), generator=gen, device=dev).to(tdt).float()
            dout = torch.randn((n_out, K), generator=gen, device=dev).to(tdt).float()
        else:
            x, dout = _grid(gen, (n_in, C), dev), _grid(gen, (n_out, K), dev)
        self.x, self.dout = x.to(tdt), dout.to(tdt)
        if self.conv is None:
            self.dw = self.dw_abs = torch.zeros((K, kv, C), dtype=torch.float64, device=dev)
            self.t_k = torch.zeros(kv, dtype=torch.float64, device=dev)
        else:
            r = _reference(x, w.float(), dout, self.conv.ref_pair, dev)
            self.dw, self.dw_abs, self.t_k = r["dw"], r["dw_abs"], r["t_k"]
        empty = lambda *s: torch.empty(s, dtype=torch.int32, device=dev)      # noqa: E731
        if algo == "igemm":
            if self.conv is None:
                pf = pb = empty(kv, 0)
                mf = sf = mb = sb = empty(0)
            else:
                pf, mf, sf, _ = self.conv.fwd
                pb, mb, sb, _ = self.conv.bwd if not subm else (pf, None, None, None)
            self.tables = (pf, pb, [mf], [] if subm else [mb], [sf], [] if subm else [sb], [])
        elif algo == "native":
            if self.conv is None:
                self.pairs = torch.full((2, kv, 1), -1, dtype=torch.int32, device=dev)
                self.num = torch.zeros(kv, dtype=torch.int32, device=dev)
            else:
                out, self.pairs, self.num = ops.get_indice_pairs(
                    torch.from_numpy(inds).to(dev), int(inds[:, 0].max()) + 1, shape, ConvAlgo.Native, list(ks),
                    [st] * nd, [pd] * nd, [dilation] * nd, [0] * nd, subm)
                assert out.shape[0] == n_out
                assert np.array_equal(out.cpu().numpy(), self._oracle_out(oracle, inds, shape, ks, st, pd, dilation))
        else:
            assert algo == "split" and self.conv is not None
            res = ops.get_indice_pairs_implicit_gemm(
                torch.from_numpy(inds).to(dev), int(inds[:, 0].max()) + 1, shape, ConvAlgo.MaskSplitImplicitGemm,
                list(ks), [st] * nd, [pd] * nd, [dilation] * nd, [0] * nd, subm, False, is_train=True)
            out, _, pf, pb, mfs, mbs, sfs, sbs, masks = res
            assert len(mfs) == 2 and out.shape[0] == n_out
            assert np.array_equal(out.cpu().numpy(), self._oracle_out(oracle, inds, shape, ks, st, pd, dilation))
            self.tables = (pf, pb, mfs, mbs, sfs, sbs, masks)

    def _oracle_out(self, oracle, inds, shape, ks, st, pd, dilation):
        nd = len(shape)
        if self.subm:
            return inds
        return oracle.get_indice_pairs(inds, int(inds[:, 0].max()) + 1, shape, list(ks), [st] * nd, [pd] * nd,
                                       [dilation] * nd, [0] * nd, False)[0]

    @property
    def parts(self):
        """mask splits of the rulebook (hook calls per layer)"""
        return len(self.tables[2]) if self.algo != "native" else 1

    def backward(self, w):
        """the op's weight gradient (the input gradient is computed too)"""
        from spconv_b200.pytorch import ops
        if self.algo == "native":
            return ops.indice_conv_backward(self.x, w, self.dout, self.pairs, self.num, False, self.subm)[1]
        pf, pb, mf, mb, sf, sb, masks = self.tables
        return ops.implicit_gemm_backward(self.x, w, self.dout, pf, pb, mf, mb, sf, sb, None, masks, 128,
                                          self.subm)[1]

    def split_backward(self, w, j):
        """dW of mask split j alone, as the op computes it before masking it to the split's offsets"""
        from spconv_b200.pytorch import ops
        pf, pb, mf, mb, sf, sb, masks = self.tables
        return ops.implicit_gemm_backward(self.x, w, self.dout, pf, pb, [mf[j]], [mb[j]] if mb else [], [sf[j]],
                                          [sb[j]] if sb else [], None, masks, 128, self.subm)[1]


def _assert_fused(name, got, refs, abs_sums, dt, scale, fma, q=Q):
    """got == the exchange of the per-rank float64 weight gradients `refs` (sums of |terms| `abs_sums`),
    whose products are multiples of q"""
    tdt = TORCH_DT[dt]
    for a in abs_sums:
        assert float(a.max()) < 2.0 ** 24 * q, f"{name}: a rank's sum of |terms| reaches 2^24 q"
    if not fma:
        _assert_exact(name, got, sum(refs) * scale, sum(abs_sums), q, tdt)
        return
    acc = None
    for d in refs:                                     # rank order, each rank's dW rounded before its push
        v = d.to(tdt).float()
        acc = v if acc is None else acc + v
    want = (acc * scale).to(tdt)
    g = got.reshape(want.shape)
    if not torch.equal(g, want):
        bad = (g != want) | torch.isnan(g)
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements differ from the rank-order sum; "
                             f"first at {tuple(int(i) for i in bad.nonzero()[0])} (NaN = not written)")


def _same_on_every_rank(name, dws):
    for r in range(1, len(dws)):
        assert torch.equal(dws[0], dws[r]), f"{name}: rank {r} holds other bits than rank 0"


# ------------------------------------------------------------------ 1. world of one, every route
def _instance_cases():
    """one case per tc_wgrad_kernel instance the coverage cases reach, plus kernel volume 125 and 1x1
    convs with 256 columns"""
    seen, out = set(), []
    for dt, g, C, K in CASES + [("f16", "k5", 32, 16), ("f16", "k1", 32, 256)]:
        inst = wgrad_instance(dt, KV[g], C, K)
        if inst is None or (inst, g in ("k5", "k1")) in seen:
            continue
        seen.add((inst, g in ("k5", "k1")))
        out.append(("igemm", dt, g, C, K))
    return out


ROUTES = (_instance_cases()
          + [("igemm", "f16", "k3", 48, 24), ("igemm", "f16", "k3", 3, 5), ("igemm", "f32", "k3", 16, 16)]   # FMA
          + [("native", "f16", "k3", 32, 64), ("native", "f16", "k3", 48, 24), ("native", "f32", "k3", 16, 16)]
          + [("split", "f16", "k3", 32, 32), ("split", "bf16", "k3", 48, 24)])


def test_routes_reach_every_weight_gradient_instance():
    """No GPU needed: the world-of-one cases reach every tc_wgrad_kernel instance the coverage cases reach,
    kernel volume 125 and 256 columns on the tensor cores, and the FMA kernels on every route."""
    def inst(dt, g, C, K):
        return None if dt == "f32" else wgrad_instance(dt, KV[g], C, K)
    reached = {inst(*c[1:]) for c in ROUTES}
    assert {inst(*c) for c in CASES} - {None} <= reached
    assert any(KV[c[2]] == 125 and inst(*c[1:]) for c in ROUTES)
    assert any(c[4] == 256 and KV[c[2]] == 1 and inst(*c[1:]) for c in ROUTES)
    assert any(c[1] == "tf32" for c in ROUTES)
    for algo in ("igemm", "native", "split"):
        fams = {inst(*c[1:]) is None for c in ROUTES if c[0] == algo}
        assert fams == {True, False}, algo


@gpu
@pytest.mark.parametrize("mode", ["subm", "conv"])
@pytest.mark.parametrize("case", ROUTES, ids=lambda c: "-".join(map(str, c)))
def test_world_of_one_equals_the_plain_weight_gradient(case, mode, oracle, cuda_dev, monkeypatch):
    """A group of one rank returns the plain weight gradient bit for bit, on the same kernel family, through the
    push + finish of implicit_gemm_backward, of indice_conv_backward and of the two exchanges of a mask-split
    layer; and through the C ABI's push, whose kernel family is read back."""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    algo, dt, geom, C, K = case
    shape, pts, ks, dil, (st, pd) = GEOMS[geom]
    if mode == "subm" and not all(k % 2 for k in ks):
        pytest.skip("even kernel: no SubM")
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", dt == "tf32")
    _, inds = random_cloud(np.random.default_rng(C * 100 + K), shape, pts, 1)
    gen = torch.Generator(device=cuda_dev).manual_seed(C + K)
    tdt = TORCH_DT[dt]
    w = _grid(gen, (K, *ks, C), cuda_dev).to(tdt)
    s = Shard(oracle, cuda_dev, inds, mode == "subm", algo, dt, C, K, w, gen, shape=shape, ks=ks, stride=st,
              padding=pd, dilation=dil)
    fam = _family(dt, s.kv, C, K)
    _configure(ENV_FAMILY)
    plain = s.backward(w)
    assert ops.last_kernel_family() == fam, (ops.last_kernel_family(), fam)
    with _ring(1, average=True) as (pg,):
        ops.set_peer_group(pg)
        fused = s.backward(w)
        if algo == "native":
            assert ops.last_kernel_family() == fam, "the exchanged Native weight gradient ran on another family"
        ops.set_peer_group(None)
        if algo == "igemm":
            lib = _cabi.load()
            d = s.conv.desc(tdt, C, K, s.conv.fwd)
            d.f32_mode = ops._f32_mode()
            ws = torch.empty(((lib.spx_implicit_gemm_wgrad_workspace_size(ctypes.byref(d)) + 3) // 4,),
                             dtype=torch.float32, device=cuda_dev)
            abi = torch.full_like(w, float("nan"))
            _cabi.check(lib.spx_implicit_gemm_wgrad_push(ctypes.byref(d), s.x.data_ptr(), s.dout.data_ptr(),
                                                         abi.data_ptr(), ws.data_ptr(), ws.numel() * 4,
                                                         ctypes.byref(pg.group), ops._stream()), "wgrad_push")
            assert lib.spx_last_kernel_family() == fam, "the exchanged weight gradient ran on another family"
            _cabi.check(lib.spx_peer_finish(ctypes.byref(pg.group), abi.data_ptr(), abi.numel(),
                                            ops._DTYPE_CODE[tdt], pg.scale, ops._stream()), "peer_finish")
            assert torch.equal(abi, plain), "C ABI push + finish differs from the plain weight gradient"
        torch.cuda.synchronize()
    assert torch.equal(fused, plain), "the exchanged weight gradient differs from the plain one"
    _assert_fused("dW", plain.reshape(K, s.kv, C), [s.dw], [s.dw_abs], dt, 1.0, fam == 1 and algo != "split")


# ------------------------------------------------------------------ 2. several ranks, eager
# (algo, subm, dtype, C, K): SubM, strided and Native on the tensor cores, then on the FMA kernels
EAGER = [("igemm", True, "f16", 32, 32), ("igemm", False, "bf16", 64, 32), ("native", True, "f16", 32, 64),
         ("native", False, "bf16", 16, 16),
         ("igemm", True, "f16", 48, 24), ("igemm", False, "f16", 3, 5), ("native", True, "bf16", 48, 24),
         ("native", False, "f32", 16, 16)]


def _shards(oracle, dev, world, it, algo, subm, dt, C, K, w, gen, empty, normal=False):
    out = []
    for r in range(world):
        inds = None
        if r != empty:
            _, inds = random_cloud(np.random.default_rng(1000 * world + 10 * it + r), SHAPE, [700 + 130 * r], 1)
        out.append(Shard(oracle, dev, inds, subm, algo, dt, C, K, w, gen, normal=normal))
    return out


@gpu
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_ranks_exchange_weight_gradients_eagerly(world, oracle, cuda_dev):
    """Each rank backpropagates its own shard (one rank per exchange has no rows) on its stream; 16
    exchanges per group over SubM, strided and Native layers on both kernel families.  Every rank gets the
    exact mean (world 2, 4, 8) or sum (world 3)."""
    average = world != 3
    streams = [torch.cuda.Stream() for _ in range(world)]
    gen = torch.Generator(device=cuda_dev).manual_seed(world)
    with _ring(world, average) as ring:
        scale = ring[0].scale
        for it, (algo, subm, dt, C, K) in enumerate(EAGER * 2):
            w = _grid(gen, (K, 3, 3, 3, C), cuda_dev).to(TORCH_DT[dt])
            shards = _shards(oracle, cuda_dev, world, it, algo, subm, dt, C, K, w, gen, empty=it % world)
            got = _round(ring, streams, lambda r: shards[r].backward(w))
            name = f"exchange {it} ({algo}, {'subm' if subm else 'strided'}, {dt}, C {C}, K {K})"
            _same_on_every_rank(name, got)
            _assert_fused(name, got[0].reshape(K, 27, C), [s.dw for s in shards], [s.dw_abs for s in shards], dt,
                          scale, _family(dt, 27, C, K) == 1)


@gpu
@pytest.mark.parametrize("dt,C,K", [("f16", 32, 32), ("f32", 16, 16)])
def test_inputs_off_the_grid(dt, C, K, oracle, cuda_dev):
    """Normal inputs, world 3: identical bits on every rank, within one rounding of the float64 sum (plus
    the fp32 accumulation); in fp32 on the FMA kernels exactly the rank-order sum of the plain gradients,
    which a rank starting the sum at its own rank would miss."""
    from spconv_b200.pytorch import ops
    world = 3
    streams = [torch.cuda.Stream() for _ in range(world)]
    gen = torch.Generator(device=cuda_dev).manual_seed(33)
    w = torch.randn((K, 3, 3, 3, C), generator=gen, device=cuda_dev).to(TORCH_DT[dt])
    shards = _shards(oracle, cuda_dev, world, 0, "igemm", True, dt, C, K, w, gen, empty=-1, normal=True)
    plain = [s.backward(w) for s in shards]
    fma = _family(dt, 27, C, K) == 1
    with _ring(world, average=False) as ring:
        got = _round(ring, streams, lambda r: shards[r].backward(w))
    _same_on_every_rank("off-grid dW", got)
    key = "tf32" if dt == "f32" else dt
    ref_abs = sum(s.dw_abs for s in shards)
    terms = torch.stack([s.t_k for s in shards]).sum(0)[None, :, None] + world
    extra = U_OUT[key] * ref_abs if fma else 0.0        # each rank rounds before its push
    _check("off-grid dW", got[0].reshape(K, 27, C), sum(s.dw for s in shards), ref_abs, terms, key, extra=extra)
    if dt == "f32":
        want = (plain[0] + plain[1]) + plain[2]
        assert torch.equal(got[0], want), "not the rank-order fp32 sum of the plain gradients"


# ------------------------------------------------------------------ 3. graph replay with several ranks
GRAPH_SHAPE = [24, 24, 24]


def _round16(t):
    return t.to(torch.float16).double()


def _chain_reference(convs, x, ws, dy3):
    """float64 forward and backward of SubM -> strided -> SubM with every intermediate rounded to fp16 once,
    as the kernels round it; asserts that every kernel sum is exact (|terms| below 2^24 of its quantum)"""
    c1, c2, c3 = convs
    w1, w2, w3 = ws
    dev = x.device

    def ref(conv, a, w, d, q_out, q_in):
        r = _reference(a, w, d, conv.ref_pair, dev)
        assert float(r["out_abs"].max()) < 2.0 ** 24 * q_out and float(r["din_abs"].max()) < 2.0 ** 24 * q_in
        return r
    # quanta: x, dy3 2^-3; w 2^-1 -> y1 2^-4, y2 2^-5, y3 2^-6, dy2 2^-4, dy1 2^-5, every dW 2^-8
    zeros = lambda n: torch.zeros((n, w1.shape[0]), dtype=torch.float64, device=dev)    # noqa: E731
    y1 = _round16(ref(c1, x, w1, zeros(c1.n_out), 2.0 ** -4, 1.0)["out"])
    y2 = _round16(ref(c2, y1, w2, zeros(c2.n_out), 2.0 ** -5, 1.0)["out"])
    r3 = ref(c3, y2, w3, dy3, 2.0 ** -6, 2.0 ** -4)
    r2 = ref(c2, y1, w2, _round16(r3["din"]), 2.0 ** -5, 2.0 ** -5)
    r1 = ref(c1, x, w1, _round16(r2["din"]), 2.0 ** -4, 1.0)
    return r3, [r1, r2, r3]


@gpu
@pytest.mark.parametrize("world", [2, 8])
def test_graph_replay_of_a_training_step(world, oracle, cuda_dev):
    """Every rank captures forward + backward of SubM -> SparseConv3d stride 2 (output bound) -> SubM on
    padded inputs, with its group installed; the graphs keep their group after set_peer_group(None).  All
    ranks' graphs replay together 20 times on fresh grid inputs, and every replay must give the exact
    output and the exact mean weight gradients: a stale slot or a missed epoch advance would not."""
    import spconv_b200.pytorch as spconv
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    C, rows, replays = 16, 1024, 20
    algo = ConvAlgo.MaskImplicitGemm
    gen = torch.Generator(device=cuda_dev).manual_seed(7 + world)
    clouds, convs = [], []
    for r in range(world):
        _, inds = random_cloud(np.random.default_rng(700 + r), GRAPH_SHAPE, [600 + 40 * r], 1)
        c1 = Conv(oracle, cuda_dev, inds, 1, GRAPH_SHAPE, 3, 1, 0, 1, True)
        c2 = Conv(oracle, cuda_dev, inds, 1, GRAPH_SHAPE, 3, 2, 1, 1, False)
        down = oracle.get_indice_pairs(inds, 1, GRAPH_SHAPE, [3] * 3, [2] * 3, [1] * 3, [1] * 3, [0] * 3, False)[0]
        c3 = Conv(oracle, cuda_dev, down, 1, [12, 12, 12], 3, 1, 0, 1, True)
        clouds.append((inds, down))
        convs.append((c1, c2, c3))
    bound = 128 * math.ceil(max(c[1].n_out for c in convs) * 1.25 / 128)
    net = torch.nn.ModuleList([spconv.SubMConv3d(C, C, 3, bias=False, algo=algo),
                               spconv.SparseConv3d(C, C, 3, 2, 1, bias=False, algo=algo),
                               spconv.SubMConv3d(C, C, 3, bias=False, algo=algo)]).to(cuda_dev).half().train()
    net[1].num_out_act_bound = bound
    with torch.no_grad():
        for layer in net:
            layer.weight.copy_(_grid(gen, tuple(layer.weight.shape), cuda_dev) * 4)      # integers in [-2, 2] / 2
    w64 = [layer.weight.detach().double() for layer in net]
    nets = [copy.deepcopy(net) for _ in range(world)]
    xs = [torch.zeros((rows, C), dtype=torch.float16, device=cuda_dev) for _ in range(world)]
    dys = [torch.zeros((bound, C), dtype=torch.float16, device=cuda_dev) for _ in range(world)]
    bases = []
    for r, (inds, _) in enumerate(clouds):
        t = spconv.SparseConvTensor(xs[r][:len(inds)].clone(), torch.from_numpy(inds).to(cuda_dev), GRAPH_SHAPE, 1)
        bases.append(t.pad_to(rows))

    def step(r):
        y = bases[r].replace_feature(xs[r])
        for layer in nets[r]:
            y = layer(y)
        grads = torch.autograd.grad(y.features, [layer.weight for layer in nets[r]], dys[r])
        return y.features, grads

    def refill():
        for r, (inds, down) in enumerate(clouds):
            xs[r][:len(inds)] = _grid(gen, (len(inds), C), cuda_dev).half()
            dys[r][:len(down)] = _grid(gen, (len(down), C), cuda_dev).half()

    def check(results, what):
        refs = [_chain_reference(convs[r], xs[r][:len(clouds[r][0])].double(), w64,
                                 dys[r][:len(clouds[r][1])].double()) for r in range(world)]
        for r, (y, _) in enumerate(results):
            n = len(clouds[r][1])
            _assert_exact(f"{what} rank {r} output", y[:n], refs[r][0]["out"], refs[r][0]["out_abs"], 2.0 ** -6,
                          torch.float16)
        for i in range(3):
            got = [res[1][i] for res in results]
            _same_on_every_rank(f"{what} dW{i + 1}", got)
            layer_refs = [ref[1][i] for ref in refs]
            _assert_fused(f"{what} dW{i + 1}", got[0].reshape(C, 27, C), [a["dw"] for a in layer_refs],
                          [a["dw_abs"] for a in layer_refs], "f16", 1.0 / world, SIMT, q=2.0 ** -8)

    streams = [torch.cuda.Stream() for _ in range(world)]
    with _ring(world, average=True) as ring:
        refill()
        check(_round(ring, streams, step), "eager warm-up")          # all ranks together: none waits alone
        graphs, static = [], []
        for r in range(world):
            ops.set_peer_group(ring[r])
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=streams[r]):
                static.append(step(r))
            graphs.append(g)
        ops.set_peer_group(None)
        for it in range(replays):
            refill()
            torch.cuda.synchronize()
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    graphs[r].replay()
            torch.cuda.synchronize()
            check(static, f"replay {it}")
        del graphs, static


# (subm, dtype, C, K): Native SubM and strided layers, one per weight-gradient kernel family
NATIVE_GRAPH = [(True, "f16", 32, 64), (False, "bf16", 16, 16), (False, "f32", 16, 16)]


@gpu
def test_graph_replay_of_native_weight_gradients(oracle, cuda_dev):
    """ConvAlgo.Native captured with a group: each of 2 ranks captures the op-level backward of a SubM and two
    strided layers (rulebooks built before capture; input gradient and finish on the forked stream).  The graphs replay
    together 5 times on fresh grid inputs, and every replay must give the exact mean weight gradients,
    bit-identical on both ranks."""
    from spconv_b200.pytorch import ops
    world, replays = 2, 5
    gen = torch.Generator(device=cuda_dev).manual_seed(77)
    layers = []
    for it, (subm, dt, C, K) in enumerate(NATIVE_GRAPH):
        w = _grid(gen, (K, 3, 3, 3, C), cuda_dev).to(TORCH_DT[dt])
        layers.append((_shards(oracle, cuda_dev, world, it, "native", subm, dt, C, K, w, gen, empty=-1), w))

    def step(r):
        return [shards[r].backward(w) for shards, w in layers]

    def refill():
        for shards, w in layers:
            for s in shards:
                x, dout = _grid(gen, tuple(s.x.shape), cuda_dev), _grid(gen, tuple(s.dout.shape), cuda_dev)
                s.x.copy_(x)
                s.dout.copy_(dout)
                ref = _reference(x, w.float(), dout, s.conv.ref_pair, cuda_dev)
                s.dw, s.dw_abs = ref["dw"], ref["dw_abs"]

    def check(results, what):
        for i, ((shards, _), (subm, dt, C, K)) in enumerate(zip(layers, NATIVE_GRAPH)):
            name = f"{what}, layer {i} ({'subm' if subm else 'strided'}, {dt})"
            got = [res[i] for res in results]
            _same_on_every_rank(name, got)
            _assert_fused(name, got[0].reshape(K, 27, C), [s.dw for s in shards], [s.dw_abs for s in shards], dt,
                          scale, _family(dt, 27, C, K) == 1)

    streams = [torch.cuda.Stream() for _ in range(world)]
    with _ring(world, average=True) as ring:
        scale = ring[0].scale
        check(_round(ring, streams, step), "eager warm-up")
        graphs, static = [], []
        for r in range(world):
            ops.set_peer_group(ring[r])
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=streams[r]):
                static.append(step(r))
            graphs.append(g)
        ops.set_peer_group(None)
        for it in range(replays):
            refill()
            torch.cuda.synchronize()
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    graphs[r].replay()
            torch.cuda.synchronize()
            check(static, f"replay {it}")
        del graphs, static


# ------------------------------------------------------------------ 4. peer_allreduce_ edges
@gpu
@pytest.mark.parametrize("world", [8, 16])
@pytest.mark.parametrize("dt", ["f16", "bf16", "f32"])
def test_small_tensor_allreduce_edges(dt, world, cuda_dev):
    """Counts 1, 3, 4, 5 (a partial last float4), 2047 and exactly the capacity, twice so both slots are
    reused; world 8 and 16 (SPX_MAX_PEERS) take the finish kernel's shared memory above 48 KB.  Integer
    values: every mean is exact in every type.  One value more than the capacity raises before anything is
    launched, and the next exchange still succeeds on every rank."""
    from spconv_b200 import _cabi
    from spconv_b200.pytorch import ops
    if world == 16:
        assert _cabi.SPX_MAX_PEERS == 16
    tdt = TORCH_DT[dt]
    cap_bytes = 1 << 15
    cap = cap_bytes // 4
    streams = [torch.cuda.Stream() for _ in range(world)]
    gen = torch.Generator(device=cuda_dev).manual_seed(world)

    def exchange(n):
        parts = [torch.randint(-8, 9, (n,), generator=gen, device=cuda_dev).to(tdt) for _ in range(world)]
        want = (sum(p.double() for p in parts) / world).to(tdt)
        work = [p.clone() for p in parts]
        _round(ring, streams, lambda r: ops.peer_allreduce_(work[r]))
        for r in range(world):
            assert torch.equal(work[r], want), f"count {n}, rank {r}"

    with _ring(world, average=True, capacity_bytes=cap_bytes) as ring:
        for n in [1, 3, 4, 5, 2047, cap] * 2:
            exchange(n)
        over = [torch.full((cap + 1,), 3, dtype=tdt, device=cuda_dev) for _ in range(world)]
        torch.cuda.synchronize()
        for r in range(world):
            ops.set_peer_group(ring[r])
            with pytest.raises(RuntimeError, match="exchange capacity"):
                ops.peer_allreduce_(over[r])
        ops.set_peer_group(None)
        torch.cuda.synchronize()
        assert all(bool((o == 3).all()) for o in over), "a refused exchange wrote its tensor"
        exchange(5)
        exchange(cap)


# ------------------------------------------------------------------ 5. the hook
# (algo, subm, dtype, C, K, empty)
HOOK = [("igemm", True, "f16", 32, 32, False), ("igemm", False, "bf16", 64, 32, False),
        ("igemm", True, "f16", 48, 24, False), ("igemm", False, "f16", 32, 32, True),
        ("native", True, "f16", 32, 32, False), ("native", False, "f16", 3, 5, False),
        ("native", True, "f16", 32, 32, True),
        ("split", True, "f16", 32, 32, False), ("split", False, "f16", 32, 32, False)]


class _Recorder:
    """the hook: records what it sees and where, then halves dW in place"""

    def __init__(self):
        self.calls = []

    def __call__(self, dw):
        self.calls.append((dw.clone(), torch.cuda.current_stream()))
        dw.mul_(0.5)


def _hook_layers(oracle, dev, cases, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for i, (algo, subm, dt, C, K, empty) in enumerate(cases):
        w = _grid(gen, (K, 3, 3, 3, C), dev).to(TORCH_DT[dt])
        inds = None if empty else random_cloud(np.random.default_rng(seed + i), SHAPE, [900], 1)[1]
        out.append((Shard(oracle, dev, inds, subm, algo, dt, C, K, w, gen), w))
    return out


def _plain_parts(s, w):
    """what the hook must see: the layer's dW, or each split's"""
    if s.algo == "split":
        return [s.split_backward(w, j) for j in range(s.parts)]
    return [s.backward(w)]


@gpu
@pytest.mark.parametrize("case", HOOK, ids=lambda c: f"{c[0]}-{'subm' if c[1] else 'strided'}-{c[2]}-C{c[3]}K{c[4]}"
                         + ("-empty" if c[5] else ""))
def test_wgrad_hook_eager(case, oracle, cuda_dev):
    """Once per weight gradient (once per split under MaskSplitImplicitGemm), on a stream other than the
    caller's, seeing the plain dW bit for bit; the op returns what the hook left (half the plain dW).  Also
    for a layer without rows and for ConvAlgo.Native."""
    from spconv_b200.pytorch import ops
    ((s, w),) = _hook_layers(oracle, cuda_dev, [case], 40)
    parts = _plain_parts(s, w)
    plain = s.backward(w)
    rec = _Recorder()
    ops.set_wgrad_hook(rec)
    caller = torch.cuda.current_stream()
    got = s.backward(w)
    ops.set_wgrad_hook(None)
    torch.cuda.synchronize()
    assert len(rec.calls) == s.parts, f"hook called {len(rec.calls)} times, want {s.parts}"
    for (seen, stream), part in zip(rec.calls, parts):
        assert stream != caller, "the hook ran on the caller's stream"
        assert torch.equal(seen, part), "the hook saw another dW than the plain one"
    assert torch.equal(got, plain * 0.5), "the op did not return what the hook left"


@gpu
def test_wgrad_hook_graph_replay(oracle, cuda_dev):
    """The same under CUDA-graph replay: the hook runs at capture, once per layer, and every replay on new
    inputs shows it the plain dW and returns half of it."""
    from spconv_b200.pytorch import ops
    cases = [c for c in HOOK if c[0] != "split"]            # a mask-split backward synchronises the host
    layers = _hook_layers(oracle, cuda_dev, cases, 60)
    gen = torch.Generator(device=cuda_dev).manual_seed(61)
    rec = _Recorder()
    ops.set_wgrad_hook(rec)
    for s, w in layers:                                     # warm-up
        s.backward(w)
    torch.cuda.synchronize()
    rec.calls.clear()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = [s.backward(w) for s, w in layers]
    ops.set_wgrad_hook(None)
    assert len(rec.calls) == len(layers)
    for it in range(5):
        for s, _ in layers:
            s.x.copy_(_grid(gen, tuple(s.x.shape), cuda_dev))
            s.dout.copy_(_grid(gen, tuple(s.dout.shape), cuda_dev))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert len(rec.calls) == len(layers), "the hook ran again at replay"
        for (s, w), case, (seen, stream), got in zip(layers, cases, rec.calls, outs):
            plain = s.backward(w)
            torch.cuda.synchronize()
            assert torch.equal(seen, plain), f"replay {it}, {case}: the hook saw another dW than the plain one"
            assert torch.equal(got, plain * 0.5), f"replay {it}, {case}: not half the plain dW"
    del g


# ------------------------------------------------------------------ 6. module-level training step
@gpu
@pytest.mark.parametrize("world", [2, 4])
def test_module_training_step(world, cuda_dev):
    """SubM -> SparseConv3d stride 2 -> SubM -> SparseInverseConv3d, all with bias, fp16, a 4-sample batch
    split with dist.shard_batch.  Every rank's forward first (the strided layer reads its output count back),
    then every rank's backward with its group: conv weight gradients come back identical on all ranks,
    within one rounding of the float64 mean of the plain gradients.  Bias gradients stay rank-local until
    ops.peer_allreduce_ reduces them."""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    from spconv_b200.pytorch.dist import shard_batch
    C = 16
    torch.manual_seed(world)
    net = spconv.SparseSequential(
        spconv.SubMConv3d(C, C, 3, bias=True, indice_key="s0"),
        spconv.SparseConv3d(C, C, 3, 2, 1, bias=True, indice_key="down"),
        spconv.SubMConv3d(C, C, 3, bias=True, indice_key="s1"),
        spconv.SparseInverseConv3d(C, C, 3, indice_key="down", bias=True)).to(cuda_dev).half().train()
    with torch.no_grad():
        for p in net.parameters():
            p.uniform_(-0.25, 0.25)
    feats, inds = random_cloud(np.random.default_rng(90 + world), SHAPE, [500, 650, 420, 580], C)
    feats_d, inds_d = torch.from_numpy(feats).to(cuda_dev).half(), torch.from_numpy(inds).to(cuda_dev)
    nets = [copy.deepcopy(net) for _ in range(world)]
    convs = [list(n.children()) for n in nets]
    inputs, dys = [], []
    for r in range(world):
        li, lf, lbs = shard_batch(inds_d, feats_d, 4, r, world)
        inputs.append(spconv.SparseConvTensor(lf, li, SHAPE, lbs))
        dys.append(torch.randn((len(li), C), device=cuda_dev).half())

    def run(r):
        out = nets[r](inputs[r])
        assert out.features.shape == dys[r].shape
        return out

    def grads(r):
        return [(m.weight.grad.clone(), m.bias.grad.clone()) for m in convs[r]]

    plain = []
    for r in range(world):
        run(r).features.backward(dys[r])
        plain.append(grads(r))
        nets[r].zero_grad(set_to_none=True)
    streams = [torch.cuda.Stream() for _ in range(world)]
    with _ring(world, average=True) as ring:
        torch.cuda.synchronize()
        outs = []
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                outs.append(run(r))
        _round(ring, streams, lambda r: outs[r].features.backward(dys[r]))
        fused = [grads(r) for r in range(world)]
        _round(ring, streams, lambda r: [ops.peer_allreduce_(m.bias.grad) for m in convs[r]])
        reduced = [[m.bias.grad.clone() for m in convs[r]] for r in range(world)]
    u = 2.0 ** -11

    def near_mean(name, got, parts):
        want = torch.stack([p.double() for p in parts]).mean(0)
        mag = torch.stack([p.double().abs() for p in parts]).mean(0)
        tol = u * (want.abs() + mag) + 2.0 ** -16 * mag + 2.0 ** -24
        err = (got.double() - want).abs()
        assert bool((err <= tol).all()), f"{name}: off the float64 mean by {float((err - tol).max()):.3g} over tol"

    for i in range(len(convs[0])):
        _same_on_every_rank(f"layer {i} dW", [fused[r][i][0] for r in range(world)])
        near_mean(f"layer {i} dW", fused[0][i][0], [plain[r][i][0] for r in range(world)])
        assert torch.equal(fused[0][i][1], plain[0][i][1]), f"layer {i}: the backward changed the local bias grad"
        _same_on_every_rank(f"layer {i} bias grad after peer_allreduce_", [reduced[r][i] for r in range(world)])
        near_mean(f"layer {i} bias grad", reduced[0][i], [plain[r][i][1] for r in range(world)])
    assert any(not torch.equal(fused[0][i][1], fused[1][i][1]) for i in range(len(convs[0]))), \
        "bias gradients already equal before peer_allreduce_: the samples do not differ"
