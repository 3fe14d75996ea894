"""Depthwise sparse convolution (groups = in_channels = out_channels) on the GPU against the float64 reference of
tests/depthwise_ref.py: every kind and dimension, kernel volumes up to 343 on all three algos, the 16-byte and
the per-element channel paths, the inference epilogue and BN / activation fusion, determinism under padding and
bounded rulebooks, CUDA-graph replay, rulebook sharing with dense layers, the data-parallel weight-gradient
routes and AMP.

Integer-grid data makes every fp32 sum exact, so outputs and gradients must equal the reference rounded once to
the dtype, bit for bit.  Random data is checked against |got - ref| <= u |ref| + T 2^-24 sum|terms| + tiny.
"""
import copy

import numpy as np
import pytest
import torch
from torch import nn

import spconv_b200.pytorch as spconv
from spconv_b200.core import Activation, ConvAlgo
from spconv_b200.pytorch import ops
from tests.conv_ref import SparseConvRef, linear_keys
from tests.depthwise_ref import depthwise_backward, depthwise_forward
from tests.util import random_cloud

pytestmark = pytest.mark.gpu

TORCH_DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
U_OUT = {"f32": 2.0 ** -24, "f16": 2.0 ** -11, "bf16": 2.0 ** -8}
TINY = {"f32": 1e-30, "f16": 2.0 ** -24, "bf16": 1e-30}
SHAPES = {1: [2000], 2: [40, 45], 3: [19, 18, 17], 4: [9, 10, 11, 12]}
ALGOS = {"igemm": ConvAlgo.MaskImplicitGemm, "split": ConvAlgo.MaskSplitImplicitGemm, "native": ConvAlgo.Native}
CLS = {"subm": "SubMConv", "conv": "SparseConv", "transpose": "SparseConvTranspose", "inverse": "SparseInverseConv"}


@pytest.fixture(autouse=True)
def _no_hook():
    yield
    ops.set_wgrad_hook(None)
    ops.set_peer_group(None)


def _np(t):
    return t.detach().double().cpu().numpy()


def _perm(gpu_inds, ref_inds, shape):
    """row j of the GPU rows is row p[j] of the reference rows (same coordinate)"""
    g = linear_keys(np.asarray(gpu_inds, np.int64), shape)
    r = linear_keys(np.asarray(ref_inds, np.int64), shape)
    order = np.argsort(r)
    pos = np.minimum(np.searchsorted(r[order], g), len(r) - 1)
    assert len(g) == len(r) and np.array_equal(r[order][pos], g), "GPU and reference coordinates differ"
    return order[pos]


def _data(gen, shape, dev, grid, lo=-2, hi=2):
    if grid:
        return torch.randint(lo, hi + 1, shape, generator=gen, device=dev).float()
    return torch.randn(shape, generator=gen, device=dev)


def _layer(kind, nd, C, k, algo, **kw):
    cls = getattr(spconv, f"{CLS[kind]}{nd}d")
    if kind == "subm":
        return cls(C, C, k, groups=C, algo=algo, **kw)
    if kind == "inverse":
        return cls(C, C, k, indice_key="down", groups=C, algo=algo, **kw)
    return cls(C, C, k, 2, 1, groups=C, algo=algo, indice_key="down" if kind == "conv" else None, **kw)


class Case:
    """One depthwise layer on a seeded cloud: the GPU out / dx / dW / db in reference row order, and the float64
    reference of each with its sum of |terms|."""

    def __init__(self, dev, kind, nd, dt, C, k=3, algo="igemm", grid=True, seed=0, pts=(700, 500), bias=True,
                 large_kernel_fast_algo=False, cloud=None):
        tdt = TORCH_DT[dt]
        shape = SHAPES[nd]
        rng = np.random.default_rng(seed)
        inds = cloud if cloud is not None else random_cloud(rng, shape, list(pts), 1)[1]
        batch = int(inds[:, 0].max()) + 1
        gen = torch.Generator(device=dev).manual_seed(seed)
        a = ALGOS[algo]
        mod = _layer(kind, nd, C, k, a, bias=bias, large_kernel_fast_algo=large_kernel_fast_algo).to(dev)
        self.mod = mod
        with torch.no_grad():
            mod.weight.copy_(_data(gen, tuple(mod.weight.shape), dev, grid) * (1.0 if grid else 0.3))
            if bias:
                mod.bias.copy_(_data(gen, (C,), dev, grid))
        mod.to(tdt).train()
        inds_d = torch.from_numpy(inds).to(dev)
        kz = [k] * nd
        if kind == "inverse":
            down = _layer("conv", nd, C, k, a).to(dev).to(tdt)
            x0 = spconv.SparseConvTensor(torch.zeros((len(inds), C), device=dev, dtype=tdt), inds_d, shape, batch)
            with torch.no_grad():
                mid = down(x0)
            paired = SparseConvRef(inds, batch, shape, kz, [2] * nd, [1] * nd, [1] * nd, kind="conv")
            ref = SparseConvRef(inds, batch, shape, kz, [2] * nd, [1] * nd, [1] * nd, kind="inverse")
            p_in = _perm(mid.indices.cpu().numpy(), paired.out_inds, paired.out_shape)
            # values drawn per reference row, so every algo sees the same value at each coordinate
            x_ref = _data(gen, (paired.n_out, C), dev, grid).to(tdt)
            x_in = mid.replace_feature(x_ref[torch.from_numpy(p_in).to(dev)].requires_grad_(True))
        else:
            st, pd = ([1] * nd, [0] * nd) if kind == "subm" else ([2] * nd, [1] * nd)
            ref = SparseConvRef(inds, batch, shape, kz, st, pd, [1] * nd, kind=kind)
            p_in = np.arange(len(inds))
            x_in = spconv.SparseConvTensor(_data(gen, (len(inds), C), dev, grid).to(tdt).requires_grad_(True), inds_d,
                                           shape, batch)
        feats = x_in.features
        y = mod(x_in)
        out_shape = ref.out_shape
        p_out = _perm(y.indices.cpu().numpy(), ref.out_inds, out_shape)
        dy = _data(gen, (ref.n_out, C), dev, grid, -1, 1).to(tdt)[torch.from_numpy(p_out).to(dev)]
        y.features.backward(dy)
        self.y, self.dx = y.features.detach(), feats.grad
        self.dw, self.db = mod.weight.grad, (mod.bias.grad if bias else None)
        # reference on the rounded inputs, rows in reference order
        x_r = np.zeros((ref.n_in, C))
        x_r[p_in] = _np(feats)
        dy_r = np.zeros((ref.n_out, C))
        dy_r[p_out] = _np(dy)
        w = _np(mod.weight)
        b = _np(mod.bias) if bias else None
        self.ref_y, self.mag_y = depthwise_forward(ref, x_r, w, b)
        self.ref_dx, self.mag_dx, self.ref_dw, self.mag_dw = depthwise_backward(ref, x_r, w, dy_r)
        self.ref_db = dy_r.sum(0)
        self.p_in, self.p_out, self.dt, self.kv, self.rows = p_in, p_out, dt, ref.kv, ref.n_out
        self.ref = ref

    def gpu_in_ref_order(self):
        """(y, dx) with rows in reference order, dW, db (torch tensors)"""
        y = torch.empty_like(self.y)
        y[torch.from_numpy(self.p_out).to(y.device)] = self.y
        dx = torch.empty_like(self.dx)
        dx[torch.from_numpy(self.p_in).to(dx.device)] = self.dx
        return y, dx, self.dw, self.db

    def check_exact(self):
        tdt = TORCH_DT[self.dt]
        y, dx, dw, db = self.gpu_in_ref_order()
        for name, got, ref in (("out", y, self.ref_y), ("dx", dx, self.ref_dx), ("dW", dw, self.ref_dw),
                               ("db", db, self.ref_db)):
            if got is None:
                continue
            want = torch.from_numpy(np.asarray(ref)).to(got.device).to(tdt).view(got.shape)
            bad = (got != want).sum().item()
            assert bad == 0, f"{name}: {bad} of {got.numel()} elements differ from the exact reference"

    def check_close(self):
        u, tiny = U_OUT[self.dt], TINY[self.dt]
        y, dx, dw, _ = self.gpu_in_ref_order()
        for name, got, ref, mag, terms in (("out", y, self.ref_y, self.mag_y, self.kv + 1),
                                           ("dx", dx, self.ref_dx, self.mag_dx, self.kv),
                                           ("dW", dw, self.ref_dw, self.mag_dw, self.rows)):
            g = _np(got).reshape(np.shape(ref))
            tol = u * np.abs(ref) + terms * 2.0 ** -24 * mag + tiny
            if name == "out":                  # the training bias is added after the output was rounded once
                tol = tol + u * mag
            err = np.abs(g - ref)
            assert (err <= tol).all(), f"{name}: off by {float((err - tol).max()):.3g} over the bound"


# ------------------------------------------------------------------ 1. every kind and dimension
KIND_CASES = [("subm", 3), ("conv", 3), ("transpose", 3), ("inverse", 3)] + \
             [(k, nd) for nd in (1, 2, 4) for k in ("subm", "conv")]


@pytest.mark.parametrize("kind, nd", KIND_CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_every_kind_exact(kind, nd, dt, cuda_dev):
    Case(cuda_dev, kind, nd, dt, 16, seed=nd * 7 + len(kind)).check_exact()


@pytest.mark.parametrize("kind, nd", KIND_CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_every_kind_random(kind, nd, dt, cuda_dev):
    Case(cuda_dev, kind, nd, dt, 24, grid=False, seed=nd * 5 + len(kind)).check_close()


# ------------------------------------------------------------------ 2. kernel volumes and algos
@pytest.mark.parametrize("kind, k, algo, fast, want_algo", [
    ("subm", 1, "igemm", False, ConvAlgo.MaskImplicitGemm),     # kv 1, SubM: x * W[c] in torch
    ("conv", 1, "igemm", False, ConvAlgo.MaskImplicitGemm),     # kv 1, stride 2: the kernels with one offset
    ("subm", 3, "igemm", False, ConvAlgo.MaskImplicitGemm),
    ("subm", 5, None, True, ConvAlgo.MaskImplicitGemm),         # kv 125: four mask words
    ("conv", 5, None, True, ConvAlgo.MaskImplicitGemm),
    ("subm", 7, None, False, ConvAlgo.Native),                  # kv 343: the default algo is Native
    ("conv", 7, None, False, ConvAlgo.Native),
])
def test_kernel_volumes(kind, k, algo, fast, want_algo, cuda_dev):
    if algo is None:
        algo = "igemm" if want_algo == ConvAlgo.MaskImplicitGemm else "native"
    c = Case(cuda_dev, kind, 3, "f16", 16, k=k, algo=algo, seed=k, bias=False, large_kernel_fast_algo=fast)
    assert c.mod.algo == want_algo
    c.check_exact()


@pytest.mark.parametrize("kind", ["subm", "conv", "inverse"])
def test_algos_agree_bit_for_bit(kind, cuda_dev):
    """The same layer on MaskImplicitGemm, MaskSplitImplicitGemm and Native: ascending k on all three, so the
    same bits per output coordinate"""
    res = [Case(cuda_dev, kind, 3, "f16", 32, algo=a, grid=False, seed=3).gpu_in_ref_order()
           for a in ("igemm", "split", "native")]
    for other in res[1:]:
        for name, a, b in zip(("out", "dx", "dW", "db"), res[0], other):
            assert torch.equal(a, b), name


def test_default_algo_of_a_large_depthwise_layer():
    assert spconv.SubMConv3d(8, 8, 7, groups=8).algo == ConvAlgo.Native
    assert spconv.SubMConv3d(8, 8, 3, groups=8).algo == ConvAlgo.MaskImplicitGemm


# ------------------------------------------------------------------ 3. channel paths and row counts
@pytest.mark.parametrize("dt, C", [("f16", 16), ("f16", 64), ("f16", 256), ("f32", 4), ("f32", 64),
                                   ("f16", 3), ("f16", 12), ("f32", 5), ("bf16", 8)])
@pytest.mark.parametrize("kind", ["subm", "conv"])
def test_channel_paths(dt, C, kind, cuda_dev):
    Case(cuda_dev, kind, 3, dt, C, seed=C).check_exact()


def test_misaligned_rows_take_the_element_path(cuda_dev):
    """feature rows that are 16-byte multiples but start off a 16-byte boundary"""
    gen = torch.Generator(device=cuda_dev).manual_seed(1)
    C, kv, n = 16, 27, 300
    base = _data(gen, (n * C + 1,), cuda_dev, True).half()
    x = base[1:].view(n, C)
    w = _data(gen, (C, 3, 3, 3, 1), cuda_dev, True).half()
    table = torch.randint(-1, n, (kv, n), generator=gen, device=cuda_dev, dtype=torch.int32)
    got = ops.depthwise_conv(x, w, table, n)
    want = ops.depthwise_conv(x.contiguous().clone(), w, table, n)
    assert x.data_ptr() % 16 != 0 and torch.equal(got, want)


@pytest.mark.parametrize("rows", [0, 1, 511, 512, 513, 1537])
@pytest.mark.parametrize("dt, C", [("f16", 64), ("f16", 3), ("f32", 4)])
def test_row_counts_at_the_op(rows, dt, C, cuda_dev):
    """ops-level: a random table over `rows` outputs and 700 inputs, the backward table its transpose"""
    tdt = TORCH_DT[dt]
    gen = torch.Generator(device=cuda_dev).manual_seed(rows + C)
    kv, n_in = 27, 700
    rng = np.random.default_rng(rows)
    t_fwd = np.full((kv, rows), -1, np.int32)
    t_bwd = np.full((kv, n_in), -1, np.int32)
    for k in range(kv):                                  # injective per offset, as every rulebook is
        m = min(rows, n_in)
        outs = rng.permutation(rows)[: (m + 1) // 2]
        ins = rng.permutation(n_in)[: len(outs)]
        t_fwd[k, outs] = ins
        t_bwd[k, ins] = outs
    x = _data(gen, (n_in, C), cuda_dev, True).to(tdt)
    w = _data(gen, (C, 3, 3, 3, 1), cuda_dev, True).to(tdt)
    dy = _data(gen, (rows, C), cuda_dev, True, -1, 1).to(tdt)
    tf, tb = torch.from_numpy(t_fwd).to(cuda_dev), torch.from_numpy(t_bwd).to(cuda_dev)
    y = ops.depthwise_conv(x, w, tf, rows)
    dx, dw = ops.depthwise_conv_backward(x, w, dy, tf, tb)
    xr, wr, dyr = _np(x), _np(w).reshape(C, kv), _np(dy)
    y_r = np.zeros((rows, C))
    dx_r = np.zeros((n_in, C))
    dw_r = np.zeros((C, kv))
    for k in range(kv):
        o = np.nonzero(t_fwd[k] >= 0)[0]
        i = t_fwd[k, o]
        y_r[o] += xr[i] * wr[:, k]
        dx_r[i] += dyr[o] * wr[:, k]
        dw_r[:, k] = (dyr[o] * xr[i]).sum(0)
    assert torch.equal(y, torch.from_numpy(y_r).to(cuda_dev).to(tdt))
    assert torch.equal(dx, torch.from_numpy(dx_r).to(cuda_dev).to(tdt))
    assert torch.equal(dw.view(C, kv), torch.from_numpy(dw_r).to(cuda_dev).to(tdt))
    if rows == 0:                                        # an empty output: dW = 0, dx = 0
        assert bool((dw == 0).all()) and bool((dx == 0).all())


# ------------------------------------------------------------------ 4. inference epilogue and fusion
@pytest.mark.parametrize("act", [Activation.None_, Activation.ReLU, Activation.LeakyReLU, Activation.Sigmoid])
@pytest.mark.parametrize("algo", ["igemm", "native"])
def test_inference_epilogue(act, algo, cuda_dev):
    C = 32
    rng = np.random.default_rng(5)
    _, inds = random_cloud(rng, SHAPES[3], [900], 1)
    gen = torch.Generator(device=cuda_dev).manual_seed(5)
    m = spconv.SubMConv3d(C, C, 3, groups=C, algo=ALGOS[algo], act_type=act, act_alpha=0.125).to(cuda_dev).half()
    m.eval()
    x = _data(gen, (len(inds), C), cuda_dev, False).half()
    with torch.no_grad():
        y = m(spconv.SparseConvTensor(x, torch.from_numpy(inds).to(cuda_dev), SHAPES[3], 1)).features
    ref = SparseConvRef(inds, 1, SHAPES[3], [3] * 3, [1] * 3, [0] * 3, [1] * 3, kind="subm")
    r, mag = depthwise_forward(ref, _np(x), _np(m.weight), _np(m.bias))
    r = {Activation.None_: r, Activation.ReLU: np.maximum(r, 0), Activation.LeakyReLU: np.where(r >= 0, r, 0.125 * r),
         Activation.Sigmoid: 1 / (1 + np.exp(-r))}[act]
    err = np.abs(_np(y) - r)
    assert (err <= 2.0 ** -11 * np.abs(r) + 28 * 2.0 ** -24 * mag + 1e-6).all()


def test_fuse_bn_and_act(cuda_dev):
    C = 24
    rng = np.random.default_rng(6)
    _, inds = random_cloud(rng, SHAPES[3], [900], 1)
    torch.manual_seed(6)
    bn = nn.BatchNorm1d(C)
    with torch.no_grad():
        bn.running_mean.uniform_(-1, 1)
        bn.running_var.uniform_(0.5, 2)
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    net = spconv.SparseSequential(spconv.SubMConv3d(C, C, 3, groups=C), bn, nn.ReLU()).to(cuda_dev).eval()
    fused = spconv.fuse_act(spconv.fuse_bn(net[0], net[1]), net[2])
    assert fused.act_type == Activation.ReLU and list(fused.weight.shape) == [C, 3, 3, 3, 1]
    x = spconv.SparseConvTensor(torch.randn((len(inds), C), device=cuda_dev), torch.from_numpy(inds).to(cuda_dev),
                                SHAPES[3], 1)
    with torch.no_grad():
        want = net(x).features
        got = fused(x).features
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------ 5. determinism and padding
def test_two_runs_are_identical(cuda_dev):
    a = Case(cuda_dev, "subm", 3, "f16", 64, grid=False, seed=9).gpu_in_ref_order()
    b = Case(cuda_dev, "subm", 3, "f16", 64, grid=False, seed=9).gpu_in_ref_order()
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _grads(net):
    return [p.grad.detach().clone() for p in net.parameters()]


def _train_step(net, x, dy):
    for p in net.parameters():
        p.grad = None
    xf = x.features.detach().clone().requires_grad_(True)
    y = net(x.replace_feature(xf))
    y.features.backward(dy[: y.features.shape[0]] if dy.shape[0] >= y.features.shape[0] else
                        torch.cat([dy, dy.new_zeros((y.features.shape[0] - dy.shape[0], dy.shape[1]))]))
    return y, xf.grad, _grads(net)


def test_padding_and_bounded_layer_change_nothing(cuda_dev):
    C, shape = 32, SHAPES[3]
    rng = np.random.default_rng(12)
    _, inds = random_cloud(rng, shape, [1500], 1)
    torch.manual_seed(12)
    net = spconv.SparseSequential(spconv.SubMConv3d(C, C, 3, groups=C, indice_key="s0"),
                                  spconv.SparseConv3d(C, C, 3, 2, 1, groups=C)).to(cuda_dev).half().train()
    x = spconv.SparseConvTensor(torch.randn((len(inds), C), device=cuda_dev).half(),
                                torch.from_numpy(inds).to(cuda_dev), shape, 1)
    dy = torch.randn((4000, C), device=cuda_dev).half()
    y0, dx0, g0 = _train_step(net, x, dy)
    m = y0.features.shape[0]
    net.eval()
    bounds = spconv.set_output_bounds(net, x, margin=1.5)
    net.train()
    assert bounds and next(iter(bounds.values())) > m
    y1, dx1, g1 = _train_step(net, x.pad_to(len(inds) + 333), dy)
    assert y1.features.shape[0] > m
    assert torch.equal(y1.features[:m], y0.features) and torch.equal(y1.indices[:m], y0.indices)
    assert torch.equal(dx1[: len(inds)], dx0)
    for a, b in zip(g1, g0):
        assert torch.equal(a, b)
    spconv.check_bounds(net)


def test_padded_native_large_kernel(cuda_dev):
    C, shape = 16, SHAPES[3]
    rng = np.random.default_rng(13)
    _, inds = random_cloud(rng, shape, [1200], 1)
    torch.manual_seed(13)
    net = spconv.SparseSequential(spconv.SubMConv3d(C, C, 7, groups=C)).to(cuda_dev).half().train()
    assert net[0].algo == ConvAlgo.Native
    x = spconv.SparseConvTensor(torch.randn((len(inds), C), device=cuda_dev).half(),
                                torch.from_numpy(inds).to(cuda_dev), shape, 1)
    dy = torch.randn((len(inds) + 100, C), device=cuda_dev).half()
    y0, dx0, g0 = _train_step(net, x, dy)
    y1, dx1, g1 = _train_step(net, x.pad_to(len(inds) + 100), dy)
    n = len(inds)
    assert torch.equal(y1.features[:n], y0.features) and torch.equal(dx1[:n], dx0)
    for a, b in zip(g1, g0):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ 6. capture
def test_graph_replay_equals_eager(cuda_dev):
    C, shape = 32, SHAPES[3]
    rng = np.random.default_rng(14)
    clouds = [random_cloud(rng, shape, [n], 1)[1] for n in (1500, 1300)]
    torch.manual_seed(14)
    net = spconv.SparseSequential(spconv.SubMConv3d(C, C, 3, groups=C, indice_key="s0"),
                                  spconv.SparseConv3d(C, C, 3, 2, 1, groups=C, indice_key="down"),
                                  spconv.SparseInverseConv3d(C, C, 3, indice_key="down", groups=C)
                                  ).to(cuda_dev).half().train()
    params = list(net.parameters())
    feats = [torch.randn((len(c), C), device=cuda_dev).half() for c in clouds]
    n_pad = 1600
    net.eval()
    spconv.set_output_bounds(net, spconv.SparseConvTensor(feats[0], torch.from_numpy(clouds[0]).to(cuda_dev), shape, 1),
                             margin=1.5)
    net.train()
    padded = [spconv.SparseConvTensor(f, torch.from_numpy(c).to(cuda_dev), shape, 1).pad_to(n_pad)
              for f, c in zip(feats, clouds)]
    args = [(p.features, p.indices, p.num_valid) for p in padded]
    dy = torch.randn((n_pad, C), device=cuda_dev).half()

    def step(f, i, nv):
        for p in params:
            p.grad = None
        xf = f.detach().requires_grad_(True)
        x = spconv.SparseConvTensor(xf, i, shape, 1)
        x.num_valid = nv
        y = net(x)
        y.features.backward(dy)
        return [y.features.detach(), xf.grad] + [p.grad for p in params]

    want = [[t.clone() for t in step(*a)] for a in args]
    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 0):
        got = graphed(*args[k])
        for j, (a, b) in enumerate(zip(got, want[k])):
            assert torch.equal(a, b), f"replay of cloud {k}, result {j}"
    spconv.check_bounds(net)


# ------------------------------------------------------------------ 7. shared rulebooks
@pytest.mark.parametrize("dw_first", [True, False])
@pytest.mark.parametrize("algo", ["igemm", "native"])
def test_rulebook_shared_with_a_dense_layer(dw_first, algo, cuda_dev, monkeypatch):
    C, shape = 16, SHAPES[3]
    rng = np.random.default_rng(15)
    _, inds = random_cloud(rng, shape, [900], 1)
    a = ALGOS[algo]
    dw = spconv.SubMConv3d(C, C, 3, groups=C, indice_key="k", algo=a)
    dense = spconv.SubMConv3d(C, C, 3, indice_key="k", algo=a)
    net = spconv.SparseSequential(*([dw, dense] if dw_first else [dense, dw])).to(cuda_dev).half()
    builds = []
    name = "get_indice_pairs_implicit_gemm" if algo == "igemm" else "get_indice_pairs"
    orig = getattr(ops, name)
    monkeypatch.setattr(ops, name, lambda *args, **kw: builds.append(1) or orig(*args, **kw))
    x = spconv.SparseConvTensor(torch.randn((len(inds), C), device=cuda_dev).half(),
                                torch.from_numpy(inds).to(cuda_dev), shape, 1)
    with torch.no_grad():
        y = net(x)
        assert len(builds) == 1, "the second layer built its own rulebook"
        # the second layer computes on the shared rulebook what it computes on its own
        alone = copy.deepcopy(net[1])
        alone.indice_key = None
        want = alone(net[0](x)).features
    assert torch.equal(y.features, want)


# ------------------------------------------------------------------ 8. data-parallel
class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, dw):
        self.calls.append(dw.clone())
        dw.mul_(0.5)


def _dp_net(dev, C):
    torch.manual_seed(16)
    net = spconv.SparseSequential(spconv.SubMConv3d(C, C, 3, groups=C, indice_key="s0", bias=False),
                                  spconv.SparseConv3d(C, C, 3, 2, 1, groups=C, bias=False),
                                  spconv.SubMConv3d(C, C, 7, groups=C, bias=False)).to(dev).half().train()
    gen = torch.Generator(device=dev).manual_seed(16)
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(_data(gen, tuple(p.shape), dev, True))
    return net


def _dp_input(dev, C, seed):
    rng = np.random.default_rng(seed)
    _, inds = random_cloud(rng, SHAPES[3], [800], 1)
    gen = torch.Generator(device=dev).manual_seed(seed)
    return spconv.SparseConvTensor(_data(gen, (len(inds), C), dev, True).half(), torch.from_numpy(inds).to(dev),
                                   SHAPES[3], 1)


def test_wgrad_hook_eager_and_replayed(cuda_dev):
    C = 16
    net = _dp_net(cuda_dev, C)
    x = _dp_input(cuda_dev, C, 17)
    y = net(x)
    dy = torch.ones_like(y.features)
    y.features.backward(dy)
    plain = _grads(net)
    rec = _Recorder()
    ops.set_wgrad_hook(rec)
    net.zero_grad(set_to_none=True)
    net(x).features.backward(dy)
    ops.set_wgrad_hook(None)
    torch.cuda.synchronize()
    assert len(rec.calls) == 3
    for seen, want, got in zip(reversed(rec.calls), plain, _grads(net)):
        assert torch.equal(seen, want) and torch.equal(got, want * 0.5)
    # replayed: SubM 3x3x3 layers sharing one rulebook (no host read-back), the hook runs at capture
    subm = spconv.SparseSequential(copy.deepcopy(net[0]), copy.deepcopy(net[0]))
    params = list(subm.parameters())

    def step(f):
        for p in params:
            p.grad = None
        subm(x.replace_feature(f)).features.backward(torch.ones_like(f))
        return [p.grad for p in params]

    f0 = x.features.clone()
    ops.set_wgrad_hook(rec)
    graphed = spconv.graph_capture(step, f0)
    ops.set_wgrad_hook(None)
    rec.calls.clear()
    gen = torch.Generator(device=cuda_dev).manual_seed(18)
    for _ in range(2):
        f0.copy_(_data(gen, tuple(f0.shape), cuda_dev, True).half())
        got = [g.clone() for g in graphed(f0)]
        assert not rec.calls, "the hook ran again at replay"
        want = [g.clone() for g in step(f0)]
        for a, b in zip(got, want):
            assert torch.equal(a, b * 0.5)


def test_two_ranks_sum_depthwise_weight_gradients(cuda_dev):
    """two simulated ranks on streams of one GPU: every depthwise dW comes back as the rank-order sum, eagerly and
    from CUDA graphs of each rank's SubM layers (input gradient and finish on the forked stream) that replay
    together on fresh inputs"""
    from spconv_b200.pytorch.dist import PeerGroup
    C, world = 16, 2
    base = _dp_net(cuda_dev, C)
    nets = [copy.deepcopy(base) for _ in range(world)]
    xs = [_dp_input(cuda_dev, C, 20 + r) for r in range(world)]
    plain = []
    for r in range(world):
        y = nets[r](xs[r])
        y.features.backward(torch.ones_like(y.features))
        plain.append(_grads(nets[r]))
        nets[r].zero_grad(set_to_none=True)
    # captured: each rank's forward + backward of SubM 3x3x3 layers sharing one rulebook (no host read-back)
    subms = [spconv.SparseSequential(copy.deepcopy(base[0]), copy.deepcopy(base[0])) for _ in range(world)]
    feats = [x.features.clone() for x in xs]

    def step(r):
        for p in subms[r].parameters():
            p.grad = None
        y = subms[r](xs[r].replace_feature(feats[r]))
        y.features.backward(torch.ones_like(y.features))
        return [p.grad for p in subms[r].parameters()]

    def rank_order_sum(what, got, parts):
        for i in range(len(parts[0])):
            want = (parts[0][i].double() + parts[1][i].double()).half()
            assert torch.equal(got[0][i], got[1][i]), f"{what} layer {i}: ranks differ"
            assert torch.equal(got[0][i], want), f"{what} layer {i}: not the rank-order sum"

    for r in range(world):                          # warm-up
        step(r)
    streams = [torch.cuda.Stream() for _ in range(world)]
    ring = PeerGroup.local_ring(world, capacity_bytes=1 << 20, average=False)
    try:
        torch.cuda.synchronize()
        outs = []
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                outs.append(nets[r](xs[r]))
        torch.cuda.synchronize()
        for r in range(world):
            ops.set_peer_group(ring[r])
            with torch.cuda.stream(streams[r]):
                outs[r].features.backward(torch.ones_like(outs[r].features))
        ops.set_peer_group(None)
        torch.cuda.synchronize()
        rank_order_sum("eager", [_grads(n) for n in nets], plain)
        graphs, static = [], []
        for r in range(world):
            ops.set_peer_group(ring[r])
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=streams[r]):
                static.append(step(r))
            graphs.append(g)
        ops.set_peer_group(None)
        gen = torch.Generator(device=cuda_dev).manual_seed(21)
        for it in range(3):
            for f in feats:
                f.copy_(_data(gen, tuple(f.shape), cuda_dev, True).half())
            torch.cuda.synchronize()
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    graphs[r].replay()
            torch.cuda.synchronize()
            got = [[t.clone() for t in static[r]] for r in range(world)]
            rank_order_sum(f"replay {it}", got, [[t.clone() for t in step(r)] for r in range(world)])
        del graphs, static
        assert [pg.error() for pg in ring] == [0] * world
    finally:
        ops.set_peer_group(None)
        for pg in ring:
            pg.close()


# ------------------------------------------------------------------ 9. AMP
def test_autocast_equals_explicit_fp16(cuda_dev):
    C, shape = 32, SHAPES[3]
    rng = np.random.default_rng(21)
    _, inds = random_cloud(rng, shape, [900], 1)
    torch.manual_seed(21)
    m32 = spconv.SubMConv3d(C, C, 3, groups=C).to(cuda_dev).train()
    m16 = copy.deepcopy(m32).half()
    inds_d = torch.from_numpy(inds).to(cuda_dev)
    x = torch.randn((len(inds), C), device=cuda_dev)
    dy = torch.randn((len(inds), C), device=cuda_dev).half()
    x16 = x.half().requires_grad_(True)
    y16 = m16(spconv.SparseConvTensor(x16, inds_d, shape, 1)).features
    y16.backward(dy)
    x32 = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        y = m32(spconv.SparseConvTensor(x32, inds_d, shape, 1)).features
    assert y.dtype == torch.float16 and torch.equal(y, y16)
    y.backward(dy)
    assert torch.equal(x32.grad, x16.grad.float())
    assert torch.equal(m32.weight.grad, m16.weight.grad.float())
