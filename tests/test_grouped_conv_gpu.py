"""Grouped sparse convolution (1 < groups, group widths multiples of 16) on the GPU.

The main property: for every group j, out[:, j Kg:(j+1) Kg], din[:, j Cg:(j+1) Cg] and dW[j Kg:(j+1) Kg] equal bit
for bit what the dense layer of width Cg -> Kg returns on the contiguous slices of that group, on the same rulebook,
algo, dtype and fp32 mode, and on the same kernel family.  Grouped fp32 runs on the FMA kernels in both fp32 modes,
so in tf32 mode it equals the dense layer in exact mode.  Around that: float64 references, the algos, row counts,
the inference epilogue, padding, bounds and graph replay, shared rulebooks, conv onto given coordinates, the
weight-gradient hook and simulated ranks, AMP and unaligned operands."""
import numpy as np
import pytest
import torch

import spconv_b200.pytorch as spconv
from spconv_b200.core import Activation, ConvAlgo
from spconv_b200.pytorch import ops
from tests.conv_ref import SparseConvRef, linear_keys
from tests.grouped_ref import grouped_backward, grouped_forward
from tests.util import random_cloud

pytestmark = pytest.mark.gpu

TORCH_DT = {"f32": torch.float32, "tf32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
U = {"f32": 2.0 ** -24, "tf32": 2.0 ** -24, "f16": 2.0 ** -11, "bf16": 2.0 ** -8}
SHAPES = {1: [3000], 2: [50, 45], 3: [20, 18, 17], 4: [9, 10, 11, 12]}
ALGOS = {"igemm": ConvAlgo.MaskImplicitGemm, "split": ConvAlgo.MaskSplitImplicitGemm, "native": ConvAlgo.Native}
CLS = {"subm": "SubMConv", "conv": "SparseConv", "transpose": "SparseConvTranspose", "inverse": "SparseInverseConv"}


@pytest.fixture(autouse=True)
def _clean(monkeypatch):
    yield
    ops.set_wgrad_hook(None)
    ops.set_peer_group(None)


def _layer(kind, nd, C, K, k, algo, groups, stride=2, **kw):
    cls = getattr(spconv, f"{CLS[kind]}{nd}d")
    if kind == "subm":
        return cls(C, K, k, groups=groups, algo=algo, **kw)
    if kind == "inverse":
        return cls(C, K, k, indice_key="down", groups=groups, algo=algo, **kw)
    return cls(C, K, k, stride, k // 2, groups=groups, algo=algo, **kw)


def _data(gen, shape, dev, grid):
    if grid:
        return torch.randint(-2, 3, shape, generator=gen, device=dev).float()
    return torch.randn(shape, generator=gen, device=dev)


def _input(dev, kind, nd, C, k, tdt, gen, grid, pts, seed, algo=ConvAlgo.MaskImplicitGemm):
    """the input tensor of the layer: a cloud, or for an inverse layer the output of the strided conv (of the same
    algo) it walks back"""
    shape = SHAPES[nd]
    inds = random_cloud(np.random.default_rng(seed), shape, list(pts), 1)[1]
    batch = len(pts)
    inds_d = torch.from_numpy(inds).to(dev)
    if kind != "inverse":
        return spconv.SparseConvTensor(_data(gen, (len(inds), C), dev, grid).to(tdt), inds_d, shape, batch)
    down = _layer("conv", nd, 16, C, k, algo, 1, indice_key="down").to(dev).to(tdt)
    with torch.no_grad():
        mid = down(spconv.SparseConvTensor(torch.zeros((len(inds), 16), device=dev, dtype=tdt), inds_d, shape, batch))
    return mid.replace_feature(_data(gen, tuple(mid.features.shape), dev, grid).to(tdt))


def _run(mod, x, dy):
    """(out, din, dW, family of the forward)"""
    f = x.features.detach().clone().requires_grad_(True)
    y = mod(x.replace_feature(f))
    fam = ops.last_kernel_family()
    y.features.backward(dy)
    return y, f.grad, mod.weight.grad, fam


def _check_groups(dev, kind, nd, dt, C, K, g, k=3, algo="igemm", grid=False, seed=0, pts=(1500, 1100), stride=2,
                  monkeypatch=None, **kw):
    """run the grouped layer and, per group, the dense layer on the slices; assert bit equality and equal families.
    Returns the grouped (out tensor, din, dW, family)."""
    tdt = TORCH_DT[dt]
    gen = torch.Generator(device=dev).manual_seed(seed)
    a = ALGOS[algo]
    x = _input(dev, kind, nd, C, k, tdt, gen, grid, pts, seed, a)
    mod = _layer(kind, nd, C, K, k, a, g, stride, **kw).to(dev)
    with torch.no_grad():
        mod.weight.copy_(_data(gen, tuple(mod.weight.shape), dev, grid) * (1.0 if grid else 0.2))
        mod.bias.copy_(_data(gen, (K,), dev, grid))
    mod = mod.to(tdt).train()
    if monkeypatch is not None:
        monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", dt == "tf32")
    dy = _dy(gen, dev, x, mod, tdt, grid)
    y, din, dw, fam = _run(mod, x, dy)
    cg, kg = C // g, K // g
    for j in range(g):
        dense = _layer(kind, nd, cg, kg, k, a, 1, stride, **kw).to(dev).to(tdt).train()
        with torch.no_grad():
            dense.weight.copy_(mod.weight[j * kg:(j + 1) * kg])
            dense.bias.copy_(mod.bias[j * kg:(j + 1) * kg])
        if monkeypatch is not None:
            monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", False)       # grouped tf32 == dense exact
        xj = x.replace_feature(x.features[:, j * cg:(j + 1) * cg].contiguous())
        f = xj.features.detach().clone().requires_grad_(True)
        yj = dense(xj.replace_feature(f))
        fam_j = ops.last_kernel_family()
        yj.features.backward(dy[:, j * kg:(j + 1) * kg].contiguous())
        assert torch.equal(yj.indices, y.indices)
        assert fam_j == fam, f"group {j}: family {fam} grouped, {fam_j} dense"
        assert torch.equal(y.features[:, j * kg:(j + 1) * kg], yj.features), f"out of group {j}"
        assert torch.equal(din[:, j * cg:(j + 1) * cg], f.grad), f"din of group {j}"
        assert torch.equal(dw[j * kg:(j + 1) * kg], dense.weight.grad), f"dW of group {j}"
        if monkeypatch is not None:
            monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", dt == "tf32")
    return x, mod, y, din, dw, fam


_DY = [None]


def _dy(gen, dev, x, mod, tdt, grid):
    with torch.no_grad():
        n = mod(x).features.shape[0]
    _DY[0] = _data(gen, (n, mod.out_channels), dev, grid).to(tdt)
    return _DY[0]


# ------------------------------------------------------------------ 1. per-group bit equality
@pytest.mark.parametrize("kind", ["subm", "conv", "transpose", "inverse"])
@pytest.mark.parametrize("nd", [1, 2, 3, 4])
def test_every_kind_and_rank(kind, nd, cuda_dev):
    *_, fam = _check_groups(cuda_dev, kind, nd, "f16", 64, 64, 2)
    assert fam == 2


# (C, K, g) -> whether the forward runs on the tensor cores at 16 bits
SHAPE_SET = [(64, 64, 2, True), (128, 128, 4, True), (256, 256, 8, True), (256, 256, 16, True), (512, 512, 4, True),
             (64, 32, 2, True), (96, 96, 2, False), (512, 512, 2, False)]


@pytest.mark.parametrize("C, K, g, tc", SHAPE_SET)
@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_channel_shapes(C, K, g, tc, dt, cuda_dev):
    *_, fam = _check_groups(cuda_dev, "subm", 3, dt, C, K, g, pts=(900,))
    assert fam == (2 if tc else 1)


@pytest.mark.parametrize("algo", ["igemm", "split", "native"])
@pytest.mark.parametrize("kind", ["subm", "conv", "inverse"])
def test_algos(algo, kind, cuda_dev):
    _check_groups(cuda_dev, kind, 3, "f16", 128, 128, 4, algo=algo)


@pytest.mark.parametrize("dt", ["f32", "tf32"])
@pytest.mark.parametrize("kind", ["subm", "conv", "transpose"])
def test_fp32_runs_on_the_fma_kernels(dt, kind, cuda_dev, monkeypatch):
    *_, fam = _check_groups(cuda_dev, kind, 3, dt, 64, 64, 2, monkeypatch=monkeypatch)
    assert fam == 1


@pytest.mark.parametrize("k, stride, algo, fast", [(1, 2, "igemm", False), (3, 2, "igemm", False),
                                                   (5, 1, "native", False), (5, 1, "igemm", True)])
def test_kernel_volumes(k, stride, algo, fast, cuda_dev):
    kind = "conv" if stride == 2 else "subm"
    _check_groups(cuda_dev, kind, 3, "f16", 64, 64, 2, k=k, algo=algo, stride=stride, pts=(900,),
                  large_kernel_fast_algo=fast)


# ------------------------------------------------------------------ 2. against float64
def _ref(kind, x, mod, k=3):
    nd = mod.ndim
    inds = x.indices.cpu().numpy()
    kz = [k] * nd
    if kind == "subm":
        return SparseConvRef(inds, x.batch_size, x.spatial_shape, kz, [1] * nd, [k // 2] * nd, [1] * nd, kind="subm")
    return SparseConvRef(inds, x.batch_size, x.spatial_shape, kz, [2] * nd, [k // 2] * nd, [1] * nd, kind="conv")


def _perm(gpu_inds, ref_inds, shape):
    g = linear_keys(np.asarray(gpu_inds, np.int64), shape)
    r = linear_keys(np.asarray(ref_inds, np.int64), shape)
    order = np.argsort(r)
    pos = np.minimum(np.searchsorted(r[order], g), len(r) - 1)
    assert np.array_equal(r[order][pos], g)
    return order[pos]


@pytest.mark.parametrize("kind", ["subm", "conv"])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("grid", [True, False])
def test_against_float64(kind, dt, grid, cuda_dev):
    """integer-grid values: exact (bf16: bounded); random values: within the rounding bound of the sum of |terms|"""
    x, mod, y, din, dw, _ = _check_groups(cuda_dev, kind, 3, dt, 64, 64, 2, grid=grid)
    ref = _ref(kind, x, mod)
    xs, ws = x.features.double().cpu().numpy(), mod.weight.detach().double().cpu().numpy()
    b = mod.bias.detach().double().cpu().numpy()
    out, mag = grouped_forward(ref, xs, ws, 2, b)
    p = _perm(y.indices.cpu().numpy(), ref.out_inds, y.spatial_shape)
    got = y.features.detach().double().cpu().numpy()
    dy = _DY[0].double().cpu().numpy()
    dy_ref = np.zeros_like(dy)
    dy_ref[p] = dy
    dx, dxm, dwr, dwm = grouped_backward(ref, xs, ws, dy_ref, 2)
    gdx, gdw = din.double().cpu().numpy(), dw.double().cpu().numpy()
    if grid and dt != "bf16":          # integer sums stay exact in fp32 and (below 2048) in fp16, not in bf16
        assert np.array_equal(got, out[p]) and np.array_equal(gdx, dx) and np.array_equal(gdw, dwr)
    else:
        u = U[dt]
        tol = lambda m: 4 * u * (m + 1e-3) + 64 * 2.0 ** -24 * m
        assert np.all(np.abs(got - out[p]) <= tol(mag[p]))
        assert np.all(np.abs(gdx - dx) <= tol(dxm))
        assert np.all(np.abs(gdw - dwr) <= tol(dwm))


@pytest.mark.parametrize("grid", [True, False])
def test_algos_agree_and_runs_repeat(grid, cuda_dev):
    """SubM outputs of MaskImplicitGemm and Native agree bit for bit per output coordinate; on integer-grid values
    so do their input gradients (the two walk the offsets in opposite orders) and MaskSplit (its two splits' partial
    outputs are added in fp16); two runs give identical bits"""
    res = {}
    for algo in ALGOS:
        x, mod, y, din, dw, _ = _check_groups(cuda_dev, "subm", 3, "f16", 128, 128, 4, algo=algo, seed=3, grid=grid)
        res[algo] = (y.features.detach().clone(), din.clone())
        if algo == "igemm":
            dw1 = dw.clone()
            mod.weight.grad = None
            y2, din2, dw2, _ = _run(mod, x, _DY[0])
            assert torch.equal(y2.features, y.features) and torch.equal(din2, din) and torch.equal(dw2, dw1)
    assert torch.equal(res["native"][0], res["igemm"][0])
    if grid:
        for algo in ("split", "native"):
            assert torch.equal(res[algo][0], res["igemm"][0]) and torch.equal(res[algo][1], res["igemm"][1]), algo


@pytest.mark.parametrize("rows", [0, 1, 127, 129, 300])
def test_row_counts_at_the_op(rows, cuda_dev):
    """the grouped op on a SubM rulebook of `rows` rows (0: no input and an empty output) equals the dense op per
    group"""
    C, g = 64, 2
    shape = SHAPES[3]
    inds = random_cloud(np.random.default_rng(rows), shape, [max(rows, 1)], 1)[1]
    inds_d = torch.from_numpy(inds).to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(inds_d, 1, shape, ConvAlgo.MaskImplicitGemm, [3] * 3, [1] * 3, [1] * 3,
                                             [1] * 3, [0] * 3, subm=True)
    outids, _, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks = res[:9]
    n = rows
    x = torch.randn((rows, C), device=cuda_dev).half()
    w = (torch.randn((C, 27, C // g), device=cuda_dev) * 0.2).half()
    out, _, _ = ops.implicit_gemm(x, w, pair_fwd, mask_fwd, sort_fwd, n, masks, True, True, groups=g)
    assert tuple(out.shape) == (n, C)
    dy = torch.randn((n, C), device=cuda_dev).half()
    din, dw = ops.implicit_gemm_backward(x, w, dy, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, None,
                                         masks, 128, True, groups=g)
    if n == 0:
        assert torch.count_nonzero(dw) == 0
    for j in range(g):
        s = slice(j * 32, (j + 1) * 32)
        o, _, _ = ops.implicit_gemm(x[:, s].contiguous(), w[s].contiguous(), pair_fwd, mask_fwd, sort_fwd, n, masks,
                                    True, True)
        di, dj = ops.implicit_gemm_backward(x[:, s].contiguous(), w[s].contiguous(), dy[:, s].contiguous(), pair_fwd,
                                            pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, None, masks, 128, True)
        assert torch.equal(out[:, s], o) and torch.equal(din[:, s][:n], di[:n]) and torch.equal(dw[s], dj)


# ------------------------------------------------------------------ 3. module features around the GEMM
@pytest.mark.parametrize("act", [Activation.None_, Activation.ReLU, Activation.LeakyReLU])
@pytest.mark.parametrize("algo", ["igemm", "native"])
def test_inference_epilogue(act, algo, cuda_dev):
    """eval: bias and activation ride in each group's epilogue, equal to the dense eval layer per group"""
    C, K, g = 128, 64, 4
    gen = torch.Generator(device=cuda_dev).manual_seed(7)
    x = _input(cuda_dev, "subm", 3, C, 3, torch.float16, gen, False, (1200,), 7)
    mod = _layer("subm", 3, C, K, 3, ALGOS[algo], g, act_type=act, act_alpha=0.1).to(cuda_dev).half().eval()
    with torch.no_grad():
        y = mod(x).features
        for j in range(g):
            d = _layer("subm", 3, C // g, K // g, 3, ALGOS[algo], 1, act_type=act, act_alpha=0.1).to(cuda_dev).half()
            d.eval()
            d.weight.copy_(mod.weight[j * 16:(j + 1) * 16])
            d.bias.copy_(mod.bias[j * 16:(j + 1) * 16])
            yj = d(x.replace_feature(x.features[:, j * 32:(j + 1) * 32].contiguous())).features
            assert torch.equal(y[:, j * 16:(j + 1) * 16], yj)


def test_fuse_bn_and_act(cuda_dev):
    """fuse_bn scales each filter row of a grouped layer and fuse_act moves the ReLU into its epilogue"""
    from spconv_b200.pytorch.utils_fuse import fuse_act, fuse_bn
    C, g = 64, 2
    gen = torch.Generator(device=cuda_dev).manual_seed(8)
    x = _input(cuda_dev, "subm", 3, C, 3, torch.float32, gen, False, (1000,), 8)
    conv = spconv.SubMConv3d(C, C, 3, groups=g, bias=False).to(cuda_dev)
    bn = torch.nn.BatchNorm1d(C).to(cuda_dev)
    with torch.no_grad():
        bn.running_mean.uniform_(-1, 1)
        bn.running_var.uniform_(0.5, 2)
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-1, 1)
    net = spconv.SparseSequential(conv, bn, torch.nn.ReLU()).eval()
    with torch.no_grad():
        want = net(x).features
        fused = fuse_act(fuse_bn(conv, bn), torch.nn.ReLU())
        assert fused.groups == g and fused.act_type == Activation.ReLU
        got = fused(x).features
    assert torch.allclose(got, want, atol=1e-4, rtol=1e-4)


def test_one_by_one_layer_is_a_batched_matmul(cuda_dev):
    C, K, g = 64, 96, 2
    x = _input(cuda_dev, "subm", 3, C, 1, torch.float32, torch.Generator(device=cuda_dev).manual_seed(9), False,
               (500,), 9)
    m = spconv.SubMConv3d(C, K, 1, groups=g).to(cuda_dev)
    y = m(x).features
    w = m.weight.detach().view(K, C // g)
    want = torch.cat([x.features[:, j * 32:(j + 1) * 32] @ w[j * 48:(j + 1) * 48].t() for j in range(g)], 1) + m.bias
    assert torch.allclose(y, want, atol=1e-5, rtol=1e-5)


def _bounded_net(dev, C, g):
    torch.manual_seed(11)
    return spconv.SparseSequential(spconv.SubMConv3d(C, C, 3, groups=g, indice_key="s0"),
                                   spconv.SparseConv3d(C, C, 3, 2, 1, groups=g, indice_key="down"),
                                   spconv.SparseInverseConv3d(C, C, 3, indice_key="down", groups=g)
                                   ).to(dev).half().train()


def test_padding_bounds_and_graph_replay(cuda_dev):
    """a padded, bounded grouped network gives the unpadded outputs and input gradients on the valid rows with the
    same launch count for every cloud; a captured step replays the eager results bit for bit"""
    C, g, shape = 64, 4, SHAPES[3]
    net = _bounded_net(cuda_dev, C, g)
    params = list(net.parameters())
    rng = np.random.default_rng(12)
    clouds = [random_cloud(rng, shape, [n], 1)[1] for n in (1500, 1300)]
    feats = [torch.randn((len(c), C), device=cuda_dev).half() for c in clouds]
    dy_full = [torch.randn((len(c), C), device=cuda_dev).half() for c in clouds]

    def plain(f, c, dy):
        for p in params:
            p.grad = None
        xf = f.detach().clone().requires_grad_(True)
        y = net(spconv.SparseConvTensor(xf, torch.from_numpy(c).to(cuda_dev), shape, 1))
        y.features.backward(dy)
        return y.features.detach(), xf.grad, [p.grad.clone() for p in params]

    unpadded = [plain(f, c, d) for f, c, d in zip(feats, clouds, dy_full)]
    net.eval()
    spconv.set_output_bounds(net, spconv.SparseConvTensor(feats[0], torch.from_numpy(clouds[0]).to(cuda_dev), shape, 1),
                             margin=1.5)
    net.train()
    n_pad = 1600
    padded = [spconv.SparseConvTensor(f, torch.from_numpy(c).to(cuda_dev), shape, 1).pad_to(n_pad)
              for f, c in zip(feats, clouds)]
    args = [(p.features, p.indices, p.num_valid) for p in padded]
    dys = [torch.cat([d, torch.zeros((n_pad - len(d), C), device=cuda_dev).half()]) for d in dy_full]
    dy = dys[0].clone()

    def step(f, i, nv):
        for p in params:
            p.grad = None
        xf = f.detach().requires_grad_(True)
        x = spconv.SparseConvTensor(xf, i, shape, 1)
        x.num_valid = nv
        y = net(x)
        y.features.backward(dy)
        return [y.features.detach(), xf.grad] + [p.grad for p in params]

    want, launches = [], []
    for k, a in enumerate(args):
        dy.copy_(dys[k])
        ops.launch_count(reset=True)
        want.append([t.clone() for t in step(*a)])
        launches.append(ops.launch_count())
        n = len(clouds[k])
        y0, dx0, _ = unpadded[k]
        assert torch.equal(want[k][0][:n], y0) and torch.equal(want[k][1][:n], dx0)
    assert launches[0] == launches[1]
    dy.copy_(dys[0])
    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 0):
        dy.copy_(dys[k])
        got = graphed(*args[k])
        for j, (a_, b_) in enumerate(zip(got, want[k])):
            assert torch.equal(a_, b_), f"replay of cloud {k}, result {j}"
    spconv.check_bounds(net)


@pytest.mark.parametrize("grouped_first", [True, False])
def test_rulebook_shared_with_a_dense_layer(grouped_first, cuda_dev):
    C = 64
    gen = torch.Generator(device=cuda_dev).manual_seed(13)
    x = _input(cuda_dev, "subm", 3, C, 3, torch.float16, gen, False, (1200,), 13)
    grouped = spconv.SubMConv3d(C, C, 3, groups=2, indice_key="k").to(cuda_dev).half()
    dense = spconv.SubMConv3d(C, C, 3, indice_key="k").to(cuda_dev).half()
    alone = spconv.SubMConv3d(C, C, 3, groups=2).to(cuda_dev).half()
    alone.load_state_dict(grouped.state_dict())
    with torch.no_grad():
        net = spconv.SparseSequential(grouped, dense) if grouped_first else spconv.SparseSequential(dense, grouped)
        y = net(x)
        assert len(y.indice_dict) == 1
        want = dense(alone(x)) if grouped_first else alone(dense(x))
        assert torch.equal(y.features, want.features)


def test_conv_onto_a_second_cloud(cuda_dev):
    C, K, g = 64, 64, 2
    gen = torch.Generator(device=cuda_dev).manual_seed(15)
    x = _input(cuda_dev, "subm", 3, C, 3, torch.float16, gen, False, (1200,), 15)
    t = _input(cuda_dev, "subm", 3, C, 3, torch.float16, gen, False, (1000,), 16)
    mod = spconv.SubMConv3d(C, K, 3, groups=g).to(cuda_dev).half().train()
    f = x.features.detach().clone().requires_grad_(True)
    y = mod(x.replace_feature(f), target=t)
    dy = torch.randn_like(y.features)
    y.features.backward(dy)
    for j in range(g):
        d = spconv.SubMConv3d(32, 32, 3).to(cuda_dev).half().train()
        with torch.no_grad():
            d.weight.copy_(mod.weight[j * 32:(j + 1) * 32])
            d.bias.copy_(mod.bias[j * 32:(j + 1) * 32])
        fj = x.features[:, j * 32:(j + 1) * 32].detach().clone().requires_grad_(True)
        yj = d(x.replace_feature(fj), target=t)
        yj.features.backward(dy[:, j * 32:(j + 1) * 32].contiguous())
        assert torch.equal(y.features[:, j * 32:(j + 1) * 32], yj.features)
        assert torch.equal(f.grad[:, j * 32:(j + 1) * 32], fj.grad)
        assert torch.equal(mod.weight.grad[j * 32:(j + 1) * 32], d.weight.grad)


# ------------------------------------------------------------------ 4. data parallel
class _Recorder:
    def __init__(self):
        self.calls = []

    def __call__(self, dw):
        self.calls.append(dw.clone())
        dw.mul_(0.5)


@pytest.mark.parametrize("algo", ["igemm", "native"])
def test_wgrad_hook_eager_and_replayed(algo, cuda_dev):
    C = 64
    gen = torch.Generator(device=cuda_dev).manual_seed(17)
    x = _input(cuda_dev, "subm", 3, C, 3, torch.float16, gen, True, (1200,), 17)
    mod = spconv.SubMConv3d(C, C, 3, groups=4, bias=False, algo=ALGOS[algo]).to(cuda_dev).half().train()
    dy = torch.ones((x.features.shape[0], C), device=cuda_dev).half()
    mod(x).features.backward(dy)
    plain = mod.weight.grad.clone()
    rec = _Recorder()
    ops.set_wgrad_hook(rec)
    mod.weight.grad = None
    mod(x).features.backward(dy)
    torch.cuda.synchronize()
    assert len(rec.calls) == 1 and torch.equal(rec.calls[0], plain) and torch.equal(mod.weight.grad, plain * 0.5)

    def step(f):
        mod.weight.grad = None
        mod(x.replace_feature(f)).features.backward(dy)
        return [mod.weight.grad]

    f0 = x.features.clone()
    graphed = spconv.graph_capture(step, f0)
    ops.set_wgrad_hook(None)
    rec.calls.clear()
    for s in range(2):
        f0.copy_(_data(torch.Generator(device=cuda_dev).manual_seed(40 + s), tuple(f0.shape), cuda_dev, True).half())
        got = graphed(f0)[0].clone()
        assert not rec.calls
        want = step(f0)[0]
        assert torch.equal(got, want * 0.5)


def test_two_ranks_sum_grouped_weight_gradients(cuda_dev):
    """two simulated ranks on streams of one GPU: each rank's dW is pushed whole after the grouped weight gradient,
    and the finish leaves the rank-order sum on both"""
    from spconv_b200.pytorch.dist import PeerGroup
    C, g = 64, 2
    gen = torch.Generator(device=cuda_dev).manual_seed(19)
    xs = [_input(cuda_dev, "subm", 3, C, 3, torch.float16, gen, True, (900,), 19 + r) for r in range(2)]
    mods = [spconv.SubMConv3d(C, C, 3, groups=g, bias=False).to(cuda_dev).half().train() for _ in range(2)]
    mods[1].load_state_dict(mods[0].state_dict())
    local = []
    for m, x in zip(mods, xs):
        m(x).features.backward(torch.ones((x.features.shape[0], C), device=cuda_dev).half())
        local.append(m.weight.grad.clone())
        m.weight.grad = None
    streams = [torch.cuda.Stream() for _ in range(2)]
    ring = PeerGroup.local_ring(2, capacity_bytes=1 << 20, average=False)
    try:
        torch.cuda.synchronize()
        outs = []
        for r in range(2):
            with torch.cuda.stream(streams[r]):
                outs.append(mods[r](xs[r]))
        torch.cuda.synchronize()
        for r in range(2):
            ops.set_peer_group(ring[r])
            with torch.cuda.stream(streams[r]):
                outs[r].features.backward(torch.ones_like(outs[r].features))
        ops.set_peer_group(None)
        torch.cuda.synchronize()
        want = (local[0].double() + local[1].double()).half()
        for m in mods:
            assert torch.equal(m.weight.grad, want)
        assert [pg.error() for pg in ring] == [0, 0]
    finally:
        ops.set_peer_group(None)
        for pg in ring:
            pg.close()


# ------------------------------------------------------------------ 5. AMP and operand addresses
def test_autocast_equals_explicit_fp16(cuda_dev):
    C = 64
    gen = torch.Generator(device=cuda_dev).manual_seed(21)
    x = _input(cuda_dev, "subm", 3, C, 3, torch.float32, gen, False, (1000,), 21)
    mod = spconv.SubMConv3d(C, C, 3, groups=2).to(cuda_dev).train()
    with torch.autocast("cuda", dtype=torch.float16):
        ya = mod(x).features
    half = spconv.SubMConv3d(C, C, 3, groups=2).to(cuda_dev).half().train()
    half.load_state_dict({k: v.half() for k, v in mod.state_dict().items()})
    yh = half(x.replace_feature(x.features.half())).features
    assert torch.equal(ya, yh)


@pytest.mark.parametrize("offset", [2, 4, 8])
def test_unaligned_operands_give_the_same_bits(offset, cuda_dev):
    """features, filters and gradients that start `offset` bytes past a 16-byte boundary give the bits of aligned
    ones"""
    C, g = 64, 2
    gen = torch.Generator(device=cuda_dev).manual_seed(23)
    x = _input(cuda_dev, "subm", 3, C, 3, torch.float16, gen, False, (1000,), 23)
    mod = spconv.SubMConv3d(C, C, 3, groups=g).to(cuda_dev).half().train()
    dy = torch.randn((x.features.shape[0], C), device=cuda_dev).half()
    y, din, dw, _ = _run(mod, x, dy)
    want = (y.features.clone(), din.clone(), dw.clone())

    def at(t):
        raw = torch.empty(t.numel() * 2 + 64, dtype=torch.uint8, device=cuda_dev)
        base = (-raw.data_ptr()) % 16 + offset
        v = raw[base:base + t.numel() * 2].view(torch.float16).view(t.shape)
        v.copy_(t)
        return v

    mod.weight.grad = None
    f = at(x.features).requires_grad_(True)
    with torch.no_grad():
        mod.weight.data = at(mod.weight.detach())
    assert f.data_ptr() % 16 == offset and mod.weight.data_ptr() % 16 == offset
    y2 = mod(x.replace_feature(f))
    y2.features.backward(at(dy))
    assert torch.equal(y2.features, want[0]) and torch.equal(f.grad, want[1]) and torch.equal(mod.weight.grad, want[2])
