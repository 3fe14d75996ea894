"""Whole sparse networks against float64 twins (tests/net_ref.py): a U-Net, an encoder, a classifier and a
two-branch net that merges different coordinates, eager, padded and graph-replayed, in every dtype.

Every module's input and output is recorded in the run, and the gradient autograd delivers to its output and
the one it returns for each input are caught by identity taps around it.  Each twin layer then gets the GPU's
own input (upcast) and its own delivered gradient; its output, input gradients and parameter gradients must
meet the per-op bounds of the kernel tests:
  * conv and depthwise: |got - ref| <= u_out |ref| + T 2^-23 sum|terms| + tiny (test_conv_modules_gpu.py),
    with the rounded bias add of training and the rounded partial results of the mask splits;
  * BatchNorm: the bounds of test_masked_batchnorm_gpu.py;
  * ReLU, tables, max pools, ToDense: bit for bit, or one rounding in the dtype.
Output coordinates come from the twins and must equal the library's rows in order.  Rows at or beyond
num_valid must be zero in every gradient and in the outputs of BatchNorm, the pools and the masked tables.
The gradient delivered to a tensor must be what its consumers returned for it, summed with one rounding
(skip connections have two consumers).  A padded step and its graph replay must agree bit for bit, and the
BN-free merge net in exact fp32 must give the twin's loss and gradients bit for bit.
"""
import numpy as np
import pytest
import torch
from torch import nn

from bench_utils import make_encoder6, surface_cloud
from tests import net_ref
from tests.conv_ref import SparseConvRef
from tests.test_masked_batchnorm_gpu import _close_f32, _close_low, _reference as _bn_reference

pytestmark = pytest.mark.gpu

SHAPE = [32, 128, 128]
BATCH = 2
COUNTS = [(2600, 2300), (3100, 2900), (2200, 2700)]     # voxels per sample of the three clouds
TORCH_DT = {"f32": torch.float32, "tf32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16,
            "amp": torch.float32}
CAST = {"f32": torch.float32, "tf32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16,
        "amp": torch.float16}
U = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
TINY = {torch.float32: 1e-30, torch.float16: 2.0 ** -24, torch.bfloat16: 1e-30}

# (net, algo, dtype, modes)
CASES = [
    ("unet", "Native", "f32", ("eager",)),
    ("unet", "MaskImplicitGemm", "f16", ("eager", "padded", "graph")),
    ("unet", "MaskSplitImplicitGemm", "bf16", ("eager", "padded", "graph")),
    ("unet", "MaskImplicitGemm", "tf32", ("eager",)),
    ("encoder", "MaskImplicitGemm", "f16", ("padded", "graph", "eval")),
    ("encoder", "MaskImplicitGemm", "f32", ("eager", "eval")),
    ("encoder", "MaskSplitImplicitGemm", "bf16", ("eager", "eval")),
    ("classifier", "MaskImplicitGemm", "amp", ("eager", "padded", "graph")),
    ("classifier", "Native", "bf16", ("eager",)),
    ("merge", "MaskImplicitGemm", "f32", ("eager", "padded", "graph")),
    ("merge", "Native", "f16", ("eager",)),
]


# ---------------------------------------------------------------------------- networks
class _Cat(nn.Module):
    def forward(self, xs):
        return torch.cat(xs, 1)


class _ToFloat(nn.Module):
    """the dense head runs in fp32 (it is torch's, not this library's)"""

    def forward(self, x):
        return x.float()


class Net:
    """``steps``: (name, input names) in order; ``mods[name]`` runs the step (a list input for several)."""

    def __init__(self, mods, steps):
        self.mods = nn.ModuleDict(mods)
        self.steps = steps


def _algo(spconv, algo, strided, padded):
    from spconv_b200.core import ConvAlgo
    if strided and algo == "MaskSplitImplicitGemm" and padded:
        return ConvAlgo.MaskImplicitGemm          # output bounds need the one-split rulebook
    return ConvAlgo[algo]


def unet(spconv, algo, padded):
    a = lambda strided=False: _algo(spconv, algo, strided, padded)      # noqa: E731
    S = spconv.SubMConv3d
    mods = {
        "c1": S(4, 16, 3, indice_key="s1", algo=a()), "bn1": spconv.MaskedBatchNorm1d(16),
        "r1": spconv.SparseReLU(), "c2": S(16, 16, 3, indice_key="s1", algo=a()), "r2": spconv.SparseReLU(),
        "d1": spconv.SparseConv3d(16, 32, 3, 2, 1, indice_key="d1", algo=a(True)), "r3": spconv.SparseReLU(),
        "c3": S(32, 32, 3, indice_key="s2", algo=a()), "r4": spconv.SparseReLU(),
        "c4": S(32, 32, 3, indice_key="s2", algo=a()), "r5": spconv.SparseReLU(),
        "d2": spconv.SparseConv3d(32, 32, 3, 2, 1, indice_key="d2", algo=a(True)), "r6": spconv.SparseReLU(),
        "c5": S(32, 32, 3, indice_key="s3", algo=a()), "r7": spconv.SparseReLU(),
        "u2": spconv.SparseInverseConv3d(32, 32, 3, indice_key="d2", algo=a(True)),
        "j2": spconv.MaskedJoinTable(),
        "c6": S(64, 32, 3, indice_key="s2", algo=a()), "r8": spconv.SparseReLU(),
        "u1": spconv.SparseInverseConv3d(32, 16, 3, indice_key="d1", algo=a(True)),
        "a1": spconv.MaskedAddTable(),
        "dw": S(16, 16, 3, groups=16, indice_key="s1", algo=a()),
        "c7": S(16, 5, 3, indice_key="s1", algo=a()),
    }
    steps = [("c1", ["x"]), ("bn1", ["c1"]), ("r1", ["bn1"]), ("c2", ["r1"]), ("r2", ["c2"]), ("d1", ["r2"]),
             ("r3", ["d1"]), ("c3", ["r3"]), ("r4", ["c3"]), ("c4", ["r4"]), ("r5", ["c4"]), ("d2", ["r5"]),
             ("r6", ["d2"]), ("c5", ["r6"]), ("r7", ["c5"]), ("u2", ["r7"]), ("j2", ["u2", "r5"]),
             ("c6", ["j2"]), ("r8", ["c6"]), ("u1", ["r8"]), ("a1", ["u1", "r2"]), ("dw", ["a1"]), ("c7", ["dw"])]
    return Net(mods, steps), 4


def encoder(spconv, algo, padded):
    """make_encoder6 with BatchNorm and ReLU / LeakyReLU after every conv, a 2x2x2 max pool and ToDense"""
    convs = make_encoder6(spconv, bias=True)
    mods, steps, prev = {}, [], "x"
    for i, conv in enumerate(convs):
        conv.algo = _algo(spconv, algo, not conv.subm, padded)
        act = nn.LeakyReLU(0.1) if i % 2 else nn.ReLU()
        for name, mod in ((f"c{i}", conv), (f"b{i}", spconv.MaskedBatchNorm1d(conv.out_channels)),
                          (f"a{i}", spconv.SparseSequential(act))):
            mods[name] = mod
            steps.append((name, [prev]))
            prev = name
        if i == 3:
            mods["pool"] = spconv.SparseMaxPool3d(2, 2)
            steps.append(("pool", [prev]))
            prev = "pool"
    mods["dense"] = spconv.ToDense()
    steps.append(("dense", [prev]))
    return Net(mods, steps), 16


def classifier(spconv, algo, padded):
    mods = {"c1": spconv.SubMConv3d(4, 16, 3, indice_key="s1", algo=_algo(spconv, algo, False, padded)),
            "r1": spconv.SparseReLU(),
            "d1": spconv.SparseConv3d(16, 32, 3, 2, 1, algo=_algo(spconv, algo, True, padded)),
            "r2": spconv.SparseReLU(), "gmax": spconv.MaskedGlobalMaxPool(), "gavg": spconv.MaskedGlobalAvgPool(),
            "cat": _Cat(), "f": _ToFloat(), "fc": nn.Linear(64, 5)}
    steps = [("c1", ["x"]), ("r1", ["c1"]), ("d1", ["r1"]), ("r2", ["d1"]), ("gmax", ["r2"]), ("gavg", ["r2"]),
             ("cat", ["gmax", "gavg"]), ("f", ["cat"]), ("fc", ["f"])]
    return Net(mods, steps), 4


def merge(spconv, algo, padded):
    a = lambda strided=False: _algo(spconv, algo, strided, padded)      # noqa: E731
    mods = {"c1": spconv.SubMConv3d(8, 16, 3, indice_key="s1", algo=a()), "r1": spconv.SparseReLU(),
            "a": spconv.SubMConv3d(16, 16, 3, indice_key="s1", algo=a()),
            "d1": spconv.SparseConv3d(16, 16, 3, 2, 1, algo=a(True)), "r2": spconv.SparseReLU(),
            "t1": spconv.SparseConvTranspose3d(16, 16, 2, 2, algo=a(True)),
            "m": spconv.MaskedAddTableMisaligned(),
            "c2": spconv.SubMConv3d(16, 8, 3, indice_key="sm", algo=a())}
    steps = [("c1", ["x"]), ("r1", ["c1"]), ("a", ["r1"]), ("d1", ["r1"]), ("r2", ["d1"]), ("t1", ["r2"]),
             ("m", ["a", "t1"]), ("c2", ["m"])]
    return Net(mods, steps), 8


NETS = {"unet": unet, "encoder": encoder, "classifier": classifier, "merge": merge}


# ---------------------------------------------------------------------------- the recorded run
class _Tap(torch.autograd.Function):
    """identity whose backward stores the gradient it passes on"""

    @staticmethod
    def forward(ctx, x, slot):
        ctx.slot = slot
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        ctx.slot.append(g.detach().clone())
        return g, None


def _tap(v, slot):
    from spconv_b200.pytorch import SparseConvTensor
    if isinstance(v, SparseConvTensor):
        return v.replace_feature(_Tap.apply(v.features, slot))
    return _Tap.apply(v, slot)


def _feats(v):
    from spconv_b200.pytorch import SparseConvTensor
    return v.features if isinstance(v, SparseConvTensor) else v


def run(net, x, G, autocast=False):
    """forward + backward of ``sum(out * G)`` over the valid rows -> record
    ``{"y": {name: value}, "gout": {name: [grad]}, "gin": {(name, j): [grad]}}``; ``x`` carries the leaf"""
    for p in net.mods.parameters():
        p.grad = None
    rec = {"y": {"x": x}, "gout": {}, "gin": {}}
    env = {"x": x}
    with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
        for name, ins in net.steps:
            args = []
            for j, i in enumerate(ins):
                rec["gin"][(name, j)] = []
                args.append(_tap(env[i], rec["gin"][(name, j)]))
            y = net.mods[name](args if len(args) > 1 else args[0])
            rec["y"][name] = y
            rec["gout"][name] = []
            env[name] = _tap(y, rec["gout"][name])
        out = _feats(env[net.steps[-1][0]])
        loss = (out.float() * G).sum()
    loss.backward()
    rec["loss"] = loss.detach()
    return rec


def flat(net, rec):
    """every recorded tensor of a run, in a fixed order (for bit-for-bit comparisons)"""
    out = [rec["loss"], _feats(rec["y"]["x"]).grad]
    for name, ins in net.steps:
        y = rec["y"][name]
        out.append(_feats(y).detach())
        if y is not _feats(y):
            out.append(y.indices)
        out += rec["gout"][name] + [g for j in range(len(ins)) for g in rec["gin"][(name, j)]]
    out += [p.grad for p in net.mods.parameters()]
    return out


# ---------------------------------------------------------------------------- inputs
def clouds(dev):
    rng = np.random.default_rng(2024)
    out = []
    for counts in COUNTS:
        parts = [surface_cloud(rng, SHAPE, n, 1) for n in counts]
        for b, p in enumerate(parts):
            p[:, 0] = b
        inds = np.concatenate(parts, 0)
        out.append(torch.from_numpy(inds[rng.permutation(len(inds))]).to(dev))
    return out


def _exact(rng, shape, lo, hi):
    return torch.from_numpy(rng.integers(lo, hi + 1, size=shape).astype(np.float64))


def setup(name, algo, dt, padded, dev, exact=False, seed=0):
    import spconv_b200.pytorch as spconv
    torch.manual_seed(seed)
    net, c_in = NETS[name](spconv, algo, padded)
    rng = np.random.default_rng(seed + 1)
    with torch.no_grad():
        for mod in net.mods.modules():
            if isinstance(mod, spconv.MaskedBatchNorm1d):       # not the identity: a real affine map
                mod.weight.copy_(torch.from_numpy(rng.uniform(0.5, 1.5, mod.num_features)))
                mod.bias.copy_(torch.from_numpy(rng.uniform(-0.3, 0.3, mod.num_features)))
            elif exact and isinstance(mod, spconv.SparseConvolution):
                # small integers: every sum of the exact fp32 kernels is exact (the twin asserts it)
                mod.weight.copy_(_exact(rng, mod.weight.shape, -1, 1) * torch.from_numpy(
                    (rng.random(tuple(mod.weight.shape)) < 0.35).astype(np.float64)))
                mod.bias.copy_(_exact(rng, mod.bias.shape, -2, 2))
    net.mods.to(dev).to(TORCH_DT[dt])
    if name == "classifier":
        net.mods["fc"].float()
    net.mods.train()
    return net, c_in


def inputs(net, c_in, inds, dt, dev, padded_rows=None, exact=False, seed=0):
    """(x SparseConvTensor with a leaf, G) for one cloud; padded to ``padded_rows`` when given"""
    import spconv_b200.pytorch as spconv
    rng = np.random.default_rng(seed + 7)
    n = inds.shape[0]
    f = _exact(rng, (n, c_in), -2, 2) if exact else torch.from_numpy(rng.standard_normal((n, c_in)))
    x = spconv.SparseConvTensor(f.to(dev).to(TORCH_DT[dt]), inds, SHAPE, BATCH)
    if padded_rows is not None:
        x = x.pad_to(padded_rows)
    x = x.replace_feature(x.features.detach().requires_grad_(True))
    return x


def make_g(rec_out, seed, exact=False):
    """fixed dL/d(out), random on every row: on the padding rows too, which no gradient may then carry (the
    loss is checked layer by layer, never against an unpadded run, so what it adds there does not matter)"""
    out = _feats(rec_out)
    rng = np.random.default_rng(seed + 11)
    g = (_exact(rng, out.shape, -1, 1) if exact else torch.from_numpy(rng.standard_normal(out.shape)))
    return g.float().to(out.device)


# ---------------------------------------------------------------------------- per-layer checks
def _nv(v):
    nv = getattr(v, "num_valid", None)
    return _feats(v).shape[0] if nv is None else int(nv)


def _d(t):
    return t.detach().double().cpu()


def _close(got, ref, mag, terms, cast, what, ref_pre=None, extra=None):
    """|got - ref| <= u_out (|ref| + |ref_pre|) + T 2^-23 mag + extra + tiny"""
    got, ref = _d(got), ref.detach()
    u = U[cast]
    bound = u * ref.abs() + terms * 2.0 ** -23 * mag + TINY[cast]
    if ref_pre is not None:
        bound = bound + u * ref_pre.detach().abs()
    if extra is not None:
        bound = bound + extra
    err = (got - ref).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())}/{bad.numel()} out of bound; first at "
                                 f"{bad.nonzero()[0].tolist()}: got {float(got[bad][0])!r} want "
                                 f"{float(ref[bad][0])!r} bound {float(bound[bad][0]):.3g}")


def _same(got, ref, cast, what):
    """bit for bit after one rounding of the float64 reference to the dtype"""
    want = ref.detach().to(cast).cpu()
    got = got.detach().cpu()
    assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
    bad = ~((got == want) | (got.isnan() & want.isnan()))
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())}/{bad.numel()} differ; first at {bad.nonzero()[0].tolist()}"
                                 f": got {float(got[bad][0])!r} want {float(want[bad][0])!r}")


def _zero_tail(t, nv, what):
    assert bool((t[nv:] == 0).all()), f"{what}: rows at or beyond num_valid are not zero"


def _paired_input(net, rec, key):
    """the input of the strided conv that built ``key`` (whose rows an inverse conv restores)"""
    for name, ins in net.steps:
        m = net.mods[name]
        if getattr(m, "indice_key", None) == key and not m.subm and not m.inverse:
            return rec["y"][ins[0]]
    raise KeyError(key)


def _conv_ref(mod, inds, shape, net=None, rec=None):
    """the reference rulebook of conv module ``mod`` on input rows ``inds``; an inverse conv's comes from the
    strided conv that built its ``indice_key``, on that conv's input rows"""
    if mod.inverse:
        paired = next(net.mods[n] for n, _ in net.steps
                      if getattr(net.mods[n], "indice_key", None) == mod.indice_key and not net.mods[n].inverse)
        src = _paired_input(net, rec, mod.indice_key)
        ref = SparseConvRef(src.indices[:_nv(src)].cpu().numpy(), BATCH, src.spatial_shape, paired.kernel_size,
                            paired.stride, paired.padding, paired.dilation, kind="inverse")
        assert np.array_equal(ref.in_inds, inds), "inverse conv: input rows are not the paired conv's output rows"
        return ref
    kind = "subm" if mod.subm else "transpose" if mod.transposed else "conv"
    return SparseConvRef(inds, BATCH, shape, mod.kernel_size, mod.stride, mod.padding, mod.dilation,
                         mod.output_padding, kind)


def check_conv(name, mod, x, y, gy, gx, net, rec, cast, dt, eval_ref=None):
    """one conv module: coordinates, output, input, weight and bias gradients"""
    from spconv_b200.core import ConvAlgo
    nv_in, nv_out = _nv(x), _nv(y)
    inds = x.indices[:nv_in].cpu().numpy()
    ref = _conv_ref(mod, inds, x.spatial_shape, net, rec)
    assert np.array_equal(y.indices[:nv_out].cpu().numpy(), ref.out_inds), f"{name}: output coordinates"
    assert y.spatial_shape == list(ref.out_shape), f"{name}: spatial shape"
    twin = net_ref.ConvTwin(ref, depthwise=mod.depthwise)
    split = mod.algo == ConvAlgo.MaskSplitImplicitGemm and not mod.depthwise
    xd = _d(_feats(x)[:nv_in].to(cast)).requires_grad_(True)
    w = _d(mod.weight.to(cast)).requires_grad_(True)
    b = _d(mod.bias.to(cast)).requires_grad_(True) if mod.bias is not None else None
    gyd = _d(gy[:nv_out])
    pre = twin(xd, w)
    out = pre if b is None else pre + b
    y_mag, y_t, dx_mag, dx_t, dw_mag, dw_t = net_ref.conv_bounds(twin, xd, w, gyd)
    extra = 2.0 ** -9 * y_mag if dt == "tf32" else 0.0          # tf32 rounds both operands of every product
    if split:
        extra = extra + U[cast] * y_mag
    bmag = y_mag + (0 if b is None else b.detach().abs())
    _close(_feats(y)[:nv_out], out, bmag, y_t + 1, cast, f"{name} forward", ref_pre=pre, extra=extra)
    out.backward(gyd)
    _zero_tail(gx, nv_in, f"{name} dX")
    ex = lambda m: (2.0 ** -9 * m if dt == "tf32" else 0.0) + (U[cast] * m if split else 0.0)   # noqa: E731
    _close(gx[:nv_in], xd.grad, dx_mag, dx_t, cast, f"{name} dX", extra=ex(dx_mag))
    _close(mod.weight.grad, w.grad, dw_mag, dw_t, cast, f"{name} dW",
           extra=2.0 ** -9 * dw_mag if dt == "tf32" else None)
    if b is not None:
        _close(mod.bias.grad, b.grad, gyd.abs().sum(0), float(nv_out), cast, f"{name} dbias")


def check_layers(net, rec, dt):
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch.pool import MaskedGlobalMaxOrAvgPool
    cast = CAST[dt]
    for name, ins in net.steps:
        mod = net.mods[name]
        xs = [rec["y"][i] for i in ins]
        y = rec["y"][name]
        gy = rec["gout"][name][0]
        gxs = [rec["gin"][(name, j)][0] for j in range(len(ins))]
        x = xs[0]
        if isinstance(mod, spconv.SparseConvolution):
            check_conv(name, mod, x, y, gy, gxs[0], net, rec, cast, dt)
        elif isinstance(mod, spconv.MaskedBatchNorm1d):
            nv = _nv(x)
            xv = _feats(x)[:nv]
            yr, dx, dw, db, _, cond = _bn_reference(xv.double(), gy[:nv].double(), mod, 1)
            dtype = _feats(x).dtype
            close = (lambda g, r, w, c: _close_f32(g.double(), r, w, c)) if dtype == torch.float32 else \
                (lambda g, r, w, c: _close_low(g, r, dtype, w, c))
            close(_feats(y)[:nv], yr, f"{name} y", cond["y"])
            close(gxs[0][:nv], dx, f"{name} dX", cond["dx"])
            close(mod.weight.grad, dw, f"{name} dW", cond["dw"])
            close(mod.bias.grad, db, f"{name} db", cond["db"])
            _zero_tail(_feats(y), nv, f"{name} y")
            _zero_tail(gxs[0], nv, f"{name} dX")
        elif isinstance(mod, (spconv.SparseReLU, spconv.SparseSequential)):
            act = mod.inner if isinstance(mod, spconv.SparseReLU) else mod[0]
            alpha = act.negative_slope if isinstance(act, nn.LeakyReLU) else 0.0
            xd = _d(_feats(x)).requires_grad_(True)
            if alpha:
                # x * alpha: torch multiplies in fp32 by the fp32 alpha, then rounds to the dtype
                r = net_ref.leaky_relu(xd, float(np.float32(alpha)))
                dtype = _feats(y).dtype
                _close(_feats(y), r, r.detach().abs(), 1.0, dtype, f"{name} y")
                r.backward(_d(gy))
                _close(gxs[0], xd.grad, xd.grad.abs(), 1.0, dtype, f"{name} dX")
            else:
                r = net_ref.relu(xd)
                _same(_feats(y), r, _feats(y).dtype, f"{name} y")
                r.backward(_d(gy))
                _same(gxs[0], xd.grad, gxs[0].dtype, f"{name} dX")
        elif isinstance(mod, (spconv.MaskedJoinTable, spconv.MaskedAddTable)):
            assert all(v.indices is x.indices or torch.equal(v.indices, x.indices) for v in xs), name
            xd = [_d(_feats(v)).requires_grad_(True) for v in xs]
            r = net_ref.join(xd) if isinstance(mod, spconv.MaskedJoinTable) else net_ref.add(xd)
            _same(_feats(y), r, _feats(y).dtype, f"{name} y")
            r.backward(_d(gy))
            for j, (v, g) in enumerate(zip(xd, gxs)):
                _same(g, v.grad, g.dtype, f"{name} dX{j}")
        elif isinstance(mod, spconv.MaskedAddTableMisaligned):
            nvs = [_nv(v) for v in xs]
            tw = net_ref.MisalignedAdd([v.indices[:n].cpu().numpy() for v, n in zip(xs, nvs)], BATCH, SHAPE)
            nv = _nv(y)
            assert np.array_equal(y.indices[:nv].cpu().numpy(), tw.out_inds), f"{name}: union coordinates"
            xd = [_d(_feats(v)[:n]).requires_grad_(True) for v, n in zip(xs, nvs)]
            r = tw(xd)
            _same(_feats(y)[:nv], r, _feats(y).dtype, f"{name} y")
            _zero_tail(_feats(y), nv, f"{name} y")
            r.backward(_d(gy[:nv]))
            for j, (v, g, n) in enumerate(zip(xd, gxs, nvs)):
                _same(g[:n], v.grad, g.dtype, f"{name} dX{j}")
                _zero_tail(g, n, f"{name} dX{j}")
        elif isinstance(mod, spconv.SparseMaxPool3d):
            nv_in, nv_out = _nv(x), _nv(y)
            inds = x.indices[:nv_in].cpu().numpy()
            ref = SparseConvRef(inds, BATCH, x.spatial_shape, mod.kernel_size, mod.stride, mod.padding,
                                mod.dilation, kind="conv")
            assert np.array_equal(y.indices[:nv_out].cpu().numpy(), ref.out_inds), f"{name}: coordinates"
            dtype = _feats(x).dtype
            xd = _d(_feats(x)[:nv_in]).requires_grad_(True)
            r = net_ref.max_pool(ref, xd, float(torch.finfo(dtype).min))
            _same(_feats(y)[:nv_out], r, dtype, f"{name} y")
            _zero_tail(_feats(y), nv_out, f"{name} y")
            r.backward(_d(gy[:nv_out]))
            _same(gxs[0][:nv_in], xd.grad, dtype, f"{name} dX")      # 2x2x2 stride 2: one window per input
            _zero_tail(gxs[0], nv_in, f"{name} dX")
        elif isinstance(mod, MaskedGlobalMaxOrAvgPool):
            nv = _nv(x)
            inds = x.indices[:nv].cpu().numpy()
            dtype = _feats(x).dtype
            xd = _d(_feats(x)[:nv]).requires_grad_(True)
            if mod.is_mean:
                r = net_ref.global_avg(xd, inds, BATCH)
                cnt = torch.tensor([float((inds[:, 0] == s).sum()) for s in range(BATCH)], dtype=torch.float64)
                mag = net_ref.global_avg(xd.detach().abs(), inds, BATCH)
                _close(y, r, mag, cnt[:, None] + 1, dtype, f"{name} y")
                r.backward(_d(gy))
                _close(gxs[0][:nv], xd.grad, xd.grad.abs(), 1.0, dtype, f"{name} dX")
            else:
                r = net_ref.global_max(xd, inds, BATCH)
                _same(y, r, dtype, f"{name} y")
                r.backward(_d(gy))
                _same(gxs[0][:nv], xd.grad, dtype, f"{name} dX")
            _zero_tail(gxs[0], nv, f"{name} dX")
        elif isinstance(mod, spconv.ToDense):
            nv = _nv(x)
            xd = _d(_feats(x)[:nv]).requires_grad_(True)
            r = net_ref.to_dense(xd, x.indices[:nv].cpu().numpy(), BATCH, x.spatial_shape)
            _same(y, r, y.dtype, f"{name} y")
            r.backward(_d(gy))
            _same(gxs[0][:nv], xd.grad, gxs[0].dtype, f"{name} dX")
            _zero_tail(gxs[0], nv, f"{name} dX")
        elif isinstance(mod, _Cat):
            xd = [_d(v).requires_grad_(True) for v in xs]
            r = torch.cat(xd, 1)
            _same(y, r, y.dtype, f"{name} y")
            r.backward(_d(gy))
            for j, (v, g) in enumerate(zip(xd, gxs)):
                _same(g, v.grad, g.dtype, f"{name} dX{j}")
        elif isinstance(mod, _ToFloat):
            _same(y, _d(x), torch.float32, f"{name} y")
            _same(gxs[0], _d(gy), x.dtype, f"{name} dX")
        elif isinstance(mod, nn.Linear):
            lin_cast = torch.float16 if dt == "amp" else torch.float32
            xd = _d(x.to(lin_cast)).requires_grad_(True)
            w = _d(mod.weight.to(lin_cast)).requires_grad_(True)
            bb = _d(mod.bias.to(lin_cast)).requires_grad_(True)
            r = xd @ w.t() + bb
            mag = xd.detach().abs() @ w.detach().abs().t() + bb.detach().abs()
            # torch's GEMM (cuBLAS), not this library's: its own summation order and split
            _close(y, r, mag, 2.0 * (xd.shape[1] + 1) * (2 ** 13 if lin_cast == torch.float16 else 1),
                   lin_cast, f"{name} y")
        else:
            raise AssertionError(f"no twin for {name}: {type(mod).__name__}")


def check_wiring(net, rec):
    """what autograd delivered to every tensor == the sum of what its consumers returned for it"""
    names = ["x"] + [n for n, _ in net.steps]
    for t in names:
        parts = [rec["gin"][(n, j)][0] for n, ins in net.steps for j, i in enumerate(ins) if i == t]
        if t == "x":
            got = _feats(rec["y"]["x"]).grad
        elif t == net.steps[-1][0]:
            continue
        else:
            got = rec["gout"][t][0]
        assert len(parts) >= 1, t
        want = sum(_d(p) for p in parts)
        assert torch.equal(got.detach().cpu(), want.to(got.dtype)), \
            f"gradient delivered to {t} is not the sum of its {len(parts)} consumers' gradients"


def check_record(net, rec, dt):
    assert len(rec["gout"][net.steps[-1][0]]) == 1
    check_wiring(net, rec)
    check_layers(net, rec, dt)


# ---------------------------------------------------------------------------- eval: fused BN + activation
def check_eval(net, x, dt):
    """eval mode after fuse_bn_act_sequential: every fused conv (BatchNorm and ReLU / LeakyReLU in its epilogue)
    against the unfused float64 twin conv -> BatchNorm with running stats -> activation, on the GPU's input"""
    import collections
    import spconv_b200.pytorch as spconv
    seq = spconv.SparseSequential(collections.OrderedDict(
        (n, net.mods[n][0] if n.startswith("a") else net.mods[n]) for n, _ in net.steps))
    seq.eval()
    fused = spconv.fuse_bn_act_sequential(seq)
    cast = CAST[dt]
    v = x.replace_feature(x.features.detach())
    with torch.no_grad():
        for name, m in fused._modules.items():
            out = m(v)
            if isinstance(m, spconv.SparseConvolution):
                assert m.act_type != spconv.Activation.None_, f"{name}: BatchNorm and activation were not fused"
                conv, bn, act = net.mods[name], net.mods["b" + name[1:]], net.mods["a" + name[1:]][0]
                nv_in, nv_out = _nv(v), _nv(out)
                ref = _conv_ref(conv, v.indices[:nv_in].cpu().numpy(), v.spatial_shape)
                assert np.array_equal(out.indices[:nv_out].cpu().numpy(), ref.out_inds), f"{name}: coordinates"
                twin = net_ref.ConvTwin(ref)
                xd = _d(v.features[:nv_in])
                z = net_ref.batch_norm_eval(twin(xd, _d(conv.weight), _d(conv.bias)), _d(bn.weight), _d(bn.bias),
                                            _d(bn.running_mean), _d(bn.running_var), bn.eps)
                r = net_ref.leaky_relu(z, act.negative_slope) if isinstance(act, nn.LeakyReLU) else net_ref.relu(z)
                scale = _d(bn.weight) / torch.sqrt(_d(bn.running_var) + bn.eps)
                wf = _d(conv.weight) * scale.view(-1, 1, 1, 1, 1)
                mag = twin(xd.abs(), wf.abs())
                terms = twin(torch.ones_like(xd), torch.ones_like(wf))
                # the folded weight and bias are rounded to the dtype once more
                fold = (_d(conv.bias).abs() + _d(bn.running_mean).abs()) * scale.abs() + _d(bn.bias).abs()
                _close(out.features[:nv_out], r, mag, terms + 1, cast, f"fused {name}",
                       extra=U[cast] * mag + 4 * U[cast] * fold)
            elif isinstance(m, spconv.SparseMaxPool3d):
                nv_in, nv_out = _nv(v), _nv(out)
                ref = SparseConvRef(v.indices[:nv_in].cpu().numpy(), BATCH, v.spatial_shape, m.kernel_size,
                                    m.stride, m.padding, m.dilation, kind="conv")
                r = net_ref.max_pool(ref, _d(v.features[:nv_in]), float(torch.finfo(v.features.dtype).min))
                _same(out.features[:nv_out], r, v.features.dtype, "fused net: pool")
            elif isinstance(m, spconv.ToDense):
                nv = _nv(v)
                r = net_ref.to_dense(_d(v.features[:nv]), v.indices[:nv].cpu().numpy(), BATCH, v.spatial_shape)
                _same(out, r, out.dtype, "fused net: dense")
            else:
                raise AssertionError(f"unexpected module {name} in the fused net: {type(m).__name__}")
            v = out


# ---------------------------------------------------------------------------- the tests
def _pad_rows(cl):
    return 128 * ((max(int(c.shape[0]) for c in cl) + 127) // 128)


@pytest.mark.parametrize("name,algo,dt,modes", CASES, ids=lambda v: v if isinstance(v, str) else "-".join(v))
def test_network_against_float64_twin(name, algo, dt, modes, cuda_dev, monkeypatch):
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", dt == "tf32")
    cl = clouds(cuda_dev)
    amp = dt == "amp"
    if "eager" in modes:
        net, c_in = setup(name, algo, dt, False, cuda_dev)
        x = inputs(net, c_in, cl[0], dt, cuda_dev)
        probe = run(net, x, 0.0, amp)
        G = make_g(probe["y"][net.steps[-1][0]], 0)
        rec = run(net, inputs(net, c_in, cl[0], dt, cuda_dev), G, amp)
        check_record(net, rec, dt)
    if "padded" in modes or "graph" in modes:
        net, c_in = setup(name, algo, dt, True, cuda_dev)
        rows = _pad_rows(cl)
        xs = [inputs(net, c_in, c, dt, cuda_dev, rows, seed=k) for k, c in enumerate(cl)]
        bounds = spconv.set_output_bounds(_Seq(net), inputs(net, c_in, cl[1], dt, cuda_dev), margin=1.3)
        assert bounds, "no bounded layer"
        probe = run(net, xs[0], 0.0, amp)
        Gs = [make_g(probe["y"][net.steps[-1][0]], 100 + k) for k in range(3)]
        probe = None          # a live autograd graph would tie the parameters' AccumulateGrad nodes to this stream
        eager = []
        for k in range(3):
            xs[k] = xs[k].replace_feature(xs[k].features.detach().requires_grad_(True))
            rec = run(net, xs[k], Gs[k], amp)
            if k == 0 and "padded" in modes:
                check_record(net, rec, dt)
            eager.append([t.detach().clone() for t in flat(net, rec)])
            rec = None
        spconv.check_bounds(net.mods)
        if "graph" in modes:
            def step(f, i, nv, g):
                x = spconv.SparseConvTensor(f.detach().requires_grad_(True), i, SHAPE, BATCH)
                x.num_valid = nv
                return flat(net, run(net, x, g, amp))
            args = [(x.features.detach(), x.indices, x.num_valid, g) for x, g in zip(xs, Gs)]
            graphed = spconv.graph_capture(step, *args[0])
            for k in (2, 0, 1):
                got = graphed(*args[k])
                assert len(got) == len(eager[k])
                for j, (a, b) in enumerate(zip(got, eager[k])):
                    assert a is not None and b is not None and torch.equal(a, b), \
                        f"replay of cloud {k}: recorded tensor {j} differs from the eager padded step"
            spconv.check_bounds(net.mods)
    if "eval" in modes:
        net, c_in = setup(name, algo, dt, False, cuda_dev)
        x = inputs(net, c_in, cl[0], dt, cuda_dev)
        for _ in range(2):                                  # running stats that are not the initial ones
            run(net, inputs(net, c_in, cl[0], dt, cuda_dev), 1.0, amp)
        check_eval(net, x, dt)


class _Seq(nn.Module):
    """a Net as one module (set_output_bounds runs it once)"""

    def __init__(self, net):
        super().__init__()
        self.net = net
        self.mods = net.mods

    def forward(self, x):
        env = {"x": x}
        for name, ins in self.net.steps:
            args = [env[i] for i in ins]
            env[name] = self.mods[name](args if len(args) > 1 else args[0])
        return env[self.net.steps[-1][0]]


def test_merge_net_exact_end_to_end(cuda_dev, monkeypatch):
    """The BN-free merge net on small integers in exact fp32: every sum of every layer is exact, so the loss,
    the input gradient and every parameter gradient equal the float64 twin's bit for bit."""
    from spconv_b200.pytorch import ops
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", False)
    cl = clouds(cuda_dev)
    for algo in ("MaskImplicitGemm", "MaskSplitImplicitGemm", "Native"):
        net, c_in = setup("merge", algo, "f32", False, cuda_dev, exact=True, seed=5)
        x = inputs(net, c_in, cl[1], "f32", cuda_dev, exact=True, seed=5)
        probe = run(net, x, 0.0)
        G = make_g(probe["y"]["c2"], 5, exact=True)
        G[_nv(probe["y"]["c2"]):] = 0               # the padding rows of the union carry the bias: not in the loss
        probe = None
        x = inputs(net, c_in, cl[1], "f32", cuda_dev, exact=True, seed=5)
        rec = run(net, x, G)
        # the twin, end to end in float64
        inds = x.indices.cpu().numpy()
        mods = net.mods
        params = {n: _d(p).requires_grad_(True) for n, p in mods.named_parameters()}
        xd = _d(x.features).requires_grad_(True)
        big = 2.0 ** 24

        def conv(mname, a, a_inds, kind, shape):
            m = mods[mname]
            ref = SparseConvRef(a_inds, BATCH, shape, m.kernel_size, m.stride, m.padding, m.dilation,
                                m.output_padding, kind)
            twin = net_ref.ConvTwin(ref)
            w, b = params[f"{mname}.weight"], params[f"{mname}.bias"]
            mag = twin(a.detach().abs(), w.detach().abs()) + b.detach().abs()
            assert float(mag.max()) < big, f"{mname}: a sum is not exact in fp32"
            return twin(a, w, b), ref

        y1, _ = conv("c1", xd, inds, "subm", SHAPE)
        r1 = net_ref.relu(y1)
        ya, _ = conv("a", r1, inds, "subm", SHAPE)
        yd, dref = conv("d1", r1, inds, "conv", SHAPE)
        yt, tref = conv("t1", net_ref.relu(yd), dref.out_inds, "transpose", dref.out_shape)
        mis = net_ref.MisalignedAdd([inds, tref.out_inds], BATCH, SHAPE)
        ym = mis([ya, yt])
        y2, _ = conv("c2", ym, mis.out_inds, "subm", SHAPE)
        got = rec["y"]["c2"]
        assert np.array_equal(got.indices[:_nv(got)].cpu().numpy(), mis.out_inds)
        loss = (y2 * _d(G[:len(mis.out_inds)])).sum()
        loss.backward()
        grads = [xd.grad] + [params[n].grad for n, _ in mods.named_parameters()]
        for g in grads:
            assert float(g.abs().max()) < big and torch.equal(g, g.float().double()), "a gradient is not exact"
        assert float(rec["loss"]) == float(loss), (algo, float(rec["loss"]), float(loss))
        assert torch.equal(x.features.grad.cpu(), xd.grad.float()), f"{algo}: input gradient"
        for n, p in mods.named_parameters():
            assert torch.equal(p.grad.cpu(), params[n].grad.float()), f"{algo}: gradient of {n}"


def test_mask_split_training_step_captures_without_host_copies(cuda_dev):
    """A MaskSplitImplicitGemm training step (rulebook, forward, input and weight gradients) makes no
    synchronising call, so it captures as a CUDA graph and replays to the eager result."""
    import spconv_b200.pytorch as spconv
    from spconv_b200.core import ConvAlgo
    cl = clouds(cuda_dev)
    torch.manual_seed(3)
    net = spconv.SparseSequential(
        spconv.SubMConv3d(16, 32, 3, indice_key="s", algo=ConvAlgo.MaskSplitImplicitGemm),
        spconv.SubMConv3d(32, 16, 3, indice_key="s", algo=ConvAlgo.MaskSplitImplicitGemm)).to(cuda_dev).half()
    rows = _pad_rows(cl)
    xs = [spconv.SparseConvTensor(torch.randn((c.shape[0], 16), device=cuda_dev).half(), c, SHAPE, BATCH).pad_to(rows)
          for c in cl]

    def step(f, i, nv):
        for p in net.parameters():
            p.grad = None
        x = spconv.SparseConvTensor(f, i, SHAPE, BATCH)
        x.num_valid = nv
        y = net(x)
        y.features.float().square().sum().backward()
        return [y.features.detach()] + [p.grad for p in net.parameters()]

    args = [(x.features, x.indices, x.num_valid) for x in xs]
    want = [[t.clone() for t in step(*a)] for a in args]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step(*args[1])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    graphed = spconv.graph_capture(step, *args[0])
    for k in (1, 2, 0):
        for a, b in zip(graphed(*args[k]), want[k]):
            assert torch.equal(a, b), f"replay of cloud {k}"


def test_cases_cover_every_net_mode_algo_and_dtype():
    seen = {(n, m) for n, _, _, modes in CASES for m in modes}
    for n in NETS:
        assert (n, "eager") in seen or (n, "padded") in seen, n
    assert {m for _, m in seen} == {"eager", "padded", "graph", "eval"}
    assert {a for n, a, _, _ in CASES if n == "unet"} == {"Native", "MaskImplicitGemm", "MaskSplitImplicitGemm"}
    assert {d for _, _, d, _ in CASES} == {"f32", "tf32", "f16", "bf16", "amp"}
    assert any(a == "MaskSplitImplicitGemm" and "graph" in modes for _, a, _, modes in CASES)
    assert any(a == "MaskSplitImplicitGemm" and "eval" in modes for _, a, _, modes in CASES)
