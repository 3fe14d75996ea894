"""The SparseConv / SubMConv / SparseConvTranspose / SparseInverseConv modules in 1-D to 4-D, with
autograd, against the float64 reference of tests/conv_ref.py.

The geometries reach every rulebook dispatch branch: the 3x3x3 SubM probe, the generic SubM probe, the
3x3x3, 3-D (FAST3) and generic regular-conv insert kernels, transposed grids with output padding, and
Table64 keys (grids of 2^31 cells or more).  Inputs, weights and dY are exactly representable in every
dtype, so each product is exact and each element is checked against
    |got - ref| <= u_out |ref| + T 2^-23 sum|terms| + tiny
(T terms summed; test_conv_tc_coverage_gpu.py).  Output coordinates must equal the oracle's rows in
order, and every call must run on the kernel family its shape implies.
"""
import numpy as np
import pytest
import torch

from tests.conv_ref import SparseConvRef
from tests.test_conv_tc_coverage_gpu import ENV_FAMILY, gemm_instance, wgrad_instance
from tests.util import random_cloud

pytestmark = pytest.mark.gpu

TORCH_DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
U_OUT = {"f32": 2.0 ** -24, "f16": 2.0 ** -11, "bf16": 2.0 ** -8}
TINY = {"f32": 1e-30, "f16": 2.0 ** -24, "bf16": 1e-30}
BIG = [1300, 1300, 1300]                       # 2.2e9 cells: int64 (Table64) keys
BIG_S2 = [2600, 2600, 2600]                    # output grid of a stride-2 conv: 2.2e9 cells


def _g(kind, shape, pts, ksize, stride=None, padding=None, dilation=None, output_padding=None, box=None):
    nd = len(shape)
    return {"kind": kind, "shape": shape, "pts": pts, "batch": len(pts), "ksize": ksize,
            "stride": stride or [1] * nd, "padding": padding or [0] * nd, "dilation": dilation or [1] * nd,
            "output_padding": output_padding or [0] * nd, "box": box}


GEOMS = {
    # subm
    "subm3d_k3": _g("subm", [20, 20, 20], [1500, 1200], [3] * 3),                      # subm_probe_k3_kernel
    "subm3d_k3d2": _g("subm", [19, 18, 17], [1500], [3] * 3, dilation=[2] * 3),
    "subm3d_k513": _g("subm", [20, 20, 20], [1800], [5, 1, 3]),                        # generic probe
    "subm1d_k5": _g("subm", [3000], [900], [5]),
    "subm2d_k7": _g("subm", [40, 50], [900], [7, 7]),                                  # kv 49: two mask words
    "subm4d_k3": _g("subm", [9, 10, 11, 12], [2000], [3] * 4),                         # kv 81
    "subm3d_k3_big": _g("subm", BIG, [2500], [3] * 3, box=[30, 30, 30]),               # Table64
    # regular conv
    "conv3d_k3s2p1": _g("conv", [19, 18, 17], [1500, 1500], [3] * 3, [2] * 3, [1] * 3),   # 3x3x3 insert kernel
    "conv3d_k3s122": _g("conv", [19, 18, 17], [1500], [3] * 3, [1, 2, 2], [1] * 3),
    "conv3d_k3s2d2": _g("conv", [19, 18, 17], [1500], [3] * 3, [2] * 3, [2] * 3, [2] * 3),
    "conv3d_k2s2": _g("conv", [19, 18, 17], [1500], [2] * 3, [2] * 3),                    # FAST3
    "conv3d_k4s3p1": _g("conv", [19, 18, 17], [1500], [4] * 3, [3] * 3, [1] * 3),        # FAST3, division by 3
    "conv3d_k313s212": _g("conv", [20, 20, 20], [1800], [3, 1, 3], [2, 1, 2], [1, 0, 1]),
    "conv1d_k3s4": _g("conv", [3000], [900], [3], [4]),                                   # some points vanish
    "conv2d_k3s2": _g("conv", [40, 50], [900, 800], [3, 3], [2, 2], [1, 1]),             # generic kernel
    "conv4d_k2s2": _g("conv", [9, 10, 11, 12], [2000], [2] * 4, [2] * 4),
    "conv4d_k3s2": _g("conv", [9, 10, 11, 12], [2000], [3] * 4, [2] * 4, [1] * 4),
    "conv3d_k2s2_big": _g("conv", BIG_S2, [2500], [2] * 3, [2] * 3, box=[30, 30, 30]),      # FAST3 + Table64
    "conv2d_k3s2_big": _g("conv", [100000, 100000], [2000], [3, 3], [2, 2], [1, 1], box=[60, 60]),  # generic + Table64
    # transposed
    "tconv3d_k3s2p1": _g("transpose", [10, 9, 8], [300, 250], [3] * 3, [2] * 3, [1] * 3),
    "tconv3d_k3s2p1op1": _g("transpose", [10, 9, 8], [300], [3] * 3, [2] * 3, [1] * 3, output_padding=[1] * 3),
    "tconv2d_k2s2": _g("transpose", [20, 25], [300], [2, 2], [2, 2]),
    "tconv1d_k4s2p1op1": _g("transpose", [400], [150], [4], [2], [1], output_padding=[1]),
    "tconv4d_k3s2p1": _g("transpose", [5, 6, 5, 6], [300], [3] * 4, [2] * 4, [1] * 4),
    "tconv3d_k3s2d2": _g("transpose", [10, 9, 8], [300], [3] * 3, [2] * 3, [1] * 3, [2] * 3),   # drops taps
    # inverse of a regular conv, through indice_key
    "inv1d_k3s4": _g("inverse", [3000], [900], [3], [4]),
    "inv2d_k3s2": _g("inverse", [40, 50], [900, 800], [3, 3], [2, 2], [1, 1]),
    "inv4d_k2s2": _g("inverse", [9, 10, 11, 12], [2000], [2] * 4, [2] * 4),
    "inv3d_k2s2": _g("inverse", [19, 18, 17], [1500], [2] * 3, [2] * 3),
}
# sparse clouds for the mask-split cases (see _split_cloud)
SPLIT_GEOMS = {
    "split_subm3d_k3": _g("subm", [64, 64, 64], [1400], [3] * 3),
    "split_conv3d_k3s2p1": _g("conv", [64, 64, 64], [400], [3] * 3, [2] * 3, [1] * 3),
}


def _split_cloud(name):
    """subm: pairs of points (p, p + (1,1,1)) far apart; the upper point's only neighbour is at offset 0,
    so its second-split mask (offsets 14..26) is zero while pair[0] >= 0.  conv: isolated odd points 4 apart;
    every output has one input, and the output (c + 1) / 2 is reached through offset 0 alone."""
    rng = np.random.default_rng(11)
    if name.startswith("split_subm"):
        base = np.stack(np.meshgrid(*[np.arange(0, 60, 4)] * 3, indexing="ij"), -1).reshape(-1, 3)
        base = base[rng.permutation(len(base))[:700]]
        pts = np.concatenate([base, base + 1], 0)[rng.permutation(1400)]
    else:
        base = np.stack(np.meshgrid(*[np.arange(1, 64, 4)] * 3, indexing="ij"), -1).reshape(-1, 3)
        pts = base[rng.permutation(len(base))[:400]]
    return np.concatenate([np.zeros((len(pts), 1), np.int64), pts], 1).astype(np.int32)


def cloud(name):
    """(indices int32 [N, 1 + ndim], batch size) of a geometry"""
    if name in SPLIT_GEOMS:
        return _split_cloud(name), 1
    g = GEOMS[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    if g["box"] is None:
        _, inds = random_cloud(rng, g["shape"], g["pts"], 1)
    else:
        _, inds = random_cloud(rng, g["box"], g["pts"], 1)
        inds[:, 1:] += np.array([s - b - 1 for s, b in zip(g["shape"], g["box"])], np.int32)
    return inds, g["batch"]


# (dtype, C, K): tensor-core pairs and FMA pairs; f32 always runs on the FMA kernels
COMBOS = [("f16", 32, 32), ("bf16", 16, 32), ("f32", 16, 32), ("f16", 3, 16), ("bf16", 16, 5), ("f32", 3, 16)]


def _cases():
    out = []
    for gi, (name, g) in enumerate(GEOMS.items()):
        kv = int(np.prod(g["ksize"]))
        algos = ["Native", "MaskImplicitGemm"] + (["MaskSplitImplicitGemm"] if kv <= 32 else [])
        for ai, algo in enumerate(algos):
            out.append((name, algo, *COMBOS[(gi * 2 + ai) % len(COMBOS)]))
    return out


CASES = _cases()


def _exact(rng, shape, scale):
    """uniform values on a grid of `scale` with at most 4 significant bits"""
    return rng.integers(-8, 9, size=shape).astype(np.float64) * scale


def _family(dt, inst):
    if ENV_FAMILY == 1 or dt == "f32":
        return 1
    return 2 if inst is not None else 1


def _check(got, ref, mag, terms, dt, what, ref_pre=None, split=False):
    """ref_pre: the value before a rounded addition (the bias in training); split: partial results of the two
    mask splits are rounded to the output type before they are summed, adding u_out (|part 1| + |part 2|)
    <= u_out sum|terms|"""
    got = got.detach().double().cpu().numpy()
    u = U_OUT[dt]
    bound = u * np.abs(ref) + (0 if ref_pre is None else u * np.abs(ref_pre)) + (u * mag if split else 0) \
        + np.reshape(terms, terms.shape + (1,) * (ref.ndim - terms.ndim)) * 2.0 ** -23 * mag + TINY[dt]
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{what}: {int(bad.sum())}/{bad.size} elements out of bound; first at "
                           f"{np.argwhere(bad)[0].tolist()}: got {got[bad][0]!r} want {ref[bad][0]!r} "
                           f"bound {bound[bad][0]:.3g}")


def _module(spconv, kind, nd, C, K, g, algo, key):
    from spconv_b200.core import ConvAlgo
    a = ConvAlgo[algo]
    if kind == "subm":
        return getattr(spconv, f"SubMConv{nd}d")(C, K, g["ksize"], dilation=g["dilation"], algo=a, indice_key=key)
    if kind == "transpose":
        return getattr(spconv, f"SparseConvTranspose{nd}d")(C, K, g["ksize"], g["stride"], g["padding"],
                                                             g["dilation"], output_padding=g["output_padding"],
                                                             algo=a, indice_key=key)
    if kind == "inverse":
        return getattr(spconv, f"SparseInverseConv{nd}d")(C, K, g["ksize"], indice_key=key, algo=a)
    return getattr(spconv, f"SparseConv{nd}d")(C, K, g["ksize"], g["stride"], g["padding"], g["dilation"],
                                               algo=a, indice_key=key)


def run_case(name, g, inds, bs, algo, dt, C, K, oracle, dev, seed=0):
    """Forward + backward of one module against the reference; returns the reference rulebook."""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    tdt = TORCH_DT[dt]
    nd = len(g["shape"])
    kind = g["kind"]
    rng = np.random.default_rng(seed)
    d_inds = torch.from_numpy(inds).to(dev)
    ref = SparseConvRef(inds, bs, g["shape"], g["ksize"], g["stride"], g["padding"], g["dilation"],
                        g["output_padding"], kind)
    if kind == "inverse":
        # the paired conv builds the rulebook under the key; the inverse layer's input is a fresh leaf on its rows
        down = _module(spconv, "conv", nd, K, C, g, algo, "key").to(dev).to(tdt)
        mid = down(spconv.SparseConvTensor(torch.zeros((len(inds), K), dtype=tdt, device=dev), d_inds, g["shape"], bs))
        assert np.array_equal(mid.indices.cpu().numpy(), ref.in_inds)
        x_np = _exact(rng, (ref.n_in, C), 1 / 8)
        x_f = torch.from_numpy(x_np).to(dev).to(tdt).requires_grad_(True)
        x = mid.replace_feature(x_f)
    else:
        x_np = _exact(rng, (ref.n_in, C), 1 / 8)
        x_f = torch.from_numpy(x_np).to(dev).to(tdt).requires_grad_(True)
        x = spconv.SparseConvTensor(x_f, d_inds, g["shape"], bs)
    layer = _module(spconv, kind, nd, C, K, g, algo, "key" if kind == "inverse" else None).to(dev).to(tdt)
    w_np = _exact(rng, tuple(layer.weight.shape), 1 / 32)
    b_np = _exact(rng, (K,), 1 / 4)
    with torch.no_grad():
        layer.weight.copy_(torch.from_numpy(w_np))
        layer.bias.copy_(torch.from_numpy(b_np))
    layer.train()
    out = layer(x)
    torch.cuda.synchronize()
    kv = ref.kv
    fam_fwd = _family(dt, gemm_instance(dt, kv, C, K) if dt != "f32" else None)
    assert ops.last_kernel_family() == fam_fwd, (ops.last_kernel_family(), fam_fwd)
    # coordinates: the oracle's rows, in order
    got_inds = out.indices.cpu().numpy()
    if kind == "subm":
        assert np.array_equal(got_inds, inds)
    elif kind == "inverse":
        assert np.array_equal(got_inds, inds) and out.spatial_shape == list(g["shape"])
    else:
        o, _, _ = oracle.get_indice_pairs(inds, bs, g["shape"], g["ksize"], g["stride"], g["padding"],
                                          g["dilation"], g["output_padding"], False, kind == "transpose")
        assert np.array_equal(got_inds, o)
        assert np.array_equal(got_inds, ref.out_inds)
        assert out.spatial_shape == list(ref.out_shape)
    y, y_mag, y_terms = ref.forward(x_np, w_np)
    split = algo == "MaskSplitImplicitGemm"
    _check(out.features, y + b_np, y_mag + np.abs(b_np), y_terms + 1, dt, f"{name} forward", ref_pre=y, split=split)
    dy_np = _exact(rng, (ref.n_out, K), 1 / 16)
    out.features.backward(torch.from_numpy(dy_np).to(dev).to(tdt))
    torch.cuda.synchronize()
    fam_w = _family(dt, wgrad_instance(dt, kv, C, K) if dt != "f32" else None)
    assert ops.last_kernel_family() == fam_w, (ops.last_kernel_family(), fam_w)
    dx, dx_mag, dx_terms, dw, dw_mag, dw_terms = ref.backward(x_np, w_np, dy_np)
    _check(x_f.grad, dx, dx_mag, dx_terms, dt, f"{name} dX", split=split)
    dw_terms_full = np.broadcast_to(np.asarray(dw_terms).reshape(1, -1, 1),
                                    (K, kv, w_np.shape[-1])).reshape(w_np.shape)
    _check(layer.weight.grad, dw, dw_mag, dw_terms_full, dt, f"{name} dW")
    db = dy_np.sum(0)
    _check(layer.bias.grad, db, np.abs(dy_np).sum(0), np.full(K, ref.n_out, float), dt, f"{name} dbias")
    return ref


@pytest.mark.parametrize("name,algo,dt,C,K", CASES, ids=lambda v: str(v))
def test_module_against_float64_reference(name, algo, dt, C, K, oracle, cuda_dev):
    inds, bs = cloud(name)
    run_case(name, GEOMS[name], inds, bs, algo, dt, C, K, oracle, cuda_dev)


def test_cases_cover_every_geometry_algo_dtype_and_family():
    seen_ga, seen_df = set(), set()
    for name, algo, dt, C, K in CASES:
        seen_ga.add((name, algo))
        kv = int(np.prod(GEOMS[name]["ksize"]))
        seen_df.add((dt, _family(dt, gemm_instance(dt, kv, C, K) if dt != "f32" else None)))
    for name, g in GEOMS.items():
        kv = int(np.prod(g["ksize"]))
        for algo in ["Native", "MaskImplicitGemm"] + (["MaskSplitImplicitGemm"] if kv <= 32 else []):
            assert (name, algo) in seen_ga
    assert {("f16", 2), ("bf16", 2), ("f16", 1), ("bf16", 1), ("f32", 1)} <= seen_df


@pytest.mark.parametrize("name", list(SPLIT_GEOMS))
def test_mask_split_on_sparse_clouds(name, oracle, cuda_dev):
    """MaskSplitImplicitGemm on the tensor cores where the second split has all-zero tiles whose rows hold
    pair[0] >= 0 (an entry of the other split).  Such a tile still runs one stage; its gather table must
    not bring in the other split's rows, or W[0] is counted twice in the forward and input gradient."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    g = SPLIT_GEOMS[name]
    inds, bs = cloud(name)
    subm = g["kind"] == "subm"
    res = ops.get_indice_pairs_implicit_gemm(torch.from_numpy(inds).to(cuda_dev), bs, g["shape"],
                                             ConvAlgo.MaskSplitImplicitGemm, g["ksize"], g["stride"], g["padding"],
                                             g["dilation"], [0] * 3, subm, False, is_train=True)
    _, _, pair_fwd, _, mask_f, _, sort_f, _, _ = res
    # preconditions, from the returned forward tables (the SubM input gradient walks the same table):
    # several empty tiles in split 2 with rows where pair[0] >= 0
    m2 = mask_f[1].cpu().numpy().reshape(-1)
    rows = sort_f[1].cpu().numpy()
    p0 = pair_fwd[0].cpu().numpy()
    empty = [t for t in range(len(m2) // 128) if not m2[t * 128:(t + 1) * 128].any()]
    leaking = sum(int((p0[rows[t * 128:(t + 1) * 128]] >= 0).sum()) for t in empty)
    assert len(empty) >= 3 and leaking >= 64, (len(empty), leaking)
    run_case(name, g, inds, bs, "MaskSplitImplicitGemm", "f16", 32, 32, oracle, cuda_dev, seed=3)
    assert gemm_instance("f16", 27, 32, 32) is not None
