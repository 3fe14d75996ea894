"""Convolution onto given output coordinates on the GPU: the cross rulebook bit for bit against the numpy oracle,
equal to the existing rulebooks and layers where the target is the layer's own output set, two different clouds
against a float64 reference on every kernel family and dtype, a padded step captured as one CUDA graph, and the
reuse of the rulebook under indice_key, forward and back."""
import numpy as np
import pytest
import torch

from tests.cross_rulebook_oracle import cross_tables
from tests.util import check_tile_table, random_cloud, rel_l2, surface_cloud

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _np(t):
    return t.detach().cpu().numpy()


def _out_shape(shape, ksize, stride, padding, dilation, kind):
    if kind == "subm":
        return list(shape)
    if kind == "transpose":
        return [(i - 1) * s - 2 * p + k for i, k, s, p in zip(shape, ksize, stride, padding)]
    return [(i + 2 * p - d * (k - 1) - 1) // s + 1 for i, k, s, p, d in zip(shape, ksize, stride, padding, dilation)]


def _relation(ksize, stride, padding, dilation, kind):
    """(stride, padding, transposed) of the relation: SubM is stride 1 with padding (k // 2) * d"""
    if kind == "subm":
        return [1] * len(ksize), [(k // 2) * d for k, d in zip(ksize, dilation)], False
    return list(stride), list(padding), kind == "transpose"


def _cloud(rng, shape, n, batch=1):
    return _cloud_per(rng, shape, [n] * batch)


def _cloud_per(rng, shape, per):
    if np.prod([float(s) for s in shape]) < 1e8:
        return random_cloud(rng, shape, per, 1)[1]
    # A grid too large to permute (>= 2^31 cells: 64-bit keys): n unique voxels in a box of ~8 n cells at the far
    # corner of the grid, so the keys use their high bits and a second such cloud on the conv's output grid
    # overlaps this one's image (pairs exist)
    rows = []
    for b, n in enumerate(per):
        side = int(np.ceil((8 * n) ** (1 / len(shape))))
        flat = rng.permutation(side ** len(shape))[:n]
        c = np.stack(np.unravel_index(flat, (side,) * len(shape)), -1) + np.asarray(shape) - side
        rows.append(np.concatenate([np.full((n, 1), b), c], 1))
    return np.concatenate(rows, 0).astype(np.int32)


def _messy(rng, inds, shape, batch):
    """duplicated rows, rows with a batch or a coordinate out of range, then padding rows of -1 (returned count)"""
    n = inds.shape[0]
    extra = [inds[rng.integers(0, n, max(n // 8, 1))] if n else inds[:0]]
    bad = np.zeros((3, inds.shape[1]), np.int32)
    bad[0, 0] = batch
    bad[1, 1] = shape[0]
    bad[2, -1] = -1
    extra.append(bad)
    rows = np.concatenate([inds, *extra]).astype(np.int32)
    rows = rows[rng.permutation(rows.shape[0])]
    return np.concatenate([rows, np.full((5, inds.shape[1]), -1, np.int32)]), rows.shape[0]


# name: (source shape, ksize, stride, padding, dilation, kind, source rows, target rows, batch)
CASES = {
    "subm_3d_k3": ([20, 30, 40], [3, 3, 3], [1] * 3, [0] * 3, [1] * 3, "subm", 1500, 1200, 2),
    "subm_1d": ([300], [5], [1], [0], [3], "subm", 130, 127, 1),
    "subm_2d_k5x5_dil": ([40, 50], [5, 5], [1, 1], [0, 0], [2, 1], "subm", 600, 500, 2),
    "conv_3d_s2": ([20, 30, 40], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], "conv", 2000, 900, 2),
    "conv_3d_dilated": ([20, 30, 40], [3, 2, 3], [1, 2, 1], [2, 0, 2], [2, 1, 2], "conv", 1000, 700, 1),
    "conv_4d": ([8, 9, 10, 11], [3, 3, 3, 3], [2, 2, 2, 2], [1, 1, 1, 1], [1] * 4, "conv", 700, 300, 1),
    "transpose_3d": ([10, 12, 14], [2, 3, 2], [2, 2, 2], [0, 1, 0], [1, 1, 1], "transpose", 300, 1500, 2),
    "transpose_2d_s3": ([20, 30], [3, 3], [3, 3], [1, 0], [1, 1], "transpose", 200, 900, 1),
    "kv125_4words": ([12, 12, 12], [5, 5, 5], [1] * 3, [0] * 3, [1] * 3, "subm", 600, 400, 1),
    "kv81_4d": ([6, 7, 8, 9], [3, 3, 3, 3], [1] * 4, [0] * 4, [1] * 4, "subm", 500, 400, 1),
    "int64_keys": ([4096, 4096, 512], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], "conv", 900, 700, 2),
    "rows_128": ([16, 16, 16], [3, 3, 3], [1] * 3, [0] * 3, [1] * 3, "subm", 128, 129, 1),
    "empty_source": ([16, 16, 16], [3, 3, 3], [1] * 3, [0] * 3, [1] * 3, "subm", 0, 200, 1),
    "empty_target": ([16, 16, 16], [3, 3, 3], [2] * 3, [1] * 3, [1] * 3, "conv", 200, 0, 1),
}


def _check_tables(res, want, n, m, kv, is_train):
    outids, _, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, _ = res
    words = (kv + 31) // 32
    assert np.array_equal(_np(pair_fwd), want["pair_fwd"])
    assert np.array_equal(_np(pair_bwd), want["pair_bwd"])
    assert np.array_equal(_np(mask_fwd[0]).view(np.uint32), want["mask_fwd"])
    assert np.array_equal(_np(sort_fwd[0]), want["argsort_fwd"])
    t, tm = sort_fwd[0]._spx_tile_cache[1:]
    if m:
        check_tile_table(_np(t), _np(tm), want["pair_fwd"], want["mask_fwd"], want["argsort_fwd"], m, kv, words,
                         "forward tile table")
    if is_train:
        assert np.array_equal(_np(mask_bwd[0]).view(np.uint32), want["mask_bwd"])
        assert np.array_equal(_np(sort_bwd[0]), want["argsort_bwd"])
        t, tm = sort_bwd[0]._spx_tile_cache[1:]
        if n:
            check_tile_table(_np(t), _np(tm), want["pair_bwd"], want["mask_bwd"], want["argsort_bwd"], n, kv, words,
                             "backward tile table")


@pytest.mark.parametrize("messy", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_tables_match_the_oracle(name, messy):
    from spconv_b200.pytorch import ops
    shape, ksize, stride, padding, dilation, kind, n, m, batch = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    out_shape = _out_shape(shape, ksize, stride, padding, dilation, kind)
    src = _cloud(rng, shape, n, batch) if n else np.zeros((0, len(shape) + 1), np.int32)
    tgt = _cloud(rng, out_shape, m, batch) if m else np.zeros((0, len(shape) + 1), np.int32)
    nv_s = nv_t = None
    if messy:
        src, nv_s = _messy(rng, src, shape, batch)
        tgt, nv_t = _messy(rng, tgt, out_shape, batch)
    s, p, tr = _relation(ksize, stride, padding, dilation, kind)
    want = cross_tables(src, tgt, batch, shape, out_shape, ksize, s, p, dilation, tr, nv_s, nv_t)
    if n and m:                                       # every case with two sides has pairs to get right
        assert (want["pair_fwd"] >= 0).sum() >= min(n, m) // 4, (want["pair_fwd"] >= 0).sum()
    if name == "int64_keys":                          # and its keys need 64 bits
        assert float(batch) * np.prod([float(d) for d in out_shape]) >= 2 ** 31 - 1
    dv = (lambda v: None if v is None else torch.tensor([v], dtype=torch.int32, device=DEV))
    for is_train in (True, False):
        res = ops.get_indice_pairs_to(torch.from_numpy(src).to(DEV), torch.from_numpy(tgt).to(DEV), batch, shape,
                                      out_shape, ksize, s, p, dilation, tr, is_train, dv(nv_s), dv(nv_t))
        _check_tables(res, want, src.shape[0], tgt.shape[0], int(np.prod(ksize)), is_train)


# ---------------------------------------------------------------------------- equal to the existing rulebooks
EQUIV = {
    "subm_3d": ([30, 40, 50], [3, 3, 3], [1] * 3, [0] * 3, [1] * 3, "subm", [2500, 1500]),
    "subm_2d_k5": ([60, 70], [5, 5], [1, 1], [0, 0], [1, 1], "subm", [1200]),
    "conv_3d_s2": ([30, 40, 50], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], "conv", [3000, 2000]),
    "conv_4d": ([8, 9, 10, 11], [3, 3, 3, 3], [2, 2, 2, 2], [1, 1, 1, 1], [1] * 4, "conv", [700]),
    "transpose_3d": ([10, 12, 14], [2, 2, 2], [2, 2, 2], [0, 0, 0], [1, 1, 1], "transpose", [600]),
    "subm_int64_keys": ([4096, 4096, 512], [3, 3, 3], [1] * 3, [0] * 3, [1] * 3, "subm", [1500, 1000]),
    "conv_int64_keys": ([4096, 4096, 512], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], "conv", [1500, 1000]),
}


def _existing(inds, case, bound=-1):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    shape, ksize, stride, padding, dilation, kind, per = case
    return ops.get_indice_pairs_implicit_gemm(inds, len(per), shape, ConvAlgo.MaskImplicitGemm, ksize, stride,
                                              padding, dilation, [0] * len(shape), kind == "subm",
                                              kind == "transpose", is_train=True, num_out_act_bound=bound)


@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("name", list(EQUIV))
def test_own_output_set_gives_the_existing_rulebook(name, bounded):
    from spconv_b200.pytorch import ops
    case = EQUIV[name]
    shape, ksize, stride, padding, dilation, kind, per = case
    if bounded and kind == "subm":
        pytest.skip("SubM has no bounded rulebook")
    inds = torch.from_numpy(_cloud_per(np.random.default_rng(3), shape, per)).to(DEV)
    ref = _existing(inds, case)
    out_nv = None
    if bounded:
        ref = _existing(inds, case, bound=ref[0].shape[0] + 300)
        out_nv = ref[0]._spx_num_valid
    out_shape = _out_shape(shape, ksize, stride, padding, dilation, kind)
    s, p, tr = _relation(ksize, stride, padding, dilation, kind)
    got = ops.get_indice_pairs_to(inds, ref[0], len(per), shape, out_shape, ksize, s, p, dilation, tr, True,
                                  None, out_nv)
    assert int((ref[2] >= 0).sum()) > inds.shape[0]   # not the centre tap or one tap per row alone
    assert torch.equal(got[2], ref[2]) and torch.equal(got[3], ref[3])
    assert torch.equal(got[4][0], ref[4][0]) and torch.equal(got[6][0], ref[6][0])
    for a, b in zip(got[6][0]._spx_tile_cache[1:], ref[6][0]._spx_tile_cache[1:]):
        assert torch.equal(a, b)
    if kind != "subm":                                # SubM has no backward mask, sort or tile table
        assert torch.equal(got[5][0], ref[5][0]) and torch.equal(got[7][0], ref[7][0])
        for a, b in zip(got[7][0]._spx_tile_cache[1:], ref[7][0]._spx_tile_cache[1:]):
            assert torch.equal(a, b)


def _int_tensor(rng, shape, lo, hi, dtype):
    return torch.from_numpy(rng.integers(lo, hi + 1, shape).astype(np.float32)).to(DEV, dtype)


@pytest.mark.parametrize("depthwise", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("name", ["subm_3d", "subm_2d_k5", "conv_3d_s2", "transpose_3d"])
def test_layer_on_its_own_output_set_equals_the_existing_layer(name, dtype, depthwise):
    """forward, input gradient and weight gradient bit for bit, on integer-valued operands (SubM's input gradient
    visits the offsets in another order)"""
    import spconv_b200.pytorch as spconv
    shape, ksize, stride, padding, dilation, kind, per = EQUIV[name]
    nd = len(shape)
    rng = np.random.default_rng(5)
    inds = torch.from_numpy(random_cloud(rng, shape, per, 1)[1]).to(DEV)
    c = 32
    cls = {"subm": f"SubMConv{nd}d", "conv": f"SparseConv{nd}d", "transpose": f"SparseConvTranspose{nd}d"}[kind]
    kw = dict(dilation=dilation) if kind == "subm" else dict(stride=stride, padding=padding, dilation=dilation)
    layer = getattr(spconv, cls)(c, c, ksize, groups=c if depthwise else 1, bias=True, **kw).to(DEV, dtype)
    with torch.no_grad():
        layer.weight.copy_(_int_tensor(rng, layer.weight.shape, -1, 1, dtype))
        layer.bias.copy_(_int_tensor(rng, layer.bias.shape, -2, 2, dtype))
    feats = _int_tensor(rng, (inds.shape[0], c), -2, 2, dtype)

    def run(target_of):
        x = spconv.SparseConvTensor(feats.clone().requires_grad_(True), inds, shape, len(per))
        layer.zero_grad()
        y = layer(x) if target_of is None else layer(x, target=target_of)
        dy = _int_tensor(np.random.default_rng(9), y.features.shape, -2, 2, dtype)
        y.features.backward(dy)
        return y, x.features.grad.clone(), layer.weight.grad.clone(), layer.bias.grad.clone()

    ref = run(None)
    tgt = spconv.SparseConvTensor(torch.zeros(ref[0].indices.shape[0], 1, device=DEV), ref[0].indices,
                                  ref[0].spatial_shape, len(per))
    got = run(tgt)
    assert torch.equal(got[0].indices, ref[0].indices) and got[0].spatial_shape == ref[0].spatial_shape
    for a, b in zip((got[0].features,) + got[1:], (ref[0].features,) + ref[1:]):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------- two clouds, float64 reference
def _reference(x, w, pair_fwd, pair_bwd, dy, depthwise):
    """float64 out, din, dW of out[o] = sum_k W_k x[pair_fwd[k][o]] (W [K, kv, C], or [C, kv] depthwise)"""
    kv = pair_fwd.shape[0]
    x, w, dy = (np.asarray(a, np.float64) for a in (x, w, dy))
    out = np.zeros((pair_fwd.shape[1], w.shape[0]))
    din = np.zeros_like(x)
    dw = np.zeros_like(w)
    for k in range(kv):
        o = np.nonzero(pair_fwd[k] >= 0)[0]
        i = pair_fwd[k][o]
        if depthwise:
            out[o] += x[i] * w[:, k]
            din[i] += dy[o] * w[:, k]
            dw[:, k] = (dy[o] * x[i]).sum(0)
        else:
            out[o] += x[i] @ w[:, k].T
            din[i] += dy[o] @ w[:, k]
            dw[:, k] = dy[o].T @ x[i]
    assert pair_bwd is not None
    return out, din, dw


@pytest.mark.parametrize("variant", ["f32", "tf32", "f16", "bf16", "f16_fma", "f32_fma", "f16_depthwise",
                                     "bf16_depthwise"])
@pytest.mark.parametrize("kind", ["subm", "conv", "transpose"])
def test_two_clouds_against_float64(kind, variant, monkeypatch):
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    if variant == "tf32":
        monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", True)
    dtype = {"f32": torch.float32, "tf32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[
        variant.split("_")[0]]
    depthwise = variant.endswith("depthwise")
    fma = variant.endswith("fma")
    c_in, c_out = (6, 10) if fma else (32, 32 if depthwise else 64)
    shape = [20, 30, 40]
    rng = np.random.default_rng({"subm": 1, "conv": 2, "transpose": 3}[kind])
    if kind == "subm":
        layer = spconv.SubMConv3d(c_in, c_out, 3, groups=c_in if depthwise else 1)
        out_shape = shape
    elif kind == "conv":
        layer = spconv.SparseConv3d(c_in, c_out, 3, 2, 1, groups=c_in if depthwise else 1)
        out_shape = _out_shape(shape, [3] * 3, [2] * 3, [1] * 3, [1] * 3, "conv")
    else:
        layer = spconv.SparseConvTranspose3d(c_in, c_out, 2, 2, groups=c_in if depthwise else 1)
        out_shape = _out_shape(shape, [2] * 3, [2] * 3, [0] * 3, [1] * 3, "transpose")
    layer = layer.to(DEV, dtype)
    src = random_cloud(rng, shape, [1500, 1000], 1)[1]
    tgt = random_cloud(rng, out_shape, [1200, 900], 1)[1]
    x = spconv.SparseConvTensor(torch.from_numpy(rng.uniform(-1, 1, (src.shape[0], c_in))).to(DEV, dtype)
                                .requires_grad_(True), torch.from_numpy(src).to(DEV), shape, 2)
    t = spconv.SparseConvTensor(torch.zeros(tgt.shape[0], 1, device=DEV), torch.from_numpy(tgt).to(DEV), out_shape, 2)
    layer.train()
    y = layer(x, target=t)
    family = ops.last_kernel_family()
    if not depthwise:                                  # exact fp32 runs on the FMA kernels
        assert family == (1 if fma or variant == "f32" else 2), family
    dy = torch.from_numpy(rng.uniform(-1, 1, tuple(y.features.shape))).to(DEV, dtype)
    y.features.backward(dy)
    assert torch.equal(y.indices, t.indices) and y.spatial_shape == out_shape
    assert y.indice_dict == {} and y.num_valid is None
    ksize, s, p, tr = ((layer.kernel_size,) + _relation(layer.kernel_size, layer.stride, layer.padding,
                                                        layer.dilation, kind))
    tab = cross_tables(src, tgt, 2, shape, out_shape, ksize, s, p, layer.dilation, tr)
    kv = int(np.prod(ksize))
    w = _np(layer.weight.float()).reshape(c_out, kv, -1)
    w = w[:, :, 0] if depthwise else w
    out, din, dw = _reference(_np(x.features.float()), w, tab["pair_fwd"], tab["pair_bwd"], _np(dy.float()),
                              depthwise)
    out += _np(layer.bias.float())
    tol = {torch.float32: 1e-5, torch.float16: 2e-3, torch.bfloat16: 1e-2}[dtype] * (100 if variant == "tf32" else 1)
    assert rel_l2(_np(y.features.float()), out) < tol
    assert rel_l2(_np(x.features.grad.float()), din) < tol
    assert rel_l2(_np(layer.weight.grad.float()).reshape(w.shape), dw) < tol
    assert rel_l2(_np(layer.bias.grad.float()), _np(dy.float()).sum(0)) < tol


# ---------------------------------------------------------------------------- capture, reuse, inverse
def test_padded_step_captures_as_one_graph_with_a_fixed_launch_count():
    """SubM -> SubM onto a second padded cloud -> bounded strided conv, forward and backward: the same native launch
    count for two clouds of one padded size, one CUDA graph (a host sync would fail the capture), replays equal to
    eager on fresh clouds"""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    shape, rows, c = [41, 400, 352], 9000, 32
    torch.manual_seed(0)
    net = spconv.SubMConv3d(c, c, 3, bias=False, indice_key="sub").to(DEV).half()
    cross = spconv.SubMConv3d(c, c, 3, bias=False, indice_key="cross").to(DEV).half()
    down = spconv.SparseConv3d(c, c, 3, 2, 1, bias=False).to(DEV).half()
    down.num_out_act_bound = rows
    params = list(net.parameters()) + list(cross.parameters()) + list(down.parameters())

    def tensors(seed):
        rng = np.random.default_rng(seed)
        a = surface_cloud(rng, shape, int(rng.integers(6000, rows)))
        b = surface_cloud(rng, shape, int(rng.integers(6000, rows)))
        fa = torch.from_numpy(rng.uniform(-1, 1, (a.shape[0], c))).to(DEV).half()
        x = spconv.SparseConvTensor(fa, torch.from_numpy(a).to(DEV), shape, 1).pad_to(rows)
        t = spconv.SparseConvTensor(torch.zeros(b.shape[0], 1, device=DEV), torch.from_numpy(b).to(DEV), shape,
                                    1).pad_to(rows)
        return x, t

    def step(x, t):
        x = x.replace_feature(x.features.detach().requires_grad_(True))
        y = cross(net(x), target=t)
        z = down(y)
        loss = (z.features.float() ** 2).sum() + (y.features.float() ** 2).sum()
        loss.backward()
        return x.features.grad, z.features, y.features

    counts = []
    for seed in (1, 2):
        x, t = tensors(seed)
        ops.launch_count(reset=True)
        step(x, t)
        torch.cuda.synchronize()
        counts.append(ops.launch_count())
    assert counts[0] == counts[1], counts
    sx, st = tensors(3)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(sx, st)                                   # warm-up on a side stream
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step(sx, st)
    static_grads = [p.grad for p in params]
    for seed in (4, 5):
        x, t = tensors(seed)
        for p in params:
            p.grad = None
        want = [o.clone() for o in step(x, t)]
        want_grads = [p.grad.clone() for p in params]
        sx.features.copy_(x.features)
        sx.indices.copy_(x.indices)
        sx.num_valid.copy_(x.num_valid)
        st.indices.copy_(t.indices)
        st.num_valid.copy_(t.num_valid)
        for gr in static_grads:
            gr.zero_()
        g.replay()
        torch.cuda.synchronize()
        for o, w in zip(outs, want):
            assert torch.equal(o, w)
        for gr, w in zip(static_grads, want_grads):
            assert torch.equal(gr, w)


def test_reuse_under_indice_key_and_the_inverse_walk_back(monkeypatch):
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    shape, c = [20, 30, 40], 32
    rng = np.random.default_rng(11)
    src = random_cloud(rng, shape, [1500], 1)[1]
    out_shape = _out_shape(shape, [3] * 3, [2] * 3, [1] * 3, [1] * 3, "conv")
    tgt = random_cloud(rng, out_shape, [800], 1)[1]
    feats = torch.from_numpy(rng.uniform(-1, 1, (src.shape[0], c))).to(DEV).half()
    x = spconv.SparseConvTensor(feats, torch.from_numpy(src).to(DEV), shape, 1)
    t = spconv.SparseConvTensor(torch.zeros(tgt.shape[0], 1, device=DEV), torch.from_numpy(tgt).to(DEV), out_shape, 1)
    a = spconv.SparseConv3d(c, c, 3, 2, 1, bias=False, indice_key="x2t").to(DEV).half().eval()
    b = spconv.SparseConv3d(c, c, 3, 2, 1, bias=False, indice_key="x2t").to(DEV).half().eval()
    inv = spconv.SparseInverseConv3d(c, c, 3, indice_key="x2t", bias=False).to(DEV).half().eval()
    with torch.no_grad():
        ops.launch_count(reset=True)
        y = a(x, target=t)
        torch.cuda.synchronize()
        first = ops.launch_count(reset=True)
        rec = y.indice_dict["x2t"]
        assert rec.cross and torch.equal(rec.out_indices, t.indices)
        monkeypatch.setattr(ops, "get_indice_pairs_to", lambda *a, **k: pytest.fail("the rulebook was rebuilt"))
        y2 = b(x, target=y)
        torch.cuda.synchronize()
        again = ops.launch_count(reset=True)
        assert again < first and y2.indice_dict["x2t"] is rec
        # the same rows and geometry on another coordinate tensor is not the rulebook's input
        other = spconv.SparseConvTensor(feats, x.indices.clone(), shape, 1)
        with pytest.raises(ValueError, match="does not match"):
            b(other, target=y)
        z = inv(y2)
    assert torch.equal(z.indices, x.indices) and z.spatial_shape == shape
    tab = cross_tables(src, tgt, 1, shape, out_shape, [3] * 3, [2] * 3, [1] * 3, [1] * 3, False)
    for layer, inp, out, table in ((a, x, y, "pair_fwd"), (b, x, y2, "pair_fwd"), (inv, y2, z, "pair_bwd")):
        w = _np(layer.weight.float()).reshape(c, 27, c)
        xi = _np(inp.features.float())
        ref = np.zeros((out.features.shape[0], c))
        for k in range(27):
            o = np.nonzero(tab[table][k] >= 0)[0]
            ref[o] += xi[tab[table][k][o]] @ w[:, k].T
        assert rel_l2(_np(out.features.float()), ref) < 2e-3
    # a SubM layer that finds the record under its key refuses it
    with pytest.raises(ValueError, match="onto given coordinates"):
        spconv.SubMConv3d(c, c, 3, indice_key="x2t").to(DEV).half()(y2)


@pytest.mark.parametrize("where", ["src", "dst"])
def test_index_rows_at_unaligned_addresses_and_as_column_slices(where):
    """spx_cross_rulebook_all reads both index arrays as 16-byte rows and refuses other addresses: the operator
    passes indices 4, 8 and 12 bytes past a 16-byte boundary, or as a column slice, through an aligned copy with the
    same tables"""
    from spconv_b200.pytorch import ops
    shape, ksize, stride, padding, dilation, kind, n, m, batch = CASES["conv_3d_s2"]
    rng = np.random.default_rng(21)
    out_shape = _out_shape(shape, ksize, stride, padding, dilation, kind)
    src = torch.from_numpy(_cloud(rng, shape, n, batch)).to(DEV)
    tgt = torch.from_numpy(_cloud(rng, out_shape, m, batch)).to(DEV)
    s, p, tr = _relation(ksize, stride, padding, dilation, kind)

    def build(a, b):
        return ops.get_indice_pairs_to(a, b, batch, shape, out_shape, ksize, s, p, dilation, tr, True)

    want = build(src, tgt)
    base = src if where == "src" else tgt
    moved = []
    for off in (1, 2, 3):
        buf = torch.empty(base.numel() + 4, dtype=torch.int32, device=DEV)
        view = buf[off:off + base.numel()].view(base.shape)
        view.copy_(base)
        moved.append(view)
    wide = torch.zeros(base.shape[0], base.shape[1] + 3, dtype=torch.int32, device=DEV)
    wide[:, 1:1 + base.shape[1]] = base
    moved.append(wide[:, 1:1 + base.shape[1]])
    for t in moved:
        got = build(t, tgt) if where == "src" else build(src, t)
        for j in (2, 3):
            assert torch.equal(got[j], want[j])
        for j in (4, 5, 6, 7):
            assert torch.equal(got[j][0], want[j][0])
            if j in (6, 7):
                for a, b in zip(got[j][0]._spx_tile_cache[1:], want[j][0]._spx_tile_cache[1:]):
                    assert torch.equal(a, b)


def test_1x1_layer_goes_through_the_rulebook():
    """a 1x1 layer given a target reads the source row at each target coordinate (zero where there is none) instead
    of multiplying its own rows"""
    import spconv_b200.pytorch as spconv
    shape = [20, 30, 40]
    rng = np.random.default_rng(13)
    src = random_cloud(rng, shape, [900], 1)[1]
    tgt = np.concatenate([src[:300], random_cloud(rng, shape, [400], 1)[1]]).astype(np.int32)
    layer = spconv.SubMConv3d(32, 64, 1, bias=False).to(DEV).half()
    x = spconv.SparseConvTensor(torch.from_numpy(rng.uniform(-1, 1, (src.shape[0], 32))).to(DEV).half()
                                .requires_grad_(True), torch.from_numpy(src).to(DEV), shape, 1)
    t = spconv.SparseConvTensor(torch.zeros(tgt.shape[0], 1, device=DEV), torch.from_numpy(tgt).to(DEV), shape, 1)
    y = layer(x, target=t)
    dy = torch.from_numpy(rng.uniform(-1, 1, (tgt.shape[0], 64))).to(DEV).half()
    y.features.backward(dy)
    tab = cross_tables(src, tgt, 1, shape, shape, [1] * 3, [1] * 3, [0] * 3, [1] * 3, False)
    assert (tab["pair_fwd"][0][:300] == np.arange(300)).all()
    out, din, dw = _reference(_np(x.features.float()), _np(layer.weight.float()).reshape(64, 1, 32), tab["pair_fwd"],
                              tab["pair_bwd"], _np(dy.float()), False)
    assert torch.equal(y.indices, t.indices) and y.features.shape == (tgt.shape[0], 64)
    assert rel_l2(_np(y.features.float()), out) < 2e-3
    assert rel_l2(_np(x.features.grad.float()), din) < 2e-3
    assert rel_l2(_np(layer.weight.grad.float()).reshape(dw.shape), dw) < 2e-3
