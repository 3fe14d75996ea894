"""Bounded regular-conv rulebook (num_out_act_bound) against the unbounded path on the same seeded clouds:
the rulebook bit for bit with its padding, the truncation when the bound is too small, the layer arithmetic
with padded rows (tiles without any active offset included), padded inputs through SubM / strided / inverse
layers, and a six-layer encoder step that runs without a host synchronisation and replays as one CUDA graph."""
import copy
import os

import numpy as np
import pytest
import torch

from bench_utils import make_encoder6
from tests.test_bounded_cpu import truncate_rulebook
from tests.util import check_tile_table, random_cloud, rel_l2, surface_cloud

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _np(t):
    return t.detach().cpu().numpy()


def _round128(m, extra_tiles=0):
    return (m + 127) // 128 * 128 + 128 * extra_tiles


# name: (spatial shape, ksize, stride, padding, dilation, transposed, points per sample)
CASES = {
    "k3_stride2": ([41, 160, 140], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], False, [6000, 5000]),
    "generic_3d": ([30, 40, 50], [2, 3, 2], [2, 1, 2], [0, 1, 0], [1, 1, 1], False, [3000]),
    "dilated_3d": ([30, 40, 50], [3, 3, 3], [1, 2, 1], [2, 2, 2], [2, 2, 2], False, [2500]),
    "conv_2d": ([200, 300], [3, 3], [2, 2], [1, 1], [1, 1], False, [4000, 100]),
    "conv_4d_81": ([10, 12, 14, 16], [3, 3, 3, 3], [2, 2, 2, 2], [1, 1, 1, 1], [1, 1, 1, 1], False, [1500]),
    "kv45_two_words": ([30, 40, 50], [3, 3, 5], [2, 2, 2], [1, 1, 2], [1, 1, 1], False, [2000]),
    "transposed_3d": ([10, 12, 14], [2, 2, 2], [2, 2, 2], [0, 0, 0], [1, 1, 1], True, [700]),
    "int64_keys": ([4096, 4096, 512], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], False, [900] * 4),
}


def _cloud(rng, case):
    shape, per_sample = case[0], case[6]
    if np.prod([float(s) for s in shape]) < 1e8:
        return random_cloud(rng, shape, per_sample, 1)[1]
    rows = []                                        # a grid too large to permute: draw coordinates, drop repeats
    for b, n in enumerate(per_sample):
        c = np.unique(np.stack([rng.integers(0, s, 2 * n) for s in shape], 1), axis=0)
        c = c[rng.permutation(c.shape[0])[:n]]
        rows.append(np.concatenate([np.full((c.shape[0], 1), b), c], 1).astype(np.int32))
    return np.concatenate(rows, 0)


def _rulebook(inds, batch, case, is_train, bound=-1):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    shape, ksize, stride, padding, dilation, transposed, _ = case
    return ops.get_indice_pairs_implicit_gemm(inds, batch, shape, ConvAlgo.MaskImplicitGemm, ksize, stride, padding,
                                              dilation, [0] * len(shape), False, transposed, is_train=is_train,
                                              num_out_act_bound=bound)


def _unsorted(mask_sorted, argsort):
    out = np.empty_like(mask_sorted)
    out[argsort] = mask_sorted
    return out


def _check_padded_rulebook(res_b, res_u, bound, kv, is_train, name):
    """rows below M equal the unbounded rulebook, rows beyond it are padding, tile tables restate the rulebook"""
    out_u, _, pf_u, pb_u, mf_u, mb_u, sf_u, sb_u, _ = res_u
    out_b, _, pf_b, pb_b, mf_b, mb_b, sf_b, sb_b, _ = res_b
    M = out_u.shape[0]
    words = (kv + 31) // 32
    assert out_b.shape[0] == bound and pf_b.shape == (kv, bound) and sf_b[0].shape == (bound,), name
    assert int(out_b._spx_num_valid) == M and int(out_b._spx_bound_status) == 0, name
    ob, pfb = _np(out_b), _np(pf_b)
    assert np.array_equal(ob[:M], _np(out_u)) and (ob[M:] == -1).all(), name
    assert np.array_equal(pfb[:, :M], _np(pf_u)) and (pfb[:, M:] == -1).all(), name
    assert np.array_equal(_np(pb_b), _np(pb_u)), name
    assert _np(pb_b).max() < M, name
    sfb, sfu = _np(sf_b[0]), _np(sf_u[0])
    # padding rows have mask 0: the stable sort puts them first, in order, and the valid rows keep their order
    assert np.array_equal(sfb[:bound - M], np.arange(M, bound)) and np.array_equal(sfb[bound - M:], sfu), name
    mfb = _unsorted(_np(mf_b[0]), sfb)
    assert np.array_equal(mfb[:M], _unsorted(_np(mf_u[0]), sfu)) and (mfb[M:] == 0).all(), name
    table, tmask = sf_b[0]._spx_tile_cache[1:]
    check_tile_table(_np(table), _np(tmask), pfb, _np(mf_b[0]), sfb, bound, kv, words, f"{name} fwd")
    if is_train:
        assert np.array_equal(_np(mb_b[0]), _np(mb_u[0])) and np.array_equal(_np(sb_b[0]), _np(sb_u[0])), name
        t_b, tm_b = sb_b[0]._spx_tile_cache[1:]
        t_u, tm_u = sb_u[0]._spx_tile_cache[1:]
        assert torch.equal(t_b, t_u) and torch.equal(tm_b, tm_u), name
    else:
        assert mb_b == [] and sb_b == [], name


def _flat(res):
    out = [res[0], res[2], res[3], res[0]._spx_num_valid, res[0]._spx_bound_status]
    for group in res[4:8]:
        out += list(group)
    return [_np(t) for t in out]


@pytest.mark.parametrize("name", list(CASES))
def test_bounded_rulebook_equals_unbounded(name, cuda_dev):
    case = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    batch = len(case[6])
    inds = torch.from_numpy(_cloud(rng, case)).to(cuda_dev)
    kv = int(np.prod(case[1]))
    for is_train in (True, False):
        res_u = _rulebook(inds, batch, case, is_train)
        M = res_u[0].shape[0]
        for bound in (M, M + 1, _round128(M, 3)):
            res_b = _rulebook(inds, batch, case, is_train, bound)
            _check_padded_rulebook(res_b, res_u, bound, kv, is_train, f"{name} train={is_train} bound={bound}")
        again = _rulebook(inds, batch, case, is_train, bound)
        for a, b in zip(_flat(res_b), _flat(again)):
            assert np.array_equal(a, b), f"{name}: two runs differ"


def test_bounded_rulebook_on_the_lidar_fixture(cuda_dev):
    g = np.load(os.path.join(GOLD, "fixture_coords.npz"))
    inds = torch.from_numpy(g["coors"]).to(cuda_dev)
    shape = [int(s) for s in g["shape"]]
    case = (shape, [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], False, None)
    res_u = _rulebook(inds, 1, case, True)
    bound = _round128(int(res_u[0].shape[0] * 1.25))
    _check_padded_rulebook(_rulebook(inds, 1, case, True, bound), res_u, bound, 27, True, "lidar fixture")


@pytest.mark.parametrize("name", ["k3_stride2", "generic_3d", "kv45_two_words"])
def test_bound_below_the_output_count_truncates(name, cuda_dev):
    case = CASES[name]
    rng = np.random.default_rng(5)
    batch = len(case[6])
    inds = torch.from_numpy(_cloud(rng, case)).to(cuda_dev)
    res_u = _rulebook(inds, batch, case, True)
    M = res_u[0].shape[0]
    bound = M - 37
    res_b = _rulebook(inds, batch, case, True, bound)
    assert int(res_b[0]._spx_bound_status) == 1 and int(res_b[0]._spx_num_valid) == bound
    oi, pf, pb, mf, mb = truncate_rulebook(_np(res_u[0]), _np(res_u[2]), _np(res_u[3]), bound)
    assert np.array_equal(_np(res_b[0]), oi) and np.array_equal(_np(res_b[2]), pf) and np.array_equal(_np(res_b[3]), pb)
    sf, sb = _np(res_b[6][0]), _np(res_b[7][0])
    assert np.array_equal(_unsorted(_np(res_b[4][0]), sf).view(np.uint32), mf)
    assert np.array_equal(_unsorted(_np(res_b[5][0]), sb).view(np.uint32), mb)
    # far too small a bound: whatever the status says, every index stays in range and nothing faults
    tiny = _rulebook(inds, batch, case, True, 128)
    assert int(tiny[0]._spx_bound_status) != 0
    assert int(_np(tiny[2]).max()) < inds.shape[0] and int(_np(tiny[3]).max()) < 128
    assert 0 <= int(tiny[0]._spx_num_valid) <= 128


def _layer_pair(spconv, C, K, dtype, dev, seed, integer):
    g = torch.Generator().manual_seed(seed)
    conv = spconv.SparseConv3d(C, K, 3, stride=2, padding=1, bias=True, indice_key="d")
    with torch.no_grad():
        if integer:       # small multiples of a power of two: every sum is exact, whatever its order
            conv.weight.copy_(torch.randint(-2, 3, conv.weight.shape, generator=g) / 8.0)
            conv.bias.copy_(torch.randint(-4, 5, conv.bias.shape, generator=g) / 4.0)
    conv = conv.to(dev).to(dtype)
    return conv, copy.deepcopy(conv)


@pytest.mark.parametrize("dtype_name", ["fp16", "bf16", "fp32", "tf32"])
@pytest.mark.parametrize("C,K", [(16, 16), (64, 32), (128, 128), (12, 20)])
@pytest.mark.parametrize("integer", [True, False])
def test_bounded_layer_equals_unbounded_layer(dtype_name, C, K, integer, cuda_dev, monkeypatch):
    """forward, input gradient, weight and bias gradient of one strided layer; the bound leaves three whole
    128-row tiles of padding, i.e. tiles without any active offset in forward, dgrad's source and wgrad"""
    import spconv_b200.pytorch as spconv
    from spconv_b200.pytorch import ops
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", dtype_name == "tf32")
    dtype = {"fp16": torch.float16, "bf16": torch.bfloat16}.get(dtype_name, torch.float32)
    rng = np.random.default_rng(C * 131 + K)
    shape = [21, 120, 100]
    inds = torch.from_numpy(surface_cloud(rng, shape, 9000)).to(cuda_dev)
    n = inds.shape[0]
    g = torch.Generator().manual_seed(C + K)
    feats = (torch.randint(-4, 5, (n, C), generator=g) / 4.0) if integer else torch.randn((n, C), generator=g)
    conv_u, conv_b = _layer_pair(spconv, C, K, dtype, cuda_dev, 3, integer)

    x_u = feats.to(cuda_dev).to(dtype).requires_grad_(True)
    y_u = conv_u(spconv.SparseConvTensor(x_u, inds, shape, 1))
    M = y_u.features.shape[0]
    bound = _round128(M, 3)
    gout = (torch.randint(-2, 3, (bound, K), generator=g) / 2.0) if integer else torch.randn((bound, K), generator=g)
    gout = gout.to(cuda_dev).to(dtype)
    (y_u.features * gout[:M]).sum().backward()

    conv_b.num_out_act_bound = bound
    x_b = feats.to(cuda_dev).to(dtype).requires_grad_(True)
    y_b = conv_b(spconv.SparseConvTensor(x_b, inds, shape, 1))
    assert y_b.features.shape == (bound, K) and int(y_b.num_valid) == M
    (y_b.features * gout).sum().backward()          # the loss reads the padding rows as well
    spconv.check_bounds(y_b)
    spconv.check_bounds(conv_b)

    assert torch.equal(y_b.features[:M], y_u.features), "forward"
    assert torch.equal(y_b.indices[:M], y_u.indices) and bool((y_b.indices[M:] == -1).all())
    assert torch.equal(y_b.features[M:], conv_b.bias.detach().expand(bound - M, K)), "padding rows hold the bias"
    assert torch.equal(x_b.grad, x_u.grad), "input gradient"
    if integer:
        assert torch.equal(conv_b.weight.grad, conv_u.weight.grad), "weight gradient"
        assert torch.equal(conv_b.bias.grad, conv_u.bias.grad), "bias gradient"
    else:
        tol = {"fp16": 2e-3, "bf16": 1e-2, "fp32": 1e-5, "tf32": 2e-3}[dtype_name]
        assert rel_l2(_np(conv_b.weight.grad.float()), _np(conv_u.weight.grad.float())) < tol
        assert rel_l2(_np(conv_b.bias.grad.float()), _np(conv_u.bias.grad.float())) < tol


def _chain(spconv, dev, dtype):
    torch.manual_seed(11)
    layers = [spconv.SubMConv3d(16, 16, 3, bias=True, indice_key="s1"),
              spconv.SparseConv3d(16, 32, 3, stride=2, padding=1, bias=True, indice_key="d"),
              spconv.SubMConv3d(32, 32, 3, bias=True, indice_key="s2"),
              spconv.SparseInverseConv3d(32, 16, 3, indice_key="d", bias=True)]
    return spconv.SparseSequential(*layers).to(dev).to(dtype)


def test_padded_input_through_subm_strided_subm_inverse(cuda_dev):
    import spconv_b200.pytorch as spconv
    rng = np.random.default_rng(21)
    shape = [21, 120, 100]
    inds = torch.from_numpy(surface_cloud(rng, shape, 5000)).to(cuda_dev)
    n = inds.shape[0]
    g = torch.Generator().manual_seed(2)
    feats = torch.randn((n, 16), generator=g).to(cuda_dev).half()
    net_u = _chain(spconv, cuda_dev, torch.float16)
    net_b = copy.deepcopy(net_u)
    gout = torch.randn((n + 300, 16), generator=g).to(cuda_dev).half()

    f_u = feats.clone().requires_grad_(True)
    y_u = net_u(spconv.SparseConvTensor(f_u, inds, shape, 1))
    (y_u.features * gout[:n]).sum().backward()

    bounds = spconv.set_output_bounds(net_b, spconv.SparseConvTensor(feats, inds, shape, 1), margin=1.1)
    assert list(bounds) == ["1"] and bounds["1"] % 128 == 0 and bounds["1"] >= net_b[1].num_out_act_bound > 0
    f_b = feats.clone().requires_grad_(True)
    y_b = net_b(spconv.SparseConvTensor(f_b, inds, shape, 1).pad_to(n + 300))
    assert y_b.features.shape[0] == n + 300 and int(y_b.num_valid) == n
    (y_b.features * gout).sum().backward()           # the loss reads the padding rows too
    spconv.check_bounds(net_b)
    assert torch.equal(y_b.features[:n], y_u.features)
    assert torch.equal(y_b.dense(), y_u.dense())
    # the tiles of the padded net differ, so the fp32 order of the weight-gradient sums differs
    assert rel_l2(_np(f_b.grad.float()), _np(f_u.grad.float())) < 2e-3
    for (name, p_b), p_u in zip(net_b.named_parameters(), net_u.parameters()):
        assert rel_l2(_np(p_b.grad.float()), _np(p_u.grad.float())) < 2e-3, name


def _encoder(spconv, dev):
    torch.manual_seed(4)
    layers = make_encoder6(spconv, bias=True, relu=True)
    return spconv.SparseSequential(*layers).to(dev).half()


def test_encoder_step_without_sync_and_as_one_graph(cuda_dev):
    import spconv_b200.pytorch as spconv
    shape = [41, 400, 352]
    rng = np.random.default_rng(8)
    counts = [20000, 17000, 18500, 40000]            # the last cloud is larger than the bounds allow
    clouds = [torch.from_numpy(surface_cloud(rng, shape, c)).to(cuda_dev) for c in counts]
    g = torch.Generator().manual_seed(6)
    feats = [torch.randn((c.shape[0], 16), generator=g).to(cuda_dev).half() for c in clouds]
    n_pad = 40064
    net = _encoder(spconv, cuda_dev)
    params = list(net.parameters())

    def step(f, i, nv=None):
        for p in params:
            p.grad = None
        x = spconv.SparseConvTensor(f, i, shape, 1)
        x.num_valid = nv
        y = net(x)
        valid = y.valid_mask().unsqueeze(1)
        loss = torch.where(valid, y.features.float(), 0.0).square().sum()
        loss.backward()
        return loss, [p.grad for p in params]

    want = []
    for f, i in zip(feats[:3], clouds[:3]):          # eager, unbounded
        loss, grads = step(f, i)
        want.append((loss.detach().clone(), [t.detach().clone() for t in grads]))

    bounds = spconv.set_output_bounds(net, spconv.SparseConvTensor(feats[0], clouds[0], shape, 1), margin=1.25)
    assert sorted(bounds) == ["10", "4", "8"]
    padded = [spconv.SparseConvTensor(f, i, shape, 1).pad_to(n_pad) for f, i in zip(feats, clouds)]
    args = [(p.features, p.indices, p.num_valid) for p in padded]

    step(*args[0])                                   # warm-up: allocator pools, status words
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss, grads = step(*args[1])                 # eager bounded: no synchronising call
    finally:
        torch.cuda.set_sync_debug_mode("default")
    def same(got, ref, what):
        loss, grads = got
        assert abs(float(loss.detach()) - float(ref[0])) <= 1e-4 * abs(float(ref[0])), what
        for (name, _), a, b in zip(net.named_parameters(), grads, ref[1]):
            assert rel_l2(_np(a.float()), _np(b.float())) < 2e-3, (what, name)

    same((loss, grads), want[1], "eager bounded")
    loss = grads = None

    graphed = spconv.graph_capture(step, *args[0])
    for k in (0, 1, 2, 1):
        same(graphed(*args[k]), want[k], f"replay of cloud {k}")
    spconv.check_bounds(net)
    graphed(*args[3])                                # more outputs than the bounds: flagged, nothing else fails
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="num_out_act_bound"):
        spconv.check_bounds(net)
    same(graphed(*args[2]), want[2], "replay after the overflow")
    spconv.check_bounds(net)


def test_max_pool_with_a_bound_and_voxel_count_record(cuda_dev):
    import spconv_b200.pytorch as spconv
    rng = np.random.default_rng(31)
    shape = [20, 60, 60]
    feats, inds = random_cloud(rng, shape, [4000], 16)
    f = torch.from_numpy(feats).to(cuda_dev).half()
    i = torch.from_numpy(inds).to(cuda_dev)
    pool_u = spconv.SparseMaxPool3d(2, 2, record_voxel_count=True).to(cuda_dev)
    pool_b = spconv.SparseMaxPool3d(2, 2, record_voxel_count=True).to(cuda_dev)
    x_u, x_b = f.clone().requires_grad_(True), f.clone().requires_grad_(True)
    y_u = pool_u(spconv.SparseConvTensor(x_u, i, shape, 1))
    M = y_u.features.shape[0]
    pool_b.num_out_act_bound = _round128(M, 1)
    y_b = pool_b(spconv.SparseConvTensor(x_b, i, shape, 1))
    assert torch.equal(y_b.features[:M], y_u.features) and bool((y_b.features[M:] == 0).all())
    assert int(pool_b.get_max_num_voxels()) == M == int(pool_u.get_max_num_voxels())
    y_u.features.float().sum().backward()
    y_b.features.float().sum().backward()
    assert torch.equal(x_b.grad, x_u.grad)
    spconv.check_bounds(pool_b)
