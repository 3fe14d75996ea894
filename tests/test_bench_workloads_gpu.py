"""The workloads of bench.py at full size, checked bit for bit.

Features, weights and output gradients are small integers times a power-of-two scale (values in
{-2, -1, 0, 1, 2} / 8).  Every product is then a multiple of one quantum q (2^-6), and so is every
partial sum, in whatever order it is formed.  Where an element's sum of |terms| stays below 2^24 q,
every partial sum is exact in fp32, so each kernel must return the float64 sum rounded once to the
output type, whatever its tiling, schedule or summation order.  The checks are torch.equal at full
size: a dropped, duplicated or misrouted tile, row or kernel offset fails them.  Every check asserts
its own precondition from the float64 |term| sums, so a change of sizes fails loudly instead of
quietly making the comparison approximate.

The clouds are bench.py's: surface_cloud(default_rng(50051 + i), shape, n, batch) with the shapes,
sizes and types of its WORKLOADS (restated below).  Each rulebook is compared bit for bit with the
oracle, and its tile tables and schedule records with a numpy restatement.  These sizes reach the
multi-chunk schedule ranking (more than 1024 tiles), the radix sort's scan carry over more than 256
blocks, and the two-job sort and tile-table launches of a strided conv with M != N.

With SPX_FORCE_SIMT=1 in the environment the same cases run on the FMA kernels, which are exact on
this grid too.
"""
import numpy as np
import pytest
import torch

from tests.test_conv_tc_coverage_gpu import ENV_FAMILY, Conv, _calls, _configure, _reference
from tests.util import check_tile_table, surface_cloud

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_forced_family():
    """Conv pins the kernel family of every call it makes; later tests get the one the environment pins"""
    yield
    if torch.cuda.is_available():
        _configure(ENV_FAMILY)

KITTI = [41, 1600, 1408]
# bench.py WORKLOADS
CONFIGS = {
    "configs1": dict(shape=KITTI, n=100_000, c_in=64, c_out=64, dt="f16", subm=True),
    "configs3": dict(shape=[41, 1440, 1440], n=300_000, c_in=64, c_out=128, dt="bf16", subm=False),
}
ENCODER_B8 = dict(shape=KITTI, n=100_000, batch=8)
TORCH_DT = {"f16": torch.float16, "bf16": torch.bfloat16}
SCALE = 0.125                          # grid values are integers in [-2, 2] times SCALE
Q = SCALE * SCALE                      # quantum of every product and partial sum
TILE_ROWS_MULTI_CHUNK = 1024 * 128     # tile_order_kernel ranks 1024 tiles per chunk
SORT_ROWS_MULTI_ROUND = 256 * 1024     # rs_scan_kernel: 256 threads, one 1024-key block each per round


def _cloud(i, shape, n, batch=1):
    return surface_cloud(np.random.default_rng(50051 + i), shape, n, batch=batch)


def _grid(gen, shape, dev):
    """integers in [-2, 2] times SCALE, as float32 on the device"""
    return torch.randint(-2, 3, shape, generator=gen, device=dev).float() * SCALE


def _assert_exact(name, got, ref, ref_abs, q, tdt):
    """got == ref rounded once to tdt, after checking that the comparison is exact: every partial sum of
    every element is a multiple of q below 2^24 q, and ref is 0 or a normal number of tdt."""
    fi = torch.finfo(tdt)
    assert float(ref_abs.max()) < 2.0 ** 24 * q, f"{name}: sum of |terms| {float(ref_abs.max())} reaches 2^24 q"
    a = ref.abs()
    assert bool(((a == 0) | ((a >= fi.tiny) & (a <= fi.max))).all()), f"{name}: reference outside the normal range"
    want = ref.to(tdt)
    assert got.shape == want.shape and got.dtype == tdt, f"{name}: {got.shape} {got.dtype}"
    g = got.reshape(want.shape)
    if not torch.equal(g, want):
        bad = (g != want) | torch.isnan(g)
        rows = bad.reshape(bad.shape[0], -1).any(1).nonzero().squeeze(1)
        idx = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements differ in {len(rows)} rows "
                             f"(first rows {rows[:8].tolist()}); at {idx}: got {float(g[idx])} want {float(want[idx])} "
                             f"(NaN = never written)")


def _check_conv_tables(conv, name):
    """the cached tile tables of a Conv's rulebook against the numpy restatement; returns the rows of
    the largest table"""
    tables = [("fwd", conv.fwd)] + ([("bwd", conv.bwd)] if conv.bwd is not None else [])
    words = (conv.kv + 31) // 32
    rows_max = 0
    for what, (pair, mask, argsort, rows) in tables:
        _, table, tile_mask = argsort._spx_tile_cache
        check_tile_table(table.cpu().numpy(), tile_mask.cpu().numpy(), pair.cpu().numpy(), mask.cpu().numpy(),
                         argsort.cpu().numpy(), rows, conv.kv, words, name=f"{name} {what} tile table")
        rows_max = max(rows_max, rows)
    return rows_max


def _conv_exact(conv, dt, C, K, x, w, dout, what, w_scale=SCALE):
    """fwd, dgrad and wgrad of one Conv on grid inputs (w on a grid of w_scale), each equal to the
    float64 sums rounded once"""
    tdt = TORCH_DT[dt]
    inst = _calls(dt, conv.kv, C, K)
    xd, wd, dd = x.to(tdt), w.to(tdt), dout.to(tdt)
    out = conv.fwd_call(xd, wd, inst["fwd"])
    din = conv.dgrad_call(dd, wd, inst["dgrad"])
    dw = conv.wgrad_call(xd, dd, wd.shape, inst["wgrad"])
    torch.cuda.synchronize()
    r = _reference(x, w, dout, conv.ref_pair, x.device)
    _assert_exact(f"{what} out", out, r["out"], r["out_abs"], SCALE * w_scale, tdt)
    _assert_exact(f"{what} din", din, r["din"], r["din_abs"], SCALE * w_scale, tdt)
    _assert_exact(f"{what} dw", dw.reshape(K, conv.kv, C), r["dw"], r["dw_abs"], Q, tdt)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_layer_workload_exact(name, oracle, cuda_dev):
    """configs[1] (SubM 3^3, 64->64, fp16, 100 k voxels) and configs[3] (stride-2 3^3, 64->128, bf16,
    300 k voxels, and its indice_key-reuse leg: a second layer with W/2 on the same tables)."""
    cfg = CONFIGS[name]
    inds = _cloud(0, cfg["shape"], cfg["n"])
    if cfg["subm"]:
        conv = Conv(oracle, cuda_dev, inds, 1, cfg["shape"], 3, 1, 1, 1, True)
    else:
        conv = Conv(oracle, cuda_dev, inds, 1, cfg["shape"], 3, 2, 1, 1, False)
    rows_max = _check_conv_tables(conv, name)
    if not cfg["subm"]:
        # the backward tables have N = 300 k rows: 2344 tiles, a mask sort of 293 blocks, M != N
        assert conv.n_in != conv.n_out
        assert rows_max > TILE_ROWS_MULTI_CHUNK and conv.n_in > SORT_ROWS_MULTI_ROUND
    C, K, dt = cfg["c_in"], cfg["c_out"], cfg["dt"]
    gen = torch.Generator(device=cuda_dev).manual_seed(1)
    x = _grid(gen, (conv.n_in, C), cuda_dev)
    w = _grid(gen, (K, conv.kv, C), cuda_dev)
    dout = _grid(gen, (conv.n_out, K), cuda_dev)
    _conv_exact(conv, dt, C, K, x, w, dout, name)
    if not cfg["subm"]:
        owners = [conv.fwd[2], conv.bwd[2]]
        cached = [o._spx_tile_cache[1] for o in owners]
        _conv_exact(conv, dt, C, K, x, w * 0.5, dout, f"{name} reuse", w_scale=SCALE / 2)
        assert all(o._spx_tile_cache[1] is t for o, t in zip(owners, cached)), "the reuse leg rebuilt a tile table"


def test_encoder_b8_exact(oracle, cuda_dev):
    """configs[2] as second_encoder6_fp16_b8 (8 samples x 100 k voxels, fp16, MaskImplicitGemm): forward
    and backward through the modules; all five rulebooks against the oracle; then every layer again on
    its own input tensor (its indice_dict included) with fresh grid features, weights and dY, since
    chained activations leave the exact grid."""
    import spconv_b200.pytorch as spconv
    from bench_utils import ENCODER6_LAYERS, make_encoder6
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    shape, batch = ENCODER_B8["shape"], ENCODER_B8["batch"]
    rng = np.random.default_rng(50051)
    inds = surface_cloud(rng, shape, ENCODER_B8["n"], batch=batch)
    feats = rng.uniform(-1, 1, size=(inds.shape[0], 16)).astype(np.float32)
    torch.manual_seed(48848)
    layers = [m.to(cuda_dev).half() for m in make_encoder6(spconv, algo=ConvAlgo.MaskImplicitGemm)]
    for m in layers:
        m.train()
    x0 = spconv.SparseConvTensor(torch.from_numpy(feats).to(cuda_dev).half().requires_grad_(True),
                                 torch.from_numpy(inds).to(cuda_dev), shape, batch)
    acts = [x0]
    for m in layers:
        acts.append(m(acts[-1]))
    acts[-1].features.float().square().mean().backward()
    torch.cuda.synchronize()
    family = 1 if ENV_FAMILY == 1 else 2
    assert ops.last_kernel_family() == family

    # ---- rulebooks: oracle bit for bit, tile tables against numpy
    cur_inds, cur_shape = inds, list(shape)
    ref_pairs, seen, tile_rows, sort_rows = [], {}, 0, 0
    for li, (kind, c_in, c_out, key) in enumerate(ENCODER6_LAYERS):
        subm = kind == "subm"
        st = [1] * 3 if subm else [2] * 3
        datas = acts[li + 1].indice_dict[key]
        if key in seen:
            assert seen[key][0] is datas, f"layer {li}: indice_key {key} was not reused"
            ref_pairs.append(seen[key][1])
            cur_inds, cur_shape = seen[key][2]
            continue
        o_inds, pairs, num = oracle.get_indice_pairs(cur_inds, batch, cur_shape, [3] * 3, st, [1] * 3, [1] * 3,
                                                     [0] * 3, subm)
        n_in, n_out = cur_inds.shape[0], o_inds.shape[0]
        tab = oracle.implicit_gemm_tables(pairs, num, n_in, n_out, subm)
        got = {"out_inds": datas.out_indices, "pair_fwd": datas.pair_fwd, "pair_bwd": datas.pair_bwd,
               "mask_fwd": datas.pair_mask_fwd_splits[0], "argsort_fwd": datas.mask_argsort_fwd_splits[0]}
        want = {"out_inds": o_inds, "pair_fwd": tab["pair_fwd"], "pair_bwd": tab["pair_bwd"],
                "mask_fwd": tab["mask_fwd"], "argsort_fwd": tab["argsort_fwd"]}
        if not subm:
            got.update(mask_bwd=datas.pair_mask_bwd_splits[0], argsort_bwd=datas.mask_argsort_bwd_splits[0])
            want.update(mask_bwd=tab["mask_bwd"], argsort_bwd=tab["argsort_bwd"])
        for what, g in got.items():
            g = g.cpu().numpy()
            w = want[what]
            if what.startswith("mask"):
                g, w = g.view(np.uint32).reshape(-1), w.reshape(-1)
            assert np.array_equal(g, w), f"layer {li} ({key}): {what} differs from the oracle"
        tables = [(datas.pair_fwd, datas.pair_mask_fwd_splits[0], datas.mask_argsort_fwd_splits[0], n_out, "fwd")]
        if not subm:
            tables.append((datas.pair_bwd, datas.pair_mask_bwd_splits[0], datas.mask_argsort_bwd_splits[0], n_in,
                           "bwd"))
        for pair, mask, argsort, rows, what in tables:
            _, table, tile_mask = argsort._spx_tile_cache
            check_tile_table(table.cpu().numpy(), tile_mask.cpu().numpy(), pair.cpu().numpy(), mask.cpu().numpy(),
                             argsort.cpu().numpy(), rows, 27, 1, name=f"layer {li} ({key}) {what} tile table")
            tile_rows = max(tile_rows, rows)
            sort_rows = max(sort_rows, rows)
        cur_shape = cur_shape if subm else oracle.get_conv_output_size(cur_shape, [3] * 3, st, [1] * 3, [1] * 3)
        cur_inds = o_inds
        seen[key] = (datas, tab["pair_fwd"], (cur_inds, cur_shape))
        ref_pairs.append(tab["pair_fwd"])
    assert len(seen) == 5
    assert tile_rows > TILE_ROWS_MULTI_CHUNK and sort_rows > SORT_ROWS_MULTI_ROUND

    # ---- every layer on grid inputs, through the module, on its own input tensor
    gen = torch.Generator(device=cuda_dev).manual_seed(2)
    for li, ((kind, c_in, c_out, key), m) in enumerate(zip(ENCODER6_LAYERS, layers)):
        src = acts[li]
        x = _grid(gen, (src.features.shape[0], c_in), cuda_dev)
        w = _grid(gen, tuple(m.weight.shape), cuda_dev)
        dy = _grid(gen, (acts[li + 1].features.shape[0], c_out), cuda_dev)
        with torch.no_grad():
            m.weight.copy_(w.half())
        m.weight.grad = None
        xin = x.half().requires_grad_(True)
        y = m(src.replace_feature(xin))
        assert torch.equal(y.indices, acts[li + 1].indices), f"layer {li}: output coordinates changed"
        y.features.backward(dy.half())
        torch.cuda.synchronize()
        assert ops.last_kernel_family() == family
        r = _reference(x, w, dy, ref_pairs[li], cuda_dev)
        kv = 27
        _assert_exact(f"layer {li} out", y.features.detach(), r["out"], r["out_abs"], Q, torch.float16)
        _assert_exact(f"layer {li} din", xin.grad, r["din"], r["din_abs"], Q, torch.float16)
        _assert_exact(f"layer {li} dw", m.weight.grad.reshape(c_out, kv, c_in), r["dw"], r["dw_abs"], Q,
                      torch.float16)


# ------------------------------------------------------------------ bench.py's depth-2 pipelined replay
NUM_CLOUDS = 4
ROUNDS = 3


def _scratch_is_zero(res):
    for owner in list(res[6]) + list(res[7]):
        table = owner._spx_tile_cache[1]
        if not bool((table[-64:] == 0).all()):
            return False
    return True


@pytest.mark.parametrize("workload", ["configs1", "configs4"])
def test_pipelined_graph_replay(workload, oracle, cuda_dev):
    """bench.py's `value` schedule: per cloud one rulebook graph and one GEMM graph; the rulebooks run
    two clouds ahead on two side streams, each behind the GEMM graph that last read that cloud's
    rulebook buffers (ge_done), beside the GEMM graph of the current cloud.  Every output is NaN-filled
    (int8: -77) on the main stream before the last round.  configs[1] (training step): every cloud's
    out, din and dW equal the float64 sums rounded once.  configs[4] (int8 inference): every cloud's
    output equals its eager output.  The scheduler scratch is zero after every round."""
    from spconv_b200.core import Activation, ConvAlgo
    from spconv_b200.pytorch import ops
    train = workload == "configs1"
    C = K = 64
    clouds = []
    for i in range(NUM_CLOUDS):
        rng = np.random.default_rng(50051 + i)
        inds = surface_cloud(rng, KITTI, 100_000)
        c = dict(inds=inds, d_inds=torch.from_numpy(inds).to(cuda_dev), n=inds.shape[0])
        if not train:
            c["feats"] = torch.from_numpy(rng.integers(-127, 128, size=(inds.shape[0], C)).astype(np.int8)).to(cuda_dev)
        clouds.append(c)
    if train:
        gen = torch.Generator(device=cuda_dev).manual_seed(3)
        w32 = _grid(gen, (K, 3, 3, 3, C), cuda_dev)
        weight = w32.half()
        for c in clouds:
            c["x32"] = _grid(gen, (c["n"], C), cuda_dev)
            c["d32"] = _grid(gen, (c["n"], K), cuda_dev)
            c["feats"], c["dout"] = c["x32"].half(), c["d32"].half()
    else:
        g = torch.Generator().manual_seed(5)
        weight = torch.randint(-127, 128, (K, 3, 3, 3, C), generator=g, dtype=torch.int8).to(cuda_dev)
        scale = (torch.rand(K, generator=g) * 2e-3 + 1e-4).to(cuda_dev)
        bias = (torch.rand(K, generator=g) - 0.5).to(cuda_dev)

    def rulebook(c):
        return ops.get_indice_pairs_implicit_gemm(c["d_inds"], 1, KITTI, ConvAlgo.MaskImplicitGemm, [3] * 3, [1] * 3,
                                                  [1] * 3, [1] * 3, [0] * 3, True, False, is_train=train)

    def compute(c, res):
        out_inds, _, pf, pb, mf, mb, sf, sb, masks = res
        if not train:
            out, _, _ = ops.implicit_gemm(c["feats"], weight, pf, mf, sf, out_inds.shape[0], masks, False, True,
                                          bias=bias, act_type=Activation.ReLU, scale=scale, output_dtype=torch.int8)
            return (out,)
        out, mask_out, mw = ops.implicit_gemm(c["feats"], weight, pf, mf, sf, out_inds.shape[0], masks, True, True)
        din, dw = ops.implicit_gemm_backward(c["feats"], weight, c["dout"], pf, pb, mf, mb, sf, sb, mask_out, masks,
                                             mw, True)
        return out, din, dw

    # eager: kernels configured before capture; int8 reference outputs
    eager = [tuple(t.clone() for t in compute(c, rulebook(c))) for c in clouds]
    torch.cuda.synchronize()
    rb_graphs, ge_graphs, rb_out, outs = [], [], [], []
    for c in clouds:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            rb_out.append(rulebook(c))
        rb_graphs.append(g)
    for c, res in zip(clouds, rb_out):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            outs.append(compute(c, res))
        ge_graphs.append(g)
    for g in rb_graphs:
        g.replay()
    torch.cuda.synchronize()

    main = torch.cuda.current_stream()
    sides = [torch.cuda.Stream(), torch.cuda.Stream()]
    ge_done = [torch.cuda.Event() for _ in range(NUM_CLOUDS)]

    def step(i):
        j, jn = i % NUM_CLOUDS, (i + 2) % NUM_CLOUDS
        sd = sides[i % 2]
        main.wait_stream(sd)
        sd.wait_event(ge_done[jn])
        with torch.cuda.stream(sd):
            rb_graphs[jn].replay()
        ge_graphs[j].replay()
        ge_done[j].record(main)

    for rnd in range(ROUNDS):
        if rnd == ROUNDS - 1:
            for o in outs:
                for t in o:
                    t.fill_(float("nan") if t.is_floating_point() else -77)
        for i in range(rnd * NUM_CLOUDS, (rnd + 1) * NUM_CLOUDS):
            step(i)
        torch.cuda.synchronize()
        for j, res in enumerate(rb_out):
            assert _scratch_is_zero(res), f"round {rnd}: scheduler scratch of cloud {j} is not zero"

    for j, (c, res, o) in enumerate(zip(clouds, rb_out, outs)):
        if not train:
            assert torch.equal(o[0], eager[j][0]), f"cloud {j}: graph replay differs from the eager int8 output"
            continue
        ref_out, pairs, num = oracle.get_indice_pairs(c["inds"], 1, KITTI, [3] * 3, [1] * 3, [1] * 3, [1] * 3,
                                                      [0] * 3, True)
        tab = oracle.implicit_gemm_tables(pairs, num, c["n"], c["n"], True)
        assert np.array_equal(res[2].cpu().numpy(), tab["pair_fwd"]), f"cloud {j}: replayed pair_fwd"
        assert np.array_equal(res[6][0].cpu().numpy(), tab["argsort_fwd"]), f"cloud {j}: replayed argsort"
        r = _reference(c["x32"], w32, c["d32"], tab["pair_fwd"], cuda_dev)
        out, din, dw = o
        _assert_exact(f"cloud {j} out", out, r["out"], r["out_abs"], Q, torch.float16)
        _assert_exact(f"cloud {j} din", din, r["din"], r["din_abs"], Q, torch.float16)
        _assert_exact(f"cloud {j} dw", dw.reshape(K, 27, C), r["dw"], r["dw_abs"], Q, torch.float16)
