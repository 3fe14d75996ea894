"""GPU conv-arithmetic parity through the operator layer (which calls the C ABI).

Tolerances are the reference's own (test/test_all_algo.py:325-329, :628-643): fp32 exact path
1e-4 abs vs the fp32 oracle (test/test_conv.py:330), fp16 ``||err||_2 < 10*max(C,K)/16`` plus a
rel-L2 <= 1e-2 bound we add; bf16 has no reference kernel ("parity unpinned"): rel-L2 <= 2e-2.
"""
import numpy as np
import pytest
import torch

from tests.util import describe_mismatch, random_cloud, rel_l2, surface_cloud

pytestmark = pytest.mark.gpu

TORCH_DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
REL_TOL = {"f32": 1e-5, "f16": 1e-2, "bf16": 2e-2}


def _round_to(x, dt):
    """values exactly representable in dt, as float32 (so oracle and kernel see the same numbers)"""
    return torch.from_numpy(x).to(TORCH_DT[dt]).float().numpy()


def _setup(oracle, dev, dt, C, K, subm, seed=50005, shape=(19, 18, 17), pts=(1500, 1500),
           ksize=3, stride=2, padding=1, dilation=1):
    rng = np.random.default_rng(seed)
    feats, inds = random_cloud(rng, list(shape), list(pts), C)
    nd = len(shape)
    ks, st, pd, dl = [ksize] * nd, [stride] * nd, [padding] * nd, [dilation] * nd
    w = rng.uniform(-1, 1, size=(K, *ks, C)).astype(np.float32)
    feats, w = _round_to(feats, dt), _round_to(w, dt)
    out_inds, pairs, num = oracle.get_indice_pairs(inds, len(pts), list(shape), ks, st, pd, dl,
                                                   [0] * nd, subm)
    dout = _round_to(rng.uniform(-0.2, 0.2, size=(out_inds.shape[0], K)).astype(np.float32), dt)
    return dict(feats=feats, inds=inds, w=w, out_inds=out_inds, pairs=pairs, num=num, dout=dout,
                ks=ks, st=st, pd=pd, dl=dl, shape=list(shape), bs=len(pts), nd=nd)


def _check(name, got, ref, dt, C, K):
    got = got.float().cpu().numpy() if isinstance(got, torch.Tensor) else got
    msg = describe_mismatch(got, ref, name)
    assert not np.isnan(got).any(), msg
    r = rel_l2(got, ref)
    assert r <= REL_TOL[dt], msg
    if dt == "f16":
        assert np.linalg.norm(got - ref) < 10 * max(C, K) / 16 * max(1.0, np.sqrt(ref.shape[0] / 1500)), msg
    if dt == "f32":
        assert np.abs(got - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max()), msg


SHAPES = [(16, 16), (16, 32), (32, 32), (32, 64), (64, 64), (64, 128), (128, 128), (128, 64),
          (3, 16), (48, 24)]


@pytest.mark.parametrize("subm", [True, False], ids=["subm", "conv"])
@pytest.mark.parametrize("dt", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("CK", SHAPES, ids=lambda ck: f"C{ck[0]}K{ck[1]}")
def test_implicit_gemm_fwd_bwd(CK, dt, subm, oracle, cuda_dev):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    C, K = CK
    s = _setup(oracle, cuda_dev, dt, C, K, subm)
    tdt = TORCH_DT[dt]
    inds = torch.from_numpy(s["inds"]).to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(inds, s["bs"], s["shape"], ConvAlgo.MaskImplicitGemm,
                                             s["ks"], s["st"], s["pd"], s["dl"], [0] * s["nd"],
                                             subm, False, is_train=True)
    out_inds, _, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks = res
    assert np.array_equal(out_inds.cpu().numpy(), s["out_inds"])
    x = torch.from_numpy(s["feats"]).to(cuda_dev, tdt)
    w = torch.from_numpy(s["w"]).to(cuda_dev, tdt)
    dout = torch.from_numpy(s["dout"]).to(cuda_dev, tdt)
    m = out_inds.shape[0]
    out, mask_out, mask_width = ops.implicit_gemm(x, w, pair_fwd, mask_fwd, sort_fwd, m, masks,
                                                  True, subm)
    fam_fwd = ops.last_kernel_family()
    din, dw = ops.implicit_gemm_backward(x, w, dout, pair_fwd, pair_bwd, mask_fwd, mask_bwd,
                                         sort_fwd, sort_bwd, mask_out, masks, mask_width, subm)
    torch.cuda.synchronize()
    ref_out = oracle.indice_conv(s["feats"], s["w"], s["pairs"], s["num"], m, False, subm)
    ref_din, ref_dw = oracle.indice_conv_backward(s["feats"], s["w"], s["dout"], s["pairs"],
                                                  s["num"], False, subm)
    tc_expected = dt != "f32" and C % 16 == 0 and K % 16 == 0 and C != 48
    import os
    if tc_expected and os.environ.get('SPX_FORCE_SIMT') != '1':
        assert fam_fwd == 2, f"expected the tensor-core kernels for {dt} C{C} K{K}, family={fam_fwd}"
    assert mask_width == 128
    # mask_output_fwd = per-128-row OR of the sorted masks
    mo = mask_out.cpu().numpy().view(np.uint32)[0, :, 0]
    ms = mask_fwd[0].cpu().numpy().view(np.uint32)[:, 0]
    ref_mo = np.array([np.bitwise_or.reduce(ms[i:i + 128]) for i in range(0, m, 128)], np.uint32)
    assert np.array_equal(mo, ref_mo)
    _check("out", out, ref_out, dt, C, K)
    _check("din", din, ref_din, dt, C, K)
    _check("dw", dw.reshape(K, -1), ref_dw.reshape(K, -1), dt, C, K)


@pytest.mark.parametrize("subm", [True, False], ids=["subm", "conv"])
@pytest.mark.parametrize("dt", ["f32", "f16"])
def test_native_indice_conv(dt, subm, oracle, cuda_dev):
    """ConvAlgo.Native operator path on oracle-order rulebooks (config 1 shape: C=K=16)."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    C = K = 16
    s = _setup(oracle, cuda_dev, dt, C, K, subm, seed=484, shape=(64, 64, 64), pts=(5000,),
               stride=1 if subm else 2)
    tdt = TORCH_DT[dt]
    inds = torch.from_numpy(s["inds"]).to(cuda_dev)
    out_inds, pairs, num = ops.get_indice_pairs(inds, 1, s["shape"], ConvAlgo.Native, s["ks"],
                                                s["st"], s["pd"], s["dl"], [0] * 3, subm)
    assert np.array_equal(pairs.cpu().numpy(), s["pairs"])
    x = torch.from_numpy(s["feats"]).to(cuda_dev, tdt)
    w = torch.from_numpy(s["w"]).to(cuda_dev, tdt)
    dout = torch.from_numpy(s["dout"]).to(cuda_dev, tdt)
    m = out_inds.shape[0]
    out = ops.indice_conv(x, w, pairs, num, m, False, subm)
    din, dw = ops.indice_conv_backward(x, w, dout, pairs, num, False, subm)
    ref_out = oracle.indice_conv(s["feats"], s["w"], s["pairs"], s["num"], m, False, subm)
    ref_din, ref_dw = oracle.indice_conv_backward(s["feats"], s["w"], s["dout"], s["pairs"],
                                                  s["num"], False, subm)
    _check("out", out, ref_out, dt, C, K)
    _check("din", din, ref_din, dt, C, K)
    _check("dw", dw.reshape(K, -1), ref_dw.reshape(K, -1), dt, C, K)
    if not subm:
        # inverse conv: swap the roles of the two pair rows (convops.py:1604-1605)
        xi = torch.from_numpy(s["dout"]).to(cuda_dev, tdt)       # [M, K] features on the outputs
        wi = torch.from_numpy(_round_to(np.random.default_rng(3).uniform(-1, 1, size=(C, 3, 3, 3, K)).astype(np.float32), dt)).to(cuda_dev, tdt)
        got = ops.indice_conv(xi, wi, pairs, num, s["feats"].shape[0], True, False)
        ref = oracle.indice_conv(s["dout"], wi.float().cpu().numpy(), s["pairs"], s["num"],
                                 s["feats"].shape[0], True, False)
        _check("inverse_out", got, ref, dt, C, K)


@pytest.mark.parametrize("act", ["relu", "leaky_relu", "sigmoid"])
def test_fused_bias_act_epilogue(act, oracle, cuda_dev):
    from spconv_b200.core import Activation, ConvAlgo
    from spconv_b200.pytorch import ops
    dt, C, K = "f16", 32, 64
    s = _setup(oracle, cuda_dev, dt, C, K, True, stride=1)
    inds = torch.from_numpy(s["inds"]).to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(inds, s["bs"], s["shape"], ConvAlgo.MaskImplicitGemm,
                                             s["ks"], s["st"], s["pd"], s["dl"], [0] * 3, True,
                                             False, is_train=False)
    x = torch.from_numpy(s["feats"]).to(cuda_dev, torch.float16)
    w = torch.from_numpy(s["w"]).to(cuda_dev, torch.float16)
    bias_np = _round_to(np.random.default_rng(5).uniform(-1, 1, size=(K,)).astype(np.float32), dt)
    bias = torch.from_numpy(bias_np).to(cuda_dev, torch.float16)
    code = {"relu": Activation.ReLU, "leaky_relu": Activation.LeakyReLU, "sigmoid": Activation.Sigmoid}[act]
    out, _, _ = ops.implicit_gemm(x, w, res[2], res[4], res[6], x.shape[0], res[8], False, True,
                                  bias=bias, act_alpha=0.1, act_type=code)
    ref = oracle.indice_conv(s["feats"], s["w"], s["pairs"], s["num"], x.shape[0], False, True,
                             bias=bias_np, act=act, act_alpha=0.1)
    _check("out", out, ref, dt, C, K)
    # standalone epilogue op (Native-algo path of the reference, inference.py:166-252)
    raw, _, _ = ops.implicit_gemm(x, w, res[2], res[4], res[6], x.shape[0], res[8], False, True)
    got = ops.bias_add_act_inplace(raw.clone(), bias, code, 0.1)
    _check("bias_act_inplace", got, ref, dt, C, K)


def test_tf32_mode_forward(oracle, cuda_dev, monkeypatch):
    """fp32 features on the tensor cores (SPCONV_ALLOW_TF32): tolerance 1e-2 (test_all_algo.py:325)."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", True)
    C, K = 32, 64
    s = _setup(oracle, cuda_dev, "f32", C, K, True, stride=1)
    inds = torch.from_numpy(s["inds"]).to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(inds, s["bs"], s["shape"], ConvAlgo.MaskImplicitGemm,
                                             s["ks"], s["st"], s["pd"], s["dl"], [0] * 3, True)
    x = torch.from_numpy(s["feats"]).to(cuda_dev)
    w = torch.from_numpy(s["w"]).to(cuda_dev)
    out, _, _ = ops.implicit_gemm(x, w, res[2], res[4], res[6], x.shape[0], res[8], True, True)
    import os
    if os.environ.get('SPX_FORCE_SIMT') != '1':
        assert ops.last_kernel_family() == 2
    ref = oracle.indice_conv(s["feats"], s["w"], s["pairs"], s["num"], x.shape[0], False, True)
    got = out.cpu().numpy()
    assert rel_l2(got, ref) < 2e-3, describe_mismatch(got, ref, "tf32 out")


def test_empty_and_tiny_inputs(oracle, cuda_dev):
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    # a single voxel: only the centre offset
    inds = torch.tensor([[0, 3, 3, 3]], dtype=torch.int32, device=cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(inds, 1, [8, 8, 8], ConvAlgo.MaskImplicitGemm, [3] * 3,
                                             [1] * 3, [1] * 3, [1] * 3, [0] * 3, True)
    x = torch.ones((1, 16), dtype=torch.float16, device=cuda_dev)
    w = torch.randn((32, 3, 3, 3, 16), dtype=torch.float16, device=cuda_dev)
    out, _, _ = ops.implicit_gemm(x, w, res[2], res[4], res[6], 1, res[8], True, True)
    ref = (x.float() @ w[:, 1, 1, 1, :].float().t())
    assert torch.allclose(out.float(), ref, atol=2e-2, rtol=1e-2)
    # 129 voxels in a line: tile boundary (128 + 1 rows)
    coords = torch.zeros((129, 4), dtype=torch.int32)
    coords[:, 3] = torch.arange(129)
    inds = coords.to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(inds, 1, [4, 4, 200], ConvAlgo.MaskImplicitGemm, [3] * 3,
                                             [1] * 3, [1] * 3, [1] * 3, [0] * 3, True)
    x = torch.randn((129, 64), dtype=torch.float16, device=cuda_dev)
    w = torch.randn((64, 3, 3, 3, 64), dtype=torch.float16, device=cuda_dev) * 0.1
    out, mo, mw = ops.implicit_gemm(x, w, res[2], res[4], res[6], 129, res[8], True, True)
    o_pairs = oracle.get_indice_pairs(coords.numpy(), 1, [4, 4, 200], [3] * 3, [1] * 3, [1] * 3,
                                      [1] * 3, [0] * 3, True)
    ref = oracle.indice_conv(x.float().cpu().numpy(), w.float().cpu().numpy(), o_pairs[1],
                             o_pairs[2], 129, False, True)
    assert rel_l2(out.float().cpu().numpy(), ref) < 1e-2


@pytest.mark.parametrize("subm", [True, False], ids=["subm", "conv"])
@pytest.mark.parametrize("CK", [(64, 64), (32, 64), (16, 16)], ids=lambda ck: f"C{ck[0]}K{ck[1]}")
@pytest.mark.parametrize("out_int8", [True, False], ids=["q8", "f32out"])
def test_int8_inference_forward(CK, subm, out_int8, oracle, cuda_dev):
    """int8 x int8 -> int32 accumulate -> per-channel scale + bias (+ residual) -> act ->
    clip(round()) : exact match with the numpy formula of test/test_all_algo.py:222-287
    (inputs randint(-1,1)-style small integers, scales U(0.5,1.5), output_add_scale 14.2)."""
    import os
    from spconv_b200.core import Activation, ConvAlgo
    from spconv_b200.pytorch import ops
    C, K = CK
    rng = np.random.default_rng(50005)
    shape = [19, 18, 17]
    _, inds = random_cloud(rng, shape, [1500, 1500], 1)
    ks, st, pd, dl = [3] * 3, [1 if subm else 2] * 3, [1] * 3, [1] * 3
    x = rng.integers(-4, 4, size=(inds.shape[0], C)).astype(np.int8)
    w = rng.integers(-4, 4, size=(K, 3, 3, 3, C)).astype(np.int8)
    out_inds, pairs, num = oracle.get_indice_pairs(inds, 2, shape, ks, st, pd, dl, [0] * 3, subm)
    m = out_inds.shape[0]
    scales = rng.uniform(0.5, 1.5, size=K).astype(np.float32) * 0.05
    bias = rng.uniform(-5, 5, size=K).astype(np.float32)
    add = rng.integers(-2, 2, size=(m, K)).astype(np.int8)
    output_scale, add_scale = 3.4, 14.2 * 0.1
    ref = oracle.int8_conv_forward(x, w, pairs, num, m, subm, scales, bias, add,
                                   np.float32(add_scale) / np.float32(output_scale), relu=True,
                                   out_int8=out_int8)
    d_inds = torch.from_numpy(inds).to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(d_inds, 2, shape, ConvAlgo.MaskImplicitGemm, ks, st, pd, dl,
                                             [0] * 3, subm, False, is_train=False)
    assert np.array_equal(res[0].cpu().numpy(), out_inds)
    out, _, _ = ops.implicit_gemm(torch.from_numpy(x).to(cuda_dev), torch.from_numpy(w).to(cuda_dev), res[2],
                                  res[4], res[6], m, res[8], False, subm, bias=torch.from_numpy(bias).to(cuda_dev),
                                  act_type=Activation.ReLU, output_scale=output_scale,
                                  scale=torch.from_numpy(scales).to(cuda_dev),
                                  output_add=torch.from_numpy(add).to(cuda_dev), output_add_scale=add_scale,
                                  output_dtype=torch.int8 if out_int8 else torch.float32)
    got = out.cpu().numpy()
    if C % 32 == 0 and K % 32 == 0 and os.environ.get("SPX_FORCE_SIMT") != "1":
        assert ops.last_kernel_family() == 2, "int8 wgmma (s8) path expected"   # docs/INT8_GUIDE.md:10
    if out_int8:
        # fp32 evaluation order can differ by 1 ulp exactly at .5 ties: allow off-by-one there only
        diff = np.abs(got.astype(np.int32) - ref.astype(np.int32))
        assert diff.max() <= 1 and (diff > 0).mean() < 1e-3, (diff.max(), (diff > 0).mean())
    else:
        assert np.abs(got - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())


def test_dynamic_scheduler_leaves_state_clean_and_is_repeatable(cuda_dev):
    """The tensor-core forward / input-gradient kernels draw tiles from an atomic ticket counter that
    lives behind the tile table; every launch must leave it zeroed (the last CTA resets it), and
    repeated launches must give bit-identical results whatever CTA ran which tile."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(11)
    shape = [24, 400, 352]
    inds = torch.from_numpy(surface_cloud(rng, shape, 40000)).to(cuda_dev)
    n = inds.shape[0]
    res = ops.get_indice_pairs_implicit_gemm(inds, 1, shape, ConvAlgo.MaskImplicitGemm, [3] * 3, [1] * 3,
                                             [1] * 3, [1] * 3, [0] * 3, True, False, is_train=True)
    _, _, pf, pb, mf, mb, sf, sb, masks = res
    g = torch.Generator(device=cuda_dev).manual_seed(3)
    x = (torch.rand((n, 64), device=cuda_dev, generator=g) - 0.5).half()
    w = ((torch.rand((64, 3, 3, 3, 64), device=cuda_dev, generator=g) - 0.5) * 0.2).half()
    dout = (torch.rand((n, 64), device=cuda_dev, generator=g) - 0.5).half()
    outs, dins = [], []
    for _ in range(5):
        out, mask_out, mw = ops.implicit_gemm(x, w, pf, mf, sf, n, masks, True, True)
        din, dw = ops.implicit_gemm_backward(x, w, dout, pf, pb, mf, mb, sf, sb, mask_out, masks, mw, True)
        outs.append(out); dins.append(din)
    torch.cuda.synchronize()
    table = sf[0]._spx_tile_cache[1]
    assert (table[-64:] == 0).all(), "scheduler scratch must be zero between launches"
    for o, d in zip(outs[1:], dins[1:]):
        assert torch.equal(o, outs[0]) and torch.equal(d, dins[0])


def test_graph_captured_backward_branches_match_eager(cuda_dev):
    """Under CUDA-graph capture implicit_gemm_backward puts the input gradient on a forked stream
    next to the weight gradient (two parallel graph branches).  Replays must give exactly what the
    sequential eager calls give, replay after replay."""
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    rng = np.random.default_rng(17)
    shape = [24, 400, 352]
    inds = torch.from_numpy(surface_cloud(rng, shape, 30000)).to(cuda_dev)
    n = inds.shape[0]
    g = torch.Generator(device=cuda_dev).manual_seed(9)
    x = (torch.rand((n, 64), device=cuda_dev, generator=g) - 0.5).half()
    w = ((torch.rand((64, 3, 3, 3, 64), device=cuda_dev, generator=g) - 0.5) * 0.2).half()
    dout = (torch.rand((n, 64), device=cuda_dev, generator=g) - 0.5).half()

    def step():
        res = ops.get_indice_pairs_implicit_gemm(inds, 1, shape, ConvAlgo.MaskImplicitGemm, [3] * 3, [1] * 3,
                                                 [1] * 3, [1] * 3, [0] * 3, True, False, is_train=True)
        _, _, pf, pb, mf, mb, sf, sb, masks = res
        out, mask_out, mw = ops.implicit_gemm(x, w, pf, mf, sf, n, masks, True, True)
        din, dw = ops.implicit_gemm_backward(x, w, dout, pf, pb, mf, mb, sf, sb, mask_out, masks, mw, True)
        return out, din, dw

    for _ in range(2):
        eager = step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for _ in range(3):
        for t in captured:
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for got, ref, name in zip(captured, eager, ("out", "din", "dw")):
            assert torch.equal(got, ref), f"{name} differs between graph replay and eager"


def test_int8_forward_at_config5_size(oracle, cuda_dev):
    """BASELINE configs[4] at its stated size: int8 SubMConv3d 3x3x3 C = K = 64 over a ~100 k-voxel
    KITTI-shaped cloud, per-channel scale + bias + ReLU + clip, exact against the numpy formula
    (test/test_all_algo.py:272-287) apart from rint ties."""
    from spconv_b200.core import Activation, ConvAlgo
    from spconv_b200.pytorch import ops
    from tests.util import surface_cloud
    rng = np.random.default_rng(50051)
    shape = [41, 1600, 1408]
    inds = surface_cloud(rng, shape, 100_000)
    C = K = 64
    x = rng.integers(-127, 128, size=(inds.shape[0], C)).astype(np.int8)
    w = rng.integers(-127, 128, size=(K, 3, 3, 3, C)).astype(np.int8)
    out_inds, pairs, num = oracle.get_indice_pairs(inds, 1, shape, [3] * 3, [1] * 3, [1] * 3, [1] * 3, [0] * 3, True)
    scales = (rng.uniform(0.5, 1.5, size=K) * 2e-4).astype(np.float32)       # per-channel
    bias = rng.uniform(-5, 5, size=K).astype(np.float32)
    ref = oracle.int8_conv_forward(x, w, pairs, num, inds.shape[0], True, scales, bias, relu=True, out_int8=True)
    d_inds = torch.from_numpy(inds).to(cuda_dev)
    res = ops.get_indice_pairs_implicit_gemm(d_inds, 1, shape, ConvAlgo.MaskImplicitGemm, [3] * 3, [1] * 3, [1] * 3,
                                             [1] * 3, [0] * 3, True, False, is_train=False)
    out, _, _ = ops.implicit_gemm(torch.from_numpy(x).to(cuda_dev), torch.from_numpy(w).to(cuda_dev), res[2], res[4],
                                  res[6], inds.shape[0], res[8], False, True, bias=torch.from_numpy(bias).to(cuda_dev),
                                  act_type=Activation.ReLU, scale=torch.from_numpy(scales).to(cuda_dev),
                                  output_dtype=torch.int8)
    import os
    if os.environ.get("SPX_FORCE_SIMT") != "1":
        assert ops.last_kernel_family() == 2, "int8 wgmma (s8) path expected"
    got = out.cpu().numpy()
    assert 0.05 < (got > 0).mean() < 0.95 and got.max() == 127            # the clip and the ReLU are both exercised
    diff = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    assert diff.max() <= 1 and (diff > 0).mean() < 1e-3, (diff.max(), (diff > 0).mean())


def test_tf32_gradients_on_tensor_cores(oracle, cuda_dev, monkeypatch):
    """fp32 + SPCONV_ALLOW_TF32: input gradient (tf32 wgmma, filter slice written transposed into a K-major operand)
    and weight gradient (both operands transposed into K-major tf32 while they are gathered) run
    on the tensor cores and match the fp32 oracle to tf32 accuracy; spx_debug_configure bits 256 / 4096 route them back to
    the FMA kernels."""
    from spconv_b200 import _cabi
    from spconv_b200.core import ConvAlgo
    from spconv_b200.pytorch import ops
    monkeypatch.setattr(ops, "SPCONV_ALLOW_TF32", True)
    lib = _cabi.load()
    try:
        for C, K, subm in ((32, 64, True), (64, 64, True), (64, 32, False), (32, 32, True)):
            s = _setup(oracle, cuda_dev, "f32", C, K, subm, stride=1 if subm else 2)
            inds = torch.from_numpy(s["inds"]).to(cuda_dev)
            res = ops.get_indice_pairs_implicit_gemm(inds, s["bs"], s["shape"], ConvAlgo.MaskImplicitGemm, s["ks"], s["st"],
                                                     s["pd"], s["dl"], [0] * 3, subm, False, is_train=True)
            m = res[0].shape[0]
            x = torch.from_numpy(s["feats"]).to(cuda_dev)
            w = torch.from_numpy(s["w"]).to(cuda_dev)
            rng = np.random.default_rng(3)
            dout = rng.uniform(-1, 1, size=(m, K)).astype(np.float32)
            args = (x, w, torch.from_numpy(dout).to(cuda_dev), res[2], res[3], res[4], res[5], res[6], res[7], None, res[8],
                    128, subm)
            ref_din, ref_dw = oracle.indice_conv_backward(s["feats"], s["w"], dout, s["pairs"], s["num"], False, subm)
            # every kernel forced onto the tensor cores: a shape it does not serve would raise
            _cabi.check(lib.spx_debug_configure(2, 0, 0, None, 0), "debug_configure")
            din, dw = ops.implicit_gemm_backward(*args)
            assert rel_l2(din.cpu().numpy(), ref_din) < 2e-3, describe_mismatch(din.cpu().numpy(), ref_din, f"tf32 din C{C}K{K}")
            assert rel_l2(dw.cpu().numpy(), ref_dw) < 2e-3, describe_mismatch(dw.cpu().numpy(), ref_dw, f"tf32 dw C{C}K{K}")
            # the off switches are honoured: with the family still forced, the refused kernel raises
            _cabi.check(lib.spx_debug_configure(2, 0, 256, None, 0), "debug_configure")
            with pytest.raises(RuntimeError, match="tensor-core path does not support"):
                ops.implicit_gemm_backward(*args)
            _cabi.check(lib.spx_debug_configure(2, 0, 4096, None, 0), "debug_configure")
            with pytest.raises(RuntimeError, match="tensor-core wgrad"):
                ops.implicit_gemm_backward(*args)
            # the FMA route gives the same answer to tf32 accuracy
            _cabi.check(lib.spx_debug_configure(0, 0, 256 | 4096, None, 0), "debug_configure")
            din_fma, dw_fma = ops.implicit_gemm_backward(*args)
            assert rel_l2(din.cpu().numpy(), din_fma.cpu().numpy()) < 2e-3
            assert rel_l2(dw.cpu().numpy(), dw_fma.cpu().numpy()) < 2e-3
    finally:
        # back to what the environment pinned (SPX_FORCE_SIMT / SPX_FORCE_TC), not to automatic dispatch
        import os
        env_family = (1 if os.environ.get("SPX_FORCE_SIMT", "").startswith("1")
                      else 2 if os.environ.get("SPX_FORCE_TC", "").startswith("1") else 0)
        _cabi.check(lib.spx_debug_configure(env_family, 0, 0, None, 0), "debug_configure")
