"""Checks of the float64 sparse-conv reference (tests/conv_ref.py) itself, without a GPU.

1-D to 3-D: against dense float64 torch convolutions on scattered inputs.  The output set must be the
support of the dense result, the values must agree there, and the dense result must be exactly 0
everywhere else.  4-D: a sum over the first axis's taps of 3-D convolutions.  Rulebooks: the reference's
pairs equal the oracle's, as sets, on every geometry the GPU module and rulebook-edge tests use.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.conv_ref import SparseConvRef, offset_taps
from tests.util import random_cloud

CONV = {1: F.conv1d, 2: F.conv2d, 3: F.conv3d}
CONV_T = {1: F.conv_transpose1d, 2: F.conv_transpose2d, 3: F.conv_transpose3d}


def _dense(inds, feats, shape, bs):
    x = torch.zeros((bs, feats.shape[1], *shape), dtype=torch.float64)
    x[(inds[:, 0], slice(None), *[inds[:, a + 1] for a in range(len(shape))])] = torch.from_numpy(feats).double()
    return x


def _at(dense, coords):
    """[rows, K] values of dense [B, K, *dims] at coords [rows, 1 + ndim]"""
    idx = (torch.from_numpy(coords[:, 0].astype(np.int64)), slice(None),
           *[torch.from_numpy(coords[:, a + 1].astype(np.int64)) for a in range(coords.shape[1] - 1)])
    return dense[idx].numpy()


def _torch_w(w):
    """KRSC [K, *k, C] -> torch conv weight [K, C, *k]"""
    nd = w.ndim - 2
    return torch.from_numpy(w).double().permute(0, nd + 1, *range(1, nd + 1)).contiguous()


def _support(dense):
    return np.stack(np.nonzero(dense.abs().sum(1).numpy() > 0), -1)


def _check_against_dense(ref, got_dense, ones_dense, out_shape, x, w):
    """ref's output set == support of ones_dense; values agree; got_dense is 0 off the set"""
    sup = _support(ones_dense)
    want = set(map(tuple, sup.tolist()))
    have = set(map(tuple, ref.out_inds.tolist()))
    assert have == want, (len(have), len(want))
    out, _, _ = ref.forward(x, w)
    np.testing.assert_allclose(out, _at(got_dense, ref.out_inds), rtol=1e-12, atol=1e-12)
    off = np.ones(got_dense.shape[:1] + got_dense.shape[2:], bool)
    off[tuple(ref.out_inds[:, a] for a in range(ref.out_inds.shape[1]))] = False
    assert (got_dense.permute(0, *range(2, got_dense.dim()), 1).numpy()[off] == 0).all()
    assert list(got_dense.shape[2:]) == list(out_shape)


def _case_data(shape, pts, C, K, ksize, seed):
    rng = np.random.default_rng(seed)
    feats, inds = random_cloud(rng, shape, pts, C, dtype=np.float64)
    w = rng.uniform(-1, 1, size=(K, *ksize, C))
    return inds, feats, w


DENSE_CASES = [
    # ndim, shape, pts, ksize, stride, padding, dilation, output_padding
    (1, [60], [20, 15], [3], [2], [1], [1], [1]),
    (1, [70], [25], [4], [3], [1], [2], [0]),
    (2, [13, 11], [30, 20], [3, 2], [2, 1], [1, 0], [1, 1], [1, 0]),
    (2, [12, 14], [35], [3, 3], [2, 3], [0, 1], [2, 1], [0, 2]),
    (3, [9, 8, 7], [40, 30], [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1], [1, 0, 1]),
    (3, [9, 10, 8], [50], [2, 3, 1], [2, 1, 1], [0, 1, 0], [1, 2, 1], [0, 0, 0]),
]


@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: f"{c[0]}d-k{c[3]}s{c[4]}")
def test_regular_conv_equals_dense(case):
    nd, shape, pts, ksize, stride, padding, dilation, _ = case
    inds, feats, w = _case_data(shape, pts, 3, 4, ksize, 1)
    ref = SparseConvRef(inds, len(pts), shape, ksize, stride, padding, dilation, kind="conv")
    x = _dense(inds, feats, shape, len(pts))
    got = CONV[nd](x, _torch_w(w), stride=stride, padding=padding, dilation=dilation)
    ones = CONV[nd]((x.abs().sum(1, keepdim=True) > 0).double(), torch.ones((1, 1, *ksize), dtype=torch.float64),
                    stride=stride, padding=padding, dilation=dilation)
    _check_against_dense(ref, got, ones, ref.out_shape, feats, w)


@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: f"{c[0]}d-k{c[3]}s{c[4]}op{c[7]}")
def test_transposed_conv_equals_dense(case):
    """torch's transposed grid counts dilation, the reference's does not: the dense result is cropped to
    the reference's grid, and the taps beyond it are the ones the reference drops."""
    nd, shape, pts, ksize, stride, padding, dilation, op = case
    op = [min(o, max(s, d) - 1) for o, s, d in zip(op, stride, dilation)]
    inds, feats, w = _case_data(shape, pts, 3, 4, ksize, 2)
    ref = SparseConvRef(inds, len(pts), shape, ksize, stride, padding, dilation, op, kind="transpose")
    x = _dense(inds, feats, shape, len(pts))
    wt = torch.from_numpy(w).double().permute(nd + 1, 0, *range(1, nd + 1)).contiguous()     # [C, K, *k]
    got = CONV_T[nd](x, wt, stride=stride, padding=padding, output_padding=op, dilation=dilation)
    ones = CONV_T[nd]((x.abs().sum(1, keepdim=True) > 0).double(), torch.ones((1, 1, *ksize), dtype=torch.float64),
                      stride=stride, padding=padding, output_padding=op, dilation=dilation)
    crop = (slice(None), slice(None), *[slice(0, o) for o in ref.out_shape])
    full = [int(v) for v in got.shape[2:]]
    assert all(f >= o for f, o in zip(full, ref.out_shape)) and (full == ref.out_shape) == (max(dilation) == 1)
    _check_against_dense(ref, got[crop], ones[crop], ref.out_shape, feats, w)


@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: f"{c[0]}d-k{c[3]}d{c[6]}")
def test_subm_equals_dense_on_active_set(case):
    nd, shape, pts, ksize, _, _, dilation, _ = case
    ksize = [k | 1 for k in ksize]
    inds, feats, w = _case_data(shape, pts, 3, 4, ksize, 3)
    ref = SparseConvRef(inds, len(pts), shape, ksize, [1] * nd, [0] * nd, dilation, kind="subm")
    assert np.array_equal(ref.out_inds, inds)
    x = _dense(inds, feats, shape, len(pts))
    pad = [(k // 2) * d for k, d in zip(ksize, dilation)]
    got = CONV[nd](x, _torch_w(w), padding=pad, dilation=dilation)
    out, _, _ = ref.forward(feats, w)
    np.testing.assert_allclose(out, _at(got, inds), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: f"{c[0]}d-k{c[3]}s{c[4]}")
def test_inverse_equals_dense_transpose_of_the_paired_output(case):
    nd, shape, pts, ksize, stride, padding, dilation, _ = case
    inds, _, w = _case_data(shape, pts, 3, 4, ksize, 4)
    fwd = SparseConvRef(inds, len(pts), shape, ksize, stride, padding, dilation, kind="conv")
    inv = SparseConvRef(inds, len(pts), shape, ksize, stride, padding, dilation, kind="inverse")
    assert np.array_equal(inv.in_inds, fwd.out_inds) and np.array_equal(inv.out_inds, inds)
    rng = np.random.default_rng(5)
    mid = rng.uniform(-1, 1, size=(fwd.n_out, 4))
    w_inv = rng.uniform(-1, 1, size=(3, *ksize, 4))
    x = _dense(fwd.out_inds, mid, fwd.out_shape, len(pts))
    wt = torch.from_numpy(w_inv).double().permute(nd + 1, 0, *range(1, nd + 1)).contiguous()
    plain = CONV_T[nd](x, wt, stride=stride, padding=padding, dilation=dilation)
    op = [max(0, i - int(g)) for i, g in zip(shape, plain.shape[2:])]
    got = CONV_T[nd](x, wt, stride=stride, padding=padding, output_padding=op, dilation=dilation)
    got = got[(slice(None), slice(None), *[slice(0, i) for i in shape])]
    out, _, _ = inv.forward(mid, w_inv)
    np.testing.assert_allclose(out, _at(got, inds), rtol=1e-12, atol=1e-12)


def _conv4d_dense(x, w, stride, padding, dilation):
    """4-D conv as a sum over the first axis's taps of 3-D convs; x [B, C, D0..D3], w KRSC [K, k0..k3, C]"""
    k0 = w.shape[1]
    xp = F.pad(x, (0, 0, 0, 0, 0, 0, padding[0], padding[0]))
    out0 = (x.shape[2] + 2 * padding[0] - dilation[0] * (k0 - 1) - 1) // stride[0] + 1
    res = None
    for o in range(out0):
        acc = None
        for r in range(k0):
            sl = xp[:, :, o * stride[0] + r * dilation[0]]
            y = F.conv3d(sl, _torch_w(np.ascontiguousarray(w[:, r])), stride=stride[1:], padding=padding[1:],
                         dilation=dilation[1:])
            acc = y if acc is None else acc + y
        res = acc[:, :, None] if res is None else torch.cat([res, acc[:, :, None]], 2)
    return res


@pytest.mark.parametrize("ksize,stride,padding,dilation", [([3] * 4, [2] * 4, [1] * 4, [1] * 4),
                                                           ([2, 3, 1, 3], [2, 1, 1, 2], [0, 1, 0, 1], [1, 1, 1, 2])])
def test_4d_conv_equals_sum_of_3d_convs(ksize, stride, padding, dilation):
    shape = [6, 7, 5, 6]
    inds, feats, w = _case_data(shape, [60, 40], 3, 4, ksize, 6)
    ref = SparseConvRef(inds, 2, shape, ksize, stride, padding, dilation, kind="conv")
    x = _dense(inds, feats, shape, 2)
    got = _conv4d_dense(x, w, stride, padding, dilation)
    ones = _conv4d_dense((x.abs().sum(1, keepdim=True) > 0).double(), np.ones((1, *ksize, 1)), stride, padding,
                         dilation)
    _check_against_dense(ref, got, ones, ref.out_shape, feats, w)
    sub = SparseConvRef(inds, 2, shape, [3] * 4, [1] * 4, [0] * 4, [1] * 4, kind="subm")
    w3 = np.random.default_rng(8).uniform(-1, 1, size=(4, 3, 3, 3, 3, 3))
    out, _, _ = sub.forward(feats, w3)
    np.testing.assert_allclose(out, _at(_conv4d_dense(x, w3, [1] * 4, [1] * 4, [1] * 4), inds), rtol=1e-12, atol=1e-12)


def test_gradients_are_the_adjoint_of_forward():
    """<dY, conv(x)> == <dX, x> and == <dW, W> for every kind (the forward is bilinear in x and W)"""
    rng = np.random.default_rng(7)
    shape = [9, 8, 7]
    _, inds = random_cloud(rng, shape, [60, 50], 1)
    for kind, ks, s, p, d in [("conv", [3, 2, 3], [2, 1, 2], [1, 0, 1], [1, 1, 2]), ("transpose", [3] * 3, [2] * 3,
                              [1] * 3, [2] * 3), ("subm", [3] * 3, [1] * 3, [0] * 3, [1] * 3),
                              ("inverse", [3] * 3, [2] * 3, [1] * 3, [1] * 3)]:
        ref = SparseConvRef(inds, 2, shape, ks, s, p, d, [1] * 3 if kind == "transpose" else None, kind)
        x = rng.uniform(-1, 1, (ref.n_in, 3))
        w = rng.uniform(-1, 1, (4, *ks, 3))
        dy = rng.uniform(-1, 1, (ref.n_out, 4))
        y, _, _ = ref.forward(x, w)
        dx, _, _, dw, _, _ = ref.backward(x, w, dy)
        e = float((dy * y).sum())
        assert abs(e - float((dx * x).sum())) < 1e-9 * max(1, abs(e)), kind
        assert abs(e - float((dw * w).sum())) < 1e-9 * max(1, abs(e)), kind


def test_duplicates_and_out_of_range_batch_rows():
    """a duplicate coordinate contributes twice to a regular conv, a subm tap lands on the first row of a
    coordinate, and a row whose batch index is out of range reaches no output (subm: only itself)"""
    inds = np.array([[0, 2, 2], [0, 2, 3], [0, 2, 2], [2, 1, 1], [-1, 1, 1]], np.int32)
    conv = SparseConvRef(inds, 2, [5, 5], [3, 3], [2, 2], [1, 1], [1, 1], kind="conv")
    for i, o in conv.pairs:
        assert not {3, 4} & set(i.tolist())
        assert sorted(o[i == 0].tolist()) == sorted(o[i == 2].tolist())
    sub = SparseConvRef(inds, 2, [5, 5], [3, 3], [1, 1], [0, 0], [1, 1], kind="subm")
    for k, (i, o) in enumerate(sub.pairs):
        if k != sub.kv // 2:
            assert not {3, 4} & (set(i.tolist()) | set(o.tolist()))
    # tap (1, 0) of (2,2) lands on (2,3): both copies of (2,2) reach row 1, row 1 reaches row 0 only
    assert sub.pair_set()[3] == {(0, 1), (2, 1)}
    assert sub.pair_set()[5] == {(1, 0), (1, 2)}


# ------------------------------------------------------------------ agreement with the oracle's rulebook
def _geometry_cases():
    from tests import test_conv_modules_gpu as M
    from tests import test_rulebook_edges_gpu as E
    out = []
    for name, g in M.GEOMS.items():
        inds, _ = M.cloud(name)
        out.append((f"module-{name}", inds, g))
    for name, (inds, g) in E.rulebook_cases().items():
        out.append((f"edge-{name}", inds, g))
    return out


@pytest.mark.parametrize("case", _geometry_cases(), ids=lambda c: c[0])
def test_pairs_equal_the_oracle_rulebook(case, oracle):
    _, inds, g = case
    kind, shape, bs = g["kind"], g["shape"], g["batch"]
    ks, s, p, d, op = g["ksize"], g["stride"], g["padding"], g["dilation"], g["output_padding"]
    nd = len(shape)
    base = "conv" if kind == "inverse" else kind
    ref = SparseConvRef(inds, bs, shape, ks, s, p, d, op, base)
    o, pairs, num = oracle.get_indice_pairs(inds, bs, shape, ks, s, p, d, op if base == "transpose" else [0] * nd,
                                            base == "subm", base == "transpose")
    assert np.array_equal(ref.out_inds, o)
    cnt = oracle._pair_counts(num, ref.kv, inds.shape[0], base == "subm")
    for k in range(ref.kv):
        want = set(zip(pairs[0, k, :cnt[k]].tolist(), pairs[1, k, :cnt[k]].tolist()))
        i, oo = ref.pairs[k]
        have = list(zip(i.tolist(), oo.tolist()))
        assert len(have) == len(want) and set(have) == want, (k, len(have), len(want))
    assert len(offset_taps(ks)) == ref.kv
