"""Depthwise sparse convolution (groups = in_channels = out_channels) without a GPU: module construction,
initialisation, repr, checkpoints, the refusals, the torch-only 1x1 path, and the float64 reference of
tests/depthwise_ref.py pinned to torch's dense grouped convolution."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch.quantized import QuantizedSparseConv
from tests.conv_ref import SparseConvRef
from tests.depthwise_ref import depthwise_backward, depthwise_forward

KINDS = {
    "subm": lambda nd, c, k, **kw: getattr(spconv, f"SubMConv{nd}d")(c, c, k, groups=c, **kw),
    "conv": lambda nd, c, k, **kw: getattr(spconv, f"SparseConv{nd}d")(c, c, k, 2, 1, groups=c, **kw),
    "transpose": lambda nd, c, k, **kw: getattr(spconv, f"SparseConvTranspose{nd}d")(c, c, k, 2, 1, groups=c, **kw),
    "inverse": lambda nd, c, k, **kw: getattr(spconv, f"SparseInverseConv{nd}d")(c, c, k, indice_key="d", groups=c,
                                                                                  **kw),
}


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("nd", [1, 2, 3, 4])
def test_construction(kind, nd):
    torch.manual_seed(nd)
    c, k = 48, 3
    m = KINDS[kind](nd, c, k)
    kv = k ** nd
    assert list(m.weight.shape) == [c] + [k] * nd + [1]
    assert m.groups == c and m.depthwise
    # kaiming-uniform(a = sqrt(5)) with torch's grouped fan-in (in_channels / groups) * kv = kv
    bound = math.sqrt(2.0 / 6.0) * math.sqrt(3.0 / kv)
    w = m.weight.detach().abs()
    assert float(w.max()) <= bound and float(w.max()) > 0.8 * bound
    assert float(m.bias.detach().abs().max()) <= 1 / math.sqrt(kv)
    assert f"groups={c}" in m.extra_repr()
    assert "groups" not in getattr(spconv, f"SubMConv{nd}d")(c, c, k).extra_repr()
    fresh = KINDS[kind](nd, c, k)
    fresh.load_state_dict(m.state_dict())
    assert torch.equal(fresh.weight, m.weight) and torch.equal(fresh.bias, m.bias)


@pytest.mark.parametrize("cin, cout, groups", [(4, 4, 2), (4, 8, 4), (8, 4, 4), (4, 4, 0), (1, 1, 1)])
def test_other_groups_raise(cin, cout, groups):
    if groups == 1:
        spconv.SubMConv3d(cin, cout, 3, groups=groups)       # groups = 1 stays the dense conv
        return
    with pytest.raises(AssertionError, match="groups"):
        spconv.SubMConv3d(cin, cout, 3, groups=groups)
    with pytest.raises(AssertionError, match="groups"):
        spconv.SparseConv3d(cin, cout, 3, 2, groups=groups)


def test_from_float_refuses_depthwise():
    m = spconv.SubMConv3d(16, 16, 3, groups=16).eval()
    with pytest.raises(NotImplementedError, match="depthwise"):
        QuantizedSparseConv.from_float(m, 0.1)


@pytest.mark.parametrize("bias", [True, False])
def test_kernel_volume_one_is_a_channel_scale(bias):
    """SubM 1x1x1 depthwise runs in torch: x * W[c] (+ b[c]), no kernel and no rulebook"""
    torch.manual_seed(3)
    m = spconv.SubMConv3d(6, 6, 1, groups=6, bias=bias)
    feats = torch.randn(10, 6)
    inds = torch.cat([torch.zeros(10, 1, dtype=torch.int32), torch.randint(0, 5, (10, 3), dtype=torch.int32)], 1)
    y = m(spconv.SparseConvTensor(feats, inds, [5, 5, 5], 1))
    want = feats * m.weight.detach().view(6) + (m.bias.detach() if bias else 0)
    assert torch.equal(y.features.detach(), want)


def _dense_case(nd, kind, seed):
    rng = np.random.default_rng(seed)
    shape = {1: [23], 2: [9, 8], 3: [6, 7, 5]}[nd]
    C = 5
    mask = rng.random(shape) < 0.45
    coords = np.argwhere(mask).astype(np.int32)
    inds = np.concatenate([np.zeros((len(coords), 1), np.int32), coords], 1)
    x = rng.standard_normal((len(inds), C))
    return shape, C, inds, x, rng


def _dense_input(shape, C, inds, x):
    X = np.zeros([1, C] + list(shape))
    X[0][(slice(None),) + tuple(inds[:, 1:].T)] = x.T
    return torch.from_numpy(X)


CONV = {1: F.conv1d, 2: F.conv2d, 3: F.conv3d}


@pytest.mark.parametrize("nd", [1, 2, 3])
@pytest.mark.parametrize("k", [3, 5])
def test_reference_subm_equals_dense_grouped_conv(nd, k):
    shape, C, inds, x, rng = _dense_case(nd, "subm", 10 * nd + k)
    w = rng.standard_normal([C] + [k] * nd + [1])
    b = rng.standard_normal(C)
    ref = SparseConvRef(inds, 1, shape, [k] * nd, [1] * nd, [0] * nd, [1] * nd, kind="subm")
    out, _ = depthwise_forward(ref, x, w, b)
    wt = torch.from_numpy(np.moveaxis(w, -1, 1))                       # [C, 1, *ksize]
    Y = CONV[nd](_dense_input(shape, C, inds, x), wt, torch.from_numpy(b), padding=k // 2, groups=C)
    want = Y[0][(slice(None),) + tuple(inds[:, 1:].T)].T.numpy()
    np.testing.assert_allclose(out, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("nd", [1, 2, 3])
@pytest.mark.parametrize("k, s, p, d", [(3, 2, 1, 1), (2, 2, 0, 1), (3, 1, 1, 2)])
def test_reference_strided_equals_dense_grouped_conv(nd, k, s, p, d):
    shape, C, inds, x, rng = _dense_case(nd, "conv", 20 * nd + k + s)
    w = rng.standard_normal([C] + [k] * nd + [1])
    ref = SparseConvRef(inds, 1, shape, [k] * nd, [s] * nd, [p] * nd, [d] * nd, kind="conv")
    out, _ = depthwise_forward(ref, x, w)
    wt = torch.from_numpy(np.moveaxis(w, -1, 1))
    Y = CONV[nd](_dense_input(shape, C, inds, x), wt, stride=s, padding=p, dilation=d, groups=C)
    want = Y[0][(slice(None),) + tuple(ref.out_inds[:, 1:].T.astype(np.int64))].T.numpy()
    np.testing.assert_allclose(out, want, rtol=1e-12, atol=1e-12)
    # every active output of the dense conv is one of the sparse outputs, the rest of the grid is 0
    reached = np.zeros(Y.shape[2:], bool)
    reached[tuple(ref.out_inds[:, 1:].T.astype(np.int64))] = True
    assert float(Y[0][:, ~torch.from_numpy(reached)].abs().sum()) == 0.0


@pytest.mark.parametrize("nd", [1, 2, 3])
def test_reference_gradients_equal_autograd_of_the_dense_conv(nd):
    """dx at the active sites and dW of the SubM reference equal torch's autograd through the dense grouped conv"""
    k = 3
    shape, C, inds, x, rng = _dense_case(nd, "subm", 40 + nd)
    w = rng.standard_normal([C] + [k] * nd + [1])
    dy = rng.standard_normal((len(inds), C))
    ref = SparseConvRef(inds, 1, shape, [k] * nd, [1] * nd, [0] * nd, [1] * nd, kind="subm")
    dx, _, dw, _ = depthwise_backward(ref, x, w, dy)
    X = _dense_input(shape, C, inds, x).requires_grad_(True)
    wt = torch.from_numpy(np.moveaxis(w, -1, 1).copy()).requires_grad_(True)
    Y = CONV[nd](X, wt, padding=k // 2, groups=C)
    sites = (slice(None),) + tuple(inds[:, 1:].T)
    Y[0][sites].T.backward(torch.from_numpy(dy))
    np.testing.assert_allclose(dx, X.grad[0][sites].T.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dw, np.moveaxis(wt.grad.numpy(), 1, -1), rtol=1e-12, atol=1e-12)
