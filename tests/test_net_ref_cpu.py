"""The float64 layer twins of tests/net_ref.py: autograd gradients against finite differences, and two small
composed nets against dense float64 convolutions on fully occupied grids, where sparse and dense agree."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import net_ref
from tests.conv_ref import SparseConvRef

F64 = torch.float64


def _cloud(rng, shape, n, batch):
    cells = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"), -1).reshape(-1, len(shape))
    out = []
    for b in range(batch):
        pick = cells[rng.permutation(len(cells))[:n]]
        out.append(np.concatenate([np.full((n, 1), b), pick], 1))
    return np.concatenate(out, 0).astype(np.int32)


def _full_grid(shape, batch):
    return _cloud(np.random.default_rng(0), shape, int(np.prod(shape)), batch)


def _leaf(rng, shape, scale=1.0):
    return torch.from_numpy(rng.standard_normal(shape) * scale).requires_grad_(True)


SHAPE = [4, 5, 3]


def _ref(kind, inds):
    if kind == "subm":
        return SparseConvRef(inds, 2, SHAPE, [3] * 3, [1] * 3, [1] * 3, [1] * 3, kind="subm")
    if kind == "transpose":
        return SparseConvRef(inds, 2, SHAPE, [2] * 3, [2] * 3, [0] * 3, [1] * 3, kind="transpose")
    return SparseConvRef(inds, 2, SHAPE, [3] * 3, [2] * 3, [1] * 3, [1] * 3, kind=kind)


@pytest.mark.parametrize("kind", ["subm", "conv", "transpose", "inverse"])
@pytest.mark.parametrize("depthwise", [False, True])
def test_conv_twin_gradcheck(kind, depthwise):
    rng = np.random.default_rng(1)
    inds = _cloud(rng, SHAPE, 12, 2)
    ref = _ref(kind, inds)
    twin = net_ref.ConvTwin(ref, depthwise=depthwise)
    C, K = (3, 3) if depthwise else (3, 2)
    x = _leaf(rng, (ref.n_in, C))
    w = _leaf(rng, (K, *ref.ksize, 1 if depthwise else C))
    b = _leaf(rng, (K,))
    assert torch.autograd.gradcheck(lambda x, w, b: twin(x, w, b), (x, w, b))


def test_conv_bounds_count_the_terms():
    rng = np.random.default_rng(2)
    inds = _cloud(rng, SHAPE, 20, 2)
    ref = _ref("subm", inds)
    twin = net_ref.ConvTwin(ref)
    x, w, dy = (torch.from_numpy(rng.standard_normal(s)) for s in ((ref.n_in, 3), (2, 3, 3, 3, 3), (ref.n_out, 2)))
    y_mag, y_t, dx_mag, dx_t, dw_mag, dw_t = net_ref.conv_bounds(twin, x, w, dy)
    out, mag, cnt = ref.forward(x.numpy(), w.numpy())
    assert np.allclose(y_mag.numpy(), mag) and np.array_equal(y_t[:, 0].numpy(), cnt)
    dx, dxm, dxc, dw, dwm, dwc = ref.backward(x.numpy(), w.numpy(), dy.numpy())
    assert np.allclose(dx_mag.numpy(), dxm) and np.array_equal(dx_t[:, 0].numpy(), dxc)
    assert np.allclose(dw_mag.numpy(), dwm) and np.array_equal(dw_t[0, ..., 0].reshape(-1).numpy(), dwc)


def test_max_pool_twin_gradcheck_and_tie_rule():
    rng = np.random.default_rng(3)
    inds = _cloud(rng, SHAPE, 14, 2)
    ref = _ref("conv", inds)
    x = _leaf(rng, (ref.n_in, 3))
    assert torch.autograd.gradcheck(lambda x: net_ref.max_pool(ref, x, -1e30), (x,))
    # every input tied with its output's max receives the gradient, as pool.cu's backward gives it
    xt = torch.zeros((ref.n_in, 1), dtype=F64, requires_grad=True)
    y = net_ref.max_pool(ref, xt, float(torch.finfo(torch.float32).min))
    y.backward(torch.ones_like(y))
    fan = np.zeros(ref.n_in)
    for i, _ in ref.pairs:
        np.add.at(fan, i, 1)
    assert np.array_equal(xt.grad[:, 0].numpy(), fan)


def test_batch_norm_twins_gradcheck_and_running_stats():
    rng = np.random.default_rng(4)
    x, w, b = _leaf(rng, (9, 4)), _leaf(rng, (4,)), _leaf(rng, (4,))
    assert torch.autograd.gradcheck(lambda x, w, b: net_ref.batch_norm_train(x, w, b, 1e-5), (x, w, b))
    rm, rv = torch.from_numpy(rng.standard_normal(4)), torch.from_numpy(rng.random(4) + 0.5)
    assert torch.autograd.gradcheck(lambda x, w, b: net_ref.batch_norm_eval(x, w, b, rm, rv, 1e-5), (x, w, b))
    bn = torch.nn.BatchNorm1d(4, momentum=0.3).double().train()
    with torch.no_grad():
        bn.weight.copy_(w)
        bn.bias.copy_(b)
        bn.running_mean.copy_(rm)
        bn.running_var.copy_(rv)
    y = bn(x.detach())
    assert torch.allclose(y, net_ref.batch_norm_train(x.detach(), w.detach(), b.detach(), bn.eps), atol=1e-12)
    m, v = net_ref.running_stats(x.detach(), rm, rv, 0.3, 1)
    assert torch.allclose(m, bn.running_mean, atol=1e-14) and torch.allclose(v, bn.running_var, atol=1e-14)


def test_pointwise_table_and_global_twins_gradcheck():
    rng = np.random.default_rng(5)
    inds = _cloud(rng, SHAPE, 10, 2)
    a, b = _leaf(rng, (20, 3)), _leaf(rng, (20, 3))
    assert torch.autograd.gradcheck(lambda a: net_ref.leaky_relu(a, 0.1), (a,))
    assert torch.autograd.gradcheck(lambda a, b: net_ref.join([a, b]), (a, b))
    assert torch.autograd.gradcheck(lambda a, b: net_ref.add([a, b]), (a, b))
    assert torch.autograd.gradcheck(lambda a: net_ref.global_max(a, inds, 3), (a,))     # sample 2 is empty
    assert torch.autograd.gradcheck(lambda a: net_ref.global_avg(a, inds, 3), (a,))
    assert torch.autograd.gradcheck(lambda a: net_ref.to_dense(a, inds, 2, SHAPE), (a,))
    other = _cloud(np.random.default_rng(6), SHAPE, 7, 2)
    mis = net_ref.MisalignedAdd([other, inds], 2, SHAPE)
    c = _leaf(rng, (14, 3))
    assert torch.autograd.gradcheck(lambda c, a: mis([c, a]), (c, a))
    # the union: the larger operand's rows first, in order, then the other's new coordinates in order
    assert np.array_equal(mis.out_inds[:20], inds)
    keys = {tuple(r) for r in inds.tolist()}
    assert mis.out_inds[20:].tolist() == [r for r in other.tolist() if tuple(r) not in keys]


def test_global_max_takes_the_first_maximum():
    inds = np.array([[0, 0, 0, 0], [1, 0, 0, 1], [0, 0, 1, 0], [0, 1, 0, 0]], np.int32)
    x = torch.tensor([[1.0], [5.0], [3.0], [3.0]], dtype=F64, requires_grad=True)
    y = net_ref.global_max(x, inds, 2)
    y.backward(torch.ones_like(y))
    assert y[:, 0].tolist() == [3.0, 5.0] and x.grad[:, 0].tolist() == [0.0, 1.0, 1.0, 0.0]


def _dense_of(x, inds, shape):
    return net_ref.to_dense(x, inds, 2, shape)


def test_subm_and_strided_net_equals_dense_conv_on_a_full_grid():
    """SubM -> ReLU -> SubM -> stride-2 conv on every cell of the grid == conv3d(padding 1) twice, then
    conv3d(stride 2, padding 1)"""
    rng = np.random.default_rng(7)
    shape = [4, 6, 5]
    inds = _full_grid(shape, 2)
    n, C = len(inds), 3
    subm = net_ref.ConvTwin(SparseConvRef(inds, 2, shape, [3] * 3, [1] * 3, [1] * 3, [1] * 3, kind="subm"))
    down_ref = SparseConvRef(inds, 2, shape, [3] * 3, [2] * 3, [1] * 3, [1] * 3, kind="conv")
    down = net_ref.ConvTwin(down_ref)
    x = torch.from_numpy(rng.standard_normal((n, C)))
    w1, w2, w3 = (torch.from_numpy(rng.standard_normal((C, 3, 3, 3, C))) for _ in range(3))
    b1 = torch.from_numpy(rng.standard_normal(C))
    y = down(subm(net_ref.relu(subm(x, w1, b1)), w2), w3)
    krsc = lambda w: w.permute(0, 4, 1, 2, 3)            # noqa: E731  KRSC -> [K, C, k, k, k]
    xd = _dense_of(x, inds, shape)
    yd = F.conv3d(F.relu(F.conv3d(xd, krsc(w1), b1, padding=1)), krsc(w2), padding=1)
    yd = F.conv3d(yd, krsc(w3), stride=2, padding=1)
    assert list(yd.shape[2:]) == down_ref.out_shape and down_ref.n_out == 2 * int(np.prod(down_ref.out_shape))
    assert torch.allclose(_dense_of(y, down_ref.out_inds, down_ref.out_shape), yd, atol=1e-10)


def test_strided_inverse_and_transposed_net_equals_dense_on_a_full_grid():
    """stride-2 conv -> inverse conv (back on the full grid) -> transposed conv k2 s2, against conv3d,
    conv_transpose3d(stride 2, padding 1, output_padding 1) and conv_transpose3d(stride 2)"""
    rng = np.random.default_rng(8)
    shape = [4, 6, 4]
    inds = _full_grid(shape, 2)
    C = 2
    down_ref = SparseConvRef(inds, 2, shape, [3] * 3, [2] * 3, [1] * 3, [1] * 3, kind="conv")
    inv_ref = SparseConvRef(inds, 2, shape, [3] * 3, [2] * 3, [1] * 3, [1] * 3, kind="inverse")
    up_ref = SparseConvRef(inds, 2, shape, [2] * 3, [2] * 3, [0] * 3, [1] * 3, kind="transpose")
    assert np.array_equal(inv_ref.in_inds, down_ref.out_inds) and np.array_equal(inv_ref.out_inds, inds)
    x = torch.from_numpy(rng.standard_normal((len(inds), C)))
    w1, w2, w3 = (torch.from_numpy(rng.standard_normal((C, *k, C))) for k in ([3] * 3, [3] * 3, [2] * 3))
    y = net_ref.ConvTwin(up_ref)(net_ref.ConvTwin(inv_ref)(net_ref.ConvTwin(down_ref)(x, w1), w2), w3)
    xd = _dense_of(x, inds, shape)
    yd = F.conv3d(xd, w1.permute(0, 4, 1, 2, 3), stride=2, padding=1)
    yd = F.conv_transpose3d(yd, w2.permute(4, 0, 1, 2, 3), stride=2, padding=1, output_padding=1)
    yd = F.conv_transpose3d(yd, w3.permute(4, 0, 1, 2, 3), stride=2)
    assert list(yd.shape[2:]) == up_ref.out_shape
    assert torch.allclose(_dense_of(y, up_ref.out_inds, up_ref.out_shape), yd, atol=1e-10)
