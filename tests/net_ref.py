"""Float64 twins of the layers of a sparse network, for whole-network tests.

Every twin is a CPU float64 torch function with autograd, built from the coordinate-level references of this
directory (``conv_ref.SparseConvRef``, ``pool_oracle``'s tie rule, ``sparse_add_oracle``'s union); none of them
uses the oracle or a kernel.  Output coordinates and row orders come from the twins, so a test can compare them
bit for bit with the library's.

Conv-like twins also give, through :func:`conv_bounds`, the size of the terms each result sums (``mag``) and
how many there are (``terms``), for the rounding-error bound ``u_out |ref| + T 2^-23 sum|terms|`` that the conv
tests use.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from tests.conv_ref import SparseConvRef
from tests import sparse_add_oracle

F64 = torch.float64


def _pairs(ref: SparseConvRef):
    return [(torch.from_numpy(np.asarray(i, np.int64)), torch.from_numpy(np.asarray(o, np.int64)))
            for i, o in ref.pairs]


class ConvTwin:
    """``y = sum over offsets k of S_k x W_k^T`` on the pairs of ``ref`` (subm, conv, transpose or inverse);
    the weight is KRSC ``[K, *ksize, C]``, or ``[C, *ksize, 1]`` with ``depthwise``."""

    def __init__(self, ref: SparseConvRef, depthwise: bool = False):
        self.ref = ref
        self.depthwise = depthwise
        self.pairs = _pairs(ref)

    @property
    def out_inds(self) -> np.ndarray:
        return self.ref.out_inds

    def __call__(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
        kv = self.ref.kv
        if self.depthwise:
            wk = w.reshape(w.shape[0], kv)
            out = x.new_zeros((self.ref.n_out, w.shape[0]))
            for k, (i, o) in enumerate(self.pairs):
                if len(i):
                    out = out.index_add(0, o, x[i] * wk[:, k])
        else:
            wk = w.reshape(w.shape[0], kv, w.shape[-1])
            out = x.new_zeros((self.ref.n_out, w.shape[0]))
            for k, (i, o) in enumerate(self.pairs):
                if len(i):
                    out = out.index_add(0, o, x[i] @ wk[:, k].t())
        return out if bias is None else out + bias


def conv_bounds(twin: ConvTwin, x, w, dy):
    """Per result, the sum of the magnitudes of its terms and the number of terms:
    ``(y_mag, y_terms, dx_mag, dx_terms, dw_mag, dw_terms)`` (the conv itself, without the bias)."""
    def run(a, b, g):
        a = a.detach().clone().requires_grad_(True)
        b = b.detach().clone().requires_grad_(True)
        y = twin(a, b)
        y.backward(g)
        return y.detach(), a.grad, b.grad
    y_mag, dx_mag, dw_mag = run(x.abs(), w.abs(), dy.abs())
    y_t, dx_t, dw_t = run(torch.ones_like(x), torch.ones_like(w), torch.ones_like(dy))
    return y_mag, y_t, dx_mag, dx_t, dw_mag, dw_t


def max_pool(ref: SparseConvRef, x: torch.Tensor, low: float) -> torch.Tensor:
    """Max over each output's inputs in offset order, from ``low``; a candidate wins only when greater
    (``pool_oracle.max_pool``).  Its gradient goes to every input equal to its output's max
    (``pool_oracle.max_pool_backward``)."""
    return _MaxPool.apply(x, ref, low)


class _MaxPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ref, low):
        out = torch.full((ref.n_out, x.shape[1]), low, dtype=x.dtype)
        for i, o in _pairs(ref):
            if len(i):
                cand, cur = x[i], out[o]
                out[o] = torch.where(cand > cur, cand, cur)
        ctx.save_for_backward(x, out)
        ctx.ref = ref
        return out

    @staticmethod
    def backward(ctx, dy):
        x, out = ctx.saved_tensors
        dx = torch.zeros_like(x)
        for i, o in _pairs(ctx.ref):
            if len(i):
                dx = dx.index_add(0, i, torch.where(x[i] == out[o], dy[o], 0.0))
        return dx, None, None


def batch_norm_train(x, weight, bias, eps):
    """training-mode BatchNorm over the rows of ``x`` (biased variance), the formula of
    ``nn.BatchNorm1d``; with autograd"""
    mean = x.mean(0)
    var = x.var(0, unbiased=False)
    return (x - mean) / torch.sqrt(var + eps) * weight + bias


def running_stats(x, running_mean, running_var, momentum, nbt_after):
    """the running stats after one training step on the rows of ``x``"""
    m = x.shape[0]
    f = 1.0 / nbt_after if momentum is None else momentum
    mean = x.mean(0)
    var = x.var(0, unbiased=False)
    return (1 - f) * running_mean + f * mean, (1 - f) * running_var + f * var * m / (m - 1)


def batch_norm_eval(x, weight, bias, running_mean, running_var, eps):
    return (x - running_mean) / torch.sqrt(running_var + eps) * weight + bias


def relu(x):
    return F.relu(x)


def leaky_relu(x, alpha):
    return F.leaky_relu(x, alpha)


def join(xs: Sequence[torch.Tensor]):
    return torch.cat(list(xs), 1)


def add(xs: Sequence[torch.Tensor]):
    out = xs[0]
    for t in xs[1:]:
        out = out + t
    return out


class MisalignedAdd:
    """The union of several operands' coordinates in ``sparse_add``'s visit order (``sparse_add_oracle``) and
    the sum of every output row's rows."""

    def __init__(self, indices: Sequence[np.ndarray], batch_size: int, spatial_shape):
        order = sparse_add_oracle.visit_order([len(i) for i in indices])
        self.out_inds, dst = sparse_add_oracle.union([indices[i] for i in order], batch_size, spatial_shape)
        rows = np.cumsum([0] + [len(indices[i]) for i in order])
        self.dst = [None] * len(indices)
        for pos, i in enumerate(order):
            self.dst[i] = torch.from_numpy(dst[rows[pos]:rows[pos + 1]].astype(np.int64))

    def __call__(self, xs: Sequence[torch.Tensor]) -> torch.Tensor:
        out = xs[0].new_zeros((len(self.out_inds), xs[0].shape[1]))
        for x, d in zip(xs, self.dst):
            keep = d >= 0
            out = out.index_add(0, d[keep], x[keep])
        return out


def _samples(indices: np.ndarray, batch_size: int) -> List[torch.Tensor]:
    b = np.asarray(indices)[:, 0]
    return [torch.from_numpy(np.nonzero(b == s)[0].astype(np.int64)) for s in range(batch_size)]


def global_max(x: torch.Tensor, indices: np.ndarray, batch_size: int) -> torch.Tensor:
    """per sample, the value of the first row (in row order) with the maximum; 0 for an empty sample.  The
    gradient goes to that row."""
    outs = []
    for rows in _samples(indices, batch_size):
        if not len(rows):
            outs.append(x.new_zeros(x.shape[1]))
            continue
        xs = x[rows]
        first = torch.from_numpy(np.argmax(xs.detach().numpy(), axis=0))     # numpy: the first maximum
        outs.append(xs.gather(0, first.view(1, -1))[0])
    return torch.stack(outs)


def global_avg(x: torch.Tensor, indices: np.ndarray, batch_size: int) -> torch.Tensor:
    outs = []
    for rows in _samples(indices, batch_size):
        outs.append(x[rows].mean(0) if len(rows) else x.new_zeros(x.shape[1]))
    return torch.stack(outs)


def to_dense(x: torch.Tensor, indices: np.ndarray, batch_size: int, spatial_shape) -> torch.Tensor:
    """``[batch, C, *spatial]``"""
    idx = torch.from_numpy(np.asarray(indices, np.int64))
    grid = x.new_zeros((batch_size, *spatial_shape, x.shape[1]))
    grid = grid.index_put(tuple(idx.t()), x)
    nd = len(spatial_shape)
    return grid.permute(0, nd + 1, *range(1, nd + 1))
