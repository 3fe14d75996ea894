"""Float64 depthwise sparse-convolution reference (groups = in_channels = out_channels = C) on the pairs of
:class:`tests.conv_ref.SparseConvRef`.

The filter is KRSC with one input channel per group, ``[C, *ksize, 1]``, read as ``W[c, k]``:
    y[o, c]  = sum over the pairs (i, o) of offset k of W[c, k] x[i, c]  (+ b[c])
    dx[i, c] = sum over the pairs (i, o) of offset k of W[c, k] dy[o, c]
    dW[c, k] = sum over the pairs (i, o) of offset k of dy[o, c] x[i, c]
Each result comes with the sum of the magnitudes of its terms, for rounding-error bounds.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from tests.conv_ref import SparseConvRef


def _taps(ref: SparseConvRef, w: np.ndarray) -> np.ndarray:
    w = np.asarray(w, np.float64)
    assert w.shape[-1] == 1 and int(np.prod(w.shape[1:-1])) == ref.kv, w.shape
    return w.reshape(w.shape[0], ref.kv)


def depthwise_forward(ref: SparseConvRef, x: np.ndarray, w: np.ndarray, bias: Optional[np.ndarray] = None):
    """(out [n_out, C], sum of |terms| [n_out, C]) in float64"""
    x = np.asarray(x, np.float64)
    wk = _taps(ref, w)
    out = np.zeros((ref.n_out, x.shape[1]))
    mag = np.zeros_like(out)
    for k, (i, o) in enumerate(ref.pairs):
        if len(i):
            np.add.at(out, o, x[i] * wk[:, k])
            np.add.at(mag, o, np.abs(x[i] * wk[:, k]))
    if bias is not None:
        out += np.asarray(bias, np.float64)
        mag += np.abs(np.asarray(bias, np.float64))
    return out, mag


def depthwise_backward(ref: SparseConvRef, x: np.ndarray, w: np.ndarray, dy: np.ndarray):
    """(dx [n_in, C], |dx terms|, dW [C, *ksize, 1], |dW terms|) in float64"""
    x = np.asarray(x, np.float64)
    dy = np.asarray(dy, np.float64)
    wk = _taps(ref, w)
    dx = np.zeros((ref.n_in, x.shape[1]))
    dx_mag = np.zeros_like(dx)
    dw = np.zeros_like(wk)
    dw_mag = np.zeros_like(wk)
    for k, (i, o) in enumerate(ref.pairs):
        if not len(i):
            continue
        np.add.at(dx, i, dy[o] * wk[:, k])
        np.add.at(dx_mag, i, np.abs(dy[o] * wk[:, k]))
        dw[:, k] = (dy[o] * x[i]).sum(0)
        dw_mag[:, k] = np.abs(dy[o] * x[i]).sum(0)
    shape = np.shape(w)
    return dx, dx_mag, dw.reshape(shape), dw_mag.reshape(shape)
