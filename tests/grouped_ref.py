"""Float64 grouped sparse-convolution reference (1 < groups) on the pairs of :class:`tests.conv_ref.SparseConvRef`.

The filter is KRSC ``[K, *ksize, C / groups]``; group j maps input channels ``[j Cg, (j+1) Cg)`` to output channels
``[j Kg, (j+1) Kg)`` with filter rows ``W[j Kg:(j+1) Kg]`` (Cg = C / groups, Kg = K / groups), torch's convention:
    y[o, j Kg + n]   = sum over the pairs (i, o) of offset k and c < Cg of W[j Kg + n, k, c] x[i, j Cg + c]  (+ b)
    dx[i, j Cg + c]  = sum over the pairs (i, o) of offset k and n < Kg of W[j Kg + n, k, c] dy[o, j Kg + n]
    dW[j Kg + n, k, c] = sum over the pairs (i, o) of offset k of dy[o, j Kg + n] x[i, j Cg + c]
Each result comes with the sum of the magnitudes of its terms, for rounding-error bounds.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from tests.conv_ref import SparseConvRef


def _split(w: np.ndarray, groups: int):
    w = np.asarray(w, np.float64)
    K = w.shape[0]
    assert groups >= 1 and K % groups == 0, (w.shape, groups)
    kg = K // groups
    return [w[j * kg:(j + 1) * kg] for j in range(groups)], kg


def grouped_forward(ref: SparseConvRef, x: np.ndarray, w: np.ndarray, groups: int,
                    bias: Optional[np.ndarray] = None):
    """(out [n_out, K], sum of |terms| [n_out, K]) in float64"""
    x = np.asarray(x, np.float64)
    ws, kg = _split(w, groups)
    cg = w.shape[-1]
    assert x.shape[1] == cg * groups, (x.shape, w.shape, groups)
    outs, mags = [], []
    for j, wj in enumerate(ws):
        bj = None if bias is None else np.asarray(bias, np.float64)[j * kg:(j + 1) * kg]
        o, m, _ = ref.forward(x[:, j * cg:(j + 1) * cg], wj, bj)
        outs.append(o)
        mags.append(m)
    return np.concatenate(outs, 1), np.concatenate(mags, 1)


def grouped_backward(ref: SparseConvRef, x: np.ndarray, w: np.ndarray, dy: np.ndarray, groups: int):
    """(dx [n_in, C], |dx terms|, dW [K, *ksize, C / groups], |dW terms|) in float64"""
    x = np.asarray(x, np.float64)
    dy = np.asarray(dy, np.float64)
    ws, kg = _split(w, groups)
    cg = w.shape[-1]
    dx, dxm, dw, dwm = [], [], [], []
    for j, wj in enumerate(ws):
        a, am, _, b, bm, _ = ref.backward(x[:, j * cg:(j + 1) * cg], wj, dy[:, j * kg:(j + 1) * kg])
        dx.append(a)
        dxm.append(am)
        dw.append(b)
        dwm.append(bm)
    return np.concatenate(dx, 1), np.concatenate(dxm, 1), np.concatenate(dw, 0), np.concatenate(dwm, 0)
