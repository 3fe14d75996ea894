"""Float64 sparse-convolution reference, built from the definition on coordinates.

It uses neither the oracle nor any rulebook kernel: every kernel offset is matched against the output
(or input) coordinates with ``np.searchsorted`` on int64 linear keys over ``[batch, *dims]``.

Semantics (those of the reference project, ``ops.get_indice_pairs``):
  * regular conv: input ``c`` reaches output ``o = (c + p - r d) / s`` through tap ``r`` when the
    division is exact and ``0 <= o < out``, ``out = (in + 2p - d (k - 1) - 1) // s + 1``;
  * transposed conv: ``o = c s - p + r d`` with ``0 <= o < out``, ``out = (in - 1) s - 2p + k + op``.
    The grid size ignores dilation, as the reference's does, so with dilation > 1 the taps that land
    beyond the grid are dropped;
  * subm: ``p = (k // 2) d``, stride 1, and the output rows are the input rows.  Tap ``r`` of input ``i``
    lands on the first input row with coordinate ``c + p - r d``, and the mirrored tap ``kv - 1 - r``
    brings that row back to ``i`` (the reference's pair order);
  * inverse: the pairs of the paired regular conv with inputs and outputs swapped; the output rows are
    the paired conv's input rows;
  * rows whose batch index lies outside ``[0, batch_size)`` reach no output.  The outputs of a regular or
    transposed conv are ranked by first touch in offset-major order (offset, then input row).

Kernel offsets are row-major over the taps, last axis fastest; the weight is KRSC ``[K, *ksize, C]``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import scipy.sparse as sp


def offset_taps(ksize: Sequence[int]) -> np.ndarray:
    """[kv, ndim] taps of every kernel offset, last axis fastest."""
    return np.stack(np.unravel_index(np.arange(int(np.prod(ksize))), tuple(ksize)), axis=-1).astype(np.int64)


def linear_keys(coords: np.ndarray, dims: Sequence[int]) -> np.ndarray:
    """int64 row-major key of [b, d0, d1, ...] rows over [batch, *dims]."""
    k = coords[:, 0].astype(np.int64)
    for a, d in enumerate(dims):
        k = k * int(d) + coords[:, a + 1].astype(np.int64)
    return k


def conv_output_size(shape, ksize, stride, padding, dilation):
    return [(i + 2 * p - d * (k - 1) - 1) // s + 1 for i, k, s, p, d in zip(shape, ksize, stride, padding, dilation)]


def deconv_output_size(shape, ksize, stride, padding, output_padding):
    return [(i - 1) * s - 2 * p + k + op for i, k, s, p, op in zip(shape, ksize, stride, padding, output_padding)]


class SparseConvRef:
    """Pairs of one sparse convolution: ``pairs[k] = (in_rows, out_rows)`` of kernel offset ``k``."""

    def __init__(self, indices, batch_size: int, spatial_shape: Sequence[int], ksize: Sequence[int],
                 stride: Sequence[int], padding: Sequence[int], dilation: Sequence[int],
                 output_padding: Optional[Sequence[int]] = None, kind: str = "conv"):
        assert kind in ("subm", "conv", "transpose", "inverse"), kind
        indices = np.asarray(indices, dtype=np.int64)
        ndim = indices.shape[1] - 1
        assert 1 <= ndim <= 4 and len(spatial_shape) == ndim
        self.kind, self.ndim, self.kv = kind, ndim, int(np.prod(ksize))
        self.ksize = list(ksize)
        output_padding = [0] * ndim if output_padding is None else list(output_padding)
        taps = offset_taps(ksize)
        ok_batch = (indices[:, 0] >= 0) & (indices[:, 0] < batch_size)
        n = indices.shape[0]
        if kind == "subm":
            pad = np.array([(k // 2) * d for k, d in zip(ksize, dilation)], np.int64)
            dil = np.asarray(dilation, np.int64)
            dims = np.asarray(spatial_shape, np.int64)
            keys = linear_keys(indices, spatial_shape)
            ukeys, first = np.unique(keys, return_index=True)        # first row of every coordinate
            pairs = [None] * self.kv
            for k in range(self.kv // 2):
                q = indices[:, 1:] + pad - taps[k] * dil
                valid = ok_batch & np.all((q >= 0) & (q < dims), axis=1)
                rows = np.nonzero(valid)[0]
                qk = linear_keys(np.concatenate([indices[rows, :1], q[rows]], 1), spatial_shape)
                pos = np.minimum(np.searchsorted(ukeys, qk), len(ukeys) - 1)
                hit = ukeys[pos] == qk
                i_rows, hits = rows[hit], first[pos[hit]]
                pairs[k] = (i_rows, hits)
                pairs[self.kv - 1 - k] = (hits, i_rows)
            pairs[self.kv // 2] = (np.arange(n), np.arange(n))
            self.out_inds = indices.astype(np.int32)
            self.out_shape = list(spatial_shape)
            self.n_in, self.n_out = n, n
            self.pairs = pairs
            return
        if kind == "inverse":
            fwd = SparseConvRef(indices, batch_size, spatial_shape, ksize, stride, padding, dilation, output_padding,
                                "conv")
            self.paired = fwd
            self.out_inds = indices.astype(np.int32)
            self.in_inds = fwd.out_inds
            self.out_shape = list(spatial_shape)
            self.n_in, self.n_out = fwd.n_out, fwd.n_in
            self.pairs = [(o, i) for i, o in fwd.pairs]
            return
        s = np.asarray(stride, np.int64)
        p = np.asarray(padding, np.int64)
        d = np.asarray(dilation, np.int64)
        if kind == "transpose":
            out_shape = deconv_output_size(spatial_shape, ksize, stride, padding, output_padding)
        else:
            out_shape = conv_output_size(spatial_shape, ksize, stride, padding, dilation)
        dims = np.asarray(out_shape, np.int64)
        cand_rows, cand_keys, cand_coords = [], [], []
        for k in range(self.kv):
            if kind == "transpose":
                o = indices[:, 1:] * s - p + taps[k] * d
                valid = np.ones(n, bool)
            else:
                h = indices[:, 1:] + p - taps[k] * d
                valid = np.all((h >= 0) & (h % s == 0), axis=1)
                o = h // s
            valid &= ok_batch & np.all((o >= 0) & (o < dims), axis=1)
            rows = np.nonzero(valid)[0]
            c = np.concatenate([indices[rows, :1], o[rows]], 1)
            cand_rows.append(rows)
            cand_coords.append(c)
            cand_keys.append(linear_keys(c, out_shape))
        all_keys = np.concatenate(cand_keys)
        all_coords = np.concatenate(cand_coords)
        ukeys, first = np.unique(all_keys, return_index=True)
        rank_order = np.argsort(first, kind="stable")              # first-touch rank of every key
        rank = np.empty_like(rank_order)
        rank[rank_order] = np.arange(len(rank_order))
        self.out_inds = all_coords[first[rank_order]].astype(np.int32).reshape(-1, ndim + 1)
        self.out_shape = out_shape
        self.n_in, self.n_out = n, len(ukeys)
        self.pairs = []
        for rows, keys in zip(cand_rows, cand_keys):
            self.pairs.append((rows, rank[np.searchsorted(ukeys, keys)] if len(keys) else keys.astype(np.int64)))

    # ------------------------------------------------------------------ values
    def _scatter(self, k: int, transpose: bool = False) -> sp.csr_matrix:
        """[n_out, n_in] 0/1 matrix of offset k (its transpose with transpose=True); repeated pairs add."""
        i, o = self.pairs[k]
        m = sp.coo_matrix((np.ones(len(i)), (o, i)), shape=(self.n_out, self.n_in)).tocsr()
        return m.T.tocsr() if transpose else m

    def forward(self, x: np.ndarray, w: np.ndarray, bias: Optional[np.ndarray] = None):
        """(out [n_out, K], sum|terms| [n_out, K], terms [n_out]) in float64; w is KRSC."""
        x = np.asarray(x, np.float64)
        K, C = w.shape[0], w.shape[-1]
        wk = np.asarray(w, np.float64).reshape(K, self.kv, C)
        out = np.zeros((self.n_out, K))
        mag = np.zeros((self.n_out, K))
        cnt = np.zeros(self.n_out)
        for k in range(self.kv):
            if not len(self.pairs[k][0]):
                continue
            s = self._scatter(k)
            out += s @ (x @ wk[:, k].T)
            mag += s @ (np.abs(x) @ np.abs(wk[:, k]).T)
            cnt += np.asarray(s.sum(axis=1)).ravel()
        if bias is not None:
            out += np.asarray(bias, np.float64)
            mag += np.abs(np.asarray(bias, np.float64))
            cnt += 1
        return out, mag, cnt * C

    def backward(self, x: np.ndarray, w: np.ndarray, dy: np.ndarray):
        """(dx, |dx| terms, dx term count, dw KRSC, |dw| terms, dw term count [kv]) in float64."""
        x = np.asarray(x, np.float64)
        dy = np.asarray(dy, np.float64)
        K, C = w.shape[0], w.shape[-1]
        wk = np.asarray(w, np.float64).reshape(K, self.kv, C)
        dx = np.zeros((self.n_in, C))
        dx_mag = np.zeros((self.n_in, C))
        dx_cnt = np.zeros(self.n_in)
        dw = np.zeros((K, self.kv, C))
        dw_mag = np.zeros((K, self.kv, C))
        dw_cnt = np.zeros(self.kv)
        for k in range(self.kv):
            i, o = self.pairs[k]
            if not len(i):
                continue
            st = self._scatter(k, transpose=True)                 # [n_in, n_out]
            dx += st @ (dy @ wk[:, k])
            dx_mag += st @ (np.abs(dy) @ np.abs(wk[:, k]))
            dx_cnt += np.asarray(st.sum(axis=1)).ravel()
            g = st.T @ x                                          # [n_out, C]: per output, sum of its inputs
            dw[:, k] = dy.T @ g
            dw_mag[:, k] = np.abs(dy).T @ (st.T @ np.abs(x))
            dw_cnt[k] = len(i)
        return dx, dx_mag, dx_cnt * K, dw.reshape(w.shape), dw_mag.reshape(w.shape), dw_cnt

    def pair_set(self) -> List[set]:
        """per offset, the set of (in_row, out_row) pairs"""
        return [set(zip(i.tolist(), o.tolist())) for i, o in self.pairs]
