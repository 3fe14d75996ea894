"""Operator layer: the drop-in boundary of the hot path.

Same function names, argument order and return shapes as ``spconv/pytorch/ops.py``
(``get_indice_pairs`` :132, ``get_indice_pairs_implicit_gemm`` :329, ``indice_conv`` :811,
``indice_conv_backward`` :1103, ``implicit_gemm`` :1450, ``implicit_gemm_backward`` :1667),
implemented as thin calls into the C-ABI library (``include/spconv_b200.h``) on the current
CUDA stream.  CUDA tensors only: there is deliberately no CPU path in the product.

Differences a reference user can observe (all documented in DESIGN.md):
  * rulebooks are deterministic and bit-equal to the reference's CPU order;
  * ``mask_width`` is always 128 (the tensor-core tile height);
  * ``ConvAlgo.MaskSplitImplicitGemm`` builds the reference's two mask splits (offsets
    ``[0, kv - kv//2)`` and the rest, ``ops.py:494-503``), sorts each on its own and runs one kernel
    pass per split, summing the partial outputs (the reference accumulates with beta = 1).
"""
from __future__ import annotations

import ctypes
import functools
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _cabi
from ..constants import SPCONV_ALLOW_TF32, SPCONV_DO_SORT
from ..core import Activation, ConvAlgo
from .core import CUDAKernelTimer, ThrustSortAllocator

INT32_MAX = 2147483647
MASK_WIDTH = 128

_DTYPE_CODE = {
    torch.float32: _cabi.SPX_F32,
    torch.float16: _cabi.SPX_F16,
    torch.bfloat16: _cabi.SPX_BF16,
    torch.int8: _cabi.SPX_I8,
    torch.float8_e4m3fn: _cabi.SPX_E4M3,
}


# ---------------------------------------------------------------------------- small helpers
def _lib():
    return _cabi.load()


_raw_stream = torch._C._cuda_getCurrentRawStream
_cur_device = torch._C._cuda_getDevice


def _stream() -> int:
    """cudaStream_t of torch's current stream on the current device.  (``torch.cuda.current_stream()``
    costs ~4 us of Python per call -- 76 calls per encoder step were a fifth of the eager host time.)"""
    return _raw_stream(_cur_device())


def _prod(xs) -> int:
    r = 1
    for x in xs:
        r *= int(x)
    return r


_SIDE_STREAMS: dict = {}


def _side_stream(device: torch.device) -> "torch.cuda.Stream":
    """One auxiliary stream per device for the input-gradient kernel (see implicit_gemm_backward)."""
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    st = _SIDE_STREAMS.get(key)
    if st is None:
        st = _SIDE_STREAMS[key] = torch.cuda.Stream(device=key)
    return st


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _dense(t: torch.Tensor) -> torch.Tensor:
    """``t`` itself when it is contiguous and 16-byte aligned, else a contiguous copy.  The tensor-core GEMMs, the
    pooling and the rulebook kernels read rows as 16-byte vectors; a contiguous view at an odd element offset
    (an autograd gradient sliced out of a ``torch.cat``, a parameter in a flat buffer) would send the GEMMs to
    the FMA kernels and make the others refuse the call.  The copy keeps every public call on the same kernels,
    with the same bits, as an aligned one."""
    if t.is_contiguous() and t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=torch.contiguous_format)


def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            f"spconv_b200: {what} must be a CUDA tensor. This engine has no CPU path "
            "(the CPU restatement under oracle/ is test infrastructure only).")


def _bytes(n: int, device, alloc: Optional[ThrustSortAllocator] = None) -> torch.Tensor:
    if alloc is not None:
        return alloc.get(n)
    return torch.empty(max(int(n), 1), dtype=torch.uint8, device=device)


def _act_code(act_type) -> int:
    if act_type is None:
        return _cabi.SPX_ACT_NONE
    if isinstance(act_type, Activation):
        return act_type.value
    return int(getattr(act_type, "value", act_type))


def get_conv_output_size(input_size, kernel_size, stride, padding, dilation):
    """``(in + 2p - d(k-1) - 1) // s + 1`` per axis; ``k == -1`` means global (size 1)."""
    return [1 if k == -1 else (i + 2 * p - d * (k - 1) - 1) // s + 1
            for i, k, s, p, d in zip(input_size, kernel_size, stride, padding, dilation)]


def get_deconv_output_size(input_size, kernel_size, stride, padding, dilation, output_padding):
    out = []
    for i, k, s, p, op in zip(input_size, kernel_size, stride, padding, output_padding):
        if k == -1:
            raise ValueError("deconv don't support kernel_size < 0")
        out.append((i - 1) * s - 2 * p + k + op)
    return out


_VANISHED = ("Your points vanished here, this usually because you provide conv params that "
             "may ignore some input points. Example: spatial_shape=[8, 200, 200] -> "
             "[3, 3, 3] kernel, [2, 2, 2] stride, no padding -> out shape [3, 99, 99]; "
             "points in z=7/8 are dropped when no point lies in z<=6.")


def _out_shape(spatial_shape, ksize, stride, padding, dilation, out_padding, subm, transpose):
    if subm:
        shape = list(spatial_shape)
    elif transpose:
        shape = get_deconv_output_size(spatial_shape, ksize, stride, padding, dilation, out_padding)
    else:
        shape = get_conv_output_size(spatial_shape, ksize, stride, padding, dilation)
    if any(x <= 0 for x in shape):
        raise ValueError(
            f"your out spatial shape {shape} reach zero!!! input shape: {spatial_shape}")
    return shape


_GEO_CACHE: dict = {}


def _geometry(indices, batch_size, spatial_shape, out_shape, ksize, stride, padding, dilation,
              transpose):
    ndim = indices.shape[1] - 1
    if not (1 <= ndim <= _cabi.SPX_MAX_NDIM):
        raise RuntimeError(f"unsupported ndim {ndim}")
    key = (ndim, int(batch_size), tuple(spatial_shape), tuple(out_shape), tuple(ksize), tuple(stride),
           tuple(padding), tuple(dilation), bool(transpose))
    geo = _GEO_CACHE.get(key)
    if geo is None:                      # the struct is immutable once built: layers re-use it every step
        if len(_GEO_CACHE) > 4096:
            _GEO_CACHE.clear()
        geo = _GEO_CACHE[key] = _cabi.make_geometry(ndim, batch_size, spatial_shape, out_shape, ksize, stride,
                                                    padding, dilation, transpose)
    return geo


_ZERO_COUNTS: dict = {}


def _zero_counts(kv: int, device) -> torch.Tensor:
    """``indice_num_per_loc`` of the implicit-GEMM rulebooks: not consumed by the GEMM (SURVEY A.5), kept
    for the shape of the reference's 9-tuple; one read-only zeros tensor per (kv, device)."""
    key = (kv, device)
    t = _ZERO_COUNTS.get(key)
    if t is None:
        t = _ZERO_COUNTS[key] = torch.zeros((kv,), dtype=torch.int32, device=device)
    return t


def _conv_stage1(geo, indices, n_in, ws) -> int:
    """Stage 1 of the regular-conv rulebook on workspace ``ws``: returns the output count M (one host sync)."""
    m_host = ctypes.c_int64(0)
    _cabi.check(_lib().spx_conv_rulebook_stage1(ctypes.byref(geo), _ptr(indices), n_in, ctypes.byref(m_host),
                                                ws.data_ptr(), ws.numel(), _stream()), "conv_rulebook_stage1")
    return int(m_host.value)


def _conv_rulebook(geo, indices, n_in, kv, words, want_masks, alloc):
    """Two-phase regular-conv rulebook; returns (out_inds, pair_fwd, pair_bwd, mask_fwd, mask_bwd).  With no outputs
    (M == 0) stage 2 does not run and pair_bwd is left unwritten: the caller decides what M == 0 means."""
    lib = _lib()
    dev = indices.device
    ws_bytes = lib.spx_rulebook_workspace_size(ctypes.byref(geo), n_in, 0, 0)
    ws = _bytes(ws_bytes, dev, alloc)
    m = _conv_stage1(geo, indices, n_in, ws)
    ndim = indices.shape[1] - 1
    out_inds = torch.empty((m, ndim + 1), dtype=torch.int32, device=dev)
    pair_fwd = torch.empty((kv, m), dtype=torch.int32, device=dev)
    pair_bwd = torch.empty((kv, n_in), dtype=torch.int32, device=dev)
    mask_fwd = torch.empty((1, m, words), dtype=torch.int32, device=dev) if want_masks else None
    mask_bwd = torch.empty((1, n_in, words), dtype=torch.int32, device=dev) if want_masks else None
    if m:
        _cabi.check(lib.spx_conv_rulebook_stage2(ctypes.byref(geo), _ptr(indices), n_in, m,
                                                 out_inds.data_ptr(), pair_fwd.data_ptr(),
                                                 pair_bwd.data_ptr(), _ptr(mask_fwd), _ptr(mask_bwd),
                                                 ws.data_ptr(), ws.numel(), _stream()),
                    "conv_rulebook_stage2")
    return out_inds, pair_fwd, pair_bwd, mask_fwd, mask_bwd


def _conv_rulebook_all(geo, indices, n_in, kv, words, is_train, do_sort, alloc, indice_num_per_loc, masks, bound=0,
                       status=None):
    """Regular-conv implicit-GEMM rulebook with its mask sorts and tile tables, as the reference's 9-tuple.

    ``bound == 0``: two native calls, stage 1 with its host read-back of the output count M, then stage 2.
    ``bound > 0`` (``spx_conv_rulebook_bounded_all``): one native call and no host read-back; every output-side
    tensor has ``bound`` rows, and the true count (device int32 ``[1]``) and the status word ride on ``out_inds`` as
    ``_spx_num_valid`` / ``_spx_bound_status``."""
    lib = _lib()
    dev = indices.device
    if bound:
        m = bound
        if n_in == 0:                    # host-known: the unbounded path raises the same error for M == 0
            raise ValueError(_VANISHED)
        ws = _bytes(lib.spx_conv_rulebook_bounded_workspace_size(ctypes.byref(geo), n_in, m), dev, alloc)
    else:
        ws = _bytes(lib.spx_conv_rulebook_all_workspace_size(ctypes.byref(geo), n_in), dev, alloc)
        m = _conv_stage1(geo, indices, n_in, ws)
        if m == 0:
            raise ValueError(_VANISHED)
    ndim = indices.shape[1] - 1
    out_inds = torch.empty((m, ndim + 1), dtype=torch.int32, device=dev)
    pair_fwd = torch.empty((kv, m), dtype=torch.int32, device=dev)
    pair_bwd = torch.empty((kv, n_in), dtype=torch.int32, device=dev)
    mask_fwd = torch.empty((1, m, words), dtype=torch.int32, device=dev)
    mask_bwd = torch.empty((1, n_in, words), dtype=torch.int32, device=dev)
    sort_fwd = torch.empty((1, m), dtype=torch.int32, device=dev)
    sort_bwd = torch.empty((1, n_in), dtype=torch.int32, device=dev) if is_train else None
    t_fwd, tm_fwd = _alloc_tile_tables(m, kv, dev)
    t_bwd, tm_bwd = _alloc_tile_tables(n_in, kv, dev) if is_train else (None, None)
    args = (ctypes.byref(geo), _ptr(indices), n_in, m, out_inds.data_ptr(), pair_fwd.data_ptr(), _ptr(pair_bwd),
            mask_fwd.data_ptr(), _ptr(mask_bwd), sort_fwd.data_ptr(), _ptr(sort_bwd), int(bool(do_sort)),
            _ptr(t_fwd), _ptr(tm_fwd), _ptr(t_bwd), _ptr(tm_bwd))
    if bound:
        num_out = torch.empty((1,), dtype=torch.int32, device=dev)
        if status is None:
            status = torch.zeros((1,), dtype=torch.int32, device=dev)
        _cabi.check(lib.spx_conv_rulebook_bounded_all(*args, num_out.data_ptr(), status.data_ptr(), ws.data_ptr(),
                                                      ws.numel(), _stream()), "conv_rulebook_bounded_all")
        out_inds._spx_num_valid = num_out
        out_inds._spx_bound_status = status
    else:
        _cabi.check(lib.spx_conv_rulebook_stage2_all(*args, ws.data_ptr(), ws.numel(), _stream()),
                    "conv_rulebook_stage2_all")
    sf = sort_fwd[0]
    sf._spx_tile_cache = (_tile_key(pair_fwd, sf, m), t_fwd, tm_fwd)
    if not is_train:
        return (out_inds, indice_num_per_loc, pair_fwd, pair_bwd, [mask_fwd[0]], [], [sf], [], masks)
    sb = sort_bwd[0]
    sb._spx_tile_cache = (_tile_key(pair_bwd, sb, n_in), t_bwd, tm_bwd)
    return (out_inds, indice_num_per_loc, pair_fwd, pair_bwd, [mask_fwd[0]], [mask_bwd[0]], [sf], [sb], masks)


def _argsort_masks(mask: torch.Tensor, kv: int, do_sort: bool, alloc) -> torch.Tensor:
    """mask [1, n, words] -> argsort [1, n]; mask is left sorted (thrust::sort_by_key semantics,
    ``spconv/csrc/sparse/all.py:935-1000``)."""
    lib = _lib()
    n, words = mask.shape[1], mask.shape[2]
    argsort = torch.empty((1, n), dtype=torch.int32, device=mask.device)
    if n == 0:
        return argsort
    ws_bytes = lib.spx_mask_argsort_workspace_size(n, words)
    ws = _bytes(ws_bytes, mask.device, alloc)
    _cabi.check(lib.spx_mask_argsort(mask.data_ptr(), argsort.data_ptr(), n, words, kv,
                                     int(bool(do_sort)), ws.data_ptr(), ws.numel(), _stream()),
                "mask_argsort")
    return argsort


def _split_and_sort(mask: torch.Tensor, masks: List[np.ndarray], kv: int, do_sort: bool, alloc):
    """mask [1, n, 1] (unsorted) -> per split j: (mask & masks[j]) sorted in place + its argsort
    (``ops.py:494-503,538-549``: every split is sorted on its own)."""
    mask_s, sort_s = [], []
    for m in masks:
        # a scalar operand, not a device tensor: no host-to-device copy, so the rulebook captures
        part = torch.bitwise_and(mask, int(m.view(np.int32)[0])).contiguous()
        sort_s.append(_argsort_masks(part, kv, do_sort, alloc)[0])
        mask_s.append(part[0])
    return mask_s, sort_s


# ---------------------------------------------------------------------------- rulebooks
def get_indice_pairs(indices: torch.Tensor, batch_size: int, spatial_shape: List[int],
                     algo: ConvAlgo, ksize: List[int], stride: List[int], padding: List[int],
                     dilation: List[int], out_padding: List[int], subm: bool = False,
                     transpose: bool = False, num_out_act_bound: int = -1):
    """ConvAlgo.Native rulebook: ``(out_inds [M, ndim+1], pairs [2, kv, N], indice_pair_num [kv])``
    with pair ORDER equal to the reference CPU implementation
    (``spconv/csrc/sparse/indices.py:1640-1778``).  ``num_out_act_bound`` is accepted and ignored: the
    Native rulebook always reads the output count back (only the masked implicit-GEMM rulebook has a
    bounded mode)."""
    _require_cuda(indices, "indices")
    lib = _lib()
    dev = indices.device
    indices = _dense(indices)
    n_in = indices.shape[0]
    kv = _prod(ksize)
    out_shape = _out_shape(spatial_shape, ksize, stride, padding, dilation, out_padding, subm,
                           transpose)
    geo = _geometry(indices, batch_size, spatial_shape, out_shape, ksize, stride, padding,
                    dilation, transpose)
    pairs = torch.empty((2, kv, n_in), dtype=torch.int32, device=dev)
    num = torch.empty((kv,), dtype=torch.int32, device=dev)
    if subm:
        for k in ksize:
            if k % 2 != 1:
                raise RuntimeError("subm only support odd ksize")
        pair_fwd = torch.empty((kv, n_in), dtype=torch.int32, device=dev)
        pair_bwd = torch.empty((kv, n_in), dtype=torch.int32, device=dev)
        ws = _bytes(lib.spx_rulebook_workspace_size(ctypes.byref(geo), n_in, 0, 1), dev)
        _cabi.check(lib.spx_subm_rulebook(ctypes.byref(geo), _ptr(indices), n_in,
                                          pair_fwd.data_ptr(), pair_bwd.data_ptr(), None,
                                          ws.data_ptr(), ws.numel(), _stream()), "subm_rulebook")
        out_inds = indices
    else:
        out_inds, pair_fwd, pair_bwd, _, _ = _conv_rulebook(geo, indices, n_in, kv,
                                                            (kv + 31) // 32, False, None)
        if out_inds.shape[0] == 0:
            raise ValueError(_VANISHED)
    ws2 = _bytes(lib.spx_native_pairs_workspace_size(n_in, kv), dev)
    _cabi.check(lib.spx_native_pairs(_ptr(pair_bwd), n_in, kv, int(subm), pairs.data_ptr(),
                                     num.data_ptr(), ws2.data_ptr(), ws2.numel(), _stream()),
                "native_pairs")
    return out_inds, pairs, num


def get_indice_pairs_implicit_gemm(indices: torch.Tensor, batch_size: int,
                                   spatial_shape: List[int], algo: ConvAlgo, ksize: List[int],
                                   stride: List[int], padding: List[int], dilation: List[int],
                                   out_padding: List[int], subm: bool = False,
                                   transpose: bool = False, is_train: bool = True,
                                   alloc: Optional[ThrustSortAllocator] = None,
                                   timer: CUDAKernelTimer = CUDAKernelTimer(False),
                                   num_out_act_bound: int = -1,
                                   direct_table: bool = True,
                                   do_sort=SPCONV_DO_SORT,
                                   bound_status: Optional[torch.Tensor] = None):
    """Masked implicit-GEMM rulebook.  Returns the reference's 9-tuple
    ``(out_inds, indice_num_per_loc, pair_fwd, pair_bwd, [mask_fwd], [mask_bwd],
    [argsort_fwd], [argsort_bwd], masks)`` (``ops.py:329-359``).

    ``num_out_act_bound = b > 0`` with ``subm=False`` and ``ConvAlgo.MaskImplicitGemm`` selects the bounded
    rulebook: no host read-back (CUDA-graph capturable), every output-side tensor has exactly ``b`` rows, the
    true count M stays on the device (``out_inds._spx_num_valid``, int32 ``[1]``) and rows ``[M, b)`` are
    padding (``out_inds`` -1, pairs -1, mask 0).  Rows below M are bit-identical to the unbounded rulebook.
    ``out_inds._spx_bound_status`` (``bound_status`` if given, which is only ever ORed into) has bit 0 set when
    more than ``b`` outputs existed (those ranked >= b were dropped) and bit 1 when the hash table sized from
    ``b`` overflowed.  SubM and ``MaskSplitImplicitGemm`` ignore the bound."""
    _require_cuda(indices, "indices")
    assert algo in (ConvAlgo.MaskImplicitGemm, ConvAlgo.MaskSplitImplicitGemm), "TODO"
    lib = _lib()
    dev = indices.device
    indices = _dense(indices)
    n_in = indices.shape[0]
    kv = _prod(ksize)
    words = (kv + 31) // 32
    if kv > 128:
        raise NotImplementedError("masked implicit gemm supports kernel volume <= 128")
    out_shape = _out_shape(spatial_shape, ksize, stride, padding, dilation, out_padding, subm,
                           transpose)
    geo = _geometry(indices, batch_size, spatial_shape, out_shape, ksize, stride, padding,
                    dilation, transpose)
    is_split = algo == ConvAlgo.MaskSplitImplicitGemm
    if is_split:
        assert words == 1, "Not Implemented"                    # reference: ops.py:495
        remain = kv - kv // 2
        masks = [np.array([(1 << remain) - 1], dtype=np.uint32),
                 np.array([((1 << (kv // 2)) - 1) << remain], dtype=np.uint32)]
    else:
        masks = [np.array([0xffffffff], dtype=np.uint32)]
    # per-offset pair counts are not consumed by the GEMM (SURVEY A.5); kept for API shape
    indice_num_per_loc = _zero_counts(kv, dev)
    if subm:
        for k in ksize:
            if k % 2 != 1:
                raise RuntimeError("subm only support odd ksize")
        pair = torch.empty((2 if is_train else 1, kv, n_in), dtype=torch.int32, device=dev)
        pair_mask = torch.empty((1, n_in, words), dtype=torch.int32, device=dev)
        pair_bwd = pair[1] if is_train else torch.Tensor()
        if is_split:
            # the splits AND the unsorted mask with their constants: separate rulebook and sort calls
            with timer.record("gen_subm_inds", _stream()):
                ws = _bytes(lib.spx_rulebook_workspace_size(ctypes.byref(geo), n_in, 0, 1), dev, alloc)
                _cabi.check(lib.spx_subm_rulebook(ctypes.byref(geo), _ptr(indices), n_in, pair[0].data_ptr(),
                                                  pair[1].data_ptr() if is_train and n_in else None,
                                                  _ptr(pair_mask), ws.data_ptr(), ws.numel(), _stream()),
                            "subm_rulebook")
            with timer.record("gen_subm_inds_sort", _stream()):
                mask_s, sort_s = _split_and_sort(pair_mask, masks, kv, do_sort, alloc)
            return (indices, indice_num_per_loc, pair[0], pair_bwd, mask_s, [], sort_s, [], masks)
        # one native call: hash + probe + mask sort + tile table
        mask_argsort = torch.empty((1, n_in), dtype=torch.int32, device=dev)
        table, tile_mask = _alloc_tile_tables(n_in, kv, dev)
        with timer.record("gen_subm_inds", _stream()):
            ws = _bytes(lib.spx_subm_rulebook_all_workspace_size(ctypes.byref(geo), n_in), dev, alloc)
            _cabi.check(lib.spx_subm_rulebook_all(
                ctypes.byref(geo), _ptr(indices), n_in, pair[0].data_ptr(), pair[1].data_ptr() if is_train else None,
                _ptr(pair_mask), _ptr(mask_argsort), int(bool(do_sort)), _ptr(table), _ptr(tile_mask),
                ws.data_ptr(), ws.numel(), _stream()), "subm_rulebook_all")
        argsort_view = mask_argsort[0]
        argsort_view._spx_tile_cache = (_tile_key(pair[0], argsort_view, n_in), table, tile_mask)
        return (indices, indice_num_per_loc, pair[0], pair_bwd, [pair_mask[0]], [], [argsort_view], [], masks)
    if is_split:
        # the splits AND the unsorted masks with their constants: separate rulebook and sort calls
        with timer.record("gen_conv_inds", _stream()):
            out_inds, pair_fwd, pair_bwd, mask_fwd, mask_bwd = _conv_rulebook(
                geo, indices, n_in, kv, words, True, alloc)
            if out_inds.shape[0] == 0:
                raise ValueError(_VANISHED)
        with timer.record("gen_conv_inds_sort", _stream()):
            mf, sf = _split_and_sort(mask_fwd, masks, kv, do_sort, alloc)
            mb, sb = _split_and_sort(mask_bwd, masks, kv, do_sort, alloc) if is_train else ([], [])
        return (out_inds, indice_num_per_loc, pair_fwd, pair_bwd, mf, mb, sf, sb, masks)
    bound = int(num_out_act_bound) if num_out_act_bound is not None and int(num_out_act_bound) > 0 else 0
    with timer.record("gen_conv_inds", _stream()):
        return _conv_rulebook_all(geo, indices, n_in, kv, words, is_train, do_sort, alloc, indice_num_per_loc, masks,
                                  bound, bound_status)


def _row_count(num_valid: Optional[torch.Tensor], what: str) -> Optional[torch.Tensor]:
    if num_valid is None:
        return None
    _require_cuda(num_valid, what)
    if num_valid.dtype != torch.int32 or num_valid.numel() != 1:
        raise ValueError(f"{what} must be a device int32 tensor of one element, got {num_valid.dtype} "
                         f"{tuple(num_valid.shape)}")
    return num_valid


def get_indice_pairs_to(indices: torch.Tensor, out_indices: torch.Tensor, batch_size: int,
                        spatial_shape: List[int], out_spatial_shape: List[int], ksize: List[int], stride: List[int],
                        padding: List[int], dilation: List[int], transpose: bool, is_train: bool,
                        num_valid: Optional[torch.Tensor] = None, out_num_valid: Optional[torch.Tensor] = None,
                        do_sort: bool = True):
    """Masked implicit-GEMM rulebook of a convolution from ``indices`` (grid ``spatial_shape``) onto the given
    coordinates ``out_indices`` (grid ``out_spatial_shape``), ``spx_cross_rulebook_all``.  Returns the 9-tuple of
    :func:`get_indice_pairs_implicit_gemm` with ``out_inds = out_indices``.

    The geometry is taken as given (a SubM layer passes stride 1 and padding ``(k // 2) * d``).  Source rows from
    ``num_valid`` on, rows whose batch or coordinates are out of range and all but the lowest row of a duplicated
    coordinate take part in no pair; the same holds for the target rows against ``out_num_valid`` and
    ``out_spatial_shape``.  Target row o reads source coordinate ``o * s - p + r * d`` per axis (regular) or
    ``(o + p - r * d) / s`` when exact (``transpose``).  ``pair_bwd`` and the backward mask are always built; their
    argsort and tile table only with ``is_train``.  The output count is the caller's, so nothing is read back and
    the call captures in a CUDA graph."""
    _require_cuda(indices, "indices")
    _require_cuda(out_indices, "out_indices")
    for t, what in ((indices, "indices"), (out_indices, "out_indices")):
        if t.dtype != torch.int32 or t.dim() != 2:
            raise ValueError(f"{what} must be int32 [rows, ndim + 1], got {t.dtype} {tuple(t.shape)}")
    ndim = indices.shape[1] - 1
    if out_indices.shape[1] != ndim + 1 or len(spatial_shape) != ndim or len(out_spatial_shape) != ndim:
        raise ValueError(f"source {tuple(indices.shape)} / target {tuple(out_indices.shape)} indices and the shapes "
                         f"{list(spatial_shape)} / {list(out_spatial_shape)} must have the same ndim")
    kv = _prod(ksize)
    if kv > 128:
        raise NotImplementedError("a rulebook onto given coordinates supports kernel volume <= 128")
    num_valid = _row_count(num_valid, "num_valid")
    out_num_valid = _row_count(out_num_valid, "out_num_valid")
    lib = _lib()
    dev = indices.device
    indices, out_indices = _dense(indices), _dense(out_indices)
    n_in, m = indices.shape[0], out_indices.shape[0]
    words = (kv + 31) // 32
    geo = _geometry(indices, batch_size, spatial_shape, out_spatial_shape, ksize, stride, padding, dilation, transpose)
    pair_fwd = torch.empty((kv, m), dtype=torch.int32, device=dev)
    pair_bwd = torch.empty((kv, n_in), dtype=torch.int32, device=dev)
    mask_fwd = torch.empty((1, m, words), dtype=torch.int32, device=dev)
    mask_bwd = torch.empty((1, n_in, words), dtype=torch.int32, device=dev)
    sort_fwd = torch.empty((1, m), dtype=torch.int32, device=dev)
    sort_bwd = torch.empty((1, n_in), dtype=torch.int32, device=dev) if is_train else None
    t_fwd, tm_fwd = _alloc_tile_tables(m, kv, dev)
    t_bwd, tm_bwd = _alloc_tile_tables(n_in, kv, dev) if is_train else (None, None)
    ws = _bytes(lib.spx_cross_rulebook_all_workspace_size(ctypes.byref(geo), n_in, m), dev)
    _cabi.check(lib.spx_cross_rulebook_all(
        ctypes.byref(geo), _ptr(indices), n_in, _ptr(num_valid), _ptr(out_indices), m, _ptr(out_num_valid),
        _ptr(pair_fwd), _ptr(pair_bwd), _ptr(mask_fwd), _ptr(mask_bwd), _ptr(sort_fwd), _ptr(sort_bwd),
        int(bool(do_sort)), _ptr(t_fwd), _ptr(tm_fwd), _ptr(t_bwd), _ptr(tm_bwd), ws.data_ptr(), ws.numel(),
        _stream()), "cross_rulebook_all")
    masks = [np.array([0xffffffff], dtype=np.uint32)]
    sf = sort_fwd[0]
    sf._spx_tile_cache = (_tile_key(pair_fwd, sf, m), t_fwd, tm_fwd)
    res = (out_indices, _zero_counts(kv, dev), pair_fwd, pair_bwd, [mask_fwd[0]])
    if not is_train:
        return (*res, [], [sf], [], masks)
    sb = sort_bwd[0]
    sb._spx_tile_cache = (_tile_key(pair_bwd, sb, n_in), t_bwd, tm_bwd)
    return (*res, [mask_bwd[0]], [sf], [sb], masks)


# ---------------------------------------------------------------------------- GEMM descriptor
def _f32_mode() -> int:
    return _cabi.SPX_F32_TF32 if SPCONV_ALLOW_TF32 else _cabi.SPX_F32_EXACT


def _tile_key(pair: torch.Tensor, argsort: Optional[torch.Tensor], rows: int):
    return (pair.data_ptr(), tuple(pair.shape), pair._version,
            None if argsort is None else (argsort.data_ptr(), argsort._version), int(rows))


def _alloc_tile_tables(rows: int, kv: int, device):
    tiles = max((int(rows) + MASK_WIDTH - 1) // MASK_WIDTH, 1)
    # layout of include/spconv_b200.h: blocks + schedule records + scheduler scratch (== spx_tile_table_elems)
    table = torch.empty((tiles * (kv + 1) * 128 + tiles * 8 + 64,), dtype=torch.int32, device=device)
    tile_mask = torch.empty((tiles, (kv + 31) // 32), dtype=torch.int32, device=device)
    return table, tile_mask


def _tile_tables(pair: torch.Tensor, mask: Optional[torch.Tensor], argsort: Optional[torch.Tensor],
                 rows: int, kv: int, owner: Optional[torch.Tensor] = None):
    """Tile-blocked gather table + per-tile OR masks for (pair, mask, argsort)
    (``spx_build_tile_table``).  Built once per rulebook and cached on ``owner`` (the argsort
    tensor that lives in the cached ``ImplicitGemmIndiceData``), so forward, input-gradient and
    weight-gradient of every layer sharing the ``indice_key`` reuse it."""
    key = _tile_key(pair, argsort, rows)
    if owner is not None:
        hit = getattr(owner, "_spx_tile_cache", None)
        if hit is not None and hit[0] == key:
            return hit[1], hit[2]
    lib = _lib()
    table, tile_mask = _alloc_tile_tables(rows, kv, pair.device)
    _cabi.check(lib.spx_build_tile_table(_ptr(pair), int(pair.stride(0)), kv, _ptr(argsort), _ptr(mask),
                                         int(rows), _ptr(table), _ptr(tile_mask), _stream()),
                "build_tile_table")
    if owner is not None:
        owner._spx_tile_cache = (key, table, tile_mask)
    return table, tile_mask


def _desc(dtype, kv, c_in, c_out, n_in, n_out, pair, mask, argsort, reverse=False, tiles=None):
    d = _cabi.GemmDesc()
    d.dtype = _DTYPE_CODE[dtype]
    d.f32_mode = _f32_mode()
    d.kv, d.c_in, d.c_out = int(kv), int(c_in), int(c_out)
    d.n_in, d.n_out = int(n_in), int(n_out)
    d.pair = _ptr(pair)
    d.pair_stride = int(pair.stride(0)) if pair is not None and pair.dim() == 2 else 0
    d.mask = _ptr(mask)
    d.argsort = _ptr(argsort)
    d.reverse_offsets = int(bool(reverse))
    if tiles is not None:
        d.tile_table = _ptr(tiles[0])
        d.tile_mask = _ptr(tiles[1])
    return d


def _check_filter(features, filters, groups=1):
    """``(kv, C, K)`` of the KRSC filter ``[K, *ksize, C / groups]``"""
    if filters.dtype != features.dtype:
        raise RuntimeError(f"features ({features.dtype}) and filters ({filters.dtype}) must have the same dtype")
    if features.dtype not in _DTYPE_CODE:
        raise RuntimeError(f"unsupported dtype {features.dtype}")
    kv = _prod(filters.shape[1:-1])
    if groups == 1:
        return kv, int(filters.shape[-1]), int(filters.shape[0])
    if groups < 1 or int(filters.shape[0]) % groups:
        raise RuntimeError(f"groups {groups} must divide the filter's {int(filters.shape[0])} output channels")
    if features.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise NotImplementedError(f"grouped conv: {features.dtype} is not supported (float32, float16, bfloat16)")
    return kv, int(filters.shape[-1]) * groups, int(filters.shape[0])


# grouped conv (groups > 1): each call runs one dense GEMM pass per group (include/spconv_b200.h)
def _grouped_fwd(d, groups, features, filters, out, bias, act_code, act_alpha, what):
    a = _cabi.GroupedGemm(features=_ptr(features), filters=_ptr(filters), bias=_ptr(bias), out=_ptr(out),
                          act=act_code, act_alpha=float(act_alpha))
    _cabi.check(_lib().spx_grouped_gemm_fwd(ctypes.byref(d), int(groups), ctypes.byref(a), _stream()), what)


def _grouped_dgrad(d, groups, out_bp, filters, din, what):
    a = _cabi.GroupedGemm(out_bp=_ptr(out_bp), filters=_ptr(filters), din=_ptr(din))
    _cabi.check(_lib().spx_grouped_gemm_dgrad(ctypes.byref(d), int(groups), ctypes.byref(a), _stream()), what)


def _grouped_wgrad(d, groups, features, out_bp, dfilters, ws, group, what):
    """``group``: None, or the peer group (``ctypes.byref``) that dW is pushed to once written"""
    a = _cabi.GroupedGemm(features=_ptr(features), out_bp=_ptr(out_bp), dfilters=_ptr(dfilters),
                          workspace=ws.data_ptr(), workspace_bytes=ws.numel())
    if group is not None:
        _cabi.check(_lib().spx_grouped_gemm_wgrad_push(ctypes.byref(d), int(groups), ctypes.byref(a), group, _stream()),
                    what + "_push")
    else:
        _cabi.check(_lib().spx_grouped_gemm_wgrad(ctypes.byref(d), int(groups), ctypes.byref(a), _stream()), what)


def _wgrad_workspace(d, groups, device):
    lib = _lib()
    if groups == 1:
        return _bytes(lib.spx_implicit_gemm_wgrad_workspace_size(ctypes.byref(d)), device)
    return _bytes(lib.spx_grouped_gemm_wgrad_workspace_size(ctypes.byref(d), int(groups)), device)


def _first(split_list):
    if isinstance(split_list, (list, tuple)):
        return split_list[0] if len(split_list) else None
    return split_list


# ---------------------------------------------------------------------------- masked implicit GEMM
def implicit_gemm(features: torch.Tensor, filters: torch.Tensor, pair_fwd: torch.Tensor,
                  pair_mask_fwd_splits: List[torch.Tensor],
                  mask_argsort_fwd_splits: List[torch.Tensor], num_activate_out: int,
                  masks: List[np.ndarray], is_train: bool, is_subm: bool,
                  timer: CUDAKernelTimer = CUDAKernelTimer(False),
                  fp32_accum: Optional[bool] = None, bias: Optional[torch.Tensor] = None,
                  act_alpha: float = 0.0, act_beta: float = 0.0,
                  act_type=Activation.None_, output_scale: float = 1.0,
                  scale: Optional[torch.Tensor] = None, output_add: Optional[torch.Tensor] = None,
                  output_add_scale: float = 0.0, output_dtype: Optional[torch.dtype] = None,
                  in_scale: Optional[torch.Tensor] = None, out_scale: Optional[torch.Tensor] = None,
                  add_scale: Optional[torch.Tensor] = None, groups: int = 1):
    """Forward masked implicit GEMM -> ``(out [M, K], mask_output_fwd, mask_width)``
    (``ops.py:1450-1469`` / ``convops.py:2075-2243``).  Accumulation is always fp32 in registers
    (``fp32_accum`` is accepted and ignored).

    ``torch.float8_e4m3fn`` features and filters run ``spx_implicit_gemm_fwd_fp8``: ``scale`` is the filter's
    per-output-channel scale, ``in_scale`` / ``out_scale`` / ``add_scale`` are device fp32 ``[1]`` scales of the
    features, an e4m3 output and an e4m3 ``output_add``; ``output_dtype`` is float32 / float16 / bfloat16 or
    float8_e4m3fn (default: float8_e4m3fn, as the features).

    ``groups > 1``: a grouped conv, filters ``[K, kv, C / groups]`` (float32 / float16 / bfloat16)."""
    _require_cuda(features, "features")
    lib = _lib()
    features = _dense(features)
    filters = _dense(filters)
    kv, c_in, c_out = _check_filter(features, filters, groups)
    assert features.shape[1] == c_in, "channel size mismatch"
    n_in, n_out = features.shape[0], int(num_activate_out)
    n_splits = len(pair_mask_fwd_splits) if isinstance(pair_mask_fwd_splits, (list, tuple)) else 1
    if n_splits > 1:
        return _implicit_gemm_splits(features, filters, pair_fwd, pair_mask_fwd_splits,
                                     mask_argsort_fwd_splits, n_out, is_train, timer, bias, act_alpha,
                                     act_type, output_add, output_dtype, groups=groups)
    mask = _first(pair_mask_fwd_splits)
    argsort = _first(mask_argsort_fwd_splits)
    is_int8 = features.dtype == torch.int8
    if output_dtype is None:
        output_dtype = features.dtype
    words = (kv + 31) // 32
    with timer.record("tile_table", _stream()):
        tiles = _tile_tables(pair_fwd, mask, argsort, n_out, kv, owner=argsort) if n_out else None
    # mask_output_fwd (per-128-row OR of the sorted masks) is the tile table's mask block
    mask_output = tiles[1].view(1, -1, words) if (is_train and tiles is not None) else torch.Tensor()
    d = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, pair_fwd, mask, argsort, tiles=tiles)
    if features.dtype == torch.float8_e4m3fn:
        out = _implicit_gemm_fp8(d, features, filters, n_out, c_out, scale, bias, output_add, output_dtype, in_scale,
                                 out_scale, add_scale, act_type, act_alpha, timer)
        return out, mask_output, MASK_WIDTH
    if is_int8:
        assert scale is not None, "int8 implicit gemm needs the per-channel scale"
        out = torch.empty((n_out, c_out), dtype=output_dtype, device=features.device)
        # reference int8 epilogue (convops.py:2176-2206): per-channel `scale` multiplies the int32
        # accumulator, the residual enters with beta = output_add_scale / output_scale
        scale_f = scale.float().contiguous()
        bias_f = bias.float().contiguous() if bias is not None else None
        if output_add is not None:
            # the epilogue reads the residual as int8 [n_out, c_out] rows
            _require_cuda(output_add, "output_add")
            if output_add.dtype != torch.int8 or tuple(output_add.shape) != (n_out, c_out):
                raise RuntimeError(f"int8 implicit gemm: output_add must be int8 of shape {(n_out, c_out)}, got "
                                   f"{output_add.dtype} {tuple(output_add.shape)}")
            output_add = _dense(output_add)
        with timer.record("implicit_gemm_int8", _stream()):
            _cabi.check(lib.spx_implicit_gemm_fwd_int8(
                ctypes.byref(d), _ptr(features), _ptr(filters), _ptr(out), _DTYPE_CODE[output_dtype],
                _ptr(scale_f), _ptr(bias_f), _ptr(output_add),
                float(output_add_scale) / float(output_scale if output_scale else 1.0),
                _act_code(act_type), float(act_alpha), _stream()), "implicit_gemm_fwd_int8")
        return out, mask_output, MASK_WIDTH
    out = torch.empty((n_out, c_out), dtype=features.dtype, device=features.device)
    if bias is not None:
        bias = bias.to(features.dtype).contiguous()
    with timer.record("implicit_gemm", _stream()):
        if groups != 1:
            _grouped_fwd(d, groups, features, filters, out, bias, _act_code(act_type), act_alpha, "grouped_gemm_fwd")
        else:
            _cabi.check(lib.spx_implicit_gemm_fwd(ctypes.byref(d), _ptr(features), _ptr(filters),
                                                  _ptr(out), _ptr(bias), _act_code(act_type),
                                                  float(act_alpha), _stream()), "implicit_gemm_fwd")
    if output_add is not None:
        out = out + output_add
    if output_dtype != out.dtype:
        out = out.to(output_dtype)
    return out, mask_output, MASK_WIDTH


_FP8_OUT = (torch.float32, torch.float16, torch.bfloat16, torch.float8_e4m3fn)


def _scale_operand(t: Optional[torch.Tensor], n: int, what: str) -> Optional[torch.Tensor]:
    if t is None:
        return None
    _require_cuda(t, what)
    if t.numel() != n:
        raise RuntimeError(f"fp8 implicit gemm: {what} must have {n} element(s), got {t.numel()}")
    return t.reshape(-1).float().contiguous()


def _implicit_gemm_fp8(d, features, filters, n_out, c_out, w_scale, bias, output_add, output_dtype, in_scale,
                       out_scale, add_scale, act_type, act_alpha, timer):
    """The fp8 route of :func:`implicit_gemm`: every scale stays on the device."""
    if output_dtype not in _FP8_OUT:
        raise RuntimeError(f"fp8 implicit gemm: output dtype {output_dtype} not supported")
    if in_scale is None or w_scale is None:
        raise RuntimeError("fp8 implicit gemm needs the features' scale (in_scale) and the filter's scale")
    if output_dtype == torch.float8_e4m3fn and out_scale is None:
        raise RuntimeError("fp8 implicit gemm: an e4m3 output needs out_scale")
    in_scale = _scale_operand(in_scale, 1, "in_scale")
    w_scale = _scale_operand(w_scale, c_out, "the filter scale")
    out_scale = _scale_operand(out_scale, 1, "out_scale")
    add_scale = _scale_operand(add_scale, 1, "add_scale")
    bias = _scale_operand(bias, c_out, "bias")
    if output_add is not None:
        _require_cuda(output_add, "output_add")
        if output_add.dtype != output_dtype or tuple(output_add.shape) != (n_out, c_out):
            raise RuntimeError(f"fp8 implicit gemm: output_add must be {output_dtype} of shape {(n_out, c_out)}, got "
                               f"{output_add.dtype} {tuple(output_add.shape)}")
        if output_dtype == torch.float8_e4m3fn and add_scale is None:
            raise RuntimeError("fp8 implicit gemm: an e4m3 output_add needs add_scale")
        output_add = _dense(output_add)
    out = torch.empty((n_out, c_out), dtype=output_dtype, device=features.device)
    with timer.record("implicit_gemm_fp8", _stream()):
        a = _cabi.Fp8Gemm(_ptr(features), _ptr(filters), _ptr(in_scale), _ptr(w_scale), _ptr(bias), _ptr(output_add),
                          _ptr(add_scale), _ptr(out), _DTYPE_CODE[output_dtype], _ptr(out_scale), _act_code(act_type),
                          float(act_alpha))
        _cabi.check(_lib().spx_implicit_gemm_fwd_fp8(ctypes.byref(d), ctypes.byref(a), _stream()), "implicit_gemm_fwd_fp8")
    return out


def fp8_quantize(x: torch.Tensor, num_valid: Optional[torch.Tensor] = None,
                 scale: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 / fp16 / bf16 rows ``x [N, C]`` -> ``(e4m3 rows, device scale fp32 [1])`` (``spx_fp8_quantize``):
    with ``scale`` the given scale, else amax / 448 of the rows below ``num_valid``.  Rows from ``num_valid`` on
    are 0."""
    _require_cuda(x, "features")
    if x.dtype not in (torch.float32, torch.float16, torch.bfloat16) or x.dim() != 2:
        raise RuntimeError(f"fp8_quantize: x must be 2-D float32 / float16 / bfloat16, got {x.dtype} {tuple(x.shape)}")
    x = _dense(x)
    rows, ch = int(x.shape[0]), int(x.shape[1])
    out = torch.empty((rows, ch), dtype=torch.float8_e4m3fn, device=x.device)
    if scale is not None:
        scale = _scale_operand(scale, 1, "scale")
        scale_out, ws = scale, None
    else:
        scale_out = torch.empty((1,), dtype=torch.float32, device=x.device)
        ws = _bytes(_lib().spx_fp8_quantize_workspace_size(rows, ch), x.device)
    if num_valid is not None:
        _require_cuda(num_valid, "num_valid")
        num_valid = num_valid.to(torch.int32)
    q = _cabi.Fp8Quant(_ptr(x), _DTYPE_CODE[x.dtype], rows if ch else 0, max(ch, 1), _ptr(num_valid), _ptr(scale),
                       _ptr(out), None if scale is not None else _ptr(scale_out))
    _cabi.check(_lib().spx_fp8_quantize(ctypes.byref(q), _ptr(ws), 0 if ws is None else ws.numel(), _stream()),
                "fp8_quantize")
    return out, scale_out


def _implicit_gemm_splits(features, filters, pair_fwd, mask_splits, argsort_splits, n_out, is_train, timer,
                          bias, act_alpha, act_type, output_add, output_dtype, groups=1):
    """ConvAlgo.MaskSplitImplicitGemm forward: one kernel pass per mask split (each visits only its
    own offsets, rows in that split's sorted order), partial outputs summed, bias / activation after
    the last split (the reference fuses them into the last pass, ``convops.py:2196-2234``)."""
    lib = _lib()
    if features.dtype == torch.int8:
        raise NotImplementedError("int8 + MaskSplitImplicitGemm: use ConvAlgo.MaskImplicitGemm")
    if features.dtype == torch.float8_e4m3fn:
        raise NotImplementedError("fp8 + MaskSplitImplicitGemm: use ConvAlgo.MaskImplicitGemm")
    kv, c_in, c_out = _check_filter(features, filters, groups)
    n_in = features.shape[0]
    words = (kv + 31) // 32
    out = None
    tile_masks = []
    for mask, argsort in zip(mask_splits, argsort_splits):
        tiles = _tile_tables(pair_fwd, mask, argsort, n_out, kv, owner=argsort) if n_out else None
        d = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, pair_fwd, mask, argsort, tiles=tiles)
        part = torch.empty((n_out, c_out), dtype=features.dtype, device=features.device)
        with timer.record("implicit_gemm", _stream()):
            if groups != 1:
                _grouped_fwd(d, groups, features, filters, part, None, _cabi.SPX_ACT_NONE, 0.0, "grouped_gemm_fwd(split)")
            else:
                _cabi.check(lib.spx_implicit_gemm_fwd(ctypes.byref(d), _ptr(features), _ptr(filters), _ptr(part),
                                                      None, _cabi.SPX_ACT_NONE, 0.0, _stream()),
                            "implicit_gemm_fwd(split)")
        out = part if out is None else out.add_(part)
        if tiles is not None:
            tile_masks.append(tiles[1].view(1, -1, words))
    if (bias is not None or _act_code(act_type) != _cabi.SPX_ACT_NONE) and n_out:
        bias_add_act_inplace(out, bias, act_type, act_alpha)
    if output_add is not None:
        out = out + output_add
    if output_dtype is not None and output_dtype != out.dtype:
        out = out.to(output_dtype)
    mask_output = torch.cat(tile_masks, 0) if (is_train and tile_masks) else torch.Tensor()
    return out, mask_output, MASK_WIDTH


def _zero_runs(mask: np.ndarray, kv: int):
    """``[(a, b), ...]``: the runs of kernel offsets ``a <= k < b`` whose bit is clear in the split mask words"""
    runs, start = [], None
    for k in range(kv + 1):
        clear = k < kv and not (int(mask[k >> 5]) >> (k & 31)) & 1
        if clear and start is None:
            start = k
        elif not clear and start is not None:
            runs.append((start, k))
            start = None
    return runs


def implicit_gemm_backward(features: torch.Tensor, filters: torch.Tensor, out_bp: torch.Tensor,
                           pair_fwd: torch.Tensor, pair_bwd: torch.Tensor,
                           pair_mask_fwd_splits: List[torch.Tensor],
                           pair_mask_bwd_splits: List[torch.Tensor],
                           mask_argsort_fwd_splits: List[torch.Tensor],
                           mask_argsort_bwd_splits: List[torch.Tensor],
                           mask_output_fwd: Optional[torch.Tensor], masks: List[np.ndarray],
                           mask_width: int, is_subm: bool,
                           timer: CUDAKernelTimer = CUDAKernelTimer(False),
                           fp32_accum: Optional[bool] = None, groups: int = 1):
    """Input gradient + weight gradient of the masked implicit GEMM -> ``(din, dfilters)``
    (``ops.py:1667-1681`` / ``convops.py:2247-2440``).  ``groups > 1``: a grouped conv (see :func:`implicit_gemm`)."""
    _require_cuda(features, "features")
    lib = _lib()
    features = _dense(features)
    filters = _dense(filters)
    out_bp = _dense(out_bp)
    if out_bp.dtype != features.dtype:
        out_bp = out_bp.to(features.dtype)
    kv, c_in, c_out = _check_filter(features, filters, groups)
    n_in, n_out = features.shape[0], out_bp.shape[0]
    n_splits = len(pair_mask_fwd_splits) if isinstance(pair_mask_fwd_splits, (list, tuple)) else 1
    if n_splits > 1:
        # MaskSplitImplicitGemm: gradients are sums over the splits (each split only visits its offsets)
        din = dfilters = None
        for j in range(n_splits):
            bwd_m = [pair_mask_bwd_splits[j]] if pair_mask_bwd_splits else []
            bwd_s = [mask_argsort_bwd_splits[j]] if mask_argsort_bwd_splits else []
            di, dw = implicit_gemm_backward(features, filters, out_bp, pair_fwd, pair_bwd,
                                            [pair_mask_fwd_splits[j]], bwd_m, [mask_argsort_fwd_splits[j]],
                                            bwd_s, None, masks, mask_width, is_subm, timer, fp32_accum, groups)
            # dW of split j is only meaningful on ITS offsets: the tensor-core kernel leaves the others zero, the
            # generic FMA kernel (odd channel counts) walks the whole pair table -- zero them either way.  The
            # offsets come from the host-side split constant, so no mask tensor is copied to the device (a
            # blocking copy per layer eagerly, refused under CUDA-graph capture)
            dw = dw.view(c_out, kv, c_in // groups)
            for a, b in _zero_runs(masks[j], kv):
                dw[:, a:b].zero_()
            din = di if din is None else din.add_(di)
            dfilters = dw if dfilters is None else dfilters.add_(dw)
        return din, dfilters.view(filters.shape)
    din = torch.empty_like(features)
    dfilters = torch.empty_like(filters)
    mask_fwd, argsort_fwd = _first(pair_mask_fwd_splits), _first(mask_argsort_fwd_splits)
    tiles_fwd = _tile_tables(pair_fwd, mask_fwd, argsort_fwd, n_out, kv, owner=argsort_fwd) if n_out else None
    if is_subm:
        # SubM pairs are symmetric: walk the FORWARD table/mask and flip the filter offset
        # (the reference's reverse_mask, convops.py:2412)
        d_dg = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, pair_fwd, mask_fwd, argsort_fwd,
                     reverse=True, tiles=tiles_fwd)
    else:
        mask_bwd, argsort_bwd = _first(pair_mask_bwd_splits), _first(mask_argsort_bwd_splits)
        tiles_bwd = _tile_tables(pair_bwd, mask_bwd, argsort_bwd, n_in, kv, owner=argsort_bwd) if n_in else None
        d_dg = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, pair_bwd, mask_bwd, argsort_bwd,
                     tiles=tiles_bwd)
    d_wg = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, pair_fwd, mask_fwd, argsort_fwd,
                 tiles=tiles_fwd)
    ws = _wgrad_workspace(d_wg, groups, features.device)

    def run_dgrad():
        with timer.record("implicit_gemm_dgrad", _stream()):
            if groups != 1:
                _grouped_dgrad(d_dg, groups, out_bp, filters, din, "grouped_gemm_dgrad")
                return
            _cabi.check(lib.spx_implicit_gemm_dgrad(ctypes.byref(d_dg), _ptr(out_bp), _ptr(filters),
                                                    _ptr(din), _stream()), "implicit_gemm_dgrad")

    def run_wgrad(group):
        with timer.record("implicit_gemm_wgrad", _stream()):
            if groups != 1:
                _grouped_wgrad(d_wg, groups, features, out_bp, dfilters, ws, group, "grouped_gemm_wgrad")
            elif group is not None:
                # data-parallel: the kernel that reduces the split-K partials pushes this rank's fp32 dW into every
                # rank's exchange buffer (csrc/peer.cu); the schedule's finish writes dfilters
                _cabi.check(lib.spx_implicit_gemm_wgrad_push(
                    ctypes.byref(d_wg), _ptr(features), _ptr(out_bp), _ptr(dfilters), ws.data_ptr(), ws.numel(),
                    group, _stream()), "implicit_gemm_wgrad_push")
            else:
                _cabi.check(lib.spx_implicit_gemm_wgrad(ctypes.byref(d_wg), _ptr(features), _ptr(out_bp),
                                                        _ptr(dfilters), ws.data_ptr(), ws.numel(),
                                                        _stream()), "implicit_gemm_wgrad")

    _backward_schedule("implicit_gemm", run_dgrad, run_wgrad, dfilters, features.device, timer, n_in and n_out)
    return din, dfilters


_WGRAD_HOOK = None


def _backward_schedule(name, run_dgrad, run_wgrad, dfilters, device, timer, rows) -> None:
    """The order of the two gradients of a conv backward and the data-parallel handling of its dW, for every route
    (implicit GEMM, Native, depthwise).  ``run_wgrad(group)`` writes dW to ``dfilters``, or, given a peer group
    (``ctypes.byref``), pushes it to the group instead; ``rows``: both sides of the layer have rows.

    * Peer group installed: weight gradient + push, input gradient, finish (which writes dfilters).  The input
      gradient between push and finish hides the NVLink latency.
    * Otherwise, a wgrad hook installed: weight gradient, then the hook on a forked stream while the input gradient
      runs on this one -- also for a layer without rows (dW = 0), so a rank with an empty shard enters the same
      collectives.
    * Otherwise: input gradient, then weight gradient.

    Eager launches stay on one stream: they are host-bound and a fork / join per call measured slower; profiling
    regions stay one kernel each.  Under CUDA-graph capture the gradients become parallel branches.  The
    weight-gradient kernel (one CTA per SM, statically assigned tiles) has a long tail -- its CTAs finish over a
    ~15 us window -- so it goes first on the caller's stream and the input gradient on a forked stream fills the SMs
    it has left.  The finish goes behind the input gradient on the forked stream: every dependent kernel on the
    caller's stream costs ~8 us of launch and queueing when the next cloud's rulebook kernels share the GPU.  (With a
    group, running the gradients one after the other measured 17 us more per config-2 step, more than the whole
    exchange.)  Joined before returning."""
    if _PEERS is None and _WGRAD_HOOK is not None:
        main = torch.cuda.current_stream()
        side = _side_stream(device)
        run_wgrad(None)
        side.wait_stream(main)
        with torch.cuda.stream(side):
            _WGRAD_HOOK(dfilters)
        run_dgrad()
        main.wait_stream(side)
        return
    group = None if _PEERS is None or _PEER_TRIAGE & 2 else ctypes.byref(_PEERS.group)

    def finish():
        if _PEER_TRIAGE & 1:
            return
        with timer.record(f"{name}_wgrad_exchange", _stream()):
            _cabi.check(_lib().spx_peer_finish(ctypes.byref(_PEERS.group), _ptr(dfilters), dfilters.numel(),
                                               _DTYPE_CODE[dfilters.dtype], _PEERS.scale, _stream()), "peer_finish")

    if timer.enable or not rows or not torch._C._cuda_isCurrentStreamCapturing():
        if _PEERS is None:
            run_dgrad()
            run_wgrad(None)
        else:
            run_wgrad(group)
            run_dgrad()
            finish()
        return
    main = torch.cuda.current_stream()
    side = _side_stream(device)
    side.wait_stream(main)
    run_wgrad(group)
    with torch.cuda.stream(side):
        run_dgrad()
        if _PEERS is not None:
            side.wait_stream(main)          # the push
            finish()
    main.wait_stream(side)


def set_wgrad_hook(fn) -> None:
    """``fn(dfilters)`` is called on a forked stream right after the weight gradient of every layer, while
    the input gradient of the same layer runs on the caller's stream (joined before the op returns).  This
    is the place for a data-parallel all-reduce of the layer's dW: it overlaps the rest of the backward pass
    instead of trailing it (DDP-style hook).  Every route, :func:`implicit_gemm_backward`,
    :func:`indice_conv_backward` (``ConvAlgo.Native``) and :func:`depthwise_conv_backward`, runs this one schedule,
    for every layer, also one without rows (its dW is zero), so every rank enters the same collectives.
    ``ConvAlgo.MaskSplitImplicitGemm`` calls it once per mask split, with that split's dW, and sums what the hook
    left of each split over that split's kernel offsets.  The hook may change ``dfilters`` in place; the op returns
    what it leaves there.  Ignored while a peer group is installed (:func:`set_peer_group`).  ``None`` removes the
    hook."""
    global _WGRAD_HOOK
    _WGRAD_HOOK = fn


_PEERS = None
_PEER_TRIAGE = 0          # bench.py --peer-triage (timing experiments only; results are wrong when set)


def set_peer_group(peers) -> None:
    """Data-parallel mode: with a :class:`spconv_b200.pytorch.dist.PeerGroup` installed, every weight
    gradient computed by :func:`implicit_gemm_backward`, :func:`indice_conv_backward` and
    :func:`depthwise_conv_backward` is returned already summed (x ``peers.scale``) over the ranks, with one
    schedule on every route: the weight gradient pushes this rank's dW to every rank (on the implicit-GEMM
    routes the push is the tail of the weight-gradient kernel: NVLink peer stores, ``csrc/peer.cu``; the
    depthwise kernels are followed by ``spx_peer_push``), the input gradient runs, then the finish sums the
    ranks' pushes in rank order into dW.  Under CUDA-graph capture the input gradient and the finish run on a
    forked stream.  Every rank must run the same sequence of layers.  Only these conv weight gradients are exchanged:
    biases (added outside the op in training) and every other parameter keep rank-local gradients until
    :func:`peer_allreduce_` sums them (one call per tensor, or one per flat ``dist.GradBucket``), on every
    rank in the same order.  ``None`` switches it off."""
    global _PEERS
    _PEERS = peers


def peer_allreduce_(t: torch.Tensor) -> torch.Tensor:
    """In-place sum (x scale) of a small tensor over the installed peer group: the step that reduces every
    gradient the conv ops do not exchange (biases, other parameters; a ``dist.GradBucket``'s ``flat``
    reduces them in one call).  Every rank calls it for the same tensors in the same order; at most the
    group's capacity (fp32 values) per call.  No-op without a group."""
    if _PEERS is None or t.numel() == 0:
        return t
    assert t.is_contiguous(), "peer_allreduce_: contiguous tensor"
    _cabi.check(_lib().spx_peer_allreduce(ctypes.byref(_PEERS.group), t.data_ptr(), t.numel(), _DTYPE_CODE[t.dtype],
                                          _PEERS.scale, _stream()), "peer_allreduce")
    return t


# ---------------------------------------------------------------------------- ConvAlgo.Native
def _native_tables(indice_pairs, indice_pair_num, n_in, n_out, kv, subm, inverse, need_fwd,
                   need_bwd):
    """compact pairs [2, kv, L] -> dense gather tables + row masks (visited in natural order)."""
    lib = _lib()
    dev = indice_pairs.device
    words = (kv + 31) // 32
    t_fwd = torch.empty((kv, n_out), dtype=torch.int32, device=dev) if need_fwd else None
    m_fwd = torch.empty((n_out, words), dtype=torch.int32, device=dev) if need_fwd else None
    t_bwd = torch.empty((kv, n_in), dtype=torch.int32, device=dev) if need_bwd else None
    m_bwd = torch.empty((n_in, words), dtype=torch.int32, device=dev) if need_bwd else None
    _cabi.check(lib.spx_pairs_to_table(_ptr(indice_pairs), _ptr(indice_pair_num), kv,
                                       int(indice_pairs.shape[2]), n_in, n_out, int(subm),
                                       int(inverse), _ptr(t_fwd), _ptr(t_bwd), _ptr(m_fwd),
                                       _ptr(m_bwd), _stream()), "pairs_to_table")
    return t_fwd, m_fwd, t_bwd, m_bwd


def indice_conv(features: torch.Tensor, filters: torch.Tensor, indice_pairs: torch.Tensor,
                indice_pair_num: torch.Tensor, num_activate_out: int, inverse: bool = False,
                subm: bool = False, algo: ConvAlgo = ConvAlgo.Native,
                timer: CUDAKernelTimer = CUDAKernelTimer(False),
                bias: Optional[torch.Tensor] = None, act_alpha: float = 0.0,
                act_beta: float = 0.0, act_type=Activation.None_, groups: int = 1):
    """Gather-GEMM-scatter forward over a compact rulebook (``ops.py:811-823`` /
    ``convops.py:1504-1747``).  The compact pairs are scattered into a dense gather table on the
    device (no ``indice_pair_num.cpu()`` sync) and the output-stationary implicit-GEMM kernel
    accumulates every offset in registers -- no atomics, deterministic."""
    _require_cuda(features, "features")
    lib = _lib()
    features = _dense(features)
    filters = _dense(filters)
    indice_pairs = indice_pairs.contiguous()
    kv, c_in, c_out = _check_filter(features, filters, groups)
    assert features.shape[1] == c_in, "channel size mismatch"
    assert indice_pairs.shape[1] == kv, "indice_pairs / filter kernel volume mismatch"
    n_in, n_out = features.shape[0], int(num_activate_out)
    with timer.record("indice_conv_table", _stream()):
        t_fwd, m_fwd, _, _ = _native_tables(indice_pairs, indice_pair_num, n_in, n_out, kv, subm,
                                            inverse, True, False)
    out = torch.empty((n_out, c_out), dtype=features.dtype, device=features.device)
    if bias is not None:
        bias = bias.to(features.dtype).contiguous()
    tiles = _tile_tables(t_fwd, m_fwd, None, n_out, kv) if n_out else None
    d = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, t_fwd, m_fwd, None, tiles=tiles)
    with timer.record("indice_conv", _stream()):
        if groups != 1:
            _grouped_fwd(d, groups, features, filters, out, bias, _act_code(act_type), act_alpha,
                         "grouped_gemm_fwd(native)")
        else:
            _cabi.check(lib.spx_implicit_gemm_fwd(ctypes.byref(d), _ptr(features), _ptr(filters),
                                                  _ptr(out), _ptr(bias), _act_code(act_type),
                                                  float(act_alpha), _stream()),
                        "implicit_gemm_fwd(native)")
    return out


def indice_conv_backward(features: torch.Tensor, filters: torch.Tensor, out_bp: torch.Tensor,
                         indice_pairs: torch.Tensor, indice_pair_num: torch.Tensor,
                         inverse: bool = False, subm: bool = False,
                         algo: ConvAlgo = ConvAlgo.Native,
                         timer: CUDAKernelTimer = CUDAKernelTimer(False), groups: int = 1):
    """Backward of :func:`indice_conv` -> ``(din, dfilters)`` (``ops.py:1103-1111`` /
    ``convops.py:1751-2071``)."""
    _require_cuda(features, "features")
    lib = _lib()
    features = _dense(features)
    filters = _dense(filters)
    out_bp = _dense(out_bp)
    if out_bp.dtype != features.dtype:
        out_bp = out_bp.to(features.dtype)
    indice_pairs = indice_pairs.contiguous()
    kv, c_in, c_out = _check_filter(features, filters, groups)
    n_in, n_out = features.shape[0], out_bp.shape[0]
    t_fwd, m_fwd, t_bwd, m_bwd = _native_tables(indice_pairs, indice_pair_num, n_in, n_out, kv,
                                                subm, inverse, True, True)
    din = torch.empty_like(features)
    dfilters = torch.empty_like(filters)
    tiles_bwd = _tile_tables(t_bwd, m_bwd, None, n_in, kv) if n_in else None
    tiles_fwd = _tile_tables(t_fwd, m_fwd, None, n_out, kv) if n_out else None
    d_dg = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, t_bwd, m_bwd, None, tiles=tiles_bwd)
    d_wg = _desc(features.dtype, kv, c_in, c_out, n_in, n_out, t_fwd, m_fwd, None, tiles=tiles_fwd)
    ws = _wgrad_workspace(d_wg, groups, features.device)

    def run_dgrad():
        with timer.record("indice_conv_dgrad", _stream()):
            if groups != 1:
                _grouped_dgrad(d_dg, groups, out_bp, filters, din, "grouped_gemm_dgrad(native)")
                return
            _cabi.check(lib.spx_implicit_gemm_dgrad(ctypes.byref(d_dg), _ptr(out_bp), _ptr(filters),
                                                    _ptr(din), _stream()), "implicit_gemm_dgrad(native)")

    def run_wgrad(group):
        with timer.record("indice_conv_wgrad", _stream()):
            if groups != 1:
                _grouped_wgrad(d_wg, groups, features, out_bp, dfilters, ws, group, "grouped_gemm_wgrad(native)")
            elif group is not None:
                _cabi.check(lib.spx_implicit_gemm_wgrad_push(
                    ctypes.byref(d_wg), _ptr(features), _ptr(out_bp), _ptr(dfilters), ws.data_ptr(), ws.numel(),
                    group, _stream()), "implicit_gemm_wgrad_push(native)")
            else:
                _cabi.check(lib.spx_implicit_gemm_wgrad(ctypes.byref(d_wg), _ptr(features), _ptr(out_bp),
                                                        _ptr(dfilters), ws.data_ptr(), ws.numel(),
                                                        _stream()), "implicit_gemm_wgrad(native)")

    _backward_schedule("indice_conv", run_dgrad, run_wgrad, dfilters, features.device, timer, n_in and n_out)
    return din, dfilters


# ---------------------------------------------------------------------------- depthwise conv
def _depthwise_check(features: torch.Tensor, filters: torch.Tensor, table: torch.Tensor) -> Tuple[int, int]:
    _require_cuda(features, "features")
    if filters.dtype != features.dtype:
        raise RuntimeError(f"features ({features.dtype}) and filters ({filters.dtype}) must have the same dtype")
    if features.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise RuntimeError(f"depthwise conv: unsupported dtype {features.dtype}")
    c = int(filters.shape[0])
    if filters.shape[-1] != 1 or features.shape[1] != c:
        raise RuntimeError(f"depthwise conv: filters [C, *ksize, 1] with C = features' channels, got "
                           f"{tuple(filters.shape)} for {tuple(features.shape)}")
    kv = _prod(filters.shape[1:-1])
    if (table.dim() != 2 or table.shape[0] != kv or table.dtype != torch.int32
            or (table.shape[1] > 1 and table.stride(1) != 1)):
        raise RuntimeError(f"depthwise conv: table must be int32 [kv = {kv}, rows] with unit column stride, got "
                           f"{tuple(table.shape)} {table.dtype}")
    return kv, c


def depthwise_conv(features: torch.Tensor, filters: torch.Tensor, table: torch.Tensor, num_activate_out: int,
                   bias: Optional[torch.Tensor] = None, act_type=Activation.None_, act_alpha: float = 0.0,
                   timer: CUDAKernelTimer = CUDAKernelTimer(False)) -> torch.Tensor:
    """Depthwise forward ``out[o, c] = act(sum_k W[c, k] x[table[k][o], c] + bias[c])`` over a dense table
    ``[kv, >= num_activate_out]`` (``pair_fwd``, or the Native forward table).  ``filters`` is KRSC
    ``[C, *ksize, 1]``.  Offsets in ascending order, fp32 sums, no atomics (``spx_depthwise_fwd``)."""
    features = features.contiguous()
    filters = filters.contiguous()
    kv, c = _depthwise_check(features, filters, table)
    n_out = int(num_activate_out)
    out = torch.empty((n_out, c), dtype=features.dtype, device=features.device)
    if bias is not None:
        bias = bias.to(features.dtype).contiguous()
    with timer.record("depthwise_conv", _stream()):
        _cabi.check(_lib().spx_depthwise_fwd(_ptr(features), _ptr(filters), _ptr(bias), _ptr(out), _ptr(table),
                                             int(table.stride(0)), kv, n_out, c, _DTYPE_CODE[features.dtype],
                                             _act_code(act_type), float(act_alpha), _stream()), "depthwise_fwd")
    return out


def depthwise_conv_backward(features: torch.Tensor, filters: torch.Tensor, out_bp: torch.Tensor,
                            table_fwd: torch.Tensor, table_bwd: Optional[torch.Tensor],
                            timer: CUDAKernelTimer = CUDAKernelTimer(False)):
    """Backward of :func:`depthwise_conv` -> ``(din, dfilters)``.  ``table_bwd`` ``[kv, >= N]`` maps inputs to
    outputs; ``None`` (SubM) walks ``table_fwd`` with the mirrored offset instead.  The weight gradient is summed
    in a fixed order of the row indices (bit-reproducible, unchanged by trailing padding rows).  Data-parallel with the
    schedule of the other convs: the wgrad hook receives dW (:func:`set_wgrad_hook`); with a peer group installed
    dW is pushed right after its kernels and summed over the ranks behind the input gradient
    (:func:`set_peer_group`)."""
    features = features.contiguous()
    filters = filters.contiguous()
    out_bp = out_bp.contiguous()
    if out_bp.dtype != features.dtype:
        out_bp = out_bp.to(features.dtype)
    kv, c = _depthwise_check(features, filters, table_fwd)
    n_in, n_out = features.shape[0], out_bp.shape[0]
    reverse = table_bwd is None
    table_dg = table_fwd if reverse else table_bwd
    if not reverse:
        _depthwise_check(features, filters, table_bwd)
    lib = _lib()
    dtype = _DTYPE_CODE[features.dtype]
    din = torch.empty_like(features)
    dfilters = torch.empty_like(filters)
    ws = _bytes(lib.spx_depthwise_wgrad_workspace_size(n_out, kv, c), features.device)

    def run_dgrad():
        with timer.record("depthwise_conv_dgrad", _stream()):
            _cabi.check(lib.spx_depthwise_dgrad(_ptr(out_bp), _ptr(filters), _ptr(din), _ptr(table_dg),
                                                int(table_dg.stride(0)), kv, n_in, c, dtype, int(reverse), _stream()),
                        "depthwise_dgrad")

    def run_wgrad(group):
        with timer.record("depthwise_conv_wgrad", _stream()):
            _cabi.check(lib.spx_depthwise_wgrad(_ptr(features), _ptr(out_bp), _ptr(dfilters), _ptr(table_fwd),
                                                int(table_fwd.stride(0)), kv, n_out, c, dtype, ws.data_ptr(),
                                                ws.numel(), _stream()), "depthwise_wgrad")
            if group is not None:
                _cabi.check(lib.spx_peer_push(group, dfilters.data_ptr(), dfilters.numel(), dtype, _stream()),
                            "peer_push")

    _backward_schedule("depthwise_conv", run_dgrad, run_wgrad, dfilters, features.device, timer, n_in and n_out)
    return din, dfilters


# ---------------------------------------------------------------------------- pooling
_POOL_MAX, _POOL_MAX_ZERO_FLOOR, _POOL_MEAN = 0, 1, 2


def _pool_check(features: torch.Tensor):
    _require_cuda(features, "features")
    if features.dtype not in _DTYPE_CODE:
        raise RuntimeError(f"unsupported dtype {features.dtype}")
    c = features.shape[1]
    if (c * features.element_size()) % 16:
        raise RuntimeError(f"pooling needs channels * element size to be a multiple of 16 bytes, got {c} x "
                           f"{features.element_size()}")


def _pool_fwd(mode, features, table, n_out, count_out=None):
    features = _dense(features)
    _pool_check(features)
    out = torch.empty((int(n_out), features.shape[1]), dtype=features.dtype, device=features.device)
    _cabi.check(_lib().spx_indice_pool_fwd(mode, _ptr(features), _ptr(out), _ptr(table), int(table.stride(0)),
                                           int(table.shape[0]), int(n_out), int(features.shape[1]),
                                           _DTYPE_CODE[features.dtype], _ptr(count_out), _stream()),
                "indice_pool_fwd")
    return out


def _pool_bwd(mode, features, out_features, out_bp, table_bwd, n_in, count_out=None):
    out_bp = _dense(out_bp)
    _pool_check(out_bp)
    din = torch.empty((int(n_in), out_bp.shape[1]), dtype=out_bp.dtype, device=out_bp.device)
    _cabi.check(_lib().spx_indice_pool_bwd(mode, _ptr(features), _ptr(out_features), _ptr(out_bp), _ptr(din),
                                           _ptr(table_bwd), int(table_bwd.stride(0)), int(table_bwd.shape[0]),
                                           int(n_in), int(out_bp.shape[1]), _DTYPE_CODE[out_bp.dtype],
                                           _ptr(count_out), _stream()), "indice_pool_bwd")
    return din


def indice_maxpool(features: torch.Tensor, indice_pairs: torch.Tensor, indice_pair_num: torch.Tensor,
                   num_activate_out):
    """ConvAlgo.Native max pooling over compact pairs (``ops.py:1899-1936``).  The reference raises a
    zero-initialised output per offset, i.e. the result is ``max(0, max over inputs)``; the compact
    pairs are scattered into a dense table on the device (no ``indice_pair_num.cpu()`` sync) and
    one kernel reduces every output row."""
    kv = int(indice_pairs.shape[1])
    t_fwd, _, _, _ = _native_tables(indice_pairs.contiguous(), indice_pair_num, features.shape[0],
                                    int(num_activate_out), kv, False, False, True, False)
    return _pool_fwd(_POOL_MAX_ZERO_FLOOR, features, t_fwd, num_activate_out)


def indice_maxpool_backward(features, out_features, out_bp, indice_pairs, indice_pair_num):
    """``din[i] += dout[o]`` where ``x[i] == y[o]`` (``ops.py:1939-1972``)."""
    kv = int(indice_pairs.shape[1])
    _, _, t_bwd, _ = _native_tables(indice_pairs.contiguous(), indice_pair_num, features.shape[0],
                                    out_features.shape[0], kv, False, False, False, True)
    return _pool_bwd(_POOL_MAX, _dense(features), _dense(out_features), out_bp, t_bwd,
                     features.shape[0])


def indice_maxpool_implicit_gemm(features: torch.Tensor, indice_pairs: torch.Tensor, num_activate_out):
    """Max pooling through the dense forward table ``pair_fwd [kv, M]`` (``ops.py:1975-2006``)."""
    return _pool_fwd(_POOL_MAX, features, indice_pairs, num_activate_out)


def indice_maxpool_implicit_gemm_backward(features, out_features, out_bp, indice_pairs):
    """``indice_pairs`` is the backward table ``pair_bwd [kv, N]`` (``ops.py:2009-2030``)."""
    return _pool_bwd(_POOL_MAX, _dense(features), _dense(out_features), out_bp, indice_pairs,
                     features.shape[0])


def indice_avgpool_implicit_gemm(features: torch.Tensor, indice_pairs: torch.Tensor, num_activate_out,
                                 calc_count: bool):
    """Mean over the valid neighbours + their count (``ops.py:2033-2074``)."""
    count_out = torch.Tensor()
    if calc_count:
        count_out = torch.empty((int(num_activate_out),), dtype=torch.int32, device=features.device)
    out = _pool_fwd(_POOL_MEAN, features, indice_pairs, num_activate_out, count_out if calc_count else None)
    return out, count_out


def indice_avgpool_implicit_gemm_backward(out_bp, indice_pairs, count_out):
    """``din[i] = sum_o dout[o] * count[o]`` -- the reference multiplies by the neighbour count
    (``maxpool.py:262-300``); kept so gradients equal the reference's (``ops.py:2077-2096``)."""
    return _pool_bwd(_POOL_MEAN, None, None, out_bp, indice_pairs, indice_pairs.shape[1], count_out)


def global_pool_rearrange(coords: torch.Tensor, batch_size: int):
    """Row indices of every sample: ``(out_indices [batch, N], counts [batch])`` (``ops.py:2108-2124``)."""
    _require_cuda(coords, "coords")
    coords = coords.contiguous()
    n = coords.shape[0]
    out_indices = torch.empty((batch_size, n), dtype=torch.int32, device=coords.device)
    counts = torch.empty((batch_size,), dtype=torch.int32, device=coords.device)
    _cabi.check(_lib().spx_global_pool_rearrange(_ptr(coords), n, int(coords.shape[1]), int(batch_size),
                                                 _ptr(out_indices) if n else out_indices.data_ptr(),
                                                 counts.data_ptr(), _stream()), "global_pool_rearrange")
    return out_indices, counts


_GLOBAL_POOL_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _global_pool_check(features: torch.Tensor, indices: torch.Tensor, batch_size: int,
                       num_valid: Optional[torch.Tensor]):
    if features.dtype not in _GLOBAL_POOL_DTYPES:
        raise RuntimeError(f"masked global pooling supports float32, float16 and bfloat16 features, got "
                           f"{features.dtype}")
    _require_cuda(features, "features")
    _require_cuda(indices, "indices")
    if features.dim() != 2 or indices.dim() != 2 or indices.dtype != torch.int32 \
            or indices.shape[0] != features.shape[0]:
        raise RuntimeError(f"masked global pooling: features [rows, C] and int32 indices [rows, ndim + 1] expected, "
                           f"got {tuple(features.shape)} and {tuple(indices.shape)} {indices.dtype}")
    if num_valid is not None and (num_valid.dtype != torch.int32 or num_valid.device != features.device):
        raise RuntimeError("masked global pooling: num_valid must be an int32 tensor on the features' device")
    if int(batch_size) < 1:
        raise RuntimeError(f"masked global pooling: batch_size must be positive, got {batch_size}")


def masked_global_pool_fwd(features: torch.Tensor, indices: torch.Tensor, batch_size: int,
                           num_valid: Optional[torch.Tensor], is_mean: bool):
    """Per-sample max or mean over rows ``[0, num_valid)`` (all rows when ``num_valid`` is None) whose batch index
    ``indices[:, 0]`` is in ``[0, batch_size)``: ``(out [batch_size, C], aux)``.  ``aux`` is what the backward
    needs: ``argmax [batch_size, C]`` int32 (max; the first row that attains the maximum, NaN counting as the
    maximum) or ``count [batch_size]`` int32 (mean).  An empty sample gives 0 (argmax -1, count 0).  No host
    synchronisation; bit-reproducible whatever the padding."""
    _global_pool_check(features, indices, batch_size, num_valid)
    features, indices = features.contiguous(), indices.contiguous()
    rows, c = features.shape
    b = int(batch_size)
    out = torch.empty((b, c), dtype=features.dtype, device=features.device)
    if is_mean:
        aux = torch.empty((b,), dtype=torch.int32, device=features.device)
    else:
        aux = torch.empty((b, c), dtype=torch.int32, device=features.device)
    lib = _lib()
    ws = _bytes(lib.spx_global_pool_workspace_size(rows, b, c), features.device)
    _cabi.check(lib.spx_global_pool_fwd(
        int(is_mean), _ptr(features), _ptr(indices), rows, int(indices.shape[1]), b, c, _DTYPE_CODE[features.dtype],
        _ptr(num_valid), out.data_ptr(), None if is_mean else aux.data_ptr(), aux.data_ptr() if is_mean else None,
        ws.data_ptr(), ws.numel(), _stream()), "global_pool_fwd")
    return out, aux


def masked_global_pool_bwd(dy: torch.Tensor, indices: torch.Tensor, batch_size: int,
                           num_valid: Optional[torch.Tensor], aux: torch.Tensor, is_mean: bool) -> torch.Tensor:
    """``din [rows, C]`` of :func:`masked_global_pool_fwd`: ``dy[b]`` at the argmax rows (max) or
    ``dy[b] / count[b]`` on every row of sample ``b`` (mean), 0 on padding and dropped rows."""
    dy = dy.contiguous()
    b = int(batch_size)
    rows = indices.shape[0]
    din = torch.empty((rows, dy.shape[1]), dtype=dy.dtype, device=dy.device)
    _global_pool_check(din, indices, b, num_valid)
    if dy.shape != (b, din.shape[1]):
        raise RuntimeError(f"masked global pooling: the output gradient must be [{b}, C], got {tuple(dy.shape)}")
    indices = indices.contiguous()
    _cabi.check(_lib().spx_global_pool_bwd(
        int(is_mean), dy.data_ptr(), _ptr(indices), rows, int(indices.shape[1]), b, int(dy.shape[1]),
        _DTYPE_CODE[dy.dtype], _ptr(num_valid), None if is_mean else aux.data_ptr(),
        aux.data_ptr() if is_mean else None, _ptr(din), _stream()), "global_pool_bwd")
    return din


# ---------------------------------------------------------------------------- sparse add
_SPARSE_ADD_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def sparse_add_union(indices: Sequence[torch.Tensor], batch_size: int, spatial_shape: List[int]):
    """Union of coordinate sets visited in the given order -> ``(out_inds [M, ndim+1], dst [sum N])``.

    ``out_inds`` holds every distinct in-range coordinate once, ranked by the first visited row that carries
    it; ``dst[g]`` is the output row of visited row ``g`` (-1: batch index or coordinate out of range).  This is
    the regular-conv rulebook of a 1x..x1, stride-1, padding-0 convolution over the concatenated coordinates
    (``dst`` is its ``pair_bwd[0]``).  One host sync (the output count).  An empty union returns 0 rows."""
    for ind in indices:
        _require_cuda(ind, "indices")
    dev = indices[0].device
    ndim = len(spatial_shape)
    cat = torch.cat([i.to(torch.int32).reshape(-1, ndim + 1) for i in indices], 0).contiguous()
    n = cat.shape[0]
    if n == 0:
        return torch.empty((0, ndim + 1), dtype=torch.int32, device=dev), torch.empty((0,), dtype=torch.int32, device=dev)
    ones, zeros = [1] * ndim, [0] * ndim
    geo = _geometry(cat, batch_size, spatial_shape, spatial_shape, ones, ones, zeros, ones, False)
    out_inds, _, pair_bwd, _, _ = _conv_rulebook(geo, cat, n, 1, 1, False, None)
    dst = pair_bwd[0]
    if out_inds.shape[0] == 0:
        dst.fill_(-1)
    return out_inds, dst


def sparse_add_group(dst: torch.Tensor, m: int):
    """``(order [N], offsets [M+1])``: the visited rows of output ``o`` are ``order[offsets[o]:offsets[o+1]]``,
    ascending; ``order[offsets[o]]`` is the row that created ``o``.  Dropped rows sort last."""
    lib = _lib()
    n = dst.shape[0]
    order = torch.empty((n,), dtype=torch.int32, device=dst.device)
    offsets = torch.empty((int(m) + 1,), dtype=torch.int32, device=dst.device)
    ws = _bytes(lib.spx_sparse_add_group_workspace_size(n), dst.device)
    _cabi.check(lib.spx_sparse_add_group(_ptr(dst), n, int(m), _ptr(order), offsets.data_ptr(), ws.data_ptr(),
                                         ws.numel(), _stream()), "sparse_add_group")
    return order, offsets


def _sparse_add_operands(rows: Sequence[int], features=None, grads=None) -> "_cabi.SparseAddOperands":
    if len(rows) > _cabi.SPX_SPARSE_ADD_MAX_OPERANDS:
        raise ValueError(f"sparse_add supports at most {_cabi.SPX_SPARSE_ADD_MAX_OPERANDS} operands, got {len(rows)}")
    ops = _cabi.SparseAddOperands()
    ops.count = len(rows)
    for t, r in enumerate(rows):
        ops.rows[t] = int(r)
        ops.features[t] = _ptr(features[t]) if features is not None else None
        ops.grads[t] = _ptr(grads[t]) if grads is not None else None
    return ops


def _sparse_add_dtype(dtype: torch.dtype) -> int:
    if dtype not in _SPARSE_ADD_DTYPES:
        raise RuntimeError(f"sparse_add supports float32, float16 and bfloat16 features, got {dtype}")
    return _DTYPE_CODE[dtype]


def sparse_add_forward(features: Sequence[torch.Tensor], order: torch.Tensor, offsets: torch.Tensor,
                       m: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out [M, C]``: per output row the fp32 sum of its visited rows in visit order, rounded once.
    ``features`` are the operands in visit order, all of one dtype; ``out`` (optional) is written in place."""
    for f in features:
        _require_cuda(f, "features")
    features = [f.contiguous() for f in features]
    c = features[0].shape[1]
    code = _sparse_add_dtype(features[0].dtype)
    if out is None:
        out = torch.empty((int(m), c), dtype=features[0].dtype, device=features[0].device)
    assert out.shape == (int(m), c) and out.dtype == features[0].dtype and out.is_contiguous()
    ops = _sparse_add_operands([f.shape[0] for f in features], features=features)
    _cabi.check(_lib().spx_sparse_add_fwd(ctypes.byref(ops), _ptr(order), _ptr(offsets), int(m), int(c), code,
                                          _ptr(out), _stream()), "sparse_add_fwd")
    return out


def sparse_add_gather(index: torch.Tensor, src: torch.Tensor, rows: Sequence[int],
                      needed: Optional[Sequence[bool]] = None,
                      outs: Optional[Sequence[torch.Tensor]] = None) -> List[Optional[torch.Tensor]]:
    """Row ``g`` of the concatenation of the returned blocks is ``src[index[g]]``, or zero where ``index[g] < 0``
    (the backward pass of :func:`sparse_add_forward` with ``index = dst``).  Blocks with ``needed[t]`` false
    are not computed and come back as None; ``outs`` (optional) are written in place."""
    _require_cuda(src, "src")
    src = src.contiguous()
    code = _sparse_add_dtype(src.dtype)
    c = src.shape[1]
    needed = [True] * len(rows) if needed is None else list(needed)
    if outs is None:
        outs = [torch.empty((int(r), c), dtype=src.dtype, device=src.device) if need else None
                for r, need in zip(rows, needed)]
    for o, r in zip(outs, rows):
        assert o is None or (o.shape == (int(r), c) and o.dtype == src.dtype and o.is_contiguous())
    ops = _sparse_add_operands(rows, grads=outs)
    _cabi.check(_lib().spx_sparse_add_gather(_ptr(index), _ptr(src), int(src.shape[0]), ctypes.byref(ops), int(c),
                                             code, _stream()), "sparse_add_gather")
    return outs


def masked_sparse_add_plan(indices: Sequence[torch.Tensor], num_valid: Sequence[Optional[torch.Tensor]],
                           batch_size: int, spatial_shape: List[int], bound: int,
                           status: Optional[torch.Tensor] = None):
    """Union and grouping of padded operands in ARGUMENT order (``spx_masked_sparse_add_plan``), no host read-back.
    Operand ``t``'s valid rows are ``[0, num_valid[t])`` (None: every row); the rest are never read.  Returns
    ``(out_inds [bound, ndim+1], dst [sum N], order [sum N], offsets [bound+1], num_out [1], status [1])``: rows
    ``[0, num_out)`` of ``out_inds`` equal :func:`sparse_add_union` of the valid rows in sparse_add's visit order,
    ``dst`` / ``order`` index the argument-order concatenation (-1 in ``dst`` for padding, out-of-range and dropped
    rows), and ``status`` (ORed into when given) gets bit 0 when more than ``bound`` outputs existed and bit 1 on a
    probe-chain overflow."""
    for ind in indices:
        _require_cuda(ind, "indices")
    dev = indices[0].device
    ndim = len(spatial_shape)
    cat = torch.cat([i.to(torch.int32).reshape(-1, ndim + 1) for i in indices], 0).contiguous()
    rows = [int(i.shape[0]) for i in indices]
    n = cat.shape[0]
    for nv in num_valid:
        if nv is not None and (nv.dtype != torch.int32 or nv.device != dev or nv.numel() < 1):
            raise RuntimeError("masked_sparse_add: num_valid must be a device int32 [1] on the indices' device")
    ones, zeros = [1] * ndim, [0] * ndim
    geo = _geometry(cat, batch_size, spatial_shape, spatial_shape, ones, ones, zeros, ones, False)
    out_inds = torch.empty((int(bound), ndim + 1), dtype=torch.int32, device=dev)
    dst = torch.empty((n,), dtype=torch.int32, device=dev)
    order = torch.empty((n,), dtype=torch.int32, device=dev)
    offsets = torch.empty((int(bound) + 1,), dtype=torch.int32, device=dev)
    num_out = torch.empty((1,), dtype=torch.int32, device=dev)
    if status is None:
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
    lib = _lib()
    ws = _bytes(lib.spx_masked_sparse_add_workspace_size(ctypes.byref(geo), n, int(bound)), dev)
    opnds = _sparse_add_operands(rows)
    nv_ptrs = (ctypes.c_void_p * len(rows))(*[None if nv is None else nv.data_ptr() for nv in num_valid])
    _cabi.check(lib.spx_masked_sparse_add_plan(
        ctypes.byref(geo), ctypes.byref(opnds), nv_ptrs, _ptr(cat), int(bound), _ptr(out_inds), _ptr(dst), _ptr(order),
        offsets.data_ptr(), num_out.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
        "masked_sparse_add_plan")
    return out_inds, dst, order, offsets, num_out, status


def masked_sparse_add_heads(order: torch.Tensor, offsets: torch.Tensor, num_out: torch.Tensor):
    """``(heads [bound], inverse [N])`` of a one-operand plan: ``heads[o]`` is the row that created output ``o``
    (-1 for ``o >= num_out``), ``inverse[heads[o]] = o`` and -1 on every other row."""
    n = order.shape[0]
    bound = offsets.shape[0] - 1
    heads = torch.empty((bound,), dtype=torch.int32, device=order.device)
    inverse = torch.empty((n,), dtype=torch.int32, device=order.device)
    _cabi.check(_lib().spx_masked_sparse_add_heads(_ptr(order), offsets.data_ptr(), num_out.data_ptr(), bound, n,
                                                   _ptr(heads), _ptr(inverse), _stream()), "masked_sparse_add_heads")
    return heads, inverse


# ---------------------------------------------------------------------------- point -> voxel reductions
POINT_SCATTER_MODES = {"max": 0, "mean": 1, "sum": 2}


def point_scatter_group(ids: torch.Tensor, rows: int):
    """``(row32 [P], order [P], offsets [rows + 1])`` of the int32 / int64 ids ``[P]`` (``spx_point_scatter_group``):
    ``row32[p]`` is the id, or -1 when it is outside ``[0, rows)`` (the point is dropped); the points of row ``r``
    are ``order[offsets[r]:offsets[r + 1]]`` in ascending point index.  No host synchronisation."""
    _require_cuda(ids, "pc_voxel_id")
    if ids.dim() != 1 or ids.dtype not in (torch.int32, torch.int64):
        raise RuntimeError(f"point scatter: the ids must be an int32 or int64 vector [P], got {ids.dtype} "
                           f"{tuple(ids.shape)}")
    ids = ids.contiguous()
    n, rows = ids.shape[0], int(rows)
    row32 = torch.empty((n,), dtype=torch.int32, device=ids.device)
    order = torch.empty((n,), dtype=torch.int32, device=ids.device)
    offsets = torch.empty((rows + 1,), dtype=torch.int32, device=ids.device)
    lib = _lib()
    ws = _bytes(lib.spx_point_scatter_group_workspace_size(n), ids.device)
    _cabi.check(lib.spx_point_scatter_group(_ptr(ids), ids.element_size(), n, rows, _ptr(row32), _ptr(order),
                                            offsets.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
                "point_scatter_group")
    return row32, order, offsets


def _point_scatter_dtype(x: torch.Tensor) -> int:
    if x.dtype not in _GLOBAL_POOL_DTYPES:
        raise RuntimeError(f"PointVoxelScatter supports float32, float16 and bfloat16 features, got {x.dtype}")
    return _DTYPE_CODE[x.dtype]


def point_scatter_fwd(x: torch.Tensor, order: torch.Tensor, offsets: torch.Tensor, mode: str):
    """``(out [rows, C], argmax)`` of the points ``x [P, C]`` grouped by :func:`point_scatter_group`: per row the max
    (``argmax [rows, C]`` int32: the first point that attains it, a NaN counting as the maximum; bit copy), the
    mean (fp32 sum in ascending point order / count, rounded once) or the sum (fp32, rounded once).  ``argmax``
    is None unless ``mode`` is ``"max"``.  A row without points gives 0 (argmax -1)."""
    code = _point_scatter_dtype(x)
    _require_cuda(x, "features")
    if x.dim() != 2 or x.shape[0] != order.shape[0]:
        raise RuntimeError(f"point scatter: features must be [{order.shape[0]}, C], got {tuple(x.shape)}")
    x = x.contiguous()
    n, c = x.shape
    rows = offsets.shape[0] - 1
    out = torch.empty((rows, c), dtype=x.dtype, device=x.device)
    argmax = torch.empty((rows, c), dtype=torch.int32, device=x.device) if mode == "max" else None
    _cabi.check(_lib().spx_point_scatter_fwd(POINT_SCATTER_MODES[mode], _ptr(x), n, c, code, _ptr(order),
                                             offsets.data_ptr(), rows, _ptr(out), _ptr(argmax), _stream()),
                "point_scatter_fwd")
    return out, argmax


def point_scatter_bwd(dy: torch.Tensor, row32: torch.Tensor, aux: Optional[torch.Tensor], mode: str) -> torch.Tensor:
    """``dx [P, C]`` of :func:`point_scatter_fwd`: ``dy[r]`` at the argmax point (max), ``dy[r] / count[r]`` (mean,
    ``aux`` = count) or ``dy[r]`` (sum) on every point of row ``r``; 0 for dropped points."""
    code = _point_scatter_dtype(dy)
    dy = dy.contiguous()
    n = row32.shape[0]
    rows, c = dy.shape
    dx = torch.empty((n, c), dtype=dy.dtype, device=dy.device)
    _cabi.check(_lib().spx_point_scatter_bwd(POINT_SCATTER_MODES[mode], _ptr(dy), _ptr(row32), n, rows, c, code,
                                             _ptr(aux) if mode == "max" else None,
                                             _ptr(aux) if mode == "mean" else None, _ptr(dx), _stream()),
                "point_scatter_bwd")
    return dx


# ---------------------------------------------------------------------------- voxel -> point interpolation
POINT_INTERP_MODES = {"trilinear": 0, "nearest": 1}


def point_interp_plan(indices: torch.Tensor, spatial_shape, batch_size: int, num_valid: Optional[torch.Tensor],
                      pos: torch.Tensor, batch_ids: torch.Tensor, mode: str = "trilinear", normalize: bool = True):
    """``(index [P, K], weight [P, K], order [P * K], offsets [rows + 1])`` of the points ``pos [P, ndim]`` (index
    space, the axis order of ``indices[:, 1:]``) in batch ``batch_ids [P]`` against the tensor ``indices
    [rows, 1 + ndim]`` (``spx_point_interp_plan``): ``K = 2^ndim`` corners (trilinear) or 1 (nearest), ``index`` -1
    and ``weight`` 0 for a missing corner; the entries ``e = p * K + j`` of row ``r`` are
    ``order[offsets[r]:offsets[r + 1]]`` in ascending ``e``.  Other float positions are cast to float32, int64
    batch ids to int32 (outside ``[0, batch_size)`` they stay dropped).  No host synchronisation."""
    for t, what in ((indices, "indices"), (pos, "pos"), (batch_ids, "batch_ids")):
        _require_cuda(t, what)
    if mode not in POINT_INTERP_MODES:
        raise ValueError(f"point interpolation: mode must be 'trilinear' or 'nearest', got {mode!r}")
    ndim = len(spatial_shape)
    if indices.dim() != 2 or indices.dtype != torch.int32 or indices.shape[1] != ndim + 1:
        raise RuntimeError(f"point interpolation: indices must be int32 [rows, {ndim + 1}], got {indices.dtype} "
                           f"{tuple(indices.shape)}")
    if pos.dim() != 2 or pos.shape[1] != ndim or not pos.is_floating_point():
        raise RuntimeError(f"point interpolation: pos must be a float tensor [P, {ndim}], got {pos.dtype} "
                           f"{tuple(pos.shape)}")
    if batch_ids.shape != (pos.shape[0],) or batch_ids.dtype not in (torch.int32, torch.int64):
        raise RuntimeError(f"point interpolation: batch_ids must be int32 or int64 [{pos.shape[0]}], got "
                           f"{batch_ids.dtype} {tuple(batch_ids.shape)}")
    if num_valid is not None:
        _require_cuda(num_valid, "num_valid")
        if num_valid.dtype != torch.int32 or num_valid.numel() != 1:
            raise RuntimeError(f"point interpolation: num_valid must be one int32, got {num_valid.dtype} "
                               f"{tuple(num_valid.shape)}")
    if batch_ids.dtype == torch.int64:
        batch_ids = torch.where((batch_ids >= 0) & (batch_ids < int(batch_size)), batch_ids, -1).int()
    indices, pos, batch_ids = indices.contiguous(), pos.float().contiguous(), batch_ids.contiguous()
    n, rows, dev = pos.shape[0], indices.shape[0], pos.device
    k = 1 if mode == "nearest" else 1 << ndim
    index = torch.empty((n, k), dtype=torch.int32, device=dev)
    weight = torch.empty((n, k), dtype=torch.float32, device=dev)
    order = torch.empty((n * k,), dtype=torch.int32, device=dev)
    offsets = torch.empty((rows + 1,), dtype=torch.int32, device=dev)
    a = _point_interp_args(ndim, mode, rows, n)
    a.batch_size, a.normalize = int(batch_size), int(bool(normalize))
    for i, v in enumerate(spatial_shape):
        a.spatial_shape[i] = int(v)
    a.indices, a.num_valid, a.pos, a.batch_ids = _ptr(indices), _ptr(num_valid), _ptr(pos), _ptr(batch_ids)
    a.index, a.weight, a.order, a.offsets = _ptr(index), _ptr(weight), _ptr(order), offsets.data_ptr()
    lib = _lib()
    nbytes = lib.spx_point_interp_plan_workspace_size(ctypes.byref(a))
    ws = _bytes(nbytes, dev)
    _cabi.check(lib.spx_point_interp_plan(ctypes.byref(a), ws.data_ptr(), nbytes, _stream()), "point_interp_plan")
    return index, weight, order, offsets


def _point_interp_args(ndim: int, mode, rows: int, n: int) -> "_cabi.PointInterp":
    a = _cabi.PointInterp()
    a.ndim, a.rows, a.num_points = int(ndim), int(rows), int(n)
    a.mode = POINT_INTERP_MODES[mode] if isinstance(mode, str) else int(mode)
    return a


def _point_interp_corners(k: int, rows: int, n: int) -> "_cabi.PointInterp":
    """the argument block of a forward / backward over a table of k corners per point (1: nearest, 2^ndim)"""
    if k not in (1, 2, 4, 8, 16):
        raise RuntimeError(f"point interpolation: {k} corners per point, expected 1, 2, 4, 8 or 16")
    return _point_interp_args(max(k.bit_length() - 1, 1), 1 if k == 1 else 0, rows, n)


def _point_interp_dtype(x: torch.Tensor) -> int:
    if x.dtype not in _GLOBAL_POOL_DTYPES:
        raise RuntimeError(f"VoxelPointInterpolator supports float32, float16 and bfloat16 features, got {x.dtype}")
    return _DTYPE_CODE[x.dtype]


def point_interp_fwd(x: torch.Tensor, index: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """``y [P, C]`` of the rows ``x [rows, C]`` at the points of :func:`point_interp_plan`: the sum over the found
    corners in ascending ``j`` of ``weight[p, j] * x[index[p, j]]`` in fp32 (no FMA), rounded once; 0 for a point
    without a found corner.  One launch."""
    code = _point_interp_dtype(x)
    _require_cuda(x, "features")
    if x.dim() != 2:
        raise RuntimeError(f"point interpolation: features must be [rows, C], got {tuple(x.shape)}")
    x = x.contiguous()
    n, k = index.shape
    rows, c = x.shape
    y = torch.empty((n, c), dtype=x.dtype, device=x.device)
    a = _point_interp_corners(k, rows, n)
    a.channels, a.dtype = c, code
    a.x, a.index, a.weight, a.y = _ptr(x), _ptr(index), _ptr(weight), _ptr(y)
    _cabi.check(_lib().spx_point_interp_fwd(ctypes.byref(a), _stream()), "point_interp_fwd")
    return y


def point_interp_bwd(dy: torch.Tensor, weight: torch.Tensor, order: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
    """``dx [rows, C]`` of :func:`point_interp_fwd`: per row the sum over its entries ``e`` in ascending order of
    ``weight[e] * dy[e / K]`` in fp32, rounded once; 0 for a row without entries.  Every element is written once, no
    atomics.  One launch."""
    code = _point_interp_dtype(dy)
    _require_cuda(dy, "grad_output")
    if dy.dim() != 2 or dy.shape[0] != weight.shape[0]:
        raise RuntimeError(f"point interpolation: grad_output must be [{weight.shape[0]}, C], got {tuple(dy.shape)}")
    dy = dy.contiguous()
    n, k = weight.shape
    rows, c = offsets.shape[0] - 1, dy.shape[1]
    dx = torch.empty((rows, c), dtype=dy.dtype, device=dy.device)
    a = _point_interp_corners(k, rows, n)
    a.channels, a.dtype = c, code
    a.dy, a.weight, a.order, a.offsets, a.dx = _ptr(dy), _ptr(weight), _ptr(order), offsets.data_ptr(), _ptr(dx)
    _cabi.check(_lib().spx_point_interp_bwd(ctypes.byref(a), _stream()), "point_interp_bwd")
    return dx


# ---------------------------------------------------------------------------- misc
def bias_add_act_inplace(x: torch.Tensor, bias: Optional[torch.Tensor], act_type=Activation.None_,
                         act_alpha: float = 0.0, act_beta: float = 0.0) -> torch.Tensor:
    """``InferenceOps.bias_add_act_inplace`` (``inference.py:166-252``)."""
    _require_cuda(x, "x")
    assert x.is_contiguous() and x.dim() == 2
    if bias is not None:
        bias = bias.to(x.dtype).contiguous()
    _cabi.check(_lib().spx_bias_act_inplace(_ptr(x), _ptr(bias), x.shape[0], x.shape[1],
                                            _DTYPE_CODE[x.dtype], _act_code(act_type),
                                            float(act_alpha), _stream()), "bias_act_inplace")
    return x


def maximum_value_int_(ten: torch.Tensor, value):
    """running max of the active-voxel count (``ops.py`` maximum_value_int_).  ``value`` is a host integer or
    a device int32 scalar (the count of a bounded rulebook: no read-back)."""
    if isinstance(value, torch.Tensor):
        torch.maximum(ten, value.to(ten.dtype).view(1), out=ten)
    else:
        ten.clamp_(min=int(value))
    return ten


def zero_rows_from_count_(x: torch.Tensor, num_valid: torch.Tensor) -> torch.Tensor:
    """Zero rows ``[num_valid, rows)`` of the contiguous matrix ``x`` in place (``num_valid``: device int32)."""
    _require_cuda(x, "x")
    assert x.is_contiguous() and x.dim() == 2 and num_valid.dtype == torch.int32
    _cabi.check(_lib().spx_zero_rows_from_count(_ptr(x), x.shape[0], x.shape[1] * x.element_size(),
                                                num_valid.data_ptr(), _stream()), "zero_rows_from_count")
    return x


_BN_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _bn_param_code(x: torch.Tensor, params: Sequence[Optional[torch.Tensor]], who: str = "masked_batch_norm") -> int:
    """dtype code of the BatchNorm / GroupNorm parameters and buffers: all float32, or all the feature dtype."""
    given = [p for p in params if p is not None]
    dt = given[0].dtype if given else torch.float32
    for p in given:
        _require_cuda(p, "BatchNorm parameters and buffers" if who == "masked_batch_norm" else "GroupNorm parameters")
        if p.dtype != dt or p.dim() != 1 or p.shape[0] != x.shape[1] or not p.is_contiguous():
            raise RuntimeError(f"{who}: parameters and buffers must be contiguous [{x.shape[1]}] tensors "
                               "of one dtype")
    if dt not in (torch.float32, x.dtype):
        raise RuntimeError(f"{who}: parameter dtype {dt} must be float32 or the feature dtype {x.dtype}")
    return _DTYPE_CODE[dt]


def _bn_features(x: torch.Tensor, num_valid: Optional[torch.Tensor]) -> torch.Tensor:
    _require_cuda(x, "features")
    if x.dim() != 2 or x.dtype not in _BN_DTYPES:
        raise RuntimeError(f"masked_batch_norm: features must be a [rows, C] float32 / float16 / bfloat16 matrix, got "
                           f"{tuple(x.shape)} {x.dtype}")
    if num_valid is not None and (num_valid.dtype != torch.int32 or num_valid.device != x.device):
        raise RuntimeError("masked_batch_norm: num_valid must be an int32 tensor on the features' device")
    return x.contiguous()


def masked_batch_norm_forward(x: torch.Tensor, num_valid: Optional[torch.Tensor], weight: Optional[torch.Tensor],
                              bias: Optional[torch.Tensor], running_mean: Optional[torch.Tensor],
                              running_var: Optional[torch.Tensor], num_batches_tracked: Optional[torch.Tensor],
                              momentum: Optional[float], eps: float):
    """Training-mode BatchNorm over rows ``[0, num_valid)`` of ``x`` (all rows when ``num_valid`` is None):
    ``(y, mean, invstd)``; rows at and beyond ``num_valid`` of ``y`` are 0.  ``running_mean`` / ``running_var``
    are updated in place; ``momentum=None`` takes ``1 / num_batches_tracked`` on the device (the caller
    increments it first, as torch does)."""
    x = _bn_features(x, num_valid)
    code = _bn_param_code(x, [weight, bias, running_mean, running_var])
    rows, c = x.shape
    cumulative = momentum is None
    if cumulative and running_mean is not None and num_batches_tracked is None:
        raise RuntimeError("masked_batch_norm: momentum=None needs num_batches_tracked")
    y = torch.empty_like(x)
    mean = torch.empty((c,), dtype=torch.float32, device=x.device)
    invstd = torch.empty((c,), dtype=torch.float32, device=x.device)
    lib = _lib()
    ws = _bytes(lib.spx_masked_bn_fwd_train_workspace_size(rows, c), x.device)
    _cabi.check(lib.spx_masked_bn_fwd_train(
        _ptr(x), _ptr(y), rows, c, _DTYPE_CODE[x.dtype], _ptr(num_valid), _ptr(weight), _ptr(bias),
        _ptr(running_mean), _ptr(running_var), _ptr(num_batches_tracked), code,
        0.0 if cumulative else float(momentum), int(cumulative), float(eps), mean.data_ptr(), invstd.data_ptr(),
        ws.data_ptr(), ws.numel(), _stream()), "masked_bn_fwd_train")
    return y, mean, invstd


def masked_batch_norm_backward(x: torch.Tensor, dy: torch.Tensor, num_valid: Optional[torch.Tensor],
                               weight: Optional[torch.Tensor], mean: torch.Tensor, invstd: torch.Tensor,
                               need_weight_grad: bool = True, need_bias_grad: bool = True):
    """``(dx, dweight, dbias)`` of :func:`masked_batch_norm_forward`; padding rows of ``dx`` are 0, the
    parameter gradients (None when not needed) have the parameters' dtype (float32 without ``weight``)."""
    x = _bn_features(x, num_valid)
    dy = dy.contiguous()
    if dy.shape != x.shape or dy.dtype != x.dtype:
        raise RuntimeError("masked_batch_norm: the output gradient must match the features' shape and dtype")
    code = _bn_param_code(x, [weight])
    pdt = weight.dtype if weight is not None else torch.float32
    rows, c = x.shape
    dx = torch.empty_like(x)
    dw = torch.empty((c,), dtype=pdt, device=x.device) if need_weight_grad else None
    db = torch.empty((c,), dtype=pdt, device=x.device) if need_bias_grad else None
    lib = _lib()
    ws = _bytes(lib.spx_masked_bn_bwd_workspace_size(rows, c), x.device)
    _cabi.check(lib.spx_masked_bn_bwd(
        _ptr(x), _ptr(dy), _ptr(dx), rows, c, _DTYPE_CODE[x.dtype], _ptr(num_valid), _ptr(weight), code,
        mean.data_ptr(), invstd.data_ptr(), _ptr(dw), _ptr(db), ws.data_ptr(), ws.numel(), _stream()),
        "masked_bn_bwd")
    return dx, dw, db


# ---------------------------------------------------------------------------- per-sample GroupNorm
GROUP_NORM_MAX_BATCH = 1 << 20
GROUP_NORM_MAX_CHANNELS = 1 << 16


def _gn_check(x: torch.Tensor, indices: torch.Tensor, batch_size: int, num_groups: int,
              num_valid: Optional[torch.Tensor]) -> None:
    _require_cuda(x, "features")
    _require_cuda(indices, "indices")
    if x.dim() != 2 or x.dtype not in _BN_DTYPES:
        raise RuntimeError(f"masked_group_norm: features must be a [rows, C] float32 / float16 / bfloat16 matrix, got "
                           f"{tuple(x.shape)} {x.dtype}")
    if indices.dim() != 2 or indices.dtype != torch.int32 or indices.shape[0] != x.shape[0] or indices.shape[1] < 1:
        raise RuntimeError(f"masked_group_norm: int32 indices [rows, ndim + 1] expected, got {tuple(indices.shape)} "
                           f"{indices.dtype}")
    if num_valid is not None and (num_valid.dtype != torch.int32 or num_valid.device != x.device):
        raise RuntimeError("masked_group_norm: num_valid must be an int32 tensor on the features' device")
    c = x.shape[1]
    if not 1 <= int(batch_size) <= GROUP_NORM_MAX_BATCH:
        raise RuntimeError(f"masked_group_norm: batch_size must be in [1, 2^20], got {batch_size}")
    if not 1 <= c <= GROUP_NORM_MAX_CHANNELS:
        raise RuntimeError(f"masked_group_norm: channels must be in [1, 65536], got {c}")
    if int(num_groups) < 1 or c % int(num_groups):
        raise RuntimeError(f"masked_group_norm: num_groups {num_groups} must divide the channels {c}")


def _gn_desc(x, indices, batch_size, num_groups, num_valid, code) -> "_cabi.MaskedGroupNorm":
    d = _cabi.MaskedGroupNorm()
    d.rows, d.row_ints, d.batch_size, d.channels = x.shape[0], indices.shape[1], int(batch_size), x.shape[1]
    d.groups, d.dtype, d.param_dtype = int(num_groups), _DTYPE_CODE[x.dtype], code
    d.coords, d.num_valid, d.x = _ptr(indices), _ptr(num_valid), _ptr(x)
    return d


GROUP_NORM_ACTS = {None: _cabi.SPX_GN_ACT_NONE, "relu": _cabi.SPX_GN_ACT_RELU, "silu": _cabi.SPX_GN_ACT_SILU}


def _gn_act_code(act: Optional[str]) -> int:
    if not isinstance(act, (str, type(None))) or act not in GROUP_NORM_ACTS:
        raise RuntimeError(f"masked_group_norm: act must be None, 'relu' or 'silu', got {act!r}")
    return GROUP_NORM_ACTS[act]


def _gn_mod_operand(t: Optional[torch.Tensor], x: torch.Tensor, batch_size: int, what: str) -> Optional[torch.Tensor]:
    """``scale`` / ``shift`` as the contiguous fp32 ``[batch_size, C]`` matrix the kernels read (a copy when it is
    not one already)."""
    if t is None:
        return None
    _require_cuda(t, f"GroupNorm {what}")
    if t.device != x.device:
        raise RuntimeError(f"masked_group_norm: {what} must be on the features' device {x.device}, got {t.device}")
    if not t.is_floating_point():
        raise RuntimeError(f"masked_group_norm: {what} must be a floating-point tensor, got {t.dtype}")
    if tuple(t.shape) != (int(batch_size), x.shape[1]):
        raise RuntimeError(f"masked_group_norm: {what} must be [batch_size, C] = [{int(batch_size)}, {x.shape[1]}], "
                           f"got {tuple(t.shape)}")
    return t.to(torch.float32).contiguous()


def _gn_mod_desc(d: "_cabi.MaskedGroupNorm", scale, shift, act_code: int) -> "_cabi.MaskedGroupNormMod":
    m = _cabi.MaskedGroupNormMod()
    m.norm = d
    m.scale, m.shift, m.act = _ptr(scale), _ptr(shift), act_code
    return m


def masked_group_norm_forward(x: torch.Tensor, indices: torch.Tensor, batch_size: int, num_valid: Optional[torch.Tensor],
                              num_groups: int, weight: Optional[torch.Tensor], bias: Optional[torch.Tensor],
                              eps: float, scale: Optional[torch.Tensor] = None, shift: Optional[torch.Tensor] = None,
                              act: Optional[str] = None):
    """Per-sample GroupNorm of the rows ``r < num_valid`` (all rows when ``num_valid`` is None) whose batch index
    ``indices[r, 0]`` is in ``[0, batch_size)``; every other row of ``y`` is 0.  Returns ``(y, mean, invstd, order,
    offsets, cstart)``: the fp32 statistics ``[batch_size, num_groups]`` and the grouping of the rows by sample,
    which :func:`masked_group_norm_backward` reuses.  No host synchronisation; bit-reproducible whatever the
    padding.

    ``scale`` / ``shift`` (``[batch_size, C]``, float; computed in fp32) modulate the normalised value h of a row of
    sample b as ``h * (1 + scale[b]) + shift[b]``, and ``act`` (None, ``"relu"`` or ``"silu"``) is applied to the
    result, in the same kernel."""
    _gn_check(x, indices, batch_size, num_groups, num_valid)
    x, indices = x.contiguous(), indices.contiguous()
    code = _bn_param_code(x, [weight, bias], "masked_group_norm")
    if not eps > 0:
        raise RuntimeError(f"masked_group_norm: eps must be positive, got {eps}")
    act_code = _gn_act_code(act)
    scale = _gn_mod_operand(scale, x, batch_size, "scale")
    shift = _gn_mod_operand(shift, x, batch_size, "shift")
    rows, c = x.shape
    b, g = int(batch_size), int(num_groups)
    y = torch.empty_like(x)
    mean = torch.empty((b, g), dtype=torch.float32, device=x.device)
    invstd = torch.empty((b, g), dtype=torch.float32, device=x.device)
    order = torch.empty((rows,), dtype=torch.int32, device=x.device)
    offsets = torch.empty((b + 1,), dtype=torch.int32, device=x.device)
    cstart = torch.empty((b + 1,), dtype=torch.int32, device=x.device)
    d = _gn_desc(x, indices, b, g, num_valid, code)
    d.eps, d.y, d.weight, d.bias = float(eps), _ptr(y), _ptr(weight), _ptr(bias)
    d.mean, d.invstd, d.order, d.offsets, d.cstart = (mean.data_ptr(), invstd.data_ptr(), _ptr(order),
                                                      offsets.data_ptr(), cstart.data_ptr())
    m = _gn_mod_desc(d, scale, shift, act_code)
    lib = _lib()
    ws = _bytes(lib.spx_masked_group_norm_workspace_size(rows, b, c), x.device)
    _cabi.check(lib.spx_masked_group_norm_mod_fwd(ctypes.byref(m), ws.data_ptr(), ws.numel(), _stream()),
                "masked_group_norm_fwd")
    return y, mean, invstd, order, offsets, cstart


def masked_group_norm_backward(x: torch.Tensor, dy: torch.Tensor, indices: torch.Tensor, batch_size: int,
                               num_valid: Optional[torch.Tensor], num_groups: int, weight: Optional[torch.Tensor],
                               mean: torch.Tensor, invstd: torch.Tensor, order: torch.Tensor, offsets: torch.Tensor,
                               cstart: torch.Tensor, need_weight_grad: bool = True, need_bias_grad: bool = True,
                               bias: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None,
                               shift: Optional[torch.Tensor] = None, act: Optional[str] = None,
                               need_scale_grad: Optional[bool] = None, need_shift_grad: Optional[bool] = None):
    """``(dx, dweight, dbias, dscale, dshift)`` of :func:`masked_group_norm_forward`, from its statistics and
    grouping (nothing is sorted again).  dx is 0 on padding and dropped rows; the parameter gradients (None when not
    needed) have the parameters' dtype (float32 without ``weight``).  ``bias``, ``scale``, ``shift`` and ``act`` are
    those of the forward (``bias`` is read when there is an activation or a scale gradient); ``dscale`` / ``dshift``
    are fp32 ``[batch_size, C]``, computed when ``need_scale_grad`` / ``need_shift_grad`` (default: when ``scale`` /
    ``shift`` is given), else None."""
    _gn_check(x, indices, batch_size, num_groups, num_valid)
    x, indices, dy = x.contiguous(), indices.contiguous(), dy.contiguous()
    if dy.shape != x.shape or dy.dtype != x.dtype:
        raise RuntimeError("masked_group_norm: the output gradient must match the features' shape and dtype")
    code = _bn_param_code(x, [weight, bias], "masked_group_norm")
    act_code = _gn_act_code(act)
    need_scale_grad = scale is not None if need_scale_grad is None else need_scale_grad
    need_shift_grad = shift is not None if need_shift_grad is None else need_shift_grad
    scale = _gn_mod_operand(scale, x, batch_size, "scale")
    shift = _gn_mod_operand(shift, x, batch_size, "shift")
    pdt = torch.float32 if code == _cabi.SPX_F32 else x.dtype
    rows, c = x.shape
    b, g = int(batch_size), int(num_groups)
    for t, shape in ((mean, (b, g)), (invstd, (b, g)), (order, (rows,)), (offsets, (b + 1,)), (cstart, (b + 1,))):
        if tuple(t.shape) != shape or not t.is_contiguous() or t.device != x.device:
            raise RuntimeError("masked_group_norm: the saved statistics and grouping do not match the features")
    dx = torch.empty_like(x)
    dw = torch.empty((c,), dtype=pdt, device=x.device) if need_weight_grad else None
    db = torch.empty((c,), dtype=pdt, device=x.device) if need_bias_grad else None
    ds = torch.empty((b, c), dtype=torch.float32, device=x.device) if need_scale_grad else None
    dt = torch.empty((b, c), dtype=torch.float32, device=x.device) if need_shift_grad else None
    d = _gn_desc(x, indices, b, g, num_valid, code)
    d.dy, d.dx, d.weight, d.bias, d.dweight, d.dbias = _ptr(dy), _ptr(dx), _ptr(weight), _ptr(bias), _ptr(dw), _ptr(db)
    d.mean, d.invstd, d.order, d.offsets, d.cstart = (mean.data_ptr(), invstd.data_ptr(), _ptr(order),
                                                      offsets.data_ptr(), cstart.data_ptr())
    m = _gn_mod_desc(d, scale, shift, act_code)
    m.dscale, m.dshift = _ptr(ds), _ptr(dt)
    lib = _lib()
    ws = _bytes(lib.spx_masked_group_norm_workspace_size(rows, b, c), x.device)
    _cabi.check(lib.spx_masked_group_norm_mod_bwd(ctypes.byref(m), ws.data_ptr(), ws.numel(), _stream()),
                "masked_group_norm_bwd")
    return dx, dw, db, ds, dt


# ---------------------------------------------------------------------------- cross-rank BatchNorm
SYNC_BN_MAX_ROWS = 1 << 24          # rows per rank and call: every count crosses the exchange as an exact fp32 value


class SyncBNTransport:
    """How the per-rank BatchNorm vectors of one :class:`MaskedSyncBatchNorm1d` call reach every rank.  ``kind`` is
    "peer" (the installed :class:`~spconv_b200.pytorch.dist.PeerGroup`, ``spx_peer_allgather``), "dist"
    (``torch.distributed.all_gather_into_tensor`` on ``group``) or "local" (one rank, no exchange).  The forward
    picks it and its backward reuses it."""

    __slots__ = ("kind", "peers", "group", "world")

    def __init__(self, kind: str, peers=None, group=None, world: int = 1):
        self.kind, self.peers, self.group, self.world = kind, peers, group, world


def sync_bn_transport(process_group=None) -> SyncBNTransport:
    """The peer route when a group is installed (:func:`set_peer_group`), else ``torch.distributed`` when
    ``process_group`` (default: the world) has more than one rank, else one rank.  Raises when ``process_group``
    and the installed peer group disagree on the number of ranks."""
    import torch.distributed as dist
    initialized = dist.is_available() and dist.is_initialized()
    if _PEERS is not None:
        if process_group is not None and initialized and dist.get_world_size(process_group) != _PEERS.world:
            raise RuntimeError(f"masked_sync_batch_norm: process_group has {dist.get_world_size(process_group)} ranks, "
                               f"the installed peer group {_PEERS.world}")
        return SyncBNTransport("peer", peers=_PEERS, world=_PEERS.world)
    if initialized:
        world = dist.get_world_size(process_group)
        if world > 1:
            return SyncBNTransport("dist", group=process_group, world=world)
    return SyncBNTransport("local")


def _sync_bn_check(x: torch.Tensor, transport: SyncBNTransport) -> None:
    rows, c = x.shape
    if rows > SYNC_BN_MAX_ROWS:
        raise RuntimeError(f"masked_sync_batch_norm: {rows} rows, at most 2^24 per rank and call")
    if transport.kind == "peer":
        if transport.world > _cabi.SPX_MAX_PEERS or not 0 <= transport.peers.rank < transport.world:
            raise RuntimeError(f"masked_sync_batch_norm: bad peer group (world {transport.world}, "
                               f"rank {transport.peers.rank})")
        need = (2 * c + 1 + 3) // 4 * 16
        if need > transport.peers.group.capacity_bytes:
            raise RuntimeError(f"masked_sync_batch_norm: {2 * c + 1} fp32 values exceed the peer group's exchange "
                               f"capacity of {transport.peers.group.capacity_bytes} bytes")


def _sync_bn_gather(local: torch.Tensor, transport: SyncBNTransport) -> torch.Tensor:
    """[world, 2 C + 1]: every rank's vector in rank order, the same bits on every rank."""
    if transport.kind == "local":
        return local.view(1, -1)
    out = torch.empty((transport.world, local.numel()), dtype=torch.float32, device=local.device)
    if transport.kind == "peer":
        _cabi.check(_lib().spx_peer_allgather(ctypes.byref(transport.peers.group), local.data_ptr(), local.numel(),
                                              out.data_ptr(), _stream()), "peer_allgather")
    else:
        import torch.distributed as dist
        dist.all_gather_into_tensor(out, local, group=transport.group)
    return out


def _sync_bn_desc(x, num_valid, weight, code, world=1) -> "_cabi.MaskedSyncBN":
    d = _cabi.MaskedSyncBN()
    d.rows, d.channels = x.shape
    d.dtype, d.param_dtype, d.world = _DTYPE_CODE[x.dtype], code, world
    d.num_valid, d.x, d.weight = _ptr(num_valid), _ptr(x), _ptr(weight)
    return d


def masked_sync_batch_norm_forward(x: torch.Tensor, num_valid: Optional[torch.Tensor], weight: Optional[torch.Tensor],
                                   bias: Optional[torch.Tensor], running_mean: Optional[torch.Tensor],
                                   running_var: Optional[torch.Tensor], num_batches_tracked: Optional[torch.Tensor],
                                   momentum: Optional[float], eps: float, transport: SyncBNTransport):
    """:func:`masked_batch_norm_forward` with statistics over the valid rows of every rank of ``transport``:
    ``(y, mean, invstd)``, where mean / invstd and the running stats come out bit-identical on every rank.  Every
    rank must call it, also one with no rows, in the same order as its other exchanges."""
    x = _bn_features(x, num_valid)
    code = _bn_param_code(x, [weight, bias, running_mean, running_var])
    _sync_bn_check(x, transport)
    rows, c = x.shape
    cumulative = momentum is None
    if cumulative and running_mean is not None and num_batches_tracked is None:
        raise RuntimeError("masked_sync_batch_norm: momentum=None needs num_batches_tracked")
    y = torch.empty_like(x)
    mean = torch.empty((c,), dtype=torch.float32, device=x.device)
    invstd = torch.empty((c,), dtype=torch.float32, device=x.device)
    local = torch.empty((2 * c + 1,), dtype=torch.float32, device=x.device)
    lib = _lib()
    ws = _bytes(lib.spx_masked_sync_bn_workspace_size(rows, c), x.device)
    d = _sync_bn_desc(x, num_valid, weight, code)
    d.local = local.data_ptr()
    _cabi.check(lib.spx_masked_sync_bn_fwd_local(ctypes.byref(d), ws.data_ptr(), ws.numel(), _stream()),
                "masked_sync_bn_fwd_local")
    gathered = _sync_bn_gather(local, transport)
    d.world, d.gathered, d.y = gathered.shape[0], gathered.data_ptr(), _ptr(y)
    d.bias, d.running_mean, d.running_var = _ptr(bias), _ptr(running_mean), _ptr(running_var)
    d.num_batches_tracked = _ptr(num_batches_tracked)
    d.momentum, d.cumulative, d.eps = 0.0 if cumulative else float(momentum), int(cumulative), float(eps)
    d.save_mean, d.save_invstd = mean.data_ptr(), invstd.data_ptr()
    _cabi.check(lib.spx_masked_sync_bn_fwd_merge(ctypes.byref(d), ws.data_ptr(), ws.numel(), _stream()),
                "masked_sync_bn_fwd_merge")
    return y, mean, invstd


def masked_sync_batch_norm_backward(x: torch.Tensor, dy: torch.Tensor, num_valid: Optional[torch.Tensor],
                                    weight: Optional[torch.Tensor], mean: torch.Tensor, invstd: torch.Tensor,
                                    transport: SyncBNTransport, need_weight_grad: bool = True,
                                    need_bias_grad: bool = True):
    """``(dx, dweight, dbias)`` of :func:`masked_sync_batch_norm_forward`: dx with the sums over every rank,
    dweight / dbias the sums over this rank's rows only (they are averaged later like any other parameter
    gradient).  Every rank must call it."""
    x = _bn_features(x, num_valid)
    dy = dy.contiguous()
    if dy.shape != x.shape or dy.dtype != x.dtype:
        raise RuntimeError("masked_sync_batch_norm: the output gradient must match the features' shape and dtype")
    code = _bn_param_code(x, [weight])
    _sync_bn_check(x, transport)
    pdt = weight.dtype if weight is not None else torch.float32
    rows, c = x.shape
    dx = torch.empty_like(x)
    dw = torch.empty((c,), dtype=pdt, device=x.device) if need_weight_grad else None
    db = torch.empty((c,), dtype=pdt, device=x.device) if need_bias_grad else None
    local = torch.empty((2 * c + 1,), dtype=torch.float32, device=x.device)
    lib = _lib()
    ws = _bytes(lib.spx_masked_sync_bn_workspace_size(rows, c), x.device)
    d = _sync_bn_desc(x, num_valid, weight, code)
    d.dy, d.dx, d.dweight, d.dbias = _ptr(dy), _ptr(dx), _ptr(dw), _ptr(db)
    d.save_mean, d.save_invstd, d.local = mean.data_ptr(), invstd.data_ptr(), local.data_ptr()
    _cabi.check(lib.spx_masked_sync_bn_bwd_local(ctypes.byref(d), ws.data_ptr(), ws.numel(), _stream()),
                "masked_sync_bn_bwd_local")
    gathered = _sync_bn_gather(local, transport)
    d.world, d.gathered = gathered.shape[0], gathered.data_ptr()
    _cabi.check(lib.spx_masked_sync_bn_bwd_merge(ctypes.byref(d), ws.data_ptr(), ws.numel(), _stream()),
                "masked_sync_bn_bwd_merge")
    return dx, dw, db


def last_kernel_family() -> int:
    """0 none, 1 generic FMA kernels, 2 wgmma tensor-core kernels (what served the last GEMM call)."""
    return int(_lib().spx_last_kernel_family())


def launch_count(reset: bool = False) -> int:
    return int(_lib().spx_launch_count(int(reset)))
