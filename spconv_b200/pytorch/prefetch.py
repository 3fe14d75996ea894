"""Rulebook prefetch: build the NEXT batch's rulebooks while the current batch computes.

A rulebook depends on coordinates only -- not on features or weights -- so, like a data loader's H2D
copy, it can run ahead of the step that consumes it:

    pre = spconv.RulebookPrefetcher(model)          # or a list of layers, in application order
    x_next = spconv.SparseConvTensor(f_next, i_next, shape, bs)
    pre.prefetch(x_next)                            # side stream (+ worker thread), returns immediately
    ... forward / backward of the current batch ...
    y = model(pre.ready(x_next))                    # the layers find their rulebooks through indice_key

Why it pays: (i) rulebook kernels are latency-bound integer work, the GEMM kernels are LSU / L2-bound --
off the critical path they cost nothing but SM time (bench.py: 0.18 -> 0.135-0.14 ms per config-2 step); (ii) a strided conv reads its
output count back to the host (``spx_conv_rulebook_stage1``, as the reference does,
``spconv/csrc/sparse/indices.py:1454-1455``) -- on the training stream that read-back drains the whole
GEMM queue three times per SECOND-encoder step; on the prefetch stream it only waits for the rulebook
kernels before it.  With ``background=True`` the host side of the chain runs in a worker thread (the
native calls release the GIL), so the training thread only issues GEMM launches.

Which layers: every sparse conv with an ``indice_key`` in APPLICATION order, following the coordinate
set through the strided layers (``out_indices`` of one layer = input of the next).  The order is the
module order, which is right for ``SparseSequential``-style encoders; pass an explicit list for other
topologies.  The chain stops at the first layer it cannot follow (no key, Native algo, inverse /
transposed conv): later layers build their rulebooks in the forward pass as usual.

The reference lets only SubM layers reuse a cached rulebook (``spconv/pytorch/conv.py:376-383``); a
strided conv accepts a cached one here only when this class built it (``prefetched`` flag) for exactly
that geometry and input.
"""
from __future__ import annotations

import concurrent.futures
from typing import List, Optional

import torch

from ..core import ConvAlgo
from . import ops
from .conv import SparseConvolution
from .core import ImplicitGemmIndiceData, SparseConvTensor


def prefetchable_chain(model_or_layers) -> List[SparseConvolution]:
    """The sparse convs whose rulebooks can be built from the input coordinates alone, in order."""
    mods = model_or_layers.modules() if isinstance(model_or_layers, torch.nn.Module) else model_or_layers
    chain = []
    for m in mods:
        if not isinstance(m, SparseConvolution) or m.conv1x1:
            continue
        if m.indice_key is None or m.algo == ConvAlgo.Native or m.inverse or m.transposed:
            break
        chain.append(m)
    return chain


def input_level_subm_layers(model) -> List[SparseConvolution]:
    """SubM layers reached before the first layer that changes the coordinate set (one per key)."""
    out, seen = [], set()
    for m in prefetchable_chain(model):
        if not m.subm:
            break
        if m.indice_key not in seen:
            seen.add(m.indice_key)
            out.append(m)
    return out


class RulebookPrefetcher:
    def __init__(self, model_or_layers, stream: Optional[torch.cuda.Stream] = None, training: bool = True,
                 background: bool = False):
        self.layers = prefetchable_chain(model_or_layers)
        self.stream = stream
        self.training = training
        self._pool = concurrent.futures.ThreadPoolExecutor(max_workers=1) if background else None

    # ------------------------------------------------------------------ the work (any thread)
    def _build(self, x: SparseConvTensor, device_index: int):
        torch.cuda.set_device(device_index)
        with torch.cuda.stream(self.stream):
            inds, shape = x.indices, list(x.spatial_shape)
            for m in self.layers:
                algo = m.algo if x.force_algo is None else x.force_algo
                done = x.indice_dict.get(m.indice_key)
                if done is None:
                    res = ops.get_indice_pairs_implicit_gemm(
                        inds, x.batch_size, shape, algo, ksize=m.kernel_size, stride=m.stride, padding=m.padding,
                        dilation=m.dilation, out_padding=m.output_padding, subm=m.subm, transpose=False,
                        is_train=(not m.subm) or self.training)
                    out_shape = shape if m.subm else ops.get_conv_output_size(shape, m.kernel_size, m.stride,
                                                                             m.padding, m.dilation)
                    done = ImplicitGemmIndiceData.from_rulebook(
                        res, inds, None, m.subm, spatial_shape=shape, out_spatial_shape=out_shape, algo=algo,
                        ksize=m.kernel_size, stride=m.stride, dilation=m.dilation, padding=m.padding, prefetched=True)
                    x.indice_dict[m.indice_key] = done
                elif not done.is_subm and not m.subm:
                    raise ValueError(f"indice_key {m.indice_key} is used by two strided layers")
                if not m.subm:
                    inds, shape = done.out_indices, list(done.out_spatial_shape)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return ev

    # ------------------------------------------------------------------ API
    def prefetch(self, x: SparseConvTensor, wait_current: bool = True) -> SparseConvTensor:
        """Start building the rulebooks of ``x`` on the prefetch stream; they land in ``x.indice_dict``.
        ``x.indices`` must be resident or its copy already queued on the prefetch stream / the current
        stream: with ``wait_current`` the prefetch stream first waits for the current stream's queue as
        of this call (pass False when the coordinates are known to be complete -- the rulebooks then
        start at once instead of behind the previous step's kernels)."""
        dev = x.indices.device
        if self.stream is None:
            self.stream = torch.cuda.Stream(device=dev)
        cur = torch.cuda.current_stream(dev)
        if wait_current and cur != self.stream:
            self.stream.wait_stream(cur)
        x.indices.record_stream(self.stream)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        if self._pool is not None:
            x._spx_prefetch = self._pool.submit(self._build, x, idx)
        else:
            x._spx_prefetch = self._build(x, idx)
        return x

    def ready(self, x: SparseConvTensor) -> SparseConvTensor:
        """Make the current stream wait for the prefetch of ``x`` (joins the worker thread if there is
        one; no device synchronisation)."""
        pending = getattr(x, "_spx_prefetch", None)
        if pending is None:
            return x
        ev = pending.result() if isinstance(pending, concurrent.futures.Future) else pending
        x._spx_prefetch = None
        cur = torch.cuda.current_stream(x.indices.device)
        cur.wait_event(ev)
        for data in x.indice_dict.values():              # tell the caching allocator about the consumer stream
            if not isinstance(data, ImplicitGemmIndiceData):
                continue
            for t in (data.out_indices, data.pair_fwd, data.pair_bwd, *data.pair_mask_fwd_splits,
                      *data.pair_mask_bwd_splits, *data.mask_argsort_fwd_splits, *data.mask_argsort_bwd_splits):
                if isinstance(t, torch.Tensor) and t.is_cuda and t.numel():
                    t.record_stream(cur)
            for owner in (*data.mask_argsort_fwd_splits, *data.mask_argsort_bwd_splits):
                cache = getattr(owner, "_spx_tile_cache", None)
                if cache is not None:
                    cache[1].record_stream(cur)
                    cache[2].record_stream(cur)
        return x

    def shutdown(self):
        if self._pool is not None:
            self._pool.shutdown(wait=True)
            self._pool = None
