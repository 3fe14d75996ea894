"""CUDA-graph replay of a fixed-shape step through the public API.

The device time of a SubM layer-step at LiDAR sizes (~0.15 ms) is several times smaller than the
host time torch + Python need to issue its ~25 launches eagerly, so a step whose SHAPES repeat
(the same cloud evaluated many times, a static calibration batch, a benchmark) is best replayed as
one graph.  ``graph_capture`` wraps the boilerplate: warm-up on a side stream, capture, static
input buffers that later calls copy into.  Every kernel of this library is capturable; the one host
read-back is the output count of an UNBOUNDED regular-conv rulebook (``spx_conv_rulebook_stage1``; the
reference syncs at the same point, ``spconv/csrc/sparse/indices.py:1454-1455``).  Give the strided layers
an output bound (``spconv.set_output_bounds``) and pad the inputs to one size
(``SparseConvTensor.pad_to``): then the rulebooks keep the count on the device and a whole encoder
step, forward and backward, captures; ``spconv.check_bounds`` tells when a bound was exceeded.  Of the
modules, ``SparseGlobalMaxPool`` / ``SparseGlobalAvgPool`` read the per-sample counts back to the host:
``MaskedGlobalMaxPool`` / ``MaskedGlobalAvgPool`` reduce on the device and capture.  Likewise
``AddTableMisaligned`` / ``functional.sparse_add`` read the size of the union back: ``MaskedAddTableMisaligned``
(``functional.masked_sparse_add``), ``MaskedRemoveDuplicate``, ``MaskedAddTable`` and ``MaskedJoinTable`` take
padded tensors and capture.  In front of the first layer, ``PointToVoxel`` reads each cloud's voxel count back:
``MaskedPointToVoxel`` voxelises a padded batch of clouds with the count on the device and captures,
``PointVoxelScatter`` (a dynamic VFE's per-voxel max / mean / sum of point features, in place of
``torch.unique`` + scatter) captures, and ``gather_features_by_pc_voxel_id`` (the per-point read-out) does not
synchronise.
"""
from __future__ import annotations

from typing import Any, Callable, Sequence

import torch


class GraphedStep:
    """``step = GraphedStep(fn, example_inputs)`` then ``out = step(*inputs)``: inputs are copied into
    the captured static buffers (shapes / dtypes must match the examples), the graph is replayed and
    the STATIC output objects are returned (clone them to keep a result across replays)."""

    def __init__(self, fn: Callable[..., Any], example_inputs: Sequence[torch.Tensor], warmup: int = 3):
        assert all(isinstance(t, torch.Tensor) and t.is_cuda for t in example_inputs), "CUDA tensor inputs only"
        self.fn = fn
        self.static_inputs = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                      # warm-up configures kernels / allocator pools
            for _ in range(max(warmup, 1)):
                fn(*self.static_inputs)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(self.graph):
                self.static_outputs = fn(*self.static_inputs)
        except Exception as e:
            torch.cuda.synchronize()
            raise RuntimeError(
                "graph_capture failed. A regular SparseConv / SparseMaxPool without an output bound builds its "
                "rulebook with one host read-back (the output count) and cannot be captured: call "
                "spconv.set_output_bounds(net, example) first and pad the inputs with SparseConvTensor.pad_to, or "
                f"capture SubM-only stacks. Original error: {type(e).__name__}: {e}") from e

    def __call__(self, *inputs: torch.Tensor):
        assert len(inputs) == len(self.static_inputs), "same number of inputs as at capture time"
        for dst, src in zip(self.static_inputs, inputs):
            if dst.data_ptr() != src.data_ptr():
                assert dst.shape == src.shape and dst.dtype == src.dtype, \
                    f"graph replay needs the captured shape {tuple(dst.shape)} / dtype, got {tuple(src.shape)}"
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_outputs


def graph_capture(fn: Callable[..., Any], *example_inputs: torch.Tensor, warmup: int = 3) -> GraphedStep:
    """Capture ``fn(*example_inputs)`` (forward, or forward + backward) into a CUDA graph."""
    return GraphedStep(fn, list(example_inputs), warmup)
