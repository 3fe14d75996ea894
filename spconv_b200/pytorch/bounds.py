"""Output bounds of the strided layers: run a net with strided convs / pools at static shapes, without a host
synchronisation, so that a whole step replays as one CUDA graph.  ``MaskedAddTableMisaligned`` and
``MaskedRemoveDuplicate`` have bounds and status words too and are covered alike.

    bounds = spconv.set_output_bounds(net, example)       # one eager forward, sets num_out_act_bound per layer
    step = spconv.graph_capture(fn, example.pad_to(N).features, ...)
    ...
    spconv.check_bounds(net)                              # every k steps: one small read-back per bounded layer
"""
from __future__ import annotations

import math
from typing import Dict, Union

from torch import nn

from .conv import SparseConvolution
from .core import SparseConvTensor
from .pool import _SparsePool
from .spatial import MaskedRemoveDuplicate
from .tables import MaskedAddTableMisaligned
from .utils import MaskedPointToVoxel

# modules whose output count depends on the data: the bound is their padded row count, num_valid the true count
_MASKED_BOUNDED = (MaskedAddTableMisaligned, MaskedRemoveDuplicate)


def _strided_modules(net: nn.Module):
    for name, mod in net.named_modules():
        if isinstance(mod, SparseConvolution) and not mod.subm and not mod.inverse and not mod.conv1x1:
            yield name, mod
        elif isinstance(mod, _SparsePool) and not mod.subm:
            yield name, mod
        elif isinstance(mod, _MASKED_BOUNDED):
            yield name, mod


def _out_count(mod: nn.Module, out: SparseConvTensor) -> int:
    """the output count of one eager forward: the row count of an unbounded strided layer, the true count (one
    read-back) of a masked module, whose unbounded output is padded to its operands' total row count"""
    if isinstance(mod, _MASKED_BOUNDED):
        return int(out.num_valid)
    return out.features.shape[0]


def set_output_bounds(net: nn.Module, example_input: SparseConvTensor, margin: float = 1.25) -> Dict[str, int]:
    """Run one eager, unbounded forward of ``net`` on ``example_input`` and set every strided module's
    ``num_out_act_bound`` to ``ceil(M * margin)`` rounded up to a multiple of 128, M being the layer's
    output count on the example.  Returns ``{module name: bound}``.  Pick the example (and the margin)
    so that no later input produces more outputs; ``check_bounds`` tells when one did."""
    counts: Dict[str, int] = {}
    hooks, saved = [], {}
    for name, mod in _strided_modules(net):
        saved[name] = mod.num_out_act_bound
        mod.num_out_act_bound = None
        hooks.append(mod.register_forward_hook(
            lambda m, inp, out, name=name: counts.__setitem__(name, max(counts.get(name, 0), _out_count(m, out)))))
    try:
        net(example_input)
    except Exception:
        for name, mod in _strided_modules(net):
            mod.num_out_act_bound = saved[name]
        raise
    finally:
        for h in hooks:
            h.remove()
    bounds = {}
    for name, mod in _strided_modules(net):
        if name in counts:
            bounds[name] = mod.num_out_act_bound = max(128, 128 * math.ceil(math.ceil(counts[name] * margin) / 128))
        else:
            mod.num_out_act_bound = saved[name]
    return bounds


def check_bounds(tensor_or_net: Union[SparseConvTensor, nn.Module, MaskedPointToVoxel]) -> None:
    """Read the status words of the bounded layers (of a net: every bounded module; of a tensor: the layers
    it went through; of a ``MaskedPointToVoxel``: its own, whose bound is ``max_num_voxels_total``) and raise
    ``RuntimeError`` naming the first layer whose bound was exceeded.  This is the one call of the bounded mode
    that synchronises; the words of a net or a voxel generator are cleared by the read."""
    if isinstance(tensor_or_net, SparseConvTensor):
        words = dict(tensor_or_net.bound_status or {})
        clear = False
    elif isinstance(tensor_or_net, MaskedPointToVoxel):
        words = {"MaskedPointToVoxel (bound: max_num_voxels_total)": tensor_or_net._bound_status}
        clear = True
    else:
        words = {name: mod._bound_status for name, mod in _strided_modules(tensor_or_net)
                 if mod._bound_status is not None}
        clear = True
    read = {name: int(word.item()) for name, word in words.items()}
    if clear:
        for name, word in words.items():
            if read[name]:
                word.zero_()
    for name, bits in read.items():
        if bits & 2:
            raise RuntimeError(f"layer {name!r}: the hash table sized from num_out_act_bound overflowed (far more "
                               "outputs than the bound); its output is empty. Raise the bound.")
        if bits & 1:
            raise RuntimeError(f"layer {name!r}: more outputs than num_out_act_bound; the outputs ranked beyond "
                               "the bound were dropped. Raise the bound (spconv.set_output_bounds).")
