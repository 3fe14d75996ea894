"""Containers that thread a :class:`SparseConvTensor` through a model
(``spconv/pytorch/modules.py:50-168`` semantics: sparse modules see the tensor, plain
``nn.Module``s see ``.features`` and are skipped on an empty tensor)."""
from __future__ import annotations

from collections import OrderedDict
from typing import Any, Optional

import torch
from torch import nn

from . import functional
from .core import SparseConvTensor


def is_spconv_module(module) -> bool:
    return isinstance(module, SparseModule)


def is_sparse_conv(module) -> bool:
    from .conv import SparseConvolution
    return isinstance(module, SparseConvolution)


class SparseModule(nn.Module):
    """Marker base: ``forward`` takes and returns a :class:`SparseConvTensor`."""

    def __init__(self, name=None):
        super().__init__()
        self.name = name
        self._sparse_unique_name = ""
        # the status word of a module with an output bound (strided conv / pool, masked sparse add, remove duplicate)
        self._bound_status: Optional[torch.Tensor] = None

    def _status_word(self, device) -> torch.Tensor:
        """This module's output-bound status word.  It lives on the module, outside any captured step, so the bits
        stay set across graph replays until spconv.check_bounds reads them."""
        if self._bound_status is None or self._bound_status.device != device:
            self._bound_status = torch.zeros((1,), dtype=torch.int32, device=device)
        return self._bound_status

    def _layer_name(self) -> str:
        """The name under which this module's status word appears in ``SparseConvTensor.bound_status``."""
        return self._sparse_unique_name or self.name or getattr(self, "indice_key", None) or type(self).__name__


def assign_name_for_sparse_modules(module: nn.Module):
    """Give every sparse module its dotted path (used as timer namespace)."""
    for qualified, child in module.named_modules():
        if isinstance(child, SparseModule):
            child._sparse_unique_name = qualified


class SparseSequential(SparseModule):
    """``nn.Sequential`` for mixed sparse / dense layers.  Accepts positional modules, one
    ``OrderedDict``, or keyword modules."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        if len(args) == 1 and isinstance(args[0], OrderedDict):
            named = list(args[0].items())
        else:
            named = [(str(i), m) for i, m in enumerate(args)]
        for key, mod in kwargs.items():
            if key in dict(named):
                raise ValueError("name exists.")
            named.append((key, mod))
        for key, mod in named:
            self.add_module(key, mod)

    def __getitem__(self, idx):
        n = len(self._modules)
        if not (-n <= idx < n):
            raise IndexError(f"index {idx} is out of range")
        return list(self._modules.values())[idx % n]

    def __len__(self):
        return len(self._modules)

    def add(self, module, name=None):
        key = str(len(self._modules)) if name is None else name
        if key in self._modules:
            raise KeyError("name exists")
        self.add_module(key, module)

    def forward(self, input: Any):
        x = input
        for layer in self._modules.values():
            if isinstance(layer, SparseModule):
                # a list comes out of ConcatTable and goes into AddTable / JoinTable (modules.py:133-134)
                assert isinstance(x, (SparseConvTensor, list))
                x = layer(x)
            elif isinstance(x, SparseConvTensor):
                # dense layers (BatchNorm1d, ReLU, ...) act on the feature matrix
                if x.indices.shape[0] != 0:
                    if isinstance(layer, nn.modules.batchnorm._BatchNorm) and layer.training:
                        x.require_unpadded("BatchNorm in training mode")
                    x = x.replace_feature(layer(x.features))
            else:
                x = layer(x)
        return x


class ToDense(SparseModule):
    """SparseConvTensor -> NC(D)HW dense tensor."""

    def forward(self, x: SparseConvTensor):
        return x.dense()


class RemoveGrid(SparseModule):
    """Drop the pre-allocated grid buffer."""

    def forward(self, x: SparseConvTensor):
        x.grid = None
        return x


class _FeatureWise(SparseModule):
    def __init__(self, inner: nn.Module):
        super().__init__()
        self.inner = inner

    def forward(self, x: SparseConvTensor):
        return x.replace_feature(self.inner(x.features))


class SparseReLU(_FeatureWise):
    def __init__(self, inplace: bool = False):
        super().__init__(nn.ReLU(inplace=inplace))


class SparseBatchNorm(_FeatureWise):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True,
                 track_running_stats=True):
        super().__init__(nn.BatchNorm1d(num_features, eps, momentum, affine, track_running_stats))

    def forward(self, x: SparseConvTensor):
        if isinstance(self.inner, (MaskedBatchNorm1d, MaskedSyncBatchNorm1d)):
            return self.inner(x)
        if self.inner.training:
            x.require_unpadded("SparseBatchNorm in training mode")
        return super().forward(x)


class SparseSyncBatchNorm(_FeatureWise):
    """``nn.SyncBatchNorm`` on the features (``spconv.pytorch.SparseSyncBatchNorm``).  It counts every row as
    data, so it refuses a padded tensor in training; :meth:`MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm`
    turns its ``inner`` into the padding-aware :class:`MaskedSyncBatchNorm1d`."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 process_group=None):
        super().__init__(nn.SyncBatchNorm(num_features, eps, momentum, affine, track_running_stats, process_group))

    def forward(self, x: SparseConvTensor):
        if isinstance(self.inner, MaskedSyncBatchNorm1d):
            return self.inner(x)
        if self.inner.training:
            x.require_unpadded("SparseSyncBatchNorm in training mode")
        return super().forward(x)


class MaskedBatchNorm1d(SparseModule, nn.BatchNorm1d):
    """``nn.BatchNorm1d`` on the features of a :class:`SparseConvTensor` whose batch statistics cover only the
    valid rows (``x.num_valid``; every row of an unpadded tensor), so a padded net trains at static shapes and
    captures as one CUDA graph.  Same constructor, parameters, buffers and ``state_dict`` keys as
    ``nn.BatchNorm1d``; convert an existing net with :meth:`convert_masked_batchnorm`.

    Training mode (and eval mode without running stats) runs the CUDA kernels of ``csrc/batchnorm.cu``: the
    results are those of ``nn.BatchNorm1d`` on the valid rows alone, computed in fp32 in a fixed order, so they
    are bit-reproducible and independent of how far the tensor is padded.  Padding rows are never read; they
    are 0 in the output and in the input gradient.  The running stats update on the device (``momentum=None``
    reads ``num_batches_tracked`` there), so nothing is read back to the host.  Eval mode with running stats
    is torch's row-wise ``F.batch_norm``, bit-identical to the unconverted module.

    Differences from ``nn.BatchNorm1d``, which raises for one value per channel where this cannot:
      * no valid row: the output is 0, every gradient is 0 and the running stats are unchanged;
      * one valid row: the normalised value is 0, so the output is ``bias``; dx = 0, dbias = dy, dweight = 0,
        and the running stats are unchanged.
    ``num_batches_tracked`` counts every training call on a non-empty tensor, as torch increments it before its
    check; a tensor without rows passes through untouched."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 device=None, dtype=None):
        nn.BatchNorm1d.__init__(self, num_features, eps, momentum, affine, track_running_stats, device, dtype)
        self.name = None
        self._sparse_unique_name = ""

    def forward(self, x: SparseConvTensor):
        feats = x.features
        if feats.shape[0] == 0:
            return x
        if feats.dim() != 2 or feats.shape[1] != self.num_features:
            raise ValueError(f"MaskedBatchNorm1d({self.num_features}): features of shape {tuple(feats.shape)}")
        momentum = self.momentum
        if self.training and self.track_running_stats and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        use_batch = self.training or (self.running_mean is None and self.running_var is None)
        if not use_batch:
            return x.replace_feature(nn.functional.batch_norm(
                feats, self.running_mean, self.running_var, self.weight, self.bias, False, 0.0, self.eps))
        track = not self.training or self.track_running_stats
        rm = self.running_mean if track else None
        rv = self.running_var if track else None
        return x.replace_feature(functional.masked_batch_norm(
            feats, self.weight, self.bias, rm, rv, self.num_batches_tracked if rm is not None else None,
            x.num_valid, momentum, self.eps))

    @classmethod
    def convert_masked_batchnorm(cls, module: nn.Module) -> nn.Module:
        """Replace, in place, every ``nn.BatchNorm1d`` (that exact type) that is a direct child of a
        :class:`SparseSequential`, and the ``inner`` BatchNorm of every :class:`SparseBatchNorm`, by a
        ``MaskedBatchNorm1d`` that takes over its parameters and buffers; returns ``module``.  ``SyncBatchNorm``,
        other subclasses and BatchNorm layers outside sparse containers (dense heads) are left alone."""
        if isinstance(module, SparseSequential):
            for key, child in list(module._modules.items()):
                if type(child) is nn.BatchNorm1d:
                    module._modules[key] = cls._from_batchnorm(child)
        elif isinstance(module, SparseBatchNorm) and type(module.inner) is nn.BatchNorm1d:
            module.inner = cls._from_batchnorm(module.inner)
        for child in module.children():
            cls.convert_masked_batchnorm(child)
        return module

    @classmethod
    def _from_batchnorm(cls, bn: nn.BatchNorm1d) -> "MaskedBatchNorm1d":
        out = cls(bn.num_features, bn.eps, bn.momentum, bn.affine, bn.track_running_stats, device="meta")
        if bn.affine:
            out.weight = bn.weight
            out.bias = bn.bias
        out.running_mean = bn.running_mean
        out.running_var = bn.running_var
        out.num_batches_tracked = bn.num_batches_tracked
        out.training = bn.training
        return out


class MaskedSyncBatchNorm1d(SparseModule, nn.SyncBatchNorm):
    """:class:`MaskedBatchNorm1d` whose training statistics cover the valid rows of every data-parallel rank, as
    ``nn.SyncBatchNorm`` does for dense tensors, but padding-aware.  Same constructor, parameters, buffers and
    ``state_dict`` keys as ``nn.SyncBatchNorm``; convert a net with :meth:`convert_masked_sync_batchnorm`.

    Each rank reduces its own valid rows (``x.num_valid``) with the kernels of ``csrc/batchnorm.cu`` into a vector
    of its count, sum and M2; the vectors are gathered in rank order and merged in that order on every rank, so
    mean, invstd, the running stats and y are computed from the same bits everywhere.  The exchange runs over the
    installed peer group (:func:`ops.set_peer_group`) when there is one, else over ``torch.distributed``
    (``process_group``, default the world) when it has more than one rank; with one rank there is no exchange
    and every result equals :class:`MaskedBatchNorm1d` bit for bit.  Nothing is read back to the host, so a
    training step captures as one CUDA graph.

    The backward exchanges the sums of dy and dy * xhat the same way, so dx uses the global sums.  The
    parameter gradients dweight / dbias are this rank's own sums, as in ``nn.SyncBatchNorm``: reduce them with
    the other parameter gradients (DDP, ``GradBucket``, ``ops.peer_allreduce_``).

    Every rank must call every training forward and backward, in the same order as its other exchanges: a
    rank whose tensor has no rows still joins, takes its running stats from the others, and gets zero
    dweight / dbias.  ``num_batches_tracked`` counts every training call.  The edge cases of the total count
    are :class:`MaskedBatchNorm1d`'s.  Eval mode with running stats is torch's ``F.batch_norm``; eval mode
    without them normalises with this rank's rows alone, like ``nn.SyncBatchNorm``."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 process_group=None, device=None, dtype=None):
        nn.SyncBatchNorm.__init__(self, num_features, eps, momentum, affine, track_running_stats, process_group,
                                  device, dtype)
        self.name = None
        self._sparse_unique_name = ""

    def forward(self, x: SparseConvTensor):
        feats = x.features
        if feats.dim() != 2 or feats.shape[1] != self.num_features:
            raise ValueError(f"MaskedSyncBatchNorm1d({self.num_features}): features of shape {tuple(feats.shape)}")
        if not self.training:
            if feats.shape[0] == 0:
                return x
            if self.running_mean is not None or self.running_var is not None:
                return x.replace_feature(nn.functional.batch_norm(
                    feats, self.running_mean, self.running_var, self.weight, self.bias, False, 0.0, self.eps))
            return x.replace_feature(functional.masked_batch_norm(
                feats, self.weight, self.bias, None, None, None, x.num_valid, self.momentum, self.eps))
        track = self.track_running_stats
        if track and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        rm = self.running_mean if track else None
        rv = self.running_var if track else None
        return x.replace_feature(functional.masked_sync_batch_norm(
            feats, self.weight, self.bias, rm, rv, self.num_batches_tracked if rm is not None else None,
            x.num_valid, self.momentum, self.eps, self.process_group))

    @classmethod
    def convert_masked_sync_batchnorm(cls, module: nn.Module, process_group=None) -> nn.Module:
        """Replace, in place, every ``nn.BatchNorm1d``, ``nn.SyncBatchNorm`` and :class:`MaskedBatchNorm1d` (those
        exact types) that is a direct child of a :class:`SparseSequential`, and the ``inner`` BatchNorm of every
        :class:`SparseBatchNorm` / :class:`SparseSyncBatchNorm`, by a ``MaskedSyncBatchNorm1d`` that takes over its
        parameters and buffers; returns ``module``.  ``process_group`` None keeps a ``SyncBatchNorm``'s own group.
        Other subclasses and BatchNorm layers outside sparse containers (dense heads) are left alone."""
        kinds = (nn.BatchNorm1d, nn.SyncBatchNorm, MaskedBatchNorm1d)
        if isinstance(module, SparseSequential):
            for key, child in list(module._modules.items()):
                if type(child) in kinds:
                    module._modules[key] = cls._from_batchnorm(child, process_group)
        elif isinstance(module, (SparseBatchNorm, SparseSyncBatchNorm)) and type(module.inner) in kinds:
            module.inner = cls._from_batchnorm(module.inner, process_group)
        for child in module.children():
            cls.convert_masked_sync_batchnorm(child, process_group)
        return module

    @classmethod
    def _from_batchnorm(cls, bn: nn.modules.batchnorm._BatchNorm, process_group=None) -> "MaskedSyncBatchNorm1d":
        group = process_group if process_group is not None else getattr(bn, "process_group", None)
        out = cls(bn.num_features, bn.eps, bn.momentum, bn.affine, bn.track_running_stats, group, device="meta")
        if bn.affine:
            out.weight = bn.weight
            out.bias = bn.bias
        out.running_mean = bn.running_mean
        out.running_var = bn.running_var
        out.num_batches_tracked = bn.num_batches_tracked
        out.training = bn.training
        return out


class MaskedGroupNorm(SparseModule, nn.GroupNorm):
    """``nn.GroupNorm`` applied per sample of a :class:`SparseConvTensor`: the statistics of sample ``b`` and group
    ``g`` (channels ``[g C/G, (g+1) C/G)``) are the mean and biased variance over every value of that group in the
    rows of sample ``b``, as ``F.group_norm(x[rows_b].T[None], G, weight, bias, eps)`` computes them.
    ``MaskedGroupNorm(C, C)`` is InstanceNorm.  Same constructor, parameters and ``state_dict`` keys as
    ``nn.GroupNorm``; :meth:`from_groupnorm` takes over an existing module's parameters.

    Row ``r`` belongs to sample ``b`` when ``r < x.num_valid`` (every row of an unpadded tensor) and
    ``x.indices[r, 0] == b`` with ``0 <= b < x.batch_size``.  Every other row (padding, or a batch index out of
    range) is dropped: never read, and 0 in the output and in the input gradient.  The kernels of
    ``csrc/group_norm.cu`` sum in fp32 in an order fixed by each sample's rows, with no float atomics and no host
    read-back, so results are bit-reproducible, independent of the padding, and a padded step captures as one CUDA
    graph.  An empty sample computes nothing; one row with one channel per group normalises to 0, so its output is
    ``bias``, as in torch.  GroupNorm has no running statistics: eval mode is the same computation.

    A plain ``nn.GroupNorm`` inside :class:`SparseSequential` sees ``x.features`` ``[N, C]`` and so treats every row
    as its own batch element, normalising it over its own C/G channels; that behaviour of dense layers is left as it
    is.  Use this module for per-sample statistics.

    Modulation and activation (AdaGN, the ResBlock norm of diffusion U-Nets): ``forward(x, scale, shift)`` with
    ``scale`` / ``shift`` of shape ``[x.batch_size, C]`` (either may be None; any float dtype, computed in fp32)
    gives, for a kept row of sample ``b``, ``act(h * (1 + scale[b]) + shift[b])`` where ``h`` is the GroupNorm output
    above.  The ``1 + scale`` convention is guided-diffusion's ``use_scale_shift_norm``: a zero scale is the
    identity.  ``act`` is None, ``"relu"`` or ``"silu"``, fixed at construction.  The modulation and the activation
    run in the same kernels, so the output is written once and the backward recomputes them from x, still four
    launches; dropped rows never read ``scale`` / ``shift`` and add nothing to their gradients, which are summed in a
    fixed order like the others.  Inside :class:`SparseSequential` the module is called with ``x`` alone."""

    def __init__(self, num_groups, num_channels, eps=1e-5, affine=True, device=None, dtype=None, *, act=None):
        if act not in (None, "relu", "silu"):
            raise ValueError(f"MaskedGroupNorm: act must be None, 'relu' or 'silu', got {act!r}")
        nn.GroupNorm.__init__(self, num_groups, num_channels, eps, affine, device, dtype)
        self.act = act
        self.name = None
        self._sparse_unique_name = ""

    def forward(self, x: SparseConvTensor, scale: Optional[torch.Tensor] = None,
                shift: Optional[torch.Tensor] = None):
        feats = x.features
        if feats.dim() != 2 or feats.shape[1] != self.num_channels:
            raise ValueError(f"MaskedGroupNorm({self.num_groups}, {self.num_channels}): features of shape "
                             f"{tuple(feats.shape)}")
        return x.replace_feature(functional.masked_group_norm(
            feats, self.weight, self.bias, x.indices, x.batch_size, x.num_valid, self.num_groups, self.eps, scale,
            shift, self.act))

    def extra_repr(self) -> str:
        r = super().extra_repr()
        return r if self.act is None else f"{r}, act={self.act!r}"

    @classmethod
    def from_groupnorm(cls, gn: nn.GroupNorm, act: Optional[str] = None) -> "MaskedGroupNorm":
        """A ``MaskedGroupNorm`` with ``gn``'s configuration and activation ``act`` that shares ``gn``'s parameters
        (the same objects)."""
        out = cls(gn.num_groups, gn.num_channels, gn.eps, gn.affine, device="meta", act=act)
        if gn.affine:
            out.weight = gn.weight
            out.bias = gn.bias
        out.training = gn.training
        return out


class SparseIdentity(SparseModule):
    def forward(self, x: SparseConvTensor):
        return x
