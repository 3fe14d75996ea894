"""Containers that thread a :class:`SparseConvTensor` through a model
(``spconv/pytorch/modules.py:50-168`` semantics: sparse modules see the tensor, plain
``nn.Module``s see ``.features`` and are skipped on an empty tensor)."""
from __future__ import annotations

from collections import OrderedDict
from typing import Any, Optional

import torch
from torch import nn

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
        if self.inner.training:
            x.require_unpadded("SparseBatchNorm in training mode")
        return super().forward(x)


class SparseIdentity(SparseModule):
    def forward(self, x: SparseConvTensor):
        return x
