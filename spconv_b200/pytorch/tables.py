"""Modules that combine several sparse tensors (``spconv/pytorch/tables.py``).

``JoinTable`` and ``AddTable`` work on tensors with the same coordinates, row for row: they concatenate
or add the feature matrices.  ``AddTableMisaligned`` adds tensors whose coordinates differ
(:func:`functional.sparse_add_hash_based`).  ``ConcatTable`` runs every child on the same input.
``MaskedAddTable``, ``MaskedJoinTable`` and ``MaskedAddTableMisaligned`` are their padding-aware twins, which
take padded tensors and never synchronise with the host (:func:`functional.masked_sparse_add`).
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import functional as F
from .core import SparseConvTensor
from .modules import SparseModule


def _check_aligned(input: List[SparseConvTensor], msg: str, masked: bool = False) -> None:
    for ten in input:
        if not masked:
            ten.require_unpadded("the table modules")
        elif ten.num_valid is not input[0].num_valid:
            raise ValueError("MaskedAddTable / MaskedJoinTable work row by row: every operand must carry the same "
                             "num_valid tensor object (or all None), as the SubM branches or inverse convs of one input "
                             "do. Use MaskedAddTableMisaligned for tensors with different coordinates.")
        assert ten.spatial_shape == input[0].spatial_shape, msg
        assert ten.batch_size == input[0].batch_size, msg
        assert ten.features.shape[1] == input[0].features.shape[1], msg
        assert ten.indices.shape[0] == input[0].indices.shape[0], msg


def _aligned_result(input: List[SparseConvTensor], features: torch.Tensor) -> SparseConvTensor:
    first = input[0]
    out = SparseConvTensor(features, first.indices, first.spatial_shape, first.batch_size, first.grid,
                           first.voxel_num, first.indice_dict)
    out.benchmark_record = input[1].benchmark_record
    out.thrust_allocator = input[1].thrust_allocator
    out._timer = input[1]._timer
    return out


class JoinTable(SparseModule):
    """Concatenate the features of tensors with the same coordinates along the channels."""

    def forward(self, input: List[SparseConvTensor]):
        _check_aligned(input, "you can't use JoinTable in two sptensor with different indices.")
        return _aligned_result(input, torch.cat([i.features for i in input], 1))

    def input_spatial_size(self, out_size):
        return out_size


class AddTable(SparseModule):
    """Add the features of tensors with the same coordinates."""

    def forward(self, input: List[SparseConvTensor]):
        _check_aligned(input, "you can't use AddTable in two sptensor with different indices. "
                              "use AddTableMisaligned instead.")
        return _aligned_result(input, sum([i.features for i in input]))

    def input_spatial_size(self, out_size):
        return out_size


class AddTableMisaligned(SparseModule):
    """Add sparse tensors with the same shape but different coordinates (slower than AddTable).

    The result keeps the largest operand's ``indice_dict`` only when its coordinates are the result's
    coordinates row for row (see :func:`functional.sparse_add`); otherwise a following
    ``SparseInverseConv`` has no rulebook to invert.
    """

    def forward(self, input: List[SparseConvTensor]):
        return F.sparse_add_hash_based(*input)

    def input_spatial_size(self, out_size):
        return out_size


def _masked_aligned_result(input: List[SparseConvTensor], features: torch.Tensor) -> SparseConvTensor:
    out = _aligned_result(input, features)
    out.num_valid = input[0].num_valid
    out.bound_status = F._merged_status(input, None, None)
    return out


class MaskedJoinTable(SparseModule):
    """``JoinTable`` for padded tensors: allowed when every operand carries the same ``num_valid`` object (or all
    None); the result carries it.  Row-wise, so padding rows never mix with valid ones."""

    def forward(self, input: List[SparseConvTensor]):
        _check_aligned(input, "you can't use MaskedJoinTable in two sptensor with different indices.", masked=True)
        return _masked_aligned_result(input, torch.cat([i.features for i in input], 1))

    def input_spatial_size(self, out_size):
        return out_size


class MaskedAddTable(SparseModule):
    """``AddTable`` for padded tensors: allowed when every operand carries the same ``num_valid`` object (or all
    None); the result carries it."""

    def forward(self, input: List[SparseConvTensor]):
        _check_aligned(input, "you can't use MaskedAddTable in two sptensor with different indices. "
                              "use MaskedAddTableMisaligned instead.", masked=True)
        return _masked_aligned_result(input, sum([i.features for i in input]))

    def input_spatial_size(self, out_size):
        return out_size


class MaskedAddTableMisaligned(SparseModule):
    """Add padded or unpadded sparse tensors whose coordinates differ, with no host synchronisation
    (:func:`functional.masked_sparse_add`): the result has ``num_out_act_bound`` rows (default: the operands' total
    row count) and ``num_valid`` = the size of the union.  With a bound, a status word is kept as the strided conv
    and pool modules keep theirs: ``spconv.check_bounds`` reports a union larger than the bound, and
    ``spconv.set_output_bounds`` sets the bound from an example.  ``indice_dict`` is not kept."""

    def __init__(self, num_out_act_bound: Optional[int] = None, name=None):
        super().__init__(name=name)
        self.num_out_act_bound = num_out_act_bound

    def forward(self, input: List[SparseConvTensor]):
        if self.num_out_act_bound is None:
            return F._masked_sparse_add(input)
        return F._masked_sparse_add(input, self.num_out_act_bound, self._status_word(input[0].indices.device),
                                    self._layer_name())

    def input_spatial_size(self, out_size):
        return out_size


class ConcatTable(SparseModule):
    """Run every child module on the same input and return the list of their outputs."""

    def forward(self, input):
        return [module(input) for module in self._modules.values()]

    def add(self, module):
        self._modules[str(len(self._modules))] = module
        return self

    def input_spatial_size(self, out_size):
        return self._modules['0'].input_spatial_size(out_size)
