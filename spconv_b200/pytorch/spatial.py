"""Coordinate clean-up (``spconv/pytorch/spatial.py``)."""
from __future__ import annotations

from typing import Optional

from . import functional as F
from .core import SparseConvTensor
from .modules import SparseModule


class RemoveDuplicate(SparseModule):
    """Keep one row per coordinate: the first row that carries it.

    The result's rows are in first-touch order (the order in which the coordinates first appear in the
    input), its features are those first rows' features, and rows whose batch index or coordinate is out of
    range are dropped.  The gradient flows to the kept rows only.  The result has an empty
    ``indice_dict``.  (The reference's version unpacks the result of ``torch.unique`` as if it returned
    indices of the unique rows, which it does not, so it cannot run.)
    """

    def forward(self, x: SparseConvTensor):
        return F.remove_duplicate(x)


class MaskedRemoveDuplicate(SparseModule):
    """``RemoveDuplicate`` of the valid rows of a padded or unpadded tensor, with no host synchronisation
    (:func:`functional.masked_remove_duplicate`): the result has ``num_out_act_bound`` rows (default: the input's row
    count) and ``num_valid`` = the number of distinct in-range coordinates.  With a bound, a status word is kept for
    ``spconv.check_bounds`` and ``spconv.set_output_bounds`` as the strided conv and pool modules keep theirs."""

    def __init__(self, num_out_act_bound: Optional[int] = None, name=None):
        super().__init__(name=name)
        self.num_out_act_bound = num_out_act_bound

    def forward(self, x: SparseConvTensor):
        if self.num_out_act_bound is None:
            return F._masked_remove_duplicate(x)
        return F._masked_remove_duplicate(x, self.num_out_act_bound, self._status_word(x.indices.device),
                                          self._layer_name())
