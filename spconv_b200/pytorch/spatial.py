"""Coordinate clean-up (``spconv/pytorch/spatial.py``)."""
from __future__ import annotations

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
