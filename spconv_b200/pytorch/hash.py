"""``spconv.pytorch.hash.HashTable`` (reference: ``spconv/pytorch/hash.py``): a fixed-size CUDA hash table
for 32- and 64-bit keys and values, with one defined, reproducible result for every call.

Same constructor, method names, argument order, return types and assertion texts as the reference.  The
semantics are those of the reference's CPU map (``spconv/csrc/hash/core.py``), which its CUDA table only
approximates, plus a defined order:

  * ``insert``: the first insertion of a key wins.  Later duplicates in the same call and re-inserts in
    later calls leave the stored value unchanged.  Without ``values`` the value is 0.
  * ``insert_exist_keys``: a key already in the table takes the value of its LAST occurrence in the call;
    missing keys are not inserted.
  * ``items`` and ``assign_arange_`` number the keys in first-insertion order: by call, then by position
    in the batch.

Differences a reference user can observe (DESIGN.md §2.5b):
  * CUDA only.  A CPU device raises the engine's "no CPU path" error.
  * ``max_size`` is at most 2^31 - 1, so insertion ordinals fit in 32 bits (the reference takes any size).
  * The largest value of the key dtype (``torch.iinfo(key_dtype).max``) marks an empty slot: a key equal
    to it is never stored, and a query for it reports the key missing.  There is no run-time check,
    since that would need a read-back to the host.

No method reads anything back to the host; counts stay on the device.  Every launch goes to torch's
current stream, so a sequence of calls can be captured in a CUDA graph.  The number of keys inserted so
far (the ordinal base) and the ``insert_exist_keys`` epoch are host state fixed at capture: a replay is
only meaningful when the graph also constructs (and so clears) the table.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _cabi
from .ops import _ptr, _require_cuda, _stream

_TORCH_DTYPE_TO_ITEMSIZE = {
    torch.int32: 4,
    torch.int64: 8,
    torch.float32: 4,
    torch.float64: 8,
}
_KEY_DTYPES = (torch.int32, torch.int64)
MAX_SIZE_LIMIT = 2147483647


def _lib():
    return _cabi.load()


class HashTable:
    """Fixed-size CUDA hash table for int32 / int64 keys and int32 / int64 / float32 / float64 values.

    ``max_size`` is the number of slots (about twice the number of keys is a good size); the number of
    keys inserted over the table's life, duplicates included, must stay below it.  ``keys_data`` and
    ``values_data`` are the slots themselves; which slot holds a key depends on thread timing, what the
    methods return does not.  The largest value of the key dtype is reserved for empty
    slots and is never stored.
    """

    def __init__(self, device: torch.device, key_dtype: torch.dtype,
                 value_dtype: torch.dtype,
                 max_size: int = -1) -> None:
        device = torch.device(device)
        _require_cuda(torch.empty(0, device=device), "the HashTable device")
        if key_dtype not in _KEY_DTYPES:
            raise ValueError(f"HashTable keys must be torch.int32 or torch.int64, got {key_dtype}")
        if value_dtype not in _TORCH_DTYPE_TO_ITEMSIZE:
            raise ValueError(f"HashTable values must be int32, int64, float32 or float64, got {value_dtype}")
        if not max_size > 0:
            raise AssertionError("you must provide max_size for fixed-size cuda hash table, usually *2 of num of keys")
        if max_size > MAX_SIZE_LIMIT:
            raise ValueError(f"HashTable max_size {max_size} exceeds 2^31 - 1 = {MAX_SIZE_LIMIT}: insertion ordinals "
                             "are 32-bit")
        self.is_cpu = False
        self.key_dtype = key_dtype
        self.value_dtype = value_dtype
        self.key_itemsize = _TORCH_DTYPE_TO_ITEMSIZE[key_dtype]
        self.value_itemsize = _TORCH_DTYPE_TO_ITEMSIZE[value_dtype]
        self._valid_value_dtype_for_arange = set([torch.int32, torch.int64])
        self.keys_data = torch.empty([max_size], dtype=key_dtype, device=device)
        self.values_data = torch.empty([max_size], dtype=value_dtype, device=device)
        self._first = torch.empty([max_size], dtype=torch.int32, device=device)     # insertion ordinal per slot
        self._tag = torch.empty([max_size], dtype=torch.int64, device=device)       # insert_exist_keys winner
        self._insert_count = 0
        self._epoch = 0
        with torch.cuda.device(device):
            _cabi.check(_lib().spx_hash_clear(self.keys_data.data_ptr(), self.values_data.data_ptr(),
                                              self._first.data_ptr(), self._tag.data_ptr(), max_size,
                                              self.key_itemsize, self.value_itemsize, _stream()), "hash_clear")

    @property
    def insert_count(self) -> int:
        """Keys inserted so far, duplicates included (the reference's ``insert_count``)."""
        return self._insert_count

    def _table_args(self):
        return self.keys_data.shape[0], self.key_itemsize, self.value_itemsize

    def _check_keys(self, keys: torch.Tensor, itemsize: bool = True) -> torch.Tensor:
        if itemsize and keys.element_size() != self.key_itemsize:
            raise RuntimeError(f"keys itemsize not equal to {self.key_itemsize}")
        if keys.dtype != self.key_dtype:
            raise RuntimeError(f"keys dtype not equal to {self.key_dtype}")
        _require_cuda(keys, "keys")
        if keys.device != self.keys_data.device:
            raise RuntimeError(f"keys are on {keys.device}, the table is on {self.keys_data.device}")
        return keys.contiguous()

    def _check_values(self, values: torch.Tensor, n: int) -> torch.Tensor:
        if values.element_size() != self.value_itemsize:
            raise RuntimeError(f"values itemsize not equal to {self.value_itemsize}")
        if values.shape[0] != n:
            raise RuntimeError("number of key and value must same")
        _require_cuda(values, "values")
        if values.device != self.keys_data.device:
            raise RuntimeError(f"values are on {values.device}, the table is on {self.keys_data.device}")
        return values

    def insert(self, keys: torch.Tensor, values: Optional[torch.Tensor] = None):
        """Insert keys with their values (0 when ``values`` is None).  The first insertion of a key wins."""
        n = keys.shape[0]
        max_size = self.keys_data.shape[0]
        if self._insert_count + n >= max_size:
            raise RuntimeError("inserted count exceed maximum hash size")
        keys = self._check_keys(keys, itemsize=False)
        if values is not None:
            values = self._check_values(values, n).contiguous()
        if n > 0:
            lib = _lib()
            ws = torch.empty(lib.spx_hash_workspace_size(n, 0), dtype=torch.uint8, device=keys.device)
            with torch.cuda.device(keys.device):
                _cabi.check(lib.spx_hash_insert(self.keys_data.data_ptr(), self.values_data.data_ptr(),
                                                self._first.data_ptr(), *self._table_args(), keys.data_ptr(),
                                                _ptr(values), n, self._insert_count, ws.data_ptr(), ws.numel(),
                                                _stream()), "hash_insert")
        self._insert_count += n

    def query(self, keys: torch.Tensor, values: Optional[torch.Tensor] = None):
        """Look keys up.  Returns ``(values, is_empty)`` with ``is_empty`` a bool tensor that is True for a
        missing key.  The value of a missing key is left as it was in a caller's ``values`` tensor, and is
        0 in a tensor this method allocates."""
        n = keys.shape[0]
        keys = self._check_keys(keys)
        if values is None:
            values = torch.zeros([n], dtype=self.value_dtype, device=keys.device)
        else:
            values = self._check_values(values, n)
            if not values.is_contiguous():
                raise RuntimeError("query: values must be contiguous (it is written in place)")
        is_empty = torch.empty([n], dtype=torch.uint8, device=keys.device)
        if n > 0:
            with torch.cuda.device(keys.device):
                _cabi.check(_lib().spx_hash_query(self.keys_data.data_ptr(), self.values_data.data_ptr(),
                                                  *self._table_args(), keys.data_ptr(), values.data_ptr(),
                                                  is_empty.data_ptr(), n, _stream()), "hash_query")
        return values, is_empty > 0

    def insert_exist_keys(self, keys: torch.Tensor, values: torch.Tensor):
        """Set the value of keys that are already in the table; a key that occurs several times takes its
        last value.  Missing keys are not inserted.  Returns ``is_empty`` (uint8, 1 = key missing)."""
        n = keys.shape[0]
        keys = self._check_keys(keys)
        values = self._check_values(values, n).contiguous()
        is_empty = torch.empty([n], dtype=torch.uint8, device=keys.device)
        if n > 0:
            self._epoch += 1
            lib = _lib()
            ws = torch.empty(lib.spx_hash_workspace_size(n, 0), dtype=torch.uint8, device=keys.device)
            with torch.cuda.device(keys.device):
                _cabi.check(lib.spx_hash_insert_exist(self.keys_data.data_ptr(), self.values_data.data_ptr(),
                                                      self._tag.data_ptr(), *self._table_args(), keys.data_ptr(),
                                                      values.data_ptr(), is_empty.data_ptr(), n, self._epoch,
                                                      ws.data_ptr(), ws.numel(), _stream()), "hash_insert_exist")
        return is_empty

    def _count(self) -> torch.Tensor:
        dtype = torch.int32 if self.key_itemsize == 4 else torch.int64
        return torch.zeros([1], dtype=dtype, device=self.values_data.device)

    def _rank(self, assign: bool, keys=None, values=None, rows: int = 0) -> torch.Tensor:
        count = self._count()
        lib = _lib()
        ws = torch.empty(max(lib.spx_hash_workspace_size(0, self._insert_count), 1), dtype=torch.uint8,
                         device=self.values_data.device)
        with torch.cuda.device(self.values_data.device):
            _cabi.check(lib.spx_hash_rank(self.keys_data.data_ptr(), self.values_data.data_ptr(),
                                          self._first.data_ptr(), *self._table_args(), self._insert_count,
                                          int(assign), _ptr(keys), _ptr(values), rows, count.data_ptr(),
                                          ws.data_ptr(), ws.numel(), _stream()), "hash_rank")
        return count

    def assign_arange_(self):
        """Set every stored key's value to its number in first-insertion order (0 .. count-1).  Returns
        ``count``, a ``[1]`` device tensor: int32 for 4-byte keys, int64 for 8-byte keys."""
        if self.value_dtype not in self._valid_value_dtype_for_arange:
            raise AssertionError(f"assign_arange_ needs int32 or int64 values, the table holds {self.value_dtype}")
        return self._rank(True)

    def items(self, max_size: int = -1):
        """``(keys, values, count)``: buffers of ``max_size`` rows (default: the table size) whose first
        ``min(count, max_size)`` rows hold the stored entries in first-insertion order.  The rows after
        them are not written."""
        if max_size == -1:
            max_size = self.values_data.shape[0]
        keys = torch.empty([max_size], dtype=self.key_dtype, device=self.values_data.device)
        values = torch.empty([max_size], dtype=self.value_dtype, device=self.values_data.device)
        count = self._rank(False, keys, values, max_size)
        return keys, values, count
