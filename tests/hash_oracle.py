"""Restatement of HashTable's semantics for the tests: the reference's CPU map (spconv/csrc/hash/core.py,
tsl::robin_map) plus first-insertion order.

  * insert: the first insertion of a key wins; later duplicates and re-inserts change nothing; without
    values the value is 0.  The reserved key (the key dtype's maximum) is never stored.
  * query: the stored value, is_empty = True for a missing key.
  * insert_exist_keys: stored keys take the value of their LAST occurrence in the call.
  * items / assign_arange_: the stored keys in first-insertion order (by call, then by position).

Values are kept as raw integer bits (int32 / int64 views of float values), so comparisons are bit for bit.
Two versions: ``DictHash`` (a plain ordered dict, for small cases) and ``NumpyHash`` (vectorised, for scale).
"""
import numpy as np


def reserved_key(key_dtype) -> int:
    return int(np.iinfo(key_dtype).max)


class DictHash:
    def __init__(self, key_dtype, value_dtype):
        self.key_dtype, self.value_dtype = np.dtype(key_dtype), np.dtype(value_dtype)
        self.d = {}

    def insert(self, keys, values=None):
        empty = reserved_key(self.key_dtype)
        for i, k in enumerate(np.asarray(keys).tolist()):
            if k != empty and k not in self.d:
                self.d[k] = 0 if values is None else int(values[i])

    def query(self, keys):
        keys = np.asarray(keys).tolist()
        vals = np.array([self.d.get(k, 0) for k in keys], dtype=self.value_dtype)
        return vals, np.array([k not in self.d for k in keys], dtype=bool)

    def insert_exist_keys(self, keys, values):
        keys = np.asarray(keys).tolist()
        for i, k in enumerate(keys):
            if k in self.d:
                self.d[k] = int(values[i])
        return np.array([k not in self.d for k in keys], dtype=np.uint8)

    def assign_arange_(self):
        for r, k in enumerate(self.d):
            self.d[k] = r
        return len(self.d)

    def items(self):
        return (np.array(list(self.d.keys()), dtype=self.key_dtype),
                np.array(list(self.d.values()), dtype=self.value_dtype))


class NumpyHash:
    def __init__(self, key_dtype, value_dtype):
        self.key_dtype, self.value_dtype = np.dtype(key_dtype), np.dtype(value_dtype)
        self.keys = np.empty(0, self.key_dtype)
        self.values = np.empty(0, self.value_dtype)

    def _find(self, keys):
        """position of every key in self.keys, and whether it is there"""
        keys = np.asarray(keys, self.key_dtype)
        if len(self.keys) == 0:
            return np.zeros(len(keys), np.int64), np.zeros(len(keys), bool)
        order = np.argsort(self.keys, kind="stable")
        pos = np.searchsorted(self.keys, keys, sorter=order)
        pos = np.minimum(pos, len(order) - 1)
        idx = order[pos]
        return idx, self.keys[idx] == keys

    def insert(self, keys, values=None):
        keys = np.asarray(keys, self.key_dtype)
        values = np.zeros(len(keys), self.value_dtype) if values is None else np.asarray(values, self.value_dtype)
        keep = keys != reserved_key(self.key_dtype)
        keys, values = keys[keep], values[keep]
        uniq, first = np.unique(keys, return_index=True)              # first occurrence in the batch
        _, found = self._find(uniq)
        new = np.sort(first[~found])                                   # new keys, in batch order
        self.keys = np.concatenate([self.keys, keys[new]])
        self.values = np.concatenate([self.values, values[new]])

    def query(self, keys):
        idx, found = self._find(keys)
        vals = np.where(found, self.values[idx] if len(self.values) else 0, 0).astype(self.value_dtype)
        return vals, ~found

    def insert_exist_keys(self, keys, values):
        keys = np.asarray(keys, self.key_dtype)
        values = np.asarray(values, self.value_dtype)
        idx, found = self._find(keys)
        rev = keys[::-1]
        uniq, first_rev = np.unique(rev, return_index=True)
        last = len(keys) - 1 - first_rev                               # last occurrence of every key
        lidx, lfound = self._find(uniq)
        self.values[lidx[lfound]] = values[last[lfound]]
        return (~found).astype(np.uint8)

    def assign_arange_(self):
        self.values = np.arange(len(self.keys)).astype(self.value_dtype)
        return len(self.keys)

    def items(self):
        return self.keys.copy(), self.values.copy()
