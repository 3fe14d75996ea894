"""HashTable without a GPU: the C ABI's argument checks (refused before any CUDA call), the no-CPU-path
error of the Python class, and the oracle of tests/hash_oracle.py against hand-worked examples."""
import numpy as np
import pytest
import torch

from tests.hash_oracle import DictHash, NumpyHash, reserved_key


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def _refused(rc, *words):
    from spconv_b200 import _cabi
    msg = _cabi.last_error()
    assert rc == 2, (rc, msg)          # 2 = argument check; a CUDA failure would return 1
    for w in words:
        assert w in msg, msg


def test_cabi_refuses_bad_itemsizes(lib):
    for ks, vs, word in ((3, 4, "key itemsize"), (2, 8, "key itemsize"), (4, 16, "value itemsize"), (8, 0, "value itemsize")):
        _refused(lib.spx_hash_clear(1, 1, 1, 1, 16, ks, vs, None), word)
        _refused(lib.spx_hash_insert(1, 1, 1, 16, ks, vs, 1, 1, 2, 0, 1, 1 << 20, None), word)
        _refused(lib.spx_hash_query(1, 1, 16, ks, vs, 1, 1, 1, 2, None), word)
        _refused(lib.spx_hash_insert_exist(1, 1, 1, 16, ks, vs, 1, 1, 1, 2, 1, 1, 1 << 20, None), word)
        _refused(lib.spx_hash_rank(1, 1, 1, 16, ks, vs, 3, 0, 1, 1, 16, 1, 1, 1 << 20, None), word)


def test_cabi_refuses_bad_max_size(lib):
    for max_size in (0, -5, 1 << 31, 1 << 40):
        _refused(lib.spx_hash_clear(1, 1, 1, 1, max_size, 4, 4, None), "max_size")
        _refused(lib.spx_hash_insert(1, 1, 1, max_size, 8, 8, 1, 1, 1, 0, 1, 1 << 20, None), "max_size")
        _refused(lib.spx_hash_query(1, 1, max_size, 4, 8, 1, 1, 1, 1, None), "max_size")
        _refused(lib.spx_hash_rank(1, 1, 1, max_size, 4, 4, 0, 1, None, None, 0, 1, 1, 1 << 20, None), "max_size")


def test_cabi_refuses_null_pointers(lib):
    _refused(lib.spx_hash_clear(None, 1, 1, 1, 16, 4, 4, None), "NULL")
    _refused(lib.spx_hash_clear(1, 1, 1, None, 16, 4, 4, None), "NULL")
    _refused(lib.spx_hash_insert(1, 1, 1, 16, 4, 4, None, None, 3, 0, 1, 1 << 20, None), "NULL")
    _refused(lib.spx_hash_insert(1, 1, None, 16, 4, 4, 1, None, 3, 0, 1, 1 << 20, None), "NULL")
    _refused(lib.spx_hash_query(1, 1, 16, 4, 4, 1, None, 1, 3, None), "NULL")
    _refused(lib.spx_hash_query(1, 1, 16, 4, 4, 1, 1, None, 3, None), "NULL")
    _refused(lib.spx_hash_insert_exist(1, 1, 1, 16, 4, 4, 1, None, 1, 3, 1, 1, 1 << 20, None), "NULL")
    _refused(lib.spx_hash_rank(1, 1, 1, 16, 4, 4, 3, 0, None, None, 4, 1, 1, 1 << 20, None), "NULL")
    _refused(lib.spx_hash_rank(1, 1, 1, 16, 4, 4, 3, 1, None, None, 0, None, 1, 1 << 20, None), "count is NULL")
    _refused(lib.spx_hash_rank(1, 1, 1, 16, 4, 4, 3, 1, None, None, 0, 1, None, 0, None), "workspace")


def test_cabi_refuses_counts_ordinals_and_workspace(lib):
    # the capacity rule: ordinal_base + n must stay below max_size (so a probe always finds a free slot)
    _refused(lib.spx_hash_insert(1, 1, 1, 16, 4, 4, 1, 1, 6, 10, 1, 1 << 20, None), "inserted count exceed maximum hash size")
    _refused(lib.spx_hash_insert(1, 1, 1, 16, 4, 4, 1, 1, 16, 0, 1, 1 << 20, None), "inserted count exceed maximum hash size")
    _refused(lib.spx_hash_insert(1, 1, 1, 16, 4, 4, 1, 1, 2, -1, 1, 1 << 20, None), "inserted count exceed")
    _refused(lib.spx_hash_insert(1, 1, 1, 16, 4, 4, 1, 1, -1, 0, 1, 1 << 20, None), "key count")
    _refused(lib.spx_hash_query(1, 1, 16, 4, 4, 1, 1, 1, 1 << 31, None), "key count")
    _refused(lib.spx_hash_insert(1, 1, 1, 16, 4, 4, 1, 1, 3, 0, 1, 8, None), "workspace too small")
    _refused(lib.spx_hash_insert_exist(1, 1, 1, 16, 4, 4, 1, 1, 1, 3, 0, 1, 1 << 20, None), "epoch")
    _refused(lib.spx_hash_insert_exist(1, 1, 1, 16, 4, 4, 1, 1, 1, 3, 1 << 32, 1, 1 << 20, None), "epoch")
    _refused(lib.spx_hash_rank(1, 1, 1, 16, 4, 4, 16, 1, None, None, 0, 1, 1, 1 << 20, None), "ordinal count")
    _refused(lib.spx_hash_rank(1, 1, 1, 16, 4, 4, 3, 1, None, None, 0, 1, 1, 16, None), "workspace too small")
    assert lib.spx_hash_workspace_size(-1, 0) == 0 and lib.spx_hash_workspace_size(0, -1) == 0
    assert lib.spx_hash_workspace_size(1000, 0) >= 4000
    assert lib.spx_hash_workspace_size(0, 1 << 20) >= (1 << 20) // 8


def test_cabi_zero_keys_launch_nothing(lib):
    """N = 0 returns success before any pointer is needed or any CUDA call is made"""
    assert lib.spx_hash_insert(None, None, None, 16, 4, 4, None, None, 0, 3, None, 0, None) == 0
    assert lib.spx_hash_query(None, None, 16, 8, 8, None, None, None, 0, None) == 0
    assert lib.spx_hash_insert_exist(None, None, None, 16, 8, 4, None, None, None, 0, 1, None, 0, None) == 0


def test_cpu_device_raises_no_cpu_path():
    from spconv_b200.pytorch.hash import HashTable
    with pytest.raises(RuntimeError, match="no CPU path"):
        HashTable(torch.device("cpu"), torch.int32, torch.int64)
    with pytest.raises(RuntimeError, match="no CPU path"):
        HashTable(torch.device("cpu"), torch.int64, torch.float32, max_size=100)


def test_oracles_on_a_hand_worked_example():
    for cls in (DictHash, NumpyHash):
        h = cls(np.int32, np.int64)
        h.insert(np.array([5, 3, 5, 7]), np.array([10, 20, 30, 40]))
        h.insert(np.array([3, 9]), np.array([50, 60]))                  # 3 is a re-insert: unchanged
        k, v = h.items()
        assert k.tolist() == [5, 3, 7, 9] and v.tolist() == [10, 20, 40, 60]
        vals, empty = h.query(np.array([9, 5, 1]))
        assert vals.tolist() == [60, 10, 0] and empty.tolist() == [False, False, True]
        assert h.insert_exist_keys(np.array([7, 1, 7, 5]), np.array([1, 2, 3, 4])).tolist() == [0, 1, 0, 0]
        k, v = h.items()
        assert k.tolist() == [5, 3, 7, 9] and v.tolist() == [4, 20, 3, 60]   # 7 takes its last occurrence
        h.insert(np.array([reserved_key(np.int32), 11]))                # reserved key dropped, 11 stores 0
        k, v = h.items()
        assert k.tolist() == [5, 3, 7, 9, 11] and v.tolist() == [4, 20, 3, 60, 0]
        assert h.assign_arange_() == 5
        assert h.items()[1].tolist() == [0, 1, 2, 3, 4]
        assert h.query(np.array([reserved_key(np.int32)]))[1].tolist() == [True]


@pytest.mark.parametrize("key_dtype", [np.int32, np.int64])
def test_numpy_oracle_matches_dict_oracle(key_dtype):
    rng = np.random.default_rng(7)
    a, b = DictHash(key_dtype, np.int64), NumpyHash(key_dtype, np.int64)
    big = np.iinfo(key_dtype)
    for step in range(6):
        keys = rng.integers(-40, 40, 60).astype(key_dtype)
        keys[:3] = [big.min, big.max, big.max - 1]
        vals = rng.integers(-1 << 40, 1 << 40, 60)
        if step % 3 == 2:
            assert a.insert_exist_keys(keys, vals).tolist() == b.insert_exist_keys(keys, vals).tolist()
        else:
            a.insert(keys, None if step == 1 else vals)
            b.insert(keys, None if step == 1 else vals)
        for x, y in zip(a.items(), b.items()):
            assert x.tolist() == y.tolist()
        q = rng.integers(-50, 50, 80).astype(key_dtype)
        for x, y in zip(a.query(q), b.query(q)):
            assert x.tolist() == y.tolist()
    assert a.assign_arange_() == b.assign_arange_()
    assert a.items()[1].tolist() == b.items()[1].tolist()
