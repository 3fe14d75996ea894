"""HashTable on the GPU, bit for bit against the oracle of tests/hash_oracle.py (float values compared through
an integer view): insert / query / insert_exist_keys / assign_arange_ / items over every key and value dtype,
nearly full and clustered tables, 4 M keys, repeatability, the checks that raise before a launch, the
reserved key, empty calls and a CUDA-graph capture."""
import numpy as np
import pytest
import torch

from tests.hash_oracle import DictHash, NumpyHash, reserved_key

pytestmark = pytest.mark.gpu

KEY_DTYPES = [torch.int32, torch.int64]
VALUE_DTYPES = [torch.int32, torch.int64, torch.float32, torch.float64]
BITS = {torch.int32: torch.int32, torch.float32: torch.int32, torch.int64: torch.int64, torch.float64: torch.int64}
NP = {torch.int32: np.int32, torch.int64: np.int64}


def _table(dev, kdt, vdt, max_size):
    from spconv_b200.pytorch.hash import HashTable
    return HashTable(dev, kdt, vdt, max_size=max_size)


def _bits(t):
    return t.view(BITS[t.dtype]).cpu().numpy()


def _values(v, vdt, dev):
    """raw integer bits -> a device tensor of the value dtype (NaN payloads and -0.0 included for floats)"""
    return torch.from_numpy(np.asarray(v).astype(NP[BITS[vdt]])).to(dev).view(vdt)


def _keys(rng, kdt, n, pool):
    return pool[rng.integers(0, len(pool), n)].astype(NP[kdt])


def _pool(rng, kdt, n):
    """n distinct keys: negatives, the type's minimum, values near 2^40 and 2^62 for int64"""
    info = np.iinfo(NP[kdt])
    parts = [np.array([info.min, info.min + 1, -1, 0, 1, info.max - 1], dtype=np.int64)]
    parts.append(rng.integers(-1000, 1000, n))
    if kdt == torch.int64:
        parts += [(1 << 40) + rng.integers(-500, 500, n), (1 << 62) + rng.integers(-500, 500, n),
                  rng.integers(info.min, info.max, n, dtype=np.int64)]
    else:
        parts.append(rng.integers(info.min, info.max, n, dtype=np.int64))
    keys = np.unique(np.concatenate(parts))
    keys = keys[keys != info.max]
    return keys[rng.permutation(len(keys))][:n].astype(NP[kdt])


def _raw_values(rng, vdt, n):
    nbits = 32 if BITS[vdt] == torch.int32 else 64
    info = np.iinfo(np.int32 if nbits == 32 else np.int64)
    v = rng.integers(info.min, info.max, n, dtype=np.int64)
    if vdt == torch.float32:                  # quiet NaN with payload, negative NaN, -0.0
        special = np.array([0x7FC00001, 0xFFC12345 - (1 << 32), -(1 << 31)], dtype=np.int64)
    elif vdt == torch.float64:
        special = np.array([0x7FF8000000000001, -0x0008000000000001, -(1 << 63)], dtype=np.int64)
    if vdt in (torch.float32, torch.float64):
        v[:len(special)] = special              # NaN payloads and -0.0
    return v


def _check_items(table, orc):
    keys, vals, count = table.items()
    ek, ev = orc.items()
    assert count.dtype == (torch.int32 if table.key_itemsize == 4 else torch.int64) and count.shape == (1,)
    c = int(count.item())
    assert c == len(ek)
    assert np.array_equal(keys[:c].cpu().numpy(), ek)
    assert np.array_equal(_bits(vals[:c]), ev.astype(NP[BITS[table.value_dtype]]))


def _check_query(table, orc, q, vdt, dev, fill=None):
    qt = torch.from_numpy(q).to(dev)
    ev, ee = orc.query(q)
    if fill is None:
        vals, empty = table.query(qt)
        want = ev
    else:
        buf = _values(np.full(len(q), fill), vdt, dev)
        vals, empty = table.query(qt, buf)
        assert vals.data_ptr() == buf.data_ptr()
        want = np.where(ee, fill, ev)
    assert empty.dtype == torch.bool
    assert np.array_equal(empty.cpu().numpy(), ee)
    assert np.array_equal(_bits(vals), want.astype(NP[BITS[vdt]]))


@pytest.mark.parametrize("vdt", VALUE_DTYPES, ids=str)
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_insert_query_items_match_the_oracle(cuda_dev, kdt, vdt):
    rng = np.random.default_rng(1)
    pool = _pool(rng, kdt, 900)
    table = _table(cuda_dev, kdt, vdt, 3001)
    orc = NumpyHash(NP[kdt], NP[BITS[vdt]])
    for step in range(4):                     # in-batch duplicates and re-inserts across calls
        keys = _keys(rng, kdt, 500, pool)
        raw = _raw_values(rng, vdt, 500)
        if step == 2:
            table.insert(torch.from_numpy(keys).to(cuda_dev))
            orc.insert(keys)
        else:
            table.insert(torch.from_numpy(keys).to(cuda_dev), _values(raw, vdt, cuda_dev))
            orc.insert(keys, raw)
        assert table.insert_count == 500 * (step + 1)
        _check_items(table, orc)
    q = np.concatenate([pool, _pool(np.random.default_rng(2), kdt, 400)])
    q = q[rng.permutation(len(q))]
    _check_query(table, orc, q, vdt, cuda_dev)
    _check_query(table, orc, q, vdt, cuda_dev, fill=12345)


def test_insert_without_values_stores_zero(cuda_dev):
    for kdt in KEY_DTYPES:
        for vdt in (torch.int64, torch.float32):
            table = _table(cuda_dev, kdt, vdt, 100)
            table.insert(torch.tensor([4, -7, 4, 9], dtype=kdt, device=cuda_dev))
            table.insert(torch.tensor([9, 5], dtype=kdt, device=cuda_dev), torch.tensor([3, 6], device=cuda_dev).to(vdt))
            keys, vals, count = table.items()
            assert int(count) == 4
            assert keys[:4].tolist() == [4, -7, 9, 5]
            assert _bits(vals[:4]).tolist() == [0, 0, 0, _bits(torch.tensor([6], dtype=vdt))[0]]


@pytest.mark.parametrize("vdt", [torch.int32, torch.float64], ids=str)
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_insert_exist_keys_last_occurrence_wins(cuda_dev, kdt, vdt):
    rng = np.random.default_rng(3)
    pool = _pool(rng, kdt, 600)
    stored, absent = pool[:300], pool[300:]
    table = _table(cuda_dev, kdt, vdt, 1000)
    orc = NumpyHash(NP[kdt], NP[BITS[vdt]])
    raw = _raw_values(rng, vdt, 300)
    table.insert(torch.from_numpy(stored).to(cuda_dev), _values(raw, vdt, cuda_dev))
    orc.insert(stored, raw)
    for call in range(3):                     # later epochs override earlier ones
        keys = np.concatenate([_keys(rng, kdt, 700, stored), _keys(rng, kdt, 100, absent)])
        keys = keys[rng.permutation(len(keys))]
        raw = _raw_values(rng, vdt, len(keys))
        empty = table.insert_exist_keys(torch.from_numpy(keys).to(cuda_dev), _values(raw, vdt, cuda_dev))
        want = orc.insert_exist_keys(keys, raw)
        assert empty.dtype == torch.uint8
        assert np.array_equal(empty.cpu().numpy(), want)
        _check_items(table, orc)              # missing keys were not inserted
    assert table.insert_count == 300
    # a key repeated in one call takes its last value, whatever the earlier calls wrote
    k = torch.tensor([stored[0], stored[0], stored[0]], dtype=kdt, device=cuda_dev)
    table.insert_exist_keys(k, _values([1, 2, 3], vdt, cuda_dev))
    vals, empty = table.query(k[:1])
    assert _bits(vals).tolist() == [3] and not bool(empty[0])


@pytest.mark.parametrize("vdt", [torch.int32, torch.int64], ids=str)
@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_assign_arange_and_items_in_first_insertion_order(cuda_dev, kdt, vdt):
    rng = np.random.default_rng(4)
    pool = _pool(rng, kdt, 2000)
    table = _table(cuda_dev, kdt, vdt, 5003)
    orc = DictHash(NP[kdt], NP[vdt])
    for _ in range(3):
        keys = _keys(rng, kdt, 1200, pool)
        raw = _raw_values(rng, vdt, 1200)
        table.insert(torch.from_numpy(keys).to(cuda_dev), _values(raw, vdt, cuda_dev))
        orc.insert(keys, raw)
    count = table.assign_arange_()
    n = orc.assign_arange_()
    assert count.dtype == (torch.int32 if kdt == torch.int32 else torch.int64) and count.shape == (1,)
    assert int(count) == n
    keys, vals, c2 = table.items()
    assert int(c2) == n
    assert np.array_equal(keys[:n].cpu().numpy(), orc.items()[0])
    assert vals[:n].tolist() == list(range(n))
    _check_query(table, orc, pool, vdt, cuda_dev)
    for m in (1, 17, n // 2, n - 1, n):       # items(max_size) below count truncates to the first rows
        keys, vals, c3 = table.items(m)
        assert keys.shape == (m,) and vals.shape == (m,) and int(c3) == n
        assert np.array_equal(keys.cpu().numpy(), orc.items()[0][:m])
        assert vals.tolist() == list(range(m))


def test_assign_arange_refuses_float_values(cuda_dev):
    for vdt in (torch.float32, torch.float64):
        table = _table(cuda_dev, torch.int32, vdt, 10)
        table.insert(torch.tensor([1, 2], dtype=torch.int32, device=cuda_dev))
        with pytest.raises(AssertionError):
            table.assign_arange_()
        assert int(table.items()[2]) == 2


def _mix32(x):
    x = x.astype(np.uint32)
    x ^= x >> np.uint32(16); x *= np.uint32(0x85EBCA6B); x ^= x >> np.uint32(13)
    x *= np.uint32(0xC2B2AE35); x ^= x >> np.uint32(16)
    return x


def _mix64(x):
    x = x.astype(np.uint64)
    x ^= x >> np.uint64(33); x *= np.uint64(0xFF51AFD7ED558CCD); x ^= x >> np.uint64(33)
    x *= np.uint64(0xC4CEB9FE1A85EC53); x ^= x >> np.uint64(33)
    return x.astype(np.uint32)


def _home(keys, kdt, cap):
    h = (_mix32 if kdt == torch.int32 else _mix64)(keys).astype(np.uint64)
    return ((h * np.uint64(cap)) >> np.uint64(32)).astype(np.int64)


@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_nearly_full_table_wraps_and_finds_every_key(cuda_dev, kdt):
    rng = np.random.default_rng(5)
    n = 4099
    keys = _pool(rng, kdt, n)
    table = _table(cuda_dev, kdt, torch.int64, n + 1)          # one free slot, not a power of two
    orc = NumpyHash(NP[kdt], np.int64)
    raw = rng.integers(-(1 << 62), 1 << 62, n)
    table.insert(torch.from_numpy(keys).to(cuda_dev), torch.from_numpy(raw).to(cuda_dev))
    orc.insert(keys, raw)
    _check_items(table, orc)
    _check_query(table, orc, keys, torch.int64, cuda_dev)
    # some probe chain ran past the last slot: a key sits below its home slot
    slots = table.keys_data.cpu().numpy()
    held = np.nonzero(slots != reserved_key(NP[kdt]))[0]
    assert len(held) == n
    assert (held < _home(slots[held], kdt, n + 1)).any()


@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_clustered_keys_at_high_load(cuda_dev, kdt):
    n = 50_000
    start, step = (-123_456, 7) if kdt == torch.int32 else ((1 << 40) - 99, 1 << 20)
    keys = (start + step * np.arange(n, dtype=np.int64)).astype(NP[kdt])
    keys = keys[np.random.default_rng(6).permutation(n)]
    table = _table(cuda_dev, kdt, torch.int32, int(n / 0.93) + 1)
    orc = NumpyHash(NP[kdt], np.int32)
    vals = np.arange(n, dtype=np.int32) * 3
    table.insert(torch.from_numpy(keys).to(cuda_dev), torch.from_numpy(vals).to(cuda_dev))
    orc.insert(keys, vals)
    _check_items(table, orc)
    miss = (start + step * np.arange(n, n + 5000, dtype=np.int64)).astype(NP[kdt])
    _check_query(table, orc, np.concatenate([keys, miss]), torch.int32, cuda_dev)


def test_four_million_keys_against_the_numpy_oracle(cuda_dev):
    rng = np.random.default_rng(7)
    n = 4_000_000
    pool = np.unique(rng.integers(-(1 << 63), (1 << 63) - 1, 5_400_000, dtype=np.int64))
    keys = pool[rng.integers(0, len(pool), n)]
    assert 0.25 < 1 - len(np.unique(keys)) / n < 0.35               # about 30 % duplicates
    vals = rng.integers(-(1 << 62), 1 << 62, n)
    table = _table(cuda_dev, torch.int64, torch.int64, (1 << 23) + 3)
    orc = NumpyHash(np.int64, np.int64)
    for part in (slice(0, n // 2), slice(n // 2, n)):
        table.insert(torch.from_numpy(keys[part]).to(cuda_dev), torch.from_numpy(vals[part]).to(cuda_dev))
        orc.insert(keys[part], vals[part])
    _check_items(table, orc)
    q = np.concatenate([keys[:1_000_000], rng.integers(-(1 << 63), (1 << 63) - 1, 500_000, dtype=np.int64)])
    _check_query(table, orc, q, torch.int64, cuda_dev)
    count = table.assign_arange_()
    assert int(count) == orc.assign_arange_()
    _check_items(table, orc)


def _sequence(dev, seed):
    rng = np.random.default_rng(seed)
    pool = _pool(rng, torch.int64, 20_000)
    table = _table(dev, torch.int64, torch.float32, 100_003)
    out = []
    for _ in range(3):
        keys = torch.from_numpy(_keys(rng, torch.int64, 25_000, pool)).to(dev)
        table.insert(keys, _values(_raw_values(rng, torch.float32, 25_000), torch.float32, dev))
        upd = torch.from_numpy(_keys(rng, torch.int64, 10_000, pool)).to(dev)
        out.append(table.insert_exist_keys(upd, _values(_raw_values(rng, torch.float32, 10_000), torch.float32, dev)))
        vals, empty = table.query(torch.from_numpy(pool).to(dev))
        out += [_bits(vals), empty]
    keys, vals, count = table.items()
    c = int(count)
    out += [keys[:c], _bits(vals[:c]), count]
    table2 = _table(dev, torch.int64, torch.int32, 100_003)
    table2.insert(torch.from_numpy(_keys(rng, torch.int64, 60_000, pool)).to(dev))
    out.append(table2.assign_arange_())
    keys, vals, count = table2.items()             # rows past count are not defined
    c = int(count)
    out += [keys[:c], vals[:c], count]
    return out


def test_repeated_sequences_are_identical(cuda_dev):
    a, b = _sequence(cuda_dev, 8), _sequence(cuda_dev, 8)
    for x, y in zip(a, b):
        x = x.cpu().numpy() if isinstance(x, torch.Tensor) else x
        y = y.cpu().numpy() if isinstance(y, torch.Tensor) else y
        assert np.array_equal(x, y)


def test_checks_raise_before_any_launch(cuda_dev):
    from spconv_b200.pytorch.hash import HashTable
    table = _table(cuda_dev, torch.int32, torch.int64, 10)
    table.insert(torch.arange(6, dtype=torch.int32, device=cuda_dev), torch.arange(6, device=cuda_dev) * 10)

    def state():
        keys, vals, count = table.items()
        c = int(count)
        return [keys[:c], vals[:c], count, table.keys_data.clone(), table.values_data.clone()]

    before = state()
    with pytest.raises(RuntimeError, match="^inserted count exceed maximum hash size$"):
        table.insert(torch.arange(100, 104, dtype=torch.int32, device=cuda_dev))     # 6 + 4 >= 10
    with pytest.raises(RuntimeError, match="keys dtype not equal to"):
        table.insert(torch.arange(2, dtype=torch.int64, device=cuda_dev))
    with pytest.raises(RuntimeError, match="number of key and value must same"):
        table.insert(torch.arange(50, 52, dtype=torch.int32, device=cuda_dev), torch.zeros(3, dtype=torch.int64, device=cuda_dev))
    with pytest.raises(RuntimeError, match="values itemsize not equal to 8"):
        table.insert(torch.arange(50, 52, dtype=torch.int32, device=cuda_dev), torch.zeros(2, dtype=torch.int32, device=cuda_dev))
    with pytest.raises(RuntimeError, match="keys itemsize not equal to 4"):
        table.query(torch.arange(2, dtype=torch.int64, device=cuda_dev))
    with pytest.raises(RuntimeError, match="number of key and value must same"):
        table.insert_exist_keys(torch.arange(2, dtype=torch.int32, device=cuda_dev), torch.zeros(3, dtype=torch.int64, device=cuda_dev))
    torch.cuda.synchronize()
    after = state()
    assert table.insert_count == 6
    for x, y in zip(before, after):
        assert torch.equal(x, y)
    table.insert(torch.arange(100, 103, dtype=torch.int32, device=cuda_dev))       # 6 + 3 < 10 still fits
    assert int(table.items()[2]) == 9
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        HashTable(cuda_dev, torch.int32, torch.int32, max_size=1 << 31)
    with pytest.raises(AssertionError, match="you must provide max_size"):
        HashTable(cuda_dev, torch.int32, torch.int32)
    with pytest.raises(ValueError):
        HashTable(cuda_dev, torch.float32, torch.int32, max_size=10)


@pytest.mark.parametrize("kdt", KEY_DTYPES, ids=str)
def test_reserved_key_is_never_stored(cuda_dev, kdt):
    top = reserved_key(NP[kdt])
    table = _table(cuda_dev, kdt, torch.int32, 50)
    table.insert(torch.tensor([top, 3, top, -2], dtype=kdt, device=cuda_dev),
                 torch.tensor([7, 8, 9, 10], dtype=torch.int32, device=cuda_dev))
    keys, vals, count = table.items()
    assert int(count) == 2 and keys[:2].tolist() == [3, -2] and vals[:2].tolist() == [8, 10]
    vals, empty = table.query(torch.tensor([top, 3], dtype=kdt, device=cuda_dev))
    assert empty.tolist() == [True, False] and vals.tolist() == [0, 8]
    assert table.insert_exist_keys(torch.tensor([top], dtype=kdt, device=cuda_dev),
                                   torch.tensor([1], dtype=torch.int32, device=cuda_dev)).tolist() == [1]
    assert int(table.assign_arange_()) == 2


def test_zero_keys_for_every_method(cuda_dev):
    for kdt in KEY_DTYPES:
        table = _table(cuda_dev, kdt, torch.float64, 8)
        none = torch.empty(0, dtype=kdt, device=cuda_dev)
        keys, vals, count = table.items()
        assert keys.shape == (8,) and int(count) == 0
        table.insert(none)
        table.insert(none, torch.empty(0, dtype=torch.float64, device=cuda_dev))
        assert table.insert_count == 0
        vals, empty = table.query(none)
        assert vals.shape == (0,) and empty.shape == (0,) and empty.dtype == torch.bool
        empty = table.insert_exist_keys(none, torch.empty(0, dtype=torch.float64, device=cuda_dev))
        assert empty.shape == (0,) and empty.dtype == torch.uint8
        k0, v0, c0 = table.items(0)
        assert k0.shape == (0,) and v0.shape == (0,) and int(c0) == 0
        itable = _table(cuda_dev, kdt, torch.int64, 8)
        assert int(itable.assign_arange_()) == 0
        itable.insert(torch.tensor([5], dtype=kdt, device=cuda_dev))
        assert int(itable.items(0)[2]) == 1


def test_cuda_graph_capture_of_construction_insert_query_items(cuda_dev):
    rng = np.random.default_rng(9)
    n, cap = 20_000, 40_009
    pool = _pool(rng, torch.int64, 30_000)
    s_keys = torch.zeros(n, dtype=torch.int64, device=cuda_dev)
    s_vals = torch.zeros(n, dtype=torch.float32, device=cuda_dev)
    s_query = torch.zeros(n, dtype=torch.int64, device=cuda_dev)

    def step():
        table = _table(cuda_dev, torch.int64, torch.float32, cap)
        table.insert(s_keys, s_vals)
        qv, qe = table.query(s_query)
        ik, iv, ic = table.items()
        return qv, qe, ik, iv, ic

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()                                 # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for _ in range(3):
        keys = torch.from_numpy(_keys(rng, torch.int64, n, pool)).to(cuda_dev)
        vals = _values(_raw_values(rng, torch.float32, n), torch.float32, cuda_dev)
        query = torch.from_numpy(_keys(np.random.default_rng(10), torch.int64, n, pool)).to(cuda_dev)
        s_keys.copy_(keys)
        s_vals.copy_(vals)
        s_query.copy_(query)
        graph.replay()
        torch.cuda.synchronize()
        eager = _table(cuda_dev, torch.int64, torch.float32, cap)
        eager.insert(keys, vals)
        qv, qe = eager.query(query)
        ik, iv, ic = eager.items()
        c = int(ic)
        assert int(outs[4]) == c
        assert np.array_equal(_bits(outs[0]), _bits(qv)) and torch.equal(outs[1], qe)
        assert torch.equal(outs[2][:c], ik[:c]) and np.array_equal(_bits(outs[3][:c]), _bits(iv[:c]))
