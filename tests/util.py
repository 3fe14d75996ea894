"""Shared helpers for the parity tests (inputs are seeded numpy -> identical for CUDA and oracle)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def random_cloud(rng, shape, num_per_batch, channels, dtype=np.float32):
    """Unique uniform-random coordinates per sample (spconv/test_utils.py:142-195 semantics)."""
    total = int(np.prod(shape))
    inds = []
    for b, n in enumerate(num_per_batch):
        flat = rng.permutation(total)[:n]
        coords = np.stack(np.unravel_index(flat, shape), axis=-1).astype(np.int32)
        inds.append(np.concatenate([np.full((n, 1), b, np.int32), coords], axis=1))
    indices = np.concatenate(inds, 0)
    feats = rng.uniform(-1, 1, size=(indices.shape[0], channels)).astype(dtype)
    return feats, indices


from bench_utils import surface_cloud  # noqa: E402,F401  (clustered LiDAR-like clouds)

REF_DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_digests.json")


def digest(arrays):
    """SHA-256 over the shapes and values of an array or a sequence of arrays (integers hashed as int64,
    floats as float64, so equal values give equal digests whatever the element type)."""
    import hashlib
    h = hashlib.sha256()
    for a in (arrays if isinstance(arrays, (tuple, list)) else [arrays]):
        a = np.asarray(a)
        a = np.ascontiguousarray(a, dtype=np.float64 if a.dtype.kind == "f" else np.int64)
        h.update(f"{a.dtype.str}{a.shape}".encode())
        h.update(a.tobytes())
    return h.hexdigest()


def assert_equals_reference(key, got, compute_ref, oracle):
    """Bit-exact check of `got` against the reference project's own CPU code (oracle/_ref).

    When oracle/_ref is built, `compute_ref()` runs it and the outputs are compared directly;
    SPX_RECORD_REF_DIGESTS=1 then also stores their digest under `key` in golden/ref_digests.json.
    Without oracle/_ref the digest of `got` must equal the stored digest of the reference's outputs."""
    import json
    stored = json.load(open(REF_DIGESTS)) if os.path.exists(REF_DIGESTS) else {}
    got = tuple(np.asarray(g) for g in (got if isinstance(got, (tuple, list)) else [got]))
    if oracle.have_ref():
        want = compute_ref()
        want = tuple(np.asarray(w) for w in (want if isinstance(want, (tuple, list)) else [want]))
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), key
        if os.environ.get("SPX_RECORD_REF_DIGESTS") == "1":
            stored[key] = digest(want)
            with open(REF_DIGESTS, "w") as f:
                json.dump(stored, f, indent=1, sort_keys=True)
        return
    assert key in stored, f"no stored reference digest for {key}"
    assert digest(got) == stored[key], f"{key}: output differs from the reference's (digest mismatch)"


def check_tile_table(table, tile_mask, pair, mask, argsort, rows, kv, words, name="tile table"):
    """Restates spx_build_tile_table's output from the rulebook it was built from (numpy arrays).

    table [tiles*(kv+1)*128 + tiles*8 + 64]: per 128-row tile one block of kv rows of gather indices
    (pair[k, argsort[j]] where bit k of the sorted mask row j is set, else -1) and one row of argsort
    (-1 past the end); then one 8-int schedule record per tile: the tiles heaviest first (most set bits
    of the tile mask, an empty tile counted as one stage with mask word 0 = 1), ties in ascending tile
    order, as (tile, mask words 0-3, 0, 0, 0); then 64 ints of scheduler scratch, zero between launches.
    tile_mask [tiles, words]: per-tile OR of the sorted masks."""
    tiles = (rows + 127) // 128
    blocks_len = tiles * (kv + 1) * 128
    assert table.shape == (blocks_len + tiles * 8 + 64,), f"{name}: {table.shape[0]} ints for {tiles} tiles"
    blocks = table[:blocks_len].reshape(tiles, kv + 1, 128)
    src = np.full(tiles * 128, -1, np.int64)
    src[:rows] = argsort
    assert np.array_equal(blocks[:, kv, :].reshape(-1), src), f"{name}: argsort row of the blocks"
    sm = np.zeros((tiles * 128, 4), np.uint32)
    sm[:rows, :words] = np.asarray(mask).view(np.uint32).reshape(rows, words)
    col = np.maximum(src, 0)
    for k in range(kv):
        hit = (((sm[:, k // 32] >> np.uint32(k % 32)) & 1) == 1) & (src >= 0)
        got = blocks[:, k, :].reshape(-1)
        want = np.where(hit, pair[k][col], -1)
        bad = np.nonzero(got != want)[0]
        assert not len(bad), (f"{name}: offset {k}: {len(bad)} gather entries differ, first at row {bad[0]} "
                              f"(tile {bad[0] // 128}): got {got[bad[0]]} want {want[bad[0]]}")
    tm = np.bitwise_or.reduce(sm.reshape(tiles, 128, 4), axis=1)
    assert np.array_equal(np.asarray(tile_mask).view(np.uint32).reshape(tiles, words), tm[:, :words]), \
        f"{name}: tile masks"
    eff = tm.copy()
    eff[~eff.any(axis=1), 0] = 1
    cost = np.bitwise_count(eff).sum(axis=1)
    order = np.argsort(-cost, kind="stable")
    rec = table[blocks_len:blocks_len + tiles * 8].reshape(tiles, 8)
    bad = np.nonzero(rec[:, 0] != order)[0]
    assert not len(bad), (f"{name}: schedule order differs at record {bad[0]} of {tiles}: tile {rec[bad[0], 0]}, "
                          f"want {order[bad[0]]}")
    assert np.array_equal(rec[:, 1:5].view(np.uint32), eff[order]), f"{name}: record masks"
    assert (rec[:, 5:] == 0).all(), f"{name}: record padding"
    assert (table[blocks_len + tiles * 8:] == 0).all(), f"{name}: scheduler scratch is not zero"


def rel_l2(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def describe_mismatch(got, ref, name="", max_rows=5):
    """Human-readable summary of where two matrices differ (used in assertion messages so one
    GPU run tells as much as possible)."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref)
    bad = err > (1e-2 + 1e-2 * np.abs(ref))
    rows = np.unique(np.nonzero(bad)[0])
    cols = np.unique(np.nonzero(bad)[1]) if bad.ndim > 1 else []
    msg = (f"{name}: shape {got.shape} max_abs_err {err.max():.4g} rel_l2 {rel_l2(got, ref):.4g} "
           f"bad {bad.sum()}/{bad.size} bad_rows {len(rows)} (first {rows[:max_rows].tolist()}) "
           f"bad_cols {len(cols)} (first {list(cols[:16])}) nan {np.isnan(got).sum()}")
    if len(rows):
        r = rows[0]
        msg += f"\n  row {r} got {np.round(got[r][:8], 3).tolist()} ref {np.round(ref[r][:8], 3).tolist()}"
    return msg
