"""Time HashTable.insert and HashTable.query, and a torch formulation of the same lookups.

    python tools/hash_timing.py [--iters 20]

Cases: 1 M and 16 M distinct random keys, int32 and int64, int32 values, table size 2 N (load 0.5).  Prints
one JSON line with the card's name and power limit, then one per case: CUDA-event medians after warm-up of
  * insert: a fresh table (construction and its clear included) and one insert of the N keys;
  * query: N lookups of the stored keys in a random order;
  * torch_build / torch_query: the same work written with torch ops -- torch.unique(return_inverse) builds the
    sorted key set and its values, and searchsorted looks keys up in it;
and the rates in keys per second.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hash_timing.py needs a CUDA device")
    from spconv_b200.pytorch.hash import HashTable
    dev = torch.device("cuda")
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit": _power_limit()}), flush=True)
    gen = torch.Generator(device=dev).manual_seed(0)
    for n in (1 << 20, 1 << 24):
        for kdt in (torch.int32, torch.int64):
            info = torch.iinfo(kdt)
            keys = torch.unique(torch.randint(info.min, info.max - 1, (int(n * 1.1),), dtype=kdt, device=dev,
                                              generator=gen))
            keys = keys[torch.randperm(keys.numel(), device=dev, generator=gen)[:n]].contiguous()
            assert keys.numel() == n
            vals = torch.arange(n, dtype=torch.int32, device=dev)
            query = keys[torch.randperm(n, device=dev, generator=gen)].contiguous()
            cap = 2 * n

            def insert():
                t = HashTable(dev, kdt, torch.int32, max_size=cap)
                t.insert(keys, vals)
                return t

            table = insert()
            t_insert = _time(insert, args.iters)
            t_query = _time(lambda: table.query(query), args.iters)
            got, empty = table.query(query)
            assert not bool(empty.any())

            def torch_build():
                uniq, inv = torch.unique(keys, return_inverse=True)
                uv = torch.empty(uniq.numel(), dtype=vals.dtype, device=dev)
                uv[inv] = vals
                return uniq, uv

            uniq, uv = torch_build()

            def torch_query():
                pos = torch.searchsorted(uniq, query).clamp_(max=uniq.numel() - 1)
                return uv[pos], uniq[pos] != query

            ref, ref_empty = torch_query()
            assert torch.equal(ref, got) and not bool(ref_empty.any())
            t_tbuild = _time(torch_build, args.iters)
            t_tquery = _time(torch_query, args.iters)
            print(json.dumps({
                "keys": n, "key_dtype": str(kdt).replace("torch.", ""), "value_dtype": "int32", "table_size": cap,
                "load": 0.5, "insert_ms": round(t_insert, 4), "query_ms": round(t_query, 4),
                "insert_Mkeys_per_s": round(n / t_insert / 1e3, 1), "query_Mkeys_per_s": round(n / t_query / 1e3, 1),
                "torch_build_ms": round(t_tbuild, 4), "torch_query_ms": round(t_tquery, 4),
                "torch_build_Mkeys_per_s": round(n / t_tbuild / 1e3, 1),
                "torch_query_Mkeys_per_s": round(n / t_tquery / 1e3, 1),
            }), flush=True)


if __name__ == "__main__":
    main()
