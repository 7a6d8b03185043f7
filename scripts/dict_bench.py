"""Time the order-preserving dictionary of a STRING column built on the device against the host encoder (baikaldb_b200/dictionary.py).

    python scripts/dict_bench.py [--workloads names] [--reps 5] [--host-max-rows 10000000]

Workloads (seeded; the strings are generated as Arrow arrays and uploaded once — the device path starts from strings already in HBM):
  customers  5M rows, 200k distinct values ("customer#000123456")
  urls       5M rows, 500k distinct URL-like values: three hosts (prefixes of 24 to 50 bytes), then shared category paths
  short      50M rows, 910k distinct values of 1 to 8 bytes

For each one line of JSON: the device encode time (encode_strings on DeviceStrings, CUDA events around the call and a synchronise, the
median of --reps runs after a warm-up run), the host encoder's time on the same strings (host clock, one run; skipped above
--host-max-rows rows), whether the two encodings are equal (dictionary, rewritten plan, codes and validity) — or, where the host run is
skipped, whether the device encoding equals the one the generator knows — and the card's name and power limit, read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import pyarrow as pa

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from baikaldb_b200 import dictionary as D, plan as P  # noqa: E402
from baikaldb_b200.plan import PrimitiveType as T  # noqa: E402


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        power = float(out.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return name, power


def _from_words(words, rows, rng, null_frac=0.01):
    """rows values drawn from `words` (a list of distinct bytes), as a large_binary array; and the drawn indices (-1 = NULL)"""
    idx = rng.integers(0, len(words), rows).astype(np.int32)
    idx[rng.random(rows) < null_frac] = -1
    dictionary = pa.array(words, pa.large_binary())
    arr = pa.DictionaryArray.from_arrays(pa.array(idx, mask=idx < 0), dictionary).dictionary_decode()
    return arr, idx


def workload(name, rng):
    if name == "customers":
        words = [f"customer#{i:09d}".encode() for i in rng.permutation(200_000)]
        rows = 5_000_000
    elif name == "urls":
        hosts = [b"https://www.example.com/", b"https://shop.example.org/catalog/", b"https://cdn.static.example.net/assets/images/2024/"]
        words = sorted({hosts[int(h)] + f"category-{int(c):03d}/product-{int(p):07d}?ref=x".encode()
                        for h, c, p in zip(rng.integers(0, 3, 600_000), rng.integers(0, 200, 600_000), rng.integers(0, 10**7, 600_000))})[:500_000]
        words = [words[i] for i in rng.permutation(len(words))]
        rows = 5_000_000
    elif name == "short":
        words = sorted({np.base_repr(int(v), 36).encode()[: 1 + int(v % 8)] for v in rng.integers(0, 36**8, 1_400_000)})[:1_000_000]
        words = [words[i] for i in rng.permutation(len(words))]
        rows = 50_000_000
    else:
        raise SystemExit(f"unknown workload {name}")
    arr, idx = _from_words(words, rows, rng)
    return words, arr, idx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="customers,urls,short")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-max-rows", type=int, default=10_000_000)
    args = ap.parse_args()
    import torch
    card, power = _card()
    plan = P.Plan(P.agg(P.scan(0), 1, [P.slot_ref(0, 1, T.STRING)], [P.agg_expr("count_star", 1, 1)]), {0: [(1, T.STRING)], 1: [(1, T.INT64)]})
    for name in args.workloads.split(","):
        rng = np.random.default_rng(2031)
        words, arr, idx = workload(name, rng)
        dev_in = D.DeviceStrings.from_arrow(arr, 0)
        torch.cuda.synchronize()
        enc = D.encode_strings(plan, [D.StringColumn(0, 1, dev_in)])   # warm-up
        times = []
        for _ in range(args.reps):
            del enc
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            enc = D.encode_strings(plan, [D.StringColumn(0, 1, dev_in)])
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        codes_t, valid_t = enc.columns[0].keepalive
        codes = codes_t.cpu().numpy()
        valid = np.ones(len(codes), bool) if valid_t is None else np.unpackbits(valid_t.cpu().numpy(), count=len(codes), bitorder="little").astype(bool)
        out = {"workload": name, "rows": len(arr), "distinct": len(enc.dictionaries[(0, 1)]), "bytes": int(arr.buffers()[2].size),
               "device_ms": round(statistics.median(times), 3), "device_ms_runs": [round(t, 3) for t in times]}
        if len(arr) <= args.host_max_rows:
            t0 = time.perf_counter()
            host = D.encode_strings(plan, [D.StringColumn(0, 1, arr)])
            out["host_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            hv = np.ones(len(codes), bool) if host.columns[0].valid is None else host.columns[0].valid
            out["equal"] = bool(host.dictionaries == enc.dictionaries and host.plan.serialize() == enc.plan.serialize()
                                and np.array_equal(host.columns[0].values, codes) and np.array_equal(hv, valid))
            out["equal_to"] = "host encoder"
        else:
            used = np.unique(idx[idx >= 0])
            ranked = sorted(used.tolist(), key=lambda i: words[i])
            rank = np.zeros(len(words), np.int64)
            rank[ranked] = np.arange(len(ranked))
            want = np.where(idx >= 0, rank[np.maximum(idx, 0)], 0)
            out["host_ms"] = None
            out["equal"] = bool(enc.dictionaries[(0, 1)] == [words[i] for i in ranked] and np.array_equal(codes, want) and np.array_equal(valid, idx >= 0))
            out["equal_to"] = "generator"
        out.update(card=card, power_limit_w=power)
        print(json.dumps(out), flush=True)
        del enc, dev_in
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
