"""Churn on one GPU: rounds of "remove 10 % random keys, add 10 % fresh rows", with slot reuse off, on, and on with
`remove(..., compact=True)`. Per round it prints capacity, memory_usage, recall@10 against the GPU exact search,
computed distances and visited members per query, kernel ms per 4096-query batch, and the add time.

    python tools/churn_check.py [--n 1000000] [--d 768] [--m 32] [--rounds 3] [--out churn.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from usearch_b200 import datagen  # noqa: E402
from usearch_b200.index import Index  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(index, queries, k=10, ef=64):
    index.expansion_search = ef
    truth = index.search(queries, k, exact=True).keys
    index.search(queries, k)  # warm-up
    res = index.search(queries, k, stats=True)
    ms = index.last_kernel_ms
    recall = float(np.mean([len(set(f) & set(t)) / k for f, t in zip(res.keys.tolist(), truth.tolist())]))
    return {"recall10": recall, "computed_per_query": float(np.mean(index.last_computed)),
            "visited_per_query": float(np.mean(index.last_visited)), "kernel_ms": ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--m", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    n, d = args.n, args.d
    base = datagen.latent(n, d, seed=42)
    queries = datagen.latent(4096, d, seed=43)
    report = {"card": card(), "n": n, "d": d, "m": args.m, "metric": "cos", "modes": {}}
    print(json.dumps({"card": report["card"], "n": n, "d": d, "m": args.m}), flush=True)
    for mode in ("reuse_off", "reuse_on", "reuse_on_compact"):
        index = Index(ndim=d, metric="cos", dtype="f32", connectivity=args.m, expansion_add=128)
        t0 = time.perf_counter()
        index.add(np.arange(n, dtype=np.uint64), base)
        build_s = time.perf_counter() - t0
        index.reuse_removed = mode != "reuse_off"
        rng = np.random.default_rng(7)
        live = np.arange(n, dtype=np.uint64)
        next_key = n
        rows = [{"round": 0, "capacity": index.capacity, "memory_usage": index.memory_usage, "build_s": build_s,
                 **measure(index, queries)}]
        print(json.dumps({"mode": mode, **rows[-1]}), flush=True)
        for rnd in range(1, args.rounds + 1):
            victims = rng.choice(live, n // 10, replace=False)
            index.remove(victims, compact=mode == "reuse_on_compact")
            pruned = index.last_pruned_edges
            live = np.setdiff1d(live, victims)
            fresh = datagen.latent(n // 10, d, seed=1000 + rnd)
            keys = np.arange(next_key, next_key + n // 10, dtype=np.uint64)
            next_key += n // 10
            t0 = time.perf_counter()
            index.add(keys, fresh)
            add_s = time.perf_counter() - t0
            live = np.concatenate([live, keys])
            rows.append({"round": rnd, "capacity": index.capacity, "memory_usage": index.memory_usage, "add_s": add_s,
                         "pruned_edges": pruned, **measure(index, queries)})
            print(json.dumps({"mode": mode, **rows[-1]}), flush=True)
        report["modes"][mode] = rows
        del index
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
