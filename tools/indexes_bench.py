"""`Indexes.search` on one GPU against the two ways to get the same rows without it.

A collection of N `datagen` rows is built on the GPU three ways per shard count S: as S shards of N/S rows, and once as
one index of all N rows. For each S in --shards and k in --counts it times, on the same --batch queries:

    indexes    `Indexes.search` over the S shards (one call: S searches, the merge kernel, one copy back)
    single     `Index.search` on the index of all N rows
    separate   S `Index.search` calls, then `merge_topk` over their rows (the merge by hand)

and reports the merge kernel's share of the `Indexes` call from the CUDA events the call records. Medians over --repeats
after one warm-up. Prints one JSON line per (S, k), each with the card's name and power limit read in the same run.

    python tools/indexes_bench.py [--n 400000] [--d 128] [--shards 2 4 8] [--counts 10 100] [--batch 4096] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from churn_check import card  # noqa: E402
from usearch_b200 import datagen  # noqa: E402
from usearch_b200.index import Index, Indexes, merge_topk  # noqa: E402


def timed(fn, repeats):
    fn()  # warm-up
    walls = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        walls.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(walls))


def build(rows, first_key, d, m, ef):
    index = Index(ndim=d, metric="cos", dtype="f32", connectivity=m, expansion_search=ef)
    index.add(np.arange(first_key, first_key + len(rows), dtype=np.uint64), rows)
    return index


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=400_000)
    p.add_argument("--d", type=int, default=128)
    p.add_argument("--m", type=int, default=16)
    p.add_argument("--ef", type=int, default=64)
    p.add_argument("--shards", type=int, nargs="+", default=[2, 4, 8])
    p.add_argument("--counts", type=int, nargs="+", default=[10, 100])
    p.add_argument("--batch", type=int, default=4096)
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--out", default=None)
    args = p.parse_args()

    rows = datagen.latent(args.n, args.d, seed=1)
    queries = datagen.latent(args.batch, args.d, seed=2)
    gpu = card()
    t0 = time.perf_counter()
    whole = build(rows, 0, args.d, args.m, args.ef)
    results = []
    for S in args.shards:
        bounds = np.linspace(0, args.n, S + 1).astype(int)
        shards = [build(rows[lo:hi], lo, args.d, args.m, args.ef) for lo, hi in zip(bounds[:-1], bounds[1:])]
        group = Indexes(shards)
        for k in args.counts:
            split = []

            def indexes_arm():
                group.search(queries, k)
                split.append(group.last_ms)

            indexes_ms = timed(indexes_arm, args.repeats)
            single_ms = timed(lambda: whole.search(queries, k), args.repeats)

            def separate_arm():
                parts = [s.search(queries, k) for s in shards]
                merge_topk([(r.keys, r.distances, r.counts) for r in parts], k)

            separate_ms = timed(separate_arm, args.repeats)
            merge_ms = float(np.median([s["merge"] for s in split[1:]]))
            search_ms = float(np.median([s["search"] for s in split[1:]]))
            result = {"card": gpu, "n": args.n, "d": args.d, "m": args.m, "ef": args.ef, "shards": S, "k": k,
                      "batch": args.batch, "repeats": args.repeats, "indexes_ms": round(indexes_ms, 3),
                      "single_ms": round(single_ms, 3), "separate_ms": round(separate_ms, 3),
                      "indexes_searches_ms": round(search_ms, 3), "indexes_merge_ms": round(merge_ms, 4),
                      "merge_share": round(merge_ms / indexes_ms, 4)}
            print(json.dumps(result), flush=True)
            results.append(result)
    print(json.dumps({"card": gpu, "build_and_bench_s": round(time.perf_counter() - t0, 1)}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
