#!/usr/bin/env python
"""Measures exact filtered search on one GPU and prints one JSON line (DESIGN.md §3.11).

The setup of §3.10: a 1M x 768 f32 cosine index (M 32, random Gaussian rows) built by the GPU builder, 4096 random queries,
k = 10. G key sets of S random keys each (S in 1K / 100K / 1M, G in 1 / 4096), query i using set i mod G. For each case:

* `exact_device_ms` / `exact_host_ms`: `grouped_filtered_search(..., exact=True)` from device arrays (queries, sets and
  outputs already in HBM) and from host arrays (uploads included);
* `graph_device_ms`: the graph's `grouped_filtered_search_device` on the same sets (`--graph-sizes` picks the set sizes it
  runs for: 1K-key sets take seconds there);
* `kernels_ms`: the GPU time of one exact device call's kernels by kind, from a `torch.profiler` run (`lists`: the slot
  lists' build, `scan`: the listed scan, `merge`, `other`: argument check, query order, gather and scatter).

The unfiltered `search(exact=True)` of the same host queries is timed once (`exact_unfiltered_ms`), and an i8
cosine index of the same shape (a linkless image: exact search reads no links) is searched with 1K-row sets (mma.sync).
Times are medians of `--repeat` rounds after a warm-up round; the calls of a round alternate between the variants, and
every call returns when its outputs are complete. The card's name, power limit and clocks are read in the same run.

  python tools/exact_filter_bench.py [--n 1000000] [--repeat 5] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.grouped_filter_bench import build  # noqa: E402  (the §3.10 index)

MAX_ENTRIES = 500_000_000  # 4096 sets of 1M keys (32 GB of keys on the host alone) are left out


def medians(calls, repeat):
    """{name: median ms} of alternated calls: one warm-up round, then `repeat` rounds of every call in turn"""
    for fn in calls.values():
        fn()
    times = {name: [] for name in calls}
    for _ in range(repeat):
        for name, fn in calls.items():
            t = time.perf_counter()
            fn()
            times[name].append((time.perf_counter() - t) * 1e3)
    return {name: round(float(np.median(v)), 3) for name, v in times.items()}


def kernel_times(torch, fn):
    """GPU milliseconds of the kernels `fn` launches, by kind"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"lists": 0.0, "scan": 0.0, "merge": 0.0, "other": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name
        if "exact_scan_kernel" in name or "exact_tiled_kernel" in name or "exact_imma_kernel" in name or "self_dot" in name:
            kind = "scan"
        elif "exact_merge" in name:
            kind = "merge"
        elif ("listed_count" in name or "listed_write" in name or "listed_rows" in name or "key_table" in name
              or ("Radix" in name and "Onesweep" in name) or "Unique" in name or "Select" in name or "Scan" in name):
            kind = "lists"
        else:
            kind = "other"
        out[kind] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def run_cases(torch, index, queries, sizes, groups_list, graph_sizes, repeat, n, k, rng, label):
    nq, dim = queries.shape
    d_q = torch.from_numpy(queries).cuda()
    row_bytes = queries.strides[0]
    keys_out = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    dists_out = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    counts_out = torch.zeros(nq, dtype=torch.int32, device="cuda")
    computed_out = torch.zeros(nq, dtype=torch.int32, device="cuda")
    cases = []
    for size in sizes:
        for G in groups_list:
            if G * size > MAX_ENTRIES:
                cases.append({"index": label, "G": G, "set_size": size, "skipped": f"{G * size} keys in all, past {MAX_ENTRIES}"})
                continue
            groups = (np.arange(nq) % G).astype(np.uint32)
            flat = rng.integers(0, n, G * size, dtype=np.uint64) if size < n else np.tile(np.arange(n, dtype=np.uint64), G)
            sets = [flat[g * size:(g + 1) * size] for g in range(G)]
            offsets = np.arange(G + 1, dtype=np.uint64) * size
            d_groups = torch.from_numpy(groups.astype(np.int32)).cuda()
            d_offsets = torch.from_numpy(offsets.view(np.int64)).cuda()
            d_keys = torch.from_numpy(flat.view(np.int64)).cuda()
            torch.cuda.synchronize()

            def exact_device():
                index.grouped_filtered_search_device(d_q.data_ptr(), nq, row_bytes, k, d_groups.data_ptr(), d_offsets.data_ptr(), G,
                                                     d_keys.data_ptr(), keys_out.data_ptr(), dists_out.data_ptr(),
                                                     counts_out.data_ptr(), computed_out.data_ptr(), exact=True)

            calls = {"exact_device_ms": exact_device,
                     "exact_host_ms": lambda: index.grouped_filtered_search(queries, k, sets, groups, exact=True)}
            if size in graph_sizes:
                calls["graph_device_ms"] = lambda: index.grouped_filtered_search_device(
                    d_q.data_ptr(), nq, row_bytes, k, d_groups.data_ptr(), d_offsets.data_ptr(), G, d_keys.data_ptr(),
                    keys_out.data_ptr(), dists_out.data_ptr(), counts_out.data_ptr())
            case = {"index": label, "G": G, "set_size": size, **medians(calls, repeat)}
            case["kernels_ms"] = kernel_times(torch, exact_device)
            case["listed_rows_per_query"] = int(computed_out.float().mean().item())
            # the device rows equal the host rows, and a sampled query equals the single-set call
            got = index.grouped_filtered_search(queries, k, sets, groups, exact=True)
            assert np.array_equal(keys_out.cpu().numpy().view(np.uint64), got.keys), (label, G, size)
            for i in (0, nq - 1):
                one = index.filtered_search(queries[i], k, sets[groups[i]], exact=True)
                assert np.array_equal(one.keys, got.keys[i, :len(one.keys)]), (label, G, size, i)
            cases.append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
            del d_keys, sets, flat
    unfiltered = medians({"exact_unfiltered_ms": lambda: index.search(queries, k, exact=True)}, repeat)
    return cases, unfiltered


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_000_000)
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--nq", type=int, default=4096)
    p.add_argument("--groups", default="1,4096")
    p.add_argument("--set-sizes", default="1000,100000,1000000")
    p.add_argument("--graph-sizes", default="100000,1000000")
    p.add_argument("--i8-set-sizes", default="1000")
    p.add_argument("--repeat", type=int, default=5)
    p.add_argument("--out", default=None, help="also write the JSON line to DIR/exact_filter_bench.json")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("exact_filter_bench needs a GPU: nothing here runs on the CPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    k = 10
    sizes = [int(s) for s in a.set_sizes.split(",") if s]
    groups_list = [int(g) for g in a.groups.split(",") if g]
    graph_sizes = {int(s) for s in a.graph_sizes.split(",") if s}
    result = {"gpu": card, "n": a.n, "dim": a.dim, "nq": a.nq, "k": k}
    t = time.perf_counter()
    index = build(torch, a.n, a.dim, seed=42)
    result["build_s"] = round(time.perf_counter() - t, 1)
    rng = np.random.default_rng(0)
    queries = rng.standard_normal((a.nq, a.dim), dtype=np.float32)
    result["cases"], unfiltered = run_cases(torch, index, queries, sizes, groups_list, graph_sizes, a.repeat, a.n, k, rng, "f32")
    result.update(unfiltered)
    del index
    i8_sizes = [int(s) for s in a.i8_set_sizes.split(",") if s]
    if i8_sizes:
        from tools.exact_bench import linkless_blob
        from usearch_b200.index import Index
        rows = rng.integers(-100, 101, (a.n, a.dim), dtype=np.int8)
        i8 = Index.restore(linkless_blob(rows, "cos", "i8", a.dim))
        del rows
        q8 = rng.integers(-100, 101, (a.nq, a.dim), dtype=np.int8)
        cases, unfiltered = run_cases(torch, i8, q8, i8_sizes, groups_list, set(), a.repeat, a.n, k, rng, "i8")
        result["cases"] += cases
        result["i8_exact_unfiltered_ms"] = unfiltered["exact_unfiltered_ms"]
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "exact_filter_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
