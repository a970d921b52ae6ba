#!/usr/bin/env python
"""Measures grouped filtered search on one GPU and prints one JSON line (DESIGN.md §3.10).

A 1M x 768 f32 cosine index (M 32, random Gaussian rows) built by the GPU builder, 4096 random queries, k = 10, G key
sets of S random keys each (G in 1 / 16 / 256 / 4096, S in 1K / 100K), query i using set i mod G. For each (G, S):

* `loop_s`: the per-set calls a caller makes today, `filtered_search(queries of set g, k, set g)` for every g, host
  buffers. At G = 4096 only the first `--loop-sets` sets are timed and the time is scaled to all G (`loop_scaled`);
* `grouped_host_s`: `grouped_filtered_search` on the same host arrays, uploads included;
* `grouped_device_s`: the device entry with queries, sets and outputs already in HBM;
* `kernels_ms`: the GPU time of that call's kernels by kind, from one more call under `torch.profiler` (`bitmap`: the
  rows' build, `search`: the search launch and its scratch retries, `other`: argument check, memsets, sort).

Each time is the best of `--repeat` calls after one warm-up; every call returns when its outputs are complete. A very
selective set (1K of 1M keys) makes each query walk much of the graph before `top` fills, so those searches take seconds:
use `--groups` / `--set-sizes` / `--loop-sets` to split the cases over runs.

  python tools/grouped_filter_bench.py [--n 1000000] [--repeat 3] [--out DIR]
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


def build(torch, n, dim, seed):
    from usearch_b200.index import Index
    index = Index(ndim=dim, metric="cos", dtype="f32", connectivity=32, expansion_add=128, expansion_search=128)
    index.reserve(n)
    g = torch.Generator(device="cuda").manual_seed(seed)
    chunk = 1 << 18
    for lo in range(0, n, chunk):
        m = min(chunk, n - lo)
        x = torch.randn((m, dim), device="cuda", dtype=torch.float32, generator=g)
        keys = torch.arange(lo, lo + m, device="cuda", dtype=torch.int64)
        index.add_device(keys.data_ptr(), x.data_ptr(), m, x.stride(0) * 4, "f32")
        torch.cuda.synchronize()
    return index


def best_of(fn, repeat):
    fn()
    best = float("inf")
    for _ in range(repeat):
        t = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t)
    return best


def kernel_times(torch, fn):
    """GPU milliseconds of the kernels `fn` launches, by kind"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"bitmap": 0.0, "search": 0.0, "other": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        kind = "bitmap" if "grouped_bits_kernel" in e.name else "search" if "hnsw_search_kernel" in e.name else "other"
        out[kind] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_000_000)
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--nq", type=int, default=4096)
    p.add_argument("--groups", default="1,16,256,4096")
    p.add_argument("--set-sizes", default="1000,100000")
    p.add_argument("--loop-sets", type=int, default=256)
    p.add_argument("--repeat", type=int, default=3)
    p.add_argument("--out", default=None, help="also write the JSON line to DIR/grouped_filter_bench.json")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("grouped_filter_bench needs a GPU: nothing here runs on the CPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    result = {"gpu": card, "n": a.n, "dim": a.dim, "nq": a.nq, "k": 10, "cases": []}
    t = time.perf_counter()
    index = build(torch, a.n, a.dim, seed=42)
    result["build_s"] = round(time.perf_counter() - t, 1)
    rng = np.random.default_rng(0)
    queries = rng.standard_normal((a.nq, a.dim), dtype=np.float32)
    d_q = torch.from_numpy(queries).cuda()
    k = 10
    keys_out = torch.zeros((a.nq, k), dtype=torch.int64, device="cuda")
    dists_out = torch.zeros((a.nq, k), dtype=torch.float32, device="cuda")
    counts_out = torch.zeros(a.nq, dtype=torch.int32, device="cuda")
    for size in (int(s) for s in a.set_sizes.split(",")):
        for G in (int(g) for g in a.groups.split(",")):
            groups = (np.arange(a.nq) % G).astype(np.uint32)
            flat = rng.integers(0, a.n, G * size, dtype=np.uint64)
            sets = [flat[g * size:(g + 1) * size] for g in range(G)]
            offsets = np.arange(G + 1, dtype=np.uint64) * size
            case = {"G": G, "set_size": size}
            timed = min(G, a.loop_sets)
            members = [np.nonzero(groups == g)[0] for g in range(timed)]
            loop = best_of(lambda: [index.filtered_search(queries[m], k, sets[g]) for g, m in enumerate(members)], a.repeat)
            case["loop_s"] = round(loop * G / timed, 4)
            case["loop_scaled"] = timed < G
            case["grouped_host_s"] = round(best_of(lambda: index.grouped_filtered_search(queries, k, sets, groups), a.repeat), 4)
            d_groups = torch.from_numpy(groups.astype(np.int32)).cuda()
            d_offsets = torch.from_numpy(offsets.view(np.int64)).cuda()
            d_keys = torch.from_numpy(flat.view(np.int64)).cuda()
            torch.cuda.synchronize()

            def device_call():
                index.grouped_filtered_search_device(d_q.data_ptr(), a.nq, a.dim * 4, k, d_groups.data_ptr(), d_offsets.data_ptr(), G,
                                                     d_keys.data_ptr(), keys_out.data_ptr(), dists_out.data_ptr(), counts_out.data_ptr())
            dev = best_of(device_call, a.repeat)
            case["grouped_device_s"] = round(dev, 4)
            case["kernels_ms"] = kernel_times(torch, device_call)
            case["speedup_device_vs_loop"] = round(case["loop_s"] / dev, 1)
            # the rows equal the per-set calls' (checked on a sample of queries)
            got = index.grouped_filtered_search(queries, k, sets, groups)
            for i in range(0, a.nq, max(a.nq // 4, 1)):
                want = index.filtered_search(queries[i], k, sets[groups[i]])
                assert np.array_equal(got.keys[i, :len(want)], want.keys), (G, size, i)
            assert np.array_equal(keys_out.cpu().numpy().view(np.uint64), got.keys), (G, size)
            result["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
            del d_keys, sets, flat
    plain = best_of(lambda: index.search_device(d_q.data_ptr(), a.nq, a.dim * 4, k, keys_out.data_ptr(), dists_out.data_ptr(),
                                                counts_out.data_ptr()), a.repeat)
    result["plain_search_device_s"] = round(plain, 4)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "grouped_filter_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
