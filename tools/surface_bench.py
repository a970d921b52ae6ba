#!/usr/bin/env python
"""Measures reading an index back out on one GPU and prints one JSON line (DESIGN.md §3.8):

* `get` of `--keys` random keys from an n x 768 f32 cosine index (M=32), the batched path against the per-key path (timed
  on a sample of `--sample` keys and scaled), and the bytes of both outputs compared;
* `vectors` of the whole index, as GB/s of output against the host link's pinned D2H rate measured in the same run;
* `copy()` of that index, as GB/s of HBM copied (bytes of the copy's arrays over the wall clock);
* `stats` of a second graph of `--stats-n` members (10M: the NS graph of bench.py, built the same way).

The collections are random Gaussian rows generated on the device and linked by the GPU builder.

  python tools/surface_bench.py [--n 1000000] [--stats-n 10000000] [--out DIR]
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


def timed(fn, repeat=3):
    best, out = float("inf"), None
    for _ in range(repeat):
        t = time.perf_counter()
        out = fn()
        best = min(best, time.perf_counter() - t)
    return best, out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_000_000)
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--keys", type=int, default=1_000_000)
    p.add_argument("--sample", type=int, default=20_000)
    p.add_argument("--stats-n", type=int, default=10_000_000)
    p.add_argument("--out", default=None, help="also write the JSON line to DIR/surface_bench.json")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("surface_bench needs a GPU: nothing here runs on the CPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    result = {"gpu": card, "n": a.n, "dim": a.dim}

    t = time.perf_counter()
    index = build(torch, a.n, a.dim, seed=42)
    result["build_s"] = round(time.perf_counter() - t, 1)
    row_bytes = a.dim * 4
    keys = np.random.default_rng(0).integers(0, a.n, a.keys, dtype=np.uint64)
    index.get(keys[:1000])  # warm-up: key map, module load
    t_new, got = timed(lambda: index.get(keys))
    sample = keys[:a.sample]
    t0 = time.perf_counter()
    old = np.stack([index.get(int(k)) for k in sample])
    t_old = (time.perf_counter() - t0) * a.keys / a.sample
    assert old.tobytes() == got[:a.sample].tobytes(), "batched and per-key rows differ"
    result["get_keys"] = a.keys
    result["get_batched_s"] = round(t_new, 4)
    result["get_per_key_s_scaled"] = round(t_old, 2)
    result["get_speedup"] = round(t_old / t_new, 1)
    result["get_batched_GBps"] = round(a.keys * row_bytes / t_new / 1e9, 2)
    t_f16, _ = timed(lambda: index.get(keys, "f16"))
    result["get_batched_f16_s"] = round(t_f16, 4)

    # host link: one pinned D2H copy of 1 GB, the ceiling `vectors` is held to
    src = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
    dst = torch.empty(1 << 30, dtype=torch.uint8, pin_memory=True)
    dst.copy_(src)
    torch.cuda.synchronize()
    t_link, _ = timed(lambda: (dst.copy_(src), torch.cuda.synchronize()))
    result["d2h_pinned_GBps"] = round((1 << 30) / t_link / 1e9, 2)
    del src, dst
    t_vec, vectors = timed(lambda: index.vectors, repeat=2)
    result["vectors_s"] = round(t_vec, 3)
    result["vectors_GBps"] = round(vectors.nbytes / t_vec / 1e9, 2)
    del vectors

    t_copy, copy = timed(lambda: index.copy(), repeat=2)
    result["copy_s"] = round(t_copy, 4)
    result["copy_bytes"] = index.memory_usage
    result["copy_GBps"] = round(index.memory_usage / t_copy / 1e9, 1)
    del copy
    t_stats, stats = timed(lambda: index.stats)
    result["stats_s"] = round(t_stats, 4)
    result["stats"] = vars(stats)
    del index

    if a.stats_n:
        t = time.perf_counter()
        big = build(torch, a.stats_n, a.dim, seed=43)
        result["stats_graph_n"] = a.stats_n
        result["stats_graph_build_s"] = round(time.perf_counter() - t, 1)
        big.levels_stats  # warm-up
        t_big, stats = timed(lambda: big.levels_stats)
        result["levels_stats_big_s"] = round(t_big, 4)
        result["levels_big"] = len(stats)
        result["edges_big"] = sum(s.edges for s in stats)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "surface_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
