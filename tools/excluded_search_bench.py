#!/usr/bin/env python
"""Measures excluded search on one GPU and prints one JSON line (DESIGN.md §3.12).

The §3.10 index: 1M x 768 f32 cosine (M 32, random Gaussian rows) built by the GPU builder, 4096 random queries, k = 10.
G excluded sets of D random keys each (G in 1 / 4096, D in 10 / 1000), query i using set i mod G. For each (G, D):

* `graph_host_s`, `graph_device_s`: `grouped_excluded_search` on host arrays (uploads included), and the device entry
  with queries, sets and outputs already in HBM;
* `exact_host_s`, `exact_device_s`: the same with `exact=True`;
* `complement_graph_host_s`, `complement_exact_host_s` (G = 1 only): the same rows asked the only way that existed
  before, `grouped_filtered_search` with the complement allowed set of about 1M keys. At G = 4096 that form would need
  G x (n - D) keys built, joined and uploaded (`complement_keys`, `complement_gb`), and is not run;
* `graph_kernels_ms`, `exact_kernels_ms`: the GPU time of one device call's kernels by kind, under `torch.profiler`
  (`rows`: the complement rows, or the slot lists' count, write, unique and offsets; `search`: the search launches and
  retries, or the exact scans; `merge`: the exact merges; `drop`: the exact form's drop; `other`: argument check, memsets,
  radix sorts, prefix sums and the query gather).

`plain_search_device_s` and `plain_exact_device_s` are the unfiltered baselines at k = 10; `exact_at_count_s` times the
unfiltered exact search at each count the exact cases ran at (k + D rounded up to a power of two), the expected cost of an
exact excluded call. Each time is the best of `--repeat` calls after one warm-up; every call returns when its outputs are
complete. The device rows are checked against the host rows, and sampled rows against `filtered_search` with the
complement.

  python tools/excluded_search_bench.py [--n 1000000] [--repeat 3] [--out DIR]
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
    out = {"rows": 0.0, "search": 0.0, "merge": 0.0, "drop": 0.0, "other": 0.0}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name  # the scan kernels' argument type names exact_listed_args_t: test the kernel names first
        if "hnsw_search_kernel" in name or any(s in name for s in ("exact_scan_kernel", "exact_tiled_kernel", "exact_imma", "exact_wgmma")):
            kind = "search"
        elif "exact_merge" in name:
            kind = "merge"
        elif "excluded_drop_kernel" in name:
            kind = "drop"
        elif any(s in name for s in ("excluded_bits_kernel", "listed_count", "listed_write", "listed_rows", "Unique", "Select")):
            kind = "rows"
        else:
            kind = "other"
        out[kind] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_000_000)
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--nq", type=int, default=4096)
    p.add_argument("--groups", default="1,4096")
    p.add_argument("--set-sizes", default="10,1000")
    p.add_argument("--repeat", type=int, default=3)
    p.add_argument("--out", default=None, help="also write the JSON line to DIR/excluded_search_bench.json")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("excluded_search_bench needs a GPU: nothing here runs on the CPU")
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
    everything = np.arange(a.n, dtype=np.uint64)
    counts_run = set()
    for size in (int(s) for s in a.set_sizes.split(",")):
        for G in (int(g) for g in a.groups.split(",")):
            groups = (np.arange(a.nq) % G).astype(np.uint32)
            flat = np.concatenate([rng.choice(a.n, size, replace=False).astype(np.uint64) for _ in range(G)])
            sets = [flat[g * size:(g + 1) * size] for g in range(G)]
            offsets = np.arange(G + 1, dtype=np.uint64) * size
            case = {"G": G, "set_size": size}
            d_groups = torch.from_numpy(groups.astype(np.int32)).cuda()
            d_offsets = torch.from_numpy(offsets.view(np.int64)).cuda()
            d_keys = torch.from_numpy(flat.view(np.int64)).cuda()
            torch.cuda.synchronize()
            for exact in (False, True):
                form = "exact" if exact else "graph"
                case[f"{form}_host_s"] = round(best_of(lambda: index.grouped_excluded_search(queries, k, sets, groups, exact=exact),
                                                       a.repeat), 4)

                def device_call():
                    index.grouped_excluded_search_device(d_q.data_ptr(), a.nq, a.dim * 4, k, d_groups.data_ptr(), d_offsets.data_ptr(), G,
                                                         d_keys.data_ptr(), keys_out.data_ptr(), dists_out.data_ptr(),
                                                         counts_out.data_ptr(), exact=exact)
                case[f"{form}_device_s"] = round(best_of(device_call, a.repeat), 4)
                case[f"{form}_kernels_ms"] = kernel_times(torch, device_call)
                got = index.grouped_excluded_search(queries, k, sets, groups, exact=exact)
                assert np.array_equal(keys_out.cpu().numpy().view(np.uint64), got.keys), (form, G, size)
                for i in range(0, a.nq, max(a.nq // 4, 1)):
                    want = index.filtered_search(queries[i], k, np.setdiff1d(everything, sets[groups[i]]), exact=exact)
                    assert np.array_equal(got.keys[i, :len(want)], want.keys), (form, G, size, i)
                if G == 1:
                    allowed = [np.setdiff1d(everything, sets[0])]
                    case[f"complement_{form}_host_s"] = round(
                        best_of(lambda: index.grouped_filtered_search(queries, k, allowed, groups, exact=exact), a.repeat), 4)
            counts_run.add(1 << (k + size - 1).bit_length())
            if G > 1:
                case["complement_keys"] = G * (a.n - size)
                case["complement_gb"] = round(G * (a.n - size) * 8 / 1e9, 1)
            result["cases"].append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
            del d_keys, sets, flat
    result["plain_search_device_s"] = round(best_of(lambda: index.search_device(
        d_q.data_ptr(), a.nq, a.dim * 4, k, keys_out.data_ptr(), dists_out.data_ptr(), counts_out.data_ptr()), a.repeat), 4)
    result["plain_exact_host_s"] = round(best_of(lambda: index.search(queries, k, exact=True), a.repeat), 4)
    result["exact_at_count_s"] = {c: round(best_of(lambda: index.search(queries, c, exact=True), a.repeat), 4) for c in sorted(counts_run)}
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "excluded_search_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
