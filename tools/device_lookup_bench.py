#!/usr/bin/env python
"""Measures the lookups by key from device memory on one GPU and prints one JSON line (DESIGN.md §3.9):

* the build of the key -> slot table at 1M and 10M entries (the first lookup on a fresh `copy()`, minus a lookup that
  finds the table built);
* `get_device` of 1M random keys from a 1M x 768 f32 index, as f32 and as f16, with the bytes the rows move and their
  share of the H100's 3.35 TB/s data-sheet HBM bandwidth;
* `count_device` of the same 1M keys;
* `filtered_search_device` with 1K / 100K / 1M device-resident allowed keys, against `filtered_search` given the same
  keys in host memory, on a 200K x 128 f32 cosine graph built by the GPU builder (1024 queries, k = 10).

Every call returns when its outputs are complete, so each time is a host clock around a finished call: the median of
`--repeat` calls after one warm-up. The two get / count indexes have no links (lookups never read them) and are loaded
from a file written here, which takes seconds where building their graphs would take minutes.

  python tools/device_lookup_bench.py [--repeat 5] [--out DIR]
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def unlinked_blob(vectors: np.ndarray, keys: np.ndarray, metric: str, scalar: str, dims: int) -> np.ndarray:
    """a v2 file whose members all sit on level 0 with empty lists (connectivity 2), written without a per-node loop"""
    from usearch_b200.v2format import METRIC_CHAR, SCALAR_CODE
    n, bpv = vectors.shape
    m, m0 = 2, 4
    head = bytearray(64)
    head[0:7] = b"usearch"
    head[7:13] = np.array([2, 21, 0], dtype=np.uint16).tobytes()
    head[13], head[14], head[15], head[16] = METRIC_CHAR[metric], SCALAR_CODE[scalar], 14, 15
    head[17:25] = np.uint64(n).tobytes()
    head[33:41] = np.uint64(dims).tobytes()
    tape = np.zeros(n, dtype=np.dtype([("key", "<u8"), ("level", "<i2"), ("list", "<u4", (m0 + 1,))]))
    tape["key"] = keys
    return np.concatenate([np.frombuffer(np.array([n, bpv], dtype=np.uint32).tobytes(), np.uint8), vectors.reshape(-1),
                           np.frombuffer(bytes(head), np.uint8),
                           np.frombuffer(np.array([n, m, m0, 0, 0], dtype=np.uint64).tobytes(), np.uint8),
                           np.zeros(2 * n, np.uint8), tape.view(np.uint8).reshape(-1)])


def median_time(fn, repeat):
    fn()
    times = []
    for _ in range(repeat):
        t = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t)
    return float(np.median(times))


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeat", type=int, default=5)
    p.add_argument("--keys", type=int, default=1_000_000)
    p.add_argument("--out", default=None, help="also write the JSON line to DIR/device_lookup_bench.json")
    args = p.parse_args()
    import torch
    from usearch_b200.index import Index
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these measurements need an H100")
    result = {"card": card()}
    rng = np.random.default_rng(0)

    def lookups(index, d_keys, n):
        counts = torch.empty(n, dtype=torch.int32, device="cuda")
        return lambda: index.count_device(d_keys.data_ptr(), n, counts.data_ptr())

    # table builds: 1M and 10M entries
    builds = {}
    for n in (1_000_000, 10_000_000):
        keys = rng.permutation(np.arange(n, dtype=np.uint64) * 7 + 1)
        index = Index.restore(unlinked_blob(np.zeros((n, 1), np.uint8), keys, "hamming", "b1", 8))
        one = torch.tensor([1], dtype=torch.int64, device="cuda")
        probe = lookups(index, one, 1)
        before = index.memory_usage
        probe()
        table_bytes = index.memory_usage - before
        steady = median_time(probe, args.repeat)
        firsts = []
        for _ in range(args.repeat):
            fresh = index.copy()
            torch.cuda.synchronize()
            t = time.perf_counter()
            lookups(fresh, one, 1)()
            firsts.append(time.perf_counter() - t)
            del fresh
        builds[f"{n // 1_000_000}M"] = {"build_ms": round((float(np.median(firsts)) - steady) * 1e3, 3),
                                        "table_mb": table_bytes / 2**20}
        del index
    result["table_build"] = builds

    # get / count of 1M random keys from a 1M x 768 f32 index
    n, dims, k = 1_000_000, 768, args.keys
    vectors = np.random.default_rng(1).standard_normal((n, dims), dtype=np.float32)
    index = Index.restore(unlinked_blob(vectors.view(np.uint8).reshape(n, -1), np.arange(n, dtype=np.uint64), "l2sq", "f32", dims))
    asked = rng.integers(0, n, k).astype(np.uint64)
    d_keys = torch.from_numpy(asked.view(np.int64)).cuda()
    counts = torch.empty(k, dtype=torch.int32, device="cuda")
    result["count_1M_keys_ms"] = round(median_time(lookups(index, d_keys, k), args.repeat) * 1e3, 3)
    gets = {}
    for kind, width in (("f32", 4), ("f16", 2)):
        out = torch.empty((k, dims * width), dtype=torch.uint8, device="cuda")
        seconds = median_time(lambda: index.get_device(d_keys.data_ptr(), k, out.data_ptr(), counts.data_ptr(), dtype=kind),
                              args.repeat)
        row_bytes = k * (dims * 4 + dims * width)  # each stored row read once, each output row written once
        sample = rng.integers(0, k, 2000)
        want = index.get(asked[sample], kind).view(np.uint8)
        gets[kind] = {"ms": round(seconds * 1e3, 3), "row_gb": round(row_bytes / 1e9, 3),
                      "row_bytes_share_of_3.35TBps": round(row_bytes / seconds / HBM_BYTES_PER_S, 3),
                      "matches_host_get": bool(np.array_equal(out[torch.from_numpy(sample).cuda()].cpu().numpy(), want))}
        del out
    result["get_1M_keys_of_1M_x_768_f32"] = gets
    del index, d_keys, counts

    # filtered search: device-resident allowed keys against the host path
    n, dims, nq, kk = 200_000, 128, 1024, 10
    index = Index(ndim=dims, metric="cos", dtype="f32", connectivity=16, expansion_search=64)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn((n, dims), device="cuda", dtype=torch.float32, generator=g)
    ids = torch.arange(n, device="cuda", dtype=torch.int64)
    index.add_device(ids.data_ptr(), x.data_ptr(), n, dims * 4, "f32")
    queries = torch.randn((nq, dims), device="cuda", dtype=torch.float32, generator=g)
    h_queries = queries.cpu().numpy()
    out_keys = torch.empty((nq, kk), dtype=torch.int64, device="cuda")
    out_dists = torch.empty((nq, kk), dtype=torch.float32, device="cuda")
    out_counts = torch.empty(nq, dtype=torch.int32, device="cuda")
    filtered = {}
    for m in (1_000, 100_000, 1_000_000):
        allowed = rng.integers(0, 2 * n, m).astype(np.uint64)
        d_allowed = torch.from_numpy(allowed.view(np.int64)).cuda()
        device_s = median_time(lambda: index.filtered_search_device(queries.data_ptr(), nq, dims * 4, kk, d_allowed.data_ptr(), m,
                                                                    out_keys.data_ptr(), out_dists.data_ptr(), out_counts.data_ptr()),
                               args.repeat)
        host_s = median_time(lambda: index.filtered_search(h_queries, kk, allowed), args.repeat)
        want = index.filtered_search(h_queries, kk, allowed)
        got = out_keys.cpu().numpy().view(np.uint64)
        same = all(np.array_equal(got[q, :int(c)], want.keys[q, :int(c)]) for q, c in enumerate(want.counts))
        filtered[f"{m}"] = {"device_ms": round(device_s * 1e3, 3), "host_keys_ms": round(host_s * 1e3, 3), "same_keys": bool(same)}
    result["filtered_search_200K_x_128_f32_cos_1024_queries"] = filtered

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_lookup_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
