"""f64 against f32 on one GPU: the same N x 768 `datagen` rows built into a cos f32 index and a cos f64 index (M = 32),
then 4096 queries at ef 128, k 10. The f32 index runs with `tune(prefilter=0)`, the like-for-like baseline of the f64
kernel, which has no int8 prefilter. Per N it prints the build time, and per alternated run the kernel ms per launch
(CUDA events), queries/s, recall@10 against each index's GPU exact search (first 1024 queries), computed distances and
visited members per query, and the reference algorithm's bytes per query (D row bytes + H 260) over the kernel time.

    python tools/f64_check.py [--n 1000000 4000000] [--runs 3] [--out f64_check.json]
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


def run(index, queries, truth, row_bytes, k=10):
    res = index.search(queries, k, stats=True)
    ms = index.last_kernel_ms
    d, h = float(np.mean(index.last_computed)), float(np.mean(index.last_visited))
    recall = float(np.mean([len(set(f) & set(t)) / k for f, t in zip(res.keys[:len(truth)].tolist(), truth.tolist())]))
    return {"kernel_ms": ms, "qps": len(queries) / ms * 1e3, "recall10": recall, "computed_per_query": d, "visited_per_query": h,
            "ref_bytes_GBps": (d * row_bytes + h * 260) * len(queries) / (ms * 1e-3) / 1e9}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, nargs="+", default=[1_000_000, 4_000_000])
    p.add_argument("--d", type=int, default=768)
    p.add_argument("--runs", type=int, default=3)
    p.add_argument("--out")
    a = p.parse_args()
    report = {"card": card(), "d": a.d, "m": 32, "ef": 128, "k": 10, "nq": 4096, "sizes": []}
    print(json.dumps({"card": report["card"]}), flush=True)
    queries32 = datagen.latent(4096, a.d, seed=43)
    for n in a.n:
        base32 = datagen.latent(n, a.d, seed=42)
        entry = {"n": n}
        indexes = {}
        for dtype in ("f32", "f64"):
            index = Index(ndim=a.d, metric="cos", dtype=dtype, connectivity=32, expansion_add=128, expansion_search=128)
            rows = base32 if dtype == "f32" else base32.astype(np.float64)
            t = time.perf_counter()
            index.add(np.arange(n, dtype=np.uint64), rows)
            entry[f"build_s_{dtype}"] = time.perf_counter() - t
            del rows
            if dtype == "f32":
                index.tune(prefilter=0)
            q = queries32 if dtype == "f32" else queries32.astype(np.float64)
            truth = index.search(q[:1024], 10, exact=True).keys
            index.search(q, 10)  # warm-up
            indexes[dtype] = (index, q, truth, a.d * (4 if dtype == "f32" else 8))
        entry["runs"] = []
        for r in range(a.runs):  # alternated: f32, f64, f32, f64, ...
            entry["runs"].append({dtype: run(*indexes[dtype]) for dtype in ("f32", "f64")})
            print(json.dumps({"n": n, "run": r, **entry["runs"][-1]}), flush=True)
        print(json.dumps({k: v for k, v in entry.items() if k != "runs"}), flush=True)
        report["sizes"].append(entry)
        del indexes
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
