"""Wall clock of the free exact search over raw f32 matrices (cos, k 10), against a parent build of the library.

    python tools/exact_chunked_bench.py --parent-lib <path to the parent's libusearch_b200.so> [--n 10000000] [--big 30000000]

A: a pageable host array of `n` x 768 rows, 1 000 and 10 000 queries, this build and the parent alternated; a single
   query gives the upload alone (the scan of one query is negligible), from which the achieved H2D rate and the share of
   the upload hidden under the scan follow. Results of the two builds are compared bit for bit.
B: the device entry over the same rows already in HBM (a torch tensor), scanned in place.
C: `big` x 768 rows, more than HBM, when the host has the memory; otherwise "not measured".
The card's name and power limit are read in the same call. Prints one JSON object.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D, K = 768, 10


def gpu_info() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in out[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def host_memory_gb() -> float:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 2**20
    return 0.0


def rows(n: int, seed: int) -> np.ndarray:
    out = np.empty((n, D), np.float32)
    rng = np.random.default_rng(seed)
    step = 1 << 20
    for i in range(0, n, step):
        out[i:i + step] = rng.standard_normal((min(step, n - i), D), dtype=np.float32)
    return out


def load(path: str) -> C.CDLL:
    lib = C.CDLL(path)
    lib.usearch_exact_search.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                         C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                         C.POINTER(C.c_char_p)]
    return lib


def run(lib: C.CDLL, data: np.ndarray, queries: np.ndarray, threads: int = 0):
    """one call: wall clock (s), keys, distances, error"""
    nq = queries.shape[0]
    keys = np.zeros((nq, K), np.uint64)
    dists = np.zeros((nq, K), np.float32)
    err = C.c_char_p()
    t0 = time.perf_counter()
    lib.usearch_exact_search(data.ctypes.data, data.shape[0], data.strides[0], queries.ctypes.data, nq, queries.strides[0], 1, D, 1, K,
                             threads, keys.ctypes.data, keys.strides[0], dists.ctypes.data, dists.strides[0], C.byref(err))
    return time.perf_counter() - t0, keys, dists, (err.value.decode() if err.value else None)


def log(*what) -> None:
    print(*what, file=sys.stderr, flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--big", type=int, default=30_000_000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--budget-s", type=float, default=330, help="skip C when A and B took longer than this")
    ap.add_argument("--queries", type=int, nargs="+", default=[1000, 10000])
    ap.add_argument("--threads", type=int, nargs="+", default=[1, 4, 16], help="host threads of the upload-only runs")
    args = ap.parse_args()
    started = time.perf_counter()
    import torch
    from usearch_b200 import index as ix
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    report = {**gpu_info(), "host_mem_available_gb": round(host_memory_gb(), 1), "n": args.n, "dims": D, "k": K}
    log(json.dumps(report))
    new, parent = load(ix.LIB_PATH), load(args.parent_lib)
    data = rows(args.n, 1)
    gb = data.nbytes / 1e9
    report["dataset_gb"] = round(gb, 2)
    qs = {nq: rows(nq, 2 + nq) for nq in [1] + args.queries}
    run(new, data[:100000], qs[1000])  # load modules on both builds
    run(parent, data[:100000], qs[1000])

    # A: host rows, alternated with the parent
    a = {}
    for nq in [1] + args.queries:
        times = {"new": [], "parent": []}
        same = True
        for _ in range(args.reps):
            tn, kn, dn, en = run(new, data, qs[nq])
            tp, kp, dp, ep = run(parent, data, qs[nq])
            assert en is None and ep is None, (en, ep)
            log(f"A nq={nq}: new {tn:.3f} s, parent {tp:.3f} s")
            times["new"].append(round(tn, 3))
            times["parent"].append(round(tp, 3))
            same &= bool(np.array_equal(kn, kp) and np.array_equal(dn.view(np.uint32), dp.view(np.uint32)))
        a[nq] = {"new_s": times["new"], "parent_s": times["parent"], "identical_results": same}
        log(f"A nq={nq}: identical results {same}")
    for threads in args.threads:
        a.setdefault("upload_only_threads", {})[threads] = round(run(new, data, qs[1], threads)[0], 3)
        log(f"A upload only, {threads} threads: {a['upload_only_threads'][threads]} s")
    upload = min(a[1]["new_s"])
    a["upload_gb_per_s"] = round(gb / upload, 1)

    # B: the same rows in HBM, scanned in place on a non-default stream
    dev = torch.from_numpy(data).cuda()
    stream = torch.cuda.Stream()
    b = {}
    for nq in args.queries:
        q = torch.from_numpy(qs[nq]).cuda()
        keys = torch.zeros((nq, K), dtype=torch.int64, device="cuda")
        dists = torch.zeros((nq, K), dtype=torch.float32, device="cuda")
        best = []
        for _ in range(args.reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ix.exact_search_device(dev.data_ptr(), args.n, D * 4, q.data_ptr(), nq, D * 4, D, K, keys.data_ptr(), dists.data_ptr(),
                                   metric="cos", stream=stream.cuda_stream)
            stream.synchronize()
            best.append(round(time.perf_counter() - t0, 3))
            log(f"B nq={nq}: {best[-1]} s")
        _, kh, dh, _ = run(new, data, qs[nq])
        b[nq] = {"device_s": best[1:], "identical_to_host_entry": bool(np.array_equal(keys.cpu().numpy().view(np.uint64), kh) and
                                                                       np.array_equal(dists.cpu().numpy().view(np.uint32), dh.view(np.uint32)))}
        scan = min(best[1:])
        t_a = min(a[nq]["new_s"])
        b[nq]["hidden_upload_share"] = round(max(0.0, min(1.0, (upload + scan - t_a) / min(upload, scan))), 3)
        log(f"B nq={nq}: {b[nq]}")
    del dev
    torch.cuda.empty_cache()
    report["A_host"] = a
    report["B_device"] = b

    # C: more rows than HBM
    free, total = torch.cuda.mem_get_info()
    big_gb = args.big * D * 4 / 1e9
    c = {"rows": args.big, "dataset_gb": round(big_gb, 1), "hbm_total_gb": round(total / 1e9, 1)}
    if not args.big:
        c["result"] = "not measured"
    elif host_memory_gb() * 2**30 / 1e9 + gb < big_gb + 8:  # the first dataset is freed before this one is made
        c["result"] = "not measured: the host has too little memory for the dataset"
    elif time.perf_counter() - started > args.budget_s:
        c["result"] = "not measured: no time left in this run"
    else:
        del data
        big = rows(args.big, 3)
        t, kb, db, e = run(new, big, qs[1000])
        c.update({"new_s": round(t, 3), "error": e, "upload_gb_per_s_effective": round(big_gb / t, 1)})
        tp, _, _, ep = run(parent, big, qs[1000])
        c["parent"] = ep or f"served in {tp:.3f} s"
        # the plan's chunk count: two buffers of rows over free HBM after about 1.9 GB of fixed needs
        per_row, fixed = 2 * D * 4 + 4, (1 << 30) * 3 // 2 + (512 << 20) + 1000 * (D * 4 + K * 24 + 8)
        c["planned_chunks"] = int(np.ceil(args.big / ((free - fixed) // per_row)))
    report["C_larger_than_hbm"] = c
    print(json.dumps(report))


if __name__ == "__main__":
    main()
