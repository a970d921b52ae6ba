"""Build one bench workload on the GPU, then time the search kernel under several launch configurations in ONE process.

    python tools/sweep.py --workload NS --configs "base;warps_per_sm=3;stage_sets=1" --steps 6

Prints one JSON line per configuration: kernel ms per launch (CUDA events inside the library), algorithmic GB/s and the
fraction of the measured HBM peak (the roofline figure of bench.py), recall on the first batch, and the launch plan the
configuration got (Index.launch_plan)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", default="C2")
    p.add_argument("--n", type=int)
    p.add_argument("--batch", type=int)
    p.add_argument("--ef", type=int)
    p.add_argument("--configs", default="base")
    p.add_argument("--steps", type=int, default=6)
    p.add_argument("--phases", action="store_true", help="also print the kernel's per-phase cycle counters")
    p.add_argument("--ncu", action="store_true", help="cudaProfilerStart/Stop around the LAST step of every configuration (ncu --profile-from-start off)")
    o = p.parse_args()
    import torch
    sys.argv = ["bench.py", "--workload", o.workload] + (["--n", str(o.n)] if o.n else []) + (["--batch", str(o.batch)] if o.batch else []) + \
               (["--ef", str(o.ef)] if o.ef else [])
    a = bench.parse_args()
    device = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    coll = bench.Collection(a, device)
    index, build_s = bench.build_index_gpu(a, coll, 0, 1)
    index.expansion_search = a.ef
    B, k = a.batch, a.k
    total = (o.steps + 2) * B
    q_dev = coll.queries(total)
    bpv = q_dev.stride(0) * q_dev.element_size()
    vs = (bpv + 15) // 16 * 16
    q_bytes = q_dev.view(torch.uint8).reshape(total, bpv)
    if vs != bpv:
        padded = torch.zeros((total, vs), dtype=torch.uint8, device=device)
        padded[:, :bpv] = q_bytes
        q_bytes = padded
    keys = torch.zeros((B, k), dtype=torch.int64, device=device)
    dist = torch.zeros((B, k), dtype=torch.float32, device=device)
    cnt = torch.zeros(B, dtype=torch.int32, device=device)
    comp = torch.zeros(B, dtype=torch.int32, device=device)
    vis = torch.zeros(B, dtype=torch.int32, device=device)
    stream = torch.cuda.Stream(device)
    torch.cuda.synchronize(device)
    torch.cuda.set_stream(stream)
    peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
    R = min(B, 1024)
    gt, _ = bench.exact_topk_gpu(a, coll, q_dev[:R], k)
    gt = gt.cpu().numpy().astype(np.uint64)
    m0 = 2 * index.connectivity
    print(json.dumps({"workload": bench.workload_name(a), "build_s": round(build_s, 1), "hbm_gb": round(index.memory_usage / 1e9, 2)}), flush=True)
    for spec in o.configs.split(";"):
        knobs = {"stage_sets": 0, "warps_per_sm": 0, "prefilter": 1, "heap_head": 0}
        if spec != "base":
            for kv in spec.split(","):
                name, value = kv.split("=")
                knobs[name] = int(value)
        index.tune(**knobs)
        ms, alg = [], []
        rec = None
        if o.phases:
            index.profile_phases(True)
        for s in range(o.steps + 2):
            qs = q_bytes[s * B:(s + 1) * B]
            if o.ncu and s == o.steps + 1:
                torch.cuda.profiler.start()
            index.search_device(qs.data_ptr(), B, vs, k, keys.data_ptr(), dist.data_ptr(), cnt.data_ptr(), comp.data_ptr(), vis.data_ptr(),
                                stream.cuda_stream)
            if o.ncu and s == o.steps + 1:
                torch.cuda.synchronize()
                torch.cuda.profiler.stop()
            if s == 0:
                rec = bench.recall_at_k(keys.cpu().numpy().astype(np.uint64)[:R], cnt.cpu().numpy()[:R], gt)
            if s >= 2:
                ms.append(index.last_kernel_ms)
                alg.append(int(comp.sum(dtype=torch.int64).item()) * index.bytes_per_vector + int(vis.sum(dtype=torch.int64).item()) * (4 + 4 * m0))
        k_ms = float(np.mean(ms))
        gbs = float(np.mean(alg)) / (k_ms * 1e-3) / 1e9
        line = {"config": spec, "kernel_ms": round(k_ms, 3), "qps": round(B / (k_ms * 1e-3)), "alg_gbs": round(gbs, 1), "frac": round(gbs / peak, 4),
                "recall_at_10": round(rec, 4), "plan": index.launch_plan(k)}
        if o.phases:
            ph = index.profile_phases(False)
            line["phases"] = {k2: round(v, 1) for k2, v in ph.items()}
            # bytes the kernel moved per query: the vectors it read, the codes and records of prefiltered candidates, the
            # lists of the hops (the algorithmic figure counts a full row for every computed distance instead)
            d_q, h_q = float(comp.sum(dtype=torch.int64).item()) / B, float(vis.sum(dtype=torch.int64).item()) / B
            line["visited_members_per_query"] = round(h_q, 1)  # hops of the last step: divides the phases into per-hop cycles
            exact = d_q - ph["prefiltered"] + ph["survivors"]
            code = (a.dim + 15) // 16 * 16 + 16
            line["physical_bytes_per_query"] = round(exact * index.bytes_per_vector + ph["prefiltered"] * code + h_q * (4 + 4 * m0))
            line["algorithmic_bytes_per_query"] = round(d_q * index.bytes_per_vector + h_q * (4 + 4 * m0))
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
