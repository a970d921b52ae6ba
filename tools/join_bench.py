"""`Index.join` on one GPU: men are `datagen` rows, women noisy, permuted copies of them, so every man has a true partner.
Both graphs are built on the GPU. One warm-up join, then --repeats timed joins; prints one JSON line with the median wall
clock of the join and of its three phases (`Index.last_join_ms`: proposal searches, pair distances, host replay), the
join's counters and kernel launches, and the share of men matched to their true partner.

--save DIR also writes both graphs and the join to DIR; --reference DIR then runs the reference's own join (`perf`
flavour, native metric, all cores; needs the reference sources, so not on a GPU machine) on those graphs and reports its
wall clock and how far its matching agrees with ours (a multi-threaded reference run depends on timing).

    python tools/join_bench.py [--n 1000000] [--d 768] [--m 32] [--noise 0.05] [--repeats 5] [--save DIR]
    python tools/join_bench.py --reference DIR [--threads 0]
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from churn_check import card  # noqa: E402
from usearch_b200 import datagen  # noqa: E402
from usearch_b200.index import Index  # noqa: E402


def reference_arm(directory, threads):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import join_reference as jr
    from oracle import bindings
    men = np.fromfile(os.path.join(directory, "men.usearch"), dtype=np.uint8)
    women = np.fromfile(os.path.join(directory, "women.usearch"), dtype=np.uint8)
    ours = np.load(os.path.join(directory, "join.npz"))
    mine = dict(zip(ours["a_keys"].tolist(), ours["b_keys"].tolist()))
    threads = threads or int(bindings.ref_lib("perf").ref_hardware_threads())
    jr.live_join(men, women, 1, 64, False, threads=threads, flavour="perf")  # compiles the driver, warms the caches
    t0 = time.perf_counter()
    theirs, stats = jr.live_join(men, women, 0, 64, False, threads=threads, flavour="perf")
    seconds = time.perf_counter() - t0
    same = sum(1 for k, v in mine.items() if theirs.get(k) == v)
    print(json.dumps({"ref_threads": threads, "ref_join_s": round(seconds, 2), **{f"ref_{k}": v for k, v in stats.items()},
                      "pairs_ours": len(mine), "pairs_ref": len(theirs), "same_pairs": same,
                      "agreement": round(same / max(len(mine), 1), 5)}))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_000_000)
    p.add_argument("--d", type=int, default=768)
    p.add_argument("--m", type=int, default=32)
    p.add_argument("--noise", type=float, default=0.05)
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--save", default=None)
    p.add_argument("--reference", default=None)
    p.add_argument("--threads", type=int, default=0)
    p.add_argument("--out", default=None)
    args = p.parse_args()
    if args.reference:
        reference_arm(args.reference, args.threads)
        return

    men_rows = datagen.latent(args.n, args.d, seed=1)
    perm = np.random.default_rng(2).permutation(args.n)
    noise = args.noise * np.random.default_rng(3).standard_normal(men_rows.shape, dtype=np.float32)
    women_rows = np.ascontiguousarray((men_rows + noise)[perm])  # woman j is the copy of man perm[j]
    t0 = time.perf_counter()
    men = Index(ndim=args.d, metric="cos", dtype="f32", connectivity=args.m)
    men.add(None, men_rows)
    women = Index(ndim=args.d, metric="cos", dtype="f32", connectivity=args.m)
    women.add(np.arange(args.n, dtype=np.uint64) + args.n, women_rows)  # woman j has key n + j
    build_s = time.perf_counter() - t0

    men.join(women)  # warm-up
    walls, phases = [], []
    for _ in range(args.repeats):
        launches = men.kernel_launches + women.kernel_launches
        t0 = time.perf_counter()
        pairs = men.join(women)
        walls.append(time.perf_counter() - t0)
        launches = men.kernel_launches + women.kernel_launches - launches
        phases.append(dict(men.last_join_ms))
    truth = {int(perm[j]): args.n + j for j in range(args.n)}
    recovered = sum(1 for a, b in pairs.items() if truth[a] == b) / args.n
    med = lambda xs: float(np.median(xs))
    result = {"card": card(), "n": args.n, "d": args.d, "m": args.m, "noise": args.noise,
              "max_proposals": int(math.log(args.n) + 1), "build_s": round(build_s, 2), "repeats": args.repeats,
              "join_ms": round(1e3 * med(walls), 1), "join_ms_range": [round(1e3 * min(walls), 1), round(1e3 * max(walls), 1)],
              **{f"{k}_ms": round(med([ph[k] for ph in phases]), 1) for k in ("search", "pair_distances", "replay")},
              "launches": launches, **men.last_join_stats, "true_partner_rate": round(recovered, 5)}
    print(json.dumps(result))
    if args.save:
        os.makedirs(args.save, exist_ok=True)
        men.save(os.path.join(args.save, "men.usearch"))
        women.save(os.path.join(args.save, "women.usearch"))
        items = sorted(pairs.items())
        np.savez(os.path.join(args.save, "join.npz"), a_keys=np.array([k for k, _ in items], dtype=np.uint64),
                 b_keys=np.array([v for _, v in items], dtype=np.uint64))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f)


if __name__ == "__main__":
    main()
