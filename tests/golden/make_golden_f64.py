"""Generate tests/golden/f64_cases.npz by RUNNING THE UNMODIFIED REFERENCE on f64 indexes (tests/native/ref_f64_driver.cpp).

Run where the reference sources are:  python tests/golden/make_golden_f64.py
Every graph is built by the reference on one thread (reproducible). Rows and queries come from seeds (tests/f64_reference.py
rebuilds them), so the file holds only the graph part of each saved index, its SHA-256, and what the reference returned:
  * ``<case>/ef<E>_k<K>_{pinned,native}``: search with the metric pinned to tests/native/f64_pinned.h, or the reference's
    own SimSIMD dispatch on the generating host (``isa``); each as keys, distances, counts, computed, visited;
  * ``<case>/exact_k<K>`` (index search, exact=True), ``<case>/free_k<K>`` (exact_search_t over the raw matrices),
    ``<case>/cluster_l<L>``, ``<case>/f32q_...`` (f32 queries), ``<case>/filtered_...`` (keys % 3 != 1), ``<case>/pairs``
    (pinned metric), and ``ip_d24/compact/...``: the graph and a search after removing COMPACT_REMOVED and `isolate`;
  * ``casts/...``: rows of other kinds added to an f64 index, and f64 rows read back with `get` in other kinds.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import f64_reference as fr  # noqa: E402

CASES = [
    # name, metric, seed, n, d, M, nq, removed (every third key from 0), searches (ef, k)
    ("cos_d768", "cos", 1, 1000, 768, 16, 32, 0, [(64, 10), (300, 50)]),
    ("l2sq_d97", "l2sq", 2, 2000, 97, 16, 32, 0, [(64, 10), (300, 50)]),
    ("ip_d24", "ip", 3, 2000, 24, 8, 32, 200, [(64, 10), (300, 50)]),
    ("l2sq_d3200", "l2sq", 4, 300, 3200, 8, 4, 0, [(64, 10)]),
]
COMPACT_REMOVED = np.arange(1000, 1200, 4, dtype=np.uint64)


def put(out, prefix, res):
    for name, v in zip(("keys", "distances", "counts", "computed", "visited"), res):
        out[f"{prefix}/{name}"] = v


def main():
    import hashlib
    out = {"cases": np.array([c[0] for c in CASES])}
    for name, metric, seed, n, d, m, nq, removed, searches in CASES:
        base, queries = fr.rows(seed, n, d), fr.rows(seed + 1, nq, d)
        ref = fr.RefF64(metric, d, connectivity=m, expansion_add=128)
        ref.pin(True)
        assert ref.add(np.arange(n), base, threads=1) == n
        for key in range(0, removed * 3, 3):
            ref.remove(key)
        blob = ref.save()
        graph_at = 8 + n * d * 8
        assert np.array_equal(blob[8:graph_at], base.view(np.uint8).ravel())
        out.update({f"{name}/metric": metric, f"{name}/seed": seed, f"{name}/n": n, f"{name}/d": d, f"{name}/m": m,
                    f"{name}/nq": nq, f"{name}/graph": blob[graph_at:], f"{name}/sha256": hashlib.sha256(blob.tobytes()).hexdigest()})
        for ef, k in searches:
            ref.change_expansion_search(ef)
            put(out, f"{name}/ef{ef}_k{k}_pinned", ref.search(queries, k))
            if k == 10:
                ref.pin(False)
                out["isa"] = ref.isa_name
                put(out, f"{name}/ef{ef}_k{k}_native", ref.search(queries, k))
                ref.pin(True)
        ref.change_expansion_search(64)
        exact_counts = [10, 300] if d <= 128 else [10]
        for k in exact_counts:
            put(out, f"{name}/exact_k{k}", ref.search(queries, k, exact=True))
            out[f"{name}/free_k{k}/keys"], out[f"{name}/free_k{k}/distances"] = fr.exact_search(base, queries, k, metric)
        if name == "l2sq_d97":
            put(out, f"{name}/f32q_ef64_k10", ref.search(queries.astype(np.float32), 10, kind="f32"))
        if name in ("l2sq_d97", "ip_d24"):  # ip_d24 has removed entries
            allowed = np.arange(n, dtype=np.uint64)[np.arange(n) % 3 != 1]
            put(out, f"{name}/filtered_ef64_k10", ref.search(queries, 10, allowed=allowed))
        if d <= 1024:
            top = int(np.frombuffer(blob[graph_at + 64 + 24:graph_at + 64 + 32].tobytes(), dtype=np.uint64)[0])
            out[f"{name}/max_level"] = top
            for level in range(top + 2):
                for tag, v in zip(("keys", "distances", "computed", "visited"), ref.cluster(queries, level)):
                    out[f"{name}/cluster_l{level}/{tag}"] = v
            rng = np.random.default_rng(seed + 7)
            pairs = rng.integers(removed * 3, n, size=(64, 2))
            out[f"{name}/pairs"] = pairs
            out[f"{name}/pairs_pinned"] = np.array([fr.distance(metric, base[i], base[j]) for i, j in pairs], dtype=np.float32)
        if name == "ip_d24":  # more removals, then isolate: what remove(keys, compact=True) must leave
            for key in COMPACT_REMOVED:
                ref.remove(int(key))
            ref.isolate()
            out[f"{name}/compact/graph"] = ref.save()[graph_at:]
            put(out, f"{name}/compact/ef64_k10", ref.search(queries, 10))
        print(f"{name}: blob {blob.size} B, graph {blob.size - graph_at} B")

    # casts into f64 (add) and out of f64 (get), against the reference's cast_gt
    d = 40
    rng = np.random.default_rng(99)
    src = {"f32": rng.standard_normal((6, d)).astype(np.float32), "f16": rng.standard_normal((6, d)).astype(np.float16),
           "i8": rng.integers(-127, 128, size=(6, d), dtype=np.int8), "b1": rng.integers(0, 256, size=(6, d // 8), dtype=np.uint8)}
    for kind, rows in src.items():
        ref = fr.RefF64("l2sq", d)
        ref.add(np.arange(len(rows)), rows, kind=kind)
        out[f"casts/in_{kind}"] = rows
        out[f"casts/in_{kind}_stored"] = np.stack([ref.get(i, "f64") for i in range(len(rows))])
    doubles = rng.standard_normal((6, d))
    doubles[0, :8] = [1e-50, -1e-50, 5e-324, 1e-46, -1e-46, 1e-3, 0.0, -0.0]  # below the f32 subnormals
    doubles[1] *= 1e-100  # zero in f32; its i8 magnitude only exists in f64
    ref = fr.RefF64("l2sq", d)
    ref.add(np.arange(len(doubles)), doubles)
    out["casts/out_rows"] = doubles
    for kind in ("f32", "f16", "i8", "b1"):
        out[f"casts/out_{kind}"] = np.stack([ref.get(i, kind) for i in range(len(doubles))])
    np.savez_compressed(os.path.join(HERE, "f64_cases.npz"), **out)
    print(f"isa {out['isa']}, {os.path.getsize(os.path.join(HERE, 'f64_cases.npz'))} B")


if __name__ == "__main__":
    main()
