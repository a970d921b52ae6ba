"""The f32, f16, bf16, f64 and b1 exact-search scans at their tile, count, query-count and length edges, under the default
kernel choice and with the one-query-per-warp scan and the tiled scan forced in turn (USEARCH_B200_EXACT is read once per
process, hence one subprocess per choice).

Inputs come from tests/float_exact_reference.edge_cases: duplicates and l2sq mirror pairs on every tile boundary,
one-ulp near ties across one, removed slots on tile edges and a whole removed tile, a short last tile, counts 1 to 700
and past the live rows, 1 to 300 queries, ragged 16-byte tails, lengths on both sides of the tiled and the staged
limits and past them (rows read in place), zero rows and queries, and cosine inputs whose norms differ by orders of
magnitude. Index mode must match the port's exact search (labels, distance bits, counts) and, where the oracle is built,
the pinned reference; the free `exact_search` must match the port's metric(row, query) in distance bits, and in labels
wherever a distance is unique in its row. Every result is also held to the float64 statement of its metric, a batch of
300 queries to its slices, and the forced tiled scan must refuse exactly where its stage ends. One `Indexes.search` and
one `join` (where the oracle is built) go through the same scans on the f32 tie case, at its length and at 4096."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

KERNELS = ["default", "scan", "tiled"]
TOO_LONG_TILED = "Vectors too long for the tiled exact-search stage"
BIG_K = "Exact search with count > 256 needs vectors that fit the tiled stage"


def _refusal(kernel, kind, d, k):
    """the message the forced kernel (or the one it hands over to) refuses this shape with, or None when it serves it"""
    import float_exact_reference as F
    fits = F.tiled_fits(kind, d)
    if k > 256 and not fits:  # lists past 256 live in global memory: the tiled scan only
        return BIG_K
    if kernel == "tiled" and not fits:
        return TOO_LONG_TILED
    return None


def _diff(what, want, got, limit=4):
    wk, wd, wc = want
    gk, gd, gc = got
    lines = []
    if not np.array_equal(np.asarray(wc, np.uint64), np.asarray(gc, np.uint64)):
        lines.append(f"{what}: counts differ in {int((np.asarray(wc, np.uint64) != np.asarray(gc, np.uint64)).sum())} queries")
    bad = np.argwhere((wk != gk) | (wd.view(np.uint32) != gd.view(np.uint32)))
    for q, pos in bad[:limit]:
        lines.append(f"{what}: query {q} position {pos}: key want {int(wk[q, pos])} got {int(gk[q, pos])}, distance bits want "
                     f"0x{int(wd.view(np.uint32)[q, pos]):08x} got 0x{int(gd.view(np.uint32)[q, pos]):08x}")
    if bad.shape[0] > limit:
        lines.append(f"{what}: ... {bad.shape[0]} mismatching positions in all")
    return lines


def _expect_refusal(what, message, call):
    try:
        call()
    except RuntimeError as e:
        return [] if message in str(e) else [f"{what}: refused with {str(e)!r}, want {message!r}"]
    return [f"{what}: served, want the refusal {message!r}"]


def _index_mode(kernel, case, metric, live):
    import float_exact_reference as F
    from oracle import bindings
    from usearch_b200.index import Index
    kind, rows, queries, d = case["kind"], case["rows"], case["queries"], case["d"]
    n = rows.shape[0]
    removed = np.zeros(n, bool)
    removed[list(case["removed"])] = True
    image = F.blob(kind, rows, metric, d)
    index = Index.restore(image)
    if case["removed"]:
        assert index.remove(np.array(case["removed"], np.uint64)) == len(case["removed"])
    ref = None
    if live and kind != "f64":
        ref = bindings.RefIndex("parity")
        ref.load(image)
        for slot in case["removed"]:
            ref.remove(int(slot))
        ref.pin_metric(True)
    matrix = F.pinned_matrix(kind, metric, rows, queries, d)
    report = []
    full = {}
    for k in case["ks"]:
        what = f"{kind} {case['name']} {metric} k={k} [{kernel}] index"
        refusal = _refusal(kernel, kind, d, k)
        if refusal:
            report += _expect_refusal(what, refusal, lambda: index.search(queries, k, exact=True))
            continue
        got = index.search(queries, k, exact=True)
        got = (got.keys, got.distances, got.counts)
        full[k] = got
        report += _diff(what + " vs port", F.top_k(matrix, k, removed), got)
        report += [f"{what} vs float64: {p}" for p in F.check_topk(kind, metric, rows, queries, d, k, *got, removed=removed)[:3]]
        if ref is not None:
            report += _diff(what + " vs reference", ref.search(queries, k, threads=8, exact=True, counters=False)[:3], got)
    if case["batches"]:  # the segment count follows the batch size: every slice must give the rows of the full batch
        for k, got in full.items():
            slices = [(0, m) for m in (1, F.qt(kind) - 1, F.qt(kind) + 1, 7, 9, F.qpc(kind) - 1, F.qpc(kind) + 1)]
            slices += [(i, i + 1) for i in range(1, queries.shape[0], 37)]
            for lo, hi in slices:
                part = index.search(queries[lo:hi], k, exact=True)
                report += _diff(f"{kind} {case['name']} {metric} k={k} [{kernel}] queries {lo}:{hi} vs the full batch",
                                tuple(x[lo:hi] for x in got), (part.keys, part.distances, part.counts))
    return report


def _free_mode(kernel, case, metric):
    import float_exact_reference as F
    from usearch_b200.index import exact_search
    kind, rows, queries, d = case["kind"], case["rows"], case["queries"], case["d"]
    n = rows.shape[0]
    matrix = F.pinned_matrix(kind, metric, rows, queries, d, swap=True)
    report = []
    for k in case["ks"]:
        if k > n:
            continue
        what = f"{kind} {case['name']} {metric} k={k} [{kernel}] free"
        refusal = _refusal(kernel, kind, d, k)
        if refusal:
            report += _expect_refusal(what, refusal, lambda: exact_search(rows, queries, k, metric=metric, dtype=kind))
            continue
        got = exact_search(rows, queries, k, metric=metric, dtype=kind)
        fk, fd, _ = F.top_k(matrix, min(k + 1, n))
        if not np.array_equal(got.distances.view(np.uint32), fd[:, :k].view(np.uint32)):
            report += _diff(what + " vs port", (fk[:, :k], fd[:, :k], np.full(len(queries), k)),
                            (got.keys, got.distances, np.full(len(queries), k)))
        u = F.unique_mask(fd, k)
        if not np.array_equal(got.keys[u], fk[:, :k][u]):
            report.append(f"{what}: labels of unique distances differ in {int((got.keys[u] != fk[:, :k][u]).sum())} places")
        report += [f"{what} vs float64: {p}" for p in F.check_topk(kind, metric, rows, queries, d, k, got.keys, got.distances,
                                                                     np.full(len(queries), k))[:3]]
    return report


def _other_callers(kernel, live):
    """Indexes.search(exact=True) against the merge model over the port's per-shard results, and join(exact=True) against
    the reference's join where the oracle is built: the f32 tie case, and the same rows widened to 4096 dims"""
    import float_exact_reference as F
    import indexes_reference as ir
    import join_reference as jr
    from usearch_b200.index import Index, Indexes
    case = next(c for c in F.edge_cases("f32", big=False) if c["name"] == "tiles")
    rows, queries = case["rows"].astype(np.float64), case["queries"].astype(np.float64)
    report = []
    for d in (case["d"], 4096):
        wide = lambda x: np.ascontiguousarray(np.pad(x, ((0, 0), (0, d - x.shape[1]))), np.float32)  # noqa: E731
        r, q = wide(rows), wide(queries)
        shards = [r[:400], np.vstack([r[300:], r[:50]])]  # rows 0-49 and 300-399 in both shards: ties across shards
        for metric in ("l2sq", "cos"):
            group = Indexes([Index.restore(F.blob("f32", s, metric, d)) for s in shards])
            for k in (1, 33, 257):
                what = f"Indexes d={d} {metric} k={k} [{kernel}]"
                if _refusal(kernel, "f32", d, k):
                    continue
                per = [F.top_k(F.pinned_matrix("f32", metric, s, q, d), k) for s in shards]
                want = ir.merge_model(np.stack([p[0] for p in per]), np.stack([p[1] for p in per]),
                                      np.stack([p[2] for p in per]), k)
                got = group.search(q, k, exact=True)
                report += _diff(what, want, (got.keys, got.distances, got.counts))
        if live and _refusal(kernel, "f32", d, 1) is None:
            a = Index.restore(F.blob("f32", np.ascontiguousarray(q[:5]), "l2sq", d))
            b = Index.restore(F.blob("f32", np.ascontiguousarray(r[:300]), "l2sq", d))
            want, want_stats = jr.reference_join(a.save(), b.save(), 0, max(a.expansion_search, b.expansion_search), True)
            got = a.join(b, exact=True)
            if got != want or a.last_join_stats != want_stats:
                report.append(f"join(exact=True) d={d} [{kernel}]: {sum(got.get(x) != y for x, y in want.items())} pairs "
                              f"differ of {len(want)}, stats {a.last_join_stats} want {want_stats}")
    return report


def run_kernel(kernel: str) -> list:
    """every edge case under the forced kernel; returns the mismatch report (empty when all agree)"""
    for p in (ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    import common
    import float_exact_reference as F
    live = common.have_reference()
    report = []
    for kind in F.KINDS:
        for case in F.edge_cases(kind):
            for metric in case["metrics"]:
                if case["index"]:
                    report += _index_mode(kernel, case, metric, live)
                if case["free"]:
                    report += _free_mode(kernel, case, metric)
    return report + _other_callers(kernel, live)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", KERNELS)
def test_float_exact_scan_at_the_edges(kernel):
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_exact_float_edges as t\n"
            "report = t.run_kernel(%r)\n"
            "print('\\n'.join(report[:80]))\n"
            "print('FLOAT_EDGES_OK' if not report else 'FLOAT_EDGES_FAILED %%d' %% len(report))\n") % (ROOT, HERE, kernel)
    env = dict(os.environ)
    env.pop("USEARCH_B200_EXACT", None)
    if kernel != "default":
        env["USEARCH_B200_EXACT"] = kernel
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert out.returncode == 0 and "FLOAT_EDGES_OK" in out.stdout, out.stdout[-8000:] + out.stderr[-3000:]
