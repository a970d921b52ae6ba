"""The four i8 exact-search scans at their numeric and tile edges, each forced in turn (USEARCH_B200_EXACT is read once per
process, hence one subprocess per kernel): wgmma (filtered, count <= 24), mma.sync, dp4a tiled and the one-query-per-warp
scan, against the numpy statement of the metric and the keyed top-k (tests/i8_exact_reference.py, itself pinned to the
live reference by the CPU tests) and, where the oracle is built, the pinned reference itself.

Inputs (i8_exact_reference.edge_cases): a constructed cos tie at distance 0.99996 across the 256-vector tile boundary,
near-orthogonal cos rows tied in bulk across tiles and segments, saturated rows whose sums pass 2^24, zero rows and
queries, duplicates / negated / scaled copies, and ragged shapes around the 128-query and 256-vector tiles with removed
slots at the tile edges. Index mode must match labels, distance bits and counts; the free `exact_search` distance bits,
and labels wherever the distance is unique in its row. One `join(exact=True)` on the tie data runs against
tests/join_reference.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

KERNELS = ["wgmma", "imma", "tiled", "scan"]


def _serves(kernel: str, d: int, k: int) -> bool:
    """whether the forced kernel (or the one it hands over to) takes this shape instead of refusing it"""
    if k > 256:  # lists beyond 256 live in global memory: the tiled kernel only
        return kernel in ("tiled", "scan")
    if kernel == "tiled":
        return d <= 2048  # the tiled stage of 32 queries and 2 x 16 vectors fits in shared memory
    return True


def _diff(what, want, got, limit=6):
    """readable first mismatches: query, position, both keys, both distance bits"""
    wk, wd, wc = want
    gk, gd, gc = got
    lines = []
    if not np.array_equal(np.asarray(wc, np.uint64), np.asarray(gc, np.uint64)):
        rows = np.nonzero(np.asarray(wc, np.uint64) != np.asarray(gc, np.uint64))[0]
        lines.append(f"{what}: counts differ in {rows.size} queries, first {rows[:5].tolist()}")
    bad = np.argwhere((wk != gk) | (wd.view(np.uint32) != gd.view(np.uint32)))
    for q, pos in bad[:limit]:
        lines.append(f"{what}: query {q} position {pos}: key want {int(wk[q, pos])} got {int(gk[q, pos])}, distance bits want "
                     f"0x{int(wd.view(np.uint32)[q, pos]):08x} got 0x{int(gd.view(np.uint32)[q, pos]):08x}")
    if bad.shape[0] > limit:
        lines.append(f"{what}: ... {bad.shape[0]} mismatching positions in all")
    return lines


def run_kernel(kernel: str) -> list:
    """every edge case under the forced kernel; returns the mismatch report (empty when all agree)"""
    sys.path.insert(0, ROOT)
    import common
    import i8_exact_reference as R
    import join_reference as jr
    from oracle import bindings
    from tools.exact_bench import linkless_blob
    from usearch_b200.index import Index, exact_search

    live = common.have_reference()
    report = []
    for case in R.edge_cases():
        rows, queries = case["rows"], case["queries"]
        n, d = rows.shape
        removed = np.zeros(n, bool)
        removed[list(case["removed"])] = True
        for metric in case["metrics"]:
            blob = linkless_blob(rows, metric, "i8", d)
            index = Index.restore(blob)
            if case["removed"]:
                assert index.remove(np.array(case["removed"], np.uint64)) == len(case["removed"])
            ref = None
            if live:
                ref = bindings.RefIndex("parity")
                ref.load(blob)
                for slot in case["removed"]:
                    ref.remove(int(slot))
                ref.pin_metric(True)
            for k in case["ks"]:
                if not _serves(kernel, d, k):
                    continue
                what = f"{case['name']} {metric} k={k} [{kernel}]"
                got = index.search(queries, k, exact=True)
                got = (got.keys, got.distances, got.counts)
                report += _diff(what + " index vs numpy", R.search(metric, rows, queries, k, removed), got)
                if ref is not None:
                    report += _diff(what + " index vs reference", ref.search(queries, k, threads=8, exact=True, counters=False)[:3], got)
                if k > n:
                    continue
                free = exact_search(rows, queries, k, metric=metric, dtype="i8")
                fk, fd, _ = R.search(metric, rows, queries, min(k + 1, n), swap=True)
                if not np.array_equal(free.distances.view(np.uint32), fd[:, :k].view(np.uint32)):
                    report += _diff(what + " free vs numpy", (fk[:, :k], fd[:, :k], np.full(len(queries), k)),
                                    (free.keys, free.distances, np.full(len(queries), k)))
                u = R.unique_mask(fd, k)
                if not np.array_equal(free.keys[u], fk[:, :k][u]):
                    report.append(f"{what} free: labels of unique distances differ in {int((free.keys[u] != fk[:, :k][u]).sum())} places")
    if live:  # the stable-marriage join proposes by exact searches through the same scans
        case = next(c for c in R.edge_cases() if c["name"] == "cos_ties")
        men = np.vstack([R.tie_pair()[0], case["queries"][:40]])
        a = Index.restore(linkless_blob(men, "cos", "i8", R.TIE_D))
        women = case["rows"][:700].copy()
        _, women[0], women[256] = R.tie_pair()  # W at slot 0, C in the second 256-vector tile
        b = Index.restore(linkless_blob(women, "cos", "i8", R.TIE_D))
        want, want_stats = jr.reference_join(a.save(), b.save(), 0, max(a.expansion_search, b.expansion_search), True)
        got = a.join(b, exact=True)
        if got != want or a.last_join_stats != want_stats:
            report.append(f"join(exact=True) [{kernel}]: {sum(got.get(x) != y for x, y in want.items())} pairs differ of {len(want)}, "
                          f"stats {a.last_join_stats} want {want_stats}")
    return report


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", KERNELS)
def test_i8_exact_scan_at_the_edges(kernel):
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_exact_i8_edges as t\n"
            "report = t.run_kernel(%r)\n"
            "print('\\n'.join(report[:60]))\n"
            "print('I8_EDGES_OK' if not report else 'I8_EDGES_FAILED %%d' %% len(report))\n") % (ROOT, HERE, kernel)
    env = dict(os.environ, USEARCH_B200_EXACT=kernel)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "I8_EDGES_OK" in out.stdout, out.stdout[-6000:] + out.stderr[-3000:]
