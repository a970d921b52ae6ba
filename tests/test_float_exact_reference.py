"""tests/float_exact_reference.py held to its claims without a GPU: the planted ties tie and the near ties are one ulp
apart under the pinned metric, no case yields a NaN, the cosine scale case makes metric(row, query) round differently
from metric(query, row), the float64 statement brackets every pinned distance, and the port's distance matrix ordered
by the keyed top-k is the port's own exact search, and the pinned reference's where the oracle is built."""
import numpy as np
import pytest

import common
import float_exact_reference as F
from oracle import bindings

CASES = [(kind, case) for kind in F.KINDS for case in F.edge_cases(kind, big=False)]


def test_stage_limits():
    """the planner's stage limits: the tiled stage (QPC queries, 2 x TV rows), the staged scan (8 queries, 2 x 32 / LPV)"""
    got = {kind: (F.limit(F.tiled_fits, kind), F.limit(F.staged_fits, kind)) for kind in F.KINDS}
    assert got == {"f32": (896, 2400), "f16": (896, 1600), "bf16": (896, 1600), "f64": (448, 1200), "b1": (19072, 46080)}


@pytest.mark.parametrize("kind,case", CASES, ids=[f"{k}-{c['name']}" for k, c in CASES])
def test_case_holds_its_claims(kind, case):
    rows, queries, d = case["rows"], case["queries"], case["d"]
    n, tv = rows.shape[0], F.tile_rows(kind)
    for metric in case["metrics"]:
        what = f"{kind} {case['name']} {metric}"
        fwd = F.pinned_matrix(kind, metric, rows, queries, d)
        sw = F.pinned_matrix(kind, metric, rows, queries, d, swap=True)
        assert not np.isnan(fwd).any() and not np.isnan(sw).any(), f"{what}: NaN distance"
        dist, bound = F.statement(kind, metric, rows, queries, d)
        for m, order in ((fwd, "metric(query, row)"), (sw, "metric(row, query)")):
            off = np.abs(m.astype(np.float64) - dist) > bound
            assert not off.any(), f"{what}: {order} outside the float64 bound at {np.argwhere(off)[:3].tolist()}"
        if case["name"] in ("tiles", "segments"):  # duplicates (and l2sq mirror pairs) across every tile boundary
            b = np.arange(tv, n, tv)
            dup = (rows[b - 1] == rows[b]).all(axis=1)
            assert dup.any()
            assert np.array_equal(fwd[:, b[dup] - 1].view(np.uint32), fwd[:, b[dup]].view(np.uint32)), what
            if metric == "l2sq" and case["name"] == "tiles" and kind != "b1":  # the others are q0 +- delta
                assert (~dup).any() and np.array_equal(fwd[0, b - 1].view(np.uint32), fwd[0, b].view(np.uint32)), what
        if case["name"].startswith("near_tie"):
            a, c = fwd[0, tv - 1], fwd[0, tv]
            assert c.view(np.uint32) == np.nextafter(a, np.float32(np.inf)).view(np.uint32), f"{what}: not one ulp apart"
            p = F.port(kind, F.blob(kind, rows, metric, d))
            q0 = queries[0]
            assert np.float32(p.distance(q0, rows[tv])) == np.nextafter(np.float32(p.distance(q0, rows[tv - 1])), np.float32(np.inf))
        if case["name"] == "swap_scales":  # rows 0 .. 8 x nq - 1 are scaled copies; most clamp to 0 either way
            par = np.arange(8 * queries.shape[0])
            diff = fwd[par % queries.shape[0], par].view(np.uint32) != sw[par % queries.shape[0], par].view(np.uint32)
            assert diff.mean() > 0.15, f"{what}: the swapped order changes only {diff.mean():.3f} of the parallel pairs"
        removed = np.zeros(n, bool)
        removed[list(case["removed"])] = True
        for k in case["ks"]:
            want = F.top_k(fwd, k, removed)
            assert not F.check_topk(kind, metric, rows, queries, d, k, *want, removed=removed), f"{what} k={k}"
        if not case["removed"] and n <= 800:  # the keyed top-k of the matrix is the port's own exact search
            k = min(n, 257)
            got = F.port(kind, F.blob(kind, rows, metric, d)).search(queries, k, exact=True)
            common.assert_same_results(F.top_k(fwd, k), got[:3], f"{what} port exact search")


LIVE = [(kind, case) for kind, case in CASES if case["rows"].shape[0] <= 800]


@pytest.mark.parametrize("kind,case", LIVE, ids=[f"{k}-{c['name']}" for k, c in LIVE])
def test_case_against_the_pinned_reference(kind, case):
    """index mode with removals against index_gt::search_exact_, the free order against exact_search_t"""
    if not common.have_reference():
        pytest.skip("reference library not built")
    rows, queries, d = case["rows"], case["queries"], case["d"]
    n = rows.shape[0]
    removed = np.zeros(n, bool)
    removed[list(case["removed"])] = True
    for metric in case["metrics"]:
        fwd = F.pinned_matrix(kind, metric, rows, queries, d)
        sw = F.pinned_matrix(kind, metric, rows, queries, d, swap=True)
        for k in case["ks"][:4]:
            if kind == "f64":
                import f64_reference
                if not f64_reference.available():
                    pytest.skip("reference sources absent")
                wk, wd = f64_reference.exact_search(rows, queries, min(k, n), metric)
            else:
                ref = bindings.RefIndex("parity")
                ref.load(F.blob(kind, rows, metric, d))
                for slot in case["removed"]:
                    assert ref.remove(int(slot)) == 1
                ref.pin_metric(True)
                got = ref.search(queries, k, exact=True, counters=False)
                common.assert_same_results(F.top_k(fwd, k, removed), got[:3], f"{kind} {case['name']} {metric} k={k} index")
                if k > n:
                    continue
                wk, wd = bindings.ref_exact_search(rows, queries, k, metric=metric, scalar=kind, dims=F.dims_of(kind, rows),
                                                   pinned=True)
            k = min(k, n)
            fk, fd, _ = F.top_k(sw, min(k + 1, n))
            assert np.array_equal(wd.view(np.uint32), fd[:, :k].view(np.uint32)), f"{kind} {case['name']} {metric} k={k} free"
            u = F.unique_mask(fd, k)
            assert np.array_equal(wk[u], fk[:, :k][u]), f"{kind} {case['name']} {metric} k={k} free labels"
