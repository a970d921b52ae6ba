"""The numpy statement of i8 exact search (tests/i8_exact_reference.py), which the GPU edge tests take as their oracle,
held bit for bit to the live pinned reference on every edge input: `search(exact=True)` of index_gt::search_exact_ on the
same image (labels, distance bits, counts, removed entries skipped, padding) and exact_search_t over the raw rows
(distance bits; labels wherever the distance is unique in its row)."""
import numpy as np
import pytest

import common
import i8_exact_reference as R
from oracle import bindings

CASES = R.edge_cases(big=False)


def _blob(rows, metric):
    import sys
    sys.path.insert(0, common.ROOT)
    from tools.exact_bench import linkless_blob
    return linkless_blob(rows, metric, "i8", rows.shape[1])


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_numpy_reference_matches_the_pinned_reference(case):
    if not common.have_reference():
        pytest.skip("reference library not built")
    rows, queries = case["rows"], case["queries"]
    n, d = rows.shape
    removed = np.zeros(n, bool)
    removed[list(case["removed"])] = True
    for metric in case["metrics"]:
        ref = bindings.RefIndex("parity")
        ref.load(_blob(rows, metric))
        for slot in case["removed"]:
            assert ref.remove(int(slot)) == 1
        ref.pin_metric(True)
        for k in case["ks"]:
            want = ref.search(queries, k, exact=True, counters=False)
            got = R.search(metric, rows, queries, k, removed)
            common.assert_same_results(want[:3], got, f"{case['name']} {metric} k={k} index")
            if k > n:
                continue
            wk, wd = bindings.ref_exact_search(rows, queries, k, metric=metric, scalar="i8", dims=d, pinned=True)
            fk, fd, _ = R.search(metric, rows, queries, min(k + 1, n), swap=True)
            assert np.array_equal(wd.view(np.uint32), fd[:, :k].view(np.uint32)), f"{case['name']} {metric} k={k} free: distance bits"
            u = R.unique_mask(fd, k)
            assert np.array_equal(wk[u], fk[:, :k][u]), f"{case['name']} {metric} k={k} free: labels"


def test_tie_pair_ties():
    """the constructed pair lies at one cos distance from its query, inside the regime the filter's slack must cover"""
    q, w, c = R.tie_pair()
    ab, a2, b2 = R.triples(q[None], np.stack([w, c]))
    assert ab.tolist() == [[33, 43]] and a2.tolist() == [1016128] and b2.tolist() == [582381, 988848]
    dist = R.distances("cos", ab, a2, b2)
    assert dist[0, 0].view(np.uint32) == dist[0, 1].view(np.uint32)
    assert 0.997 < dist[0, 0] < 1
