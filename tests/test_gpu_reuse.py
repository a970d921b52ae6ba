"""Removal with `compact=True` (isolate) and slot reuse on add, against the reference on one GPU.

The reference always reuses removed slots (index_dense_gt::add_ pops its `free_keys_` ring); with `threads=1` its order
is fixed, so the slot -> key map and the levels of reused slots must match ours exactly. Its `isolate()` erases every link
to a removed entry; the lists it leaves are restated here from its saved file (every link to a free-key slot dropped)."""
import os
import sys

import numpy as np
import pytest

import common
from oracle import bindings
from usearch_b200 import v2format

sys.path.insert(0, os.path.join(common.ROOT, "tools"))
from build_check import structure_report  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = [
    ("cos", "f32", 4000, 96, 16),
    ("l2sq", "f32", 3000, 128, 16),
    ("cos", "f16", 3000, 256, 16),
    ("ip", "i8", 3000, 256, 16),
    ("hamming", "b1", 4000, 256, 32),
    ("cos", "f32", 3000, 768, 32),
]
IDS = [f"{m}-{s}-{d}" for m, s, _, d, _ in CASES]
EF, K = 64, 10


def _isolated(blob):
    """index_gt::isolate over a saved file: lists without links to removed slots, and the number of links erased."""
    g = v2format.loads(blob)
    gone = g.keys == v2format.FREE_KEY
    pruned = 0
    lists = []
    for per_slot in g.neighbors:
        kept = []
        for lst in per_slot:
            keep = [t for t in lst if not gone[t]]
            pruned += len(lst) - len(keep)
            kept.append(keep)
        lists.append(kept)
    return lists, pruned


def _pinned_search(blob, queries, allowed=None):
    ref = bindings.RefIndex("parity")
    ref.load(blob)
    ref.pin_metric(True)
    ref.change_expansion_search(EF)
    if allowed is not None:
        return ref.filtered_search(queries, K, allowed, threads=16)
    return ref.search(queries, K, threads=16)


def _assert_search_parity(index, queries, what, filtered=True):
    """our graph search (plain and filtered) == the pinned reference's over our own saved file, bit for bit"""
    blob = index.save()
    index.expansion_search = EF
    mine = index.search(queries, K, stats=True)
    common.assert_same_results(_pinned_search(blob, queries),
                               (mine.keys, mine.distances, mine.counts, index.last_computed, index.last_visited), what)
    if filtered and index.dtype == "f32":
        live = v2format.loads(blob).keys
        live = live[live != v2format.FREE_KEY]
        allowed = np.random.default_rng(3).permutation(live)[: len(live) // 2]
        got = index.filtered_search(queries, K, allowed)
        common.assert_same_results(_pinned_search(blob, queries, allowed),
                                   (got.keys, got.distances, got.counts, index.last_computed, index.last_visited),
                                   what + " filtered")


def _fresh(n, d, scalar, seed):
    return common.make_collection(n, d, scalar, 1, seed=seed)[0]


@pytest.mark.parametrize("metric,scalar,n,d,m", CASES, ids=IDS)
def test_remove_compact_matches_reference_isolate(metric, scalar, n, d, m):
    from usearch_b200.index import Index
    base, queries = common.make_collection(n, d, scalar, 200)
    ref, blob = common.build_reference_blob(base, metric, scalar, d, m, threads=16)
    g = v2format.loads(blob)
    rng = np.random.default_rng(11)
    victims = rng.choice(g.keys, n * 15 // 100, replace=False)
    victims = np.unique(np.append(victims, g.keys[g.entry_slot]))
    rng.shuffle(victims)
    for key in victims:
        assert ref.remove(int(key)) == 1
    want_lists, want_pruned = _isolated(ref.save())
    index = Index.restore(blob)
    assert index.remove(victims, compact=True) == len(victims)
    assert index.last_pruned_edges == want_pruned > 0
    ours = v2format.loads(index.save())
    assert ours.neighbors == want_lists
    assert len(index) == n - len(victims) and not index.contains(victims).any()
    _assert_search_parity(index, queries, f"isolated {metric}/{scalar}")
    ref.pin_metric(True)
    want = ref.search(queries, K, threads=16, exact=True)
    got = index.search(queries, K, exact=True)
    common.assert_same_results(want[:3], (got.keys, got.distances, got.counts), "exact after remove")


@pytest.mark.parametrize("metric,scalar,n,d,m", CASES, ids=IDS)
def test_reused_slots_match_reference_and_churned_graph_holds_up(metric, scalar, n, d, m):
    """Slot assignment (also after save -> load), exact search after churn, and graph quality after three rounds."""
    from usearch_b200.index import Index
    base, queries = common.make_collection(n, d, scalar, 200)
    ref, blob = common.build_reference_blob(base, metric, scalar, d, m, threads=16)
    index = Index.restore(blob)
    index.reuse_removed = True
    rng = np.random.default_rng(5)
    next_key = 10**9
    for rnd in range(3):
        live = v2format.loads(ref.save()).keys
        live = live[live != v2format.FREE_KEY]
        order = rng.permutation(live)[: len(live) // 10]
        for key in order:
            ref.remove(int(key))
        assert index.remove(order) == len(order)
        if rnd == 1:  # a load rebuilds the queue in ascending slot order, as the reference's reindex does
            ref_blob = ref.save()
            ref = bindings.RefIndex("parity")
            ref.load(ref_blob)
            index = Index.restore(index.save())
            index.reuse_removed = True
        capacity = index.capacity
        fresh_n = len(order) + (0 if rnd == 0 else 25)  # N == R keeps the capacity, N > R appends the rest
        fresh = _fresh(fresh_n, d, scalar, 100 + rnd)
        keys = np.arange(next_key, next_key + fresh_n, dtype=np.uint64)
        next_key += fresh_n
        ref.add(keys, fresh, threads=1)
        index.add(keys, fresh)
        if rnd == 0:
            assert index.capacity == capacity
        gr, go = v2format.loads(ref.save()), v2format.loads(index.save())
        assert np.array_equal(gr.keys, go.keys), f"round {rnd}: slot -> key maps differ"
        assert np.array_equal(gr.levels[:n], go.levels[:n])  # appended slots draw their levels independently
        assert len(index) == ref.size
        assert index.contains(keys).all() and (index.count(keys) == 1).all()
        assert not index.contains(order).any()
        assert np.array_equal(index.get(int(keys[0])), fresh[0])
    # exact search: same slots, same rows -> same answers and tie order
    ref.pin_metric(True)
    want_exact = ref.search(queries, K, threads=16, exact=True)
    got = index.search(queries, K, exact=True)
    common.assert_same_results(want_exact[:3], (got.keys, got.distances, got.counts), "exact after churn")
    # graph quality: the reference's search over our file against its own churned file
    ours = index.save()
    rep = structure_report(ours)
    assert rep["n_problems"] == 0, rep["problems"]
    truth = want_exact[0]
    stats = {}
    for label, b in (("ref", ref.save()), ("gpu", ours)):
        s = bindings.RefIndex("parity")
        s.load(b)
        s.change_expansion_search(EF)
        found, _, _, comp, _ = s.search(queries, K, threads=16)
        stats[label] = (np.mean([len(set(f) & set(t)) / K for f, t in zip(found.tolist(), truth.tolist())]), comp.mean())
    assert stats["gpu"][0] >= stats["ref"][0] - 0.01, stats
    assert abs(stats["gpu"][1] - stats["ref"][1]) <= 0.08 * stats["ref"][1], stats
    _assert_search_parity(index, queries, f"churned {metric}/{scalar}")


def test_entry_point_slot_is_reused_and_rebuilt():
    from usearch_b200.index import Index
    n, d, m = 3000, 96, 16
    base, queries = common.make_collection(n, d, "f32", 200)
    _, blob = common.build_reference_blob(base, "cos", "f32", d, m, threads=16)
    g = v2format.loads(blob)
    entry, top = g.entry_slot, int(g.max_level)
    index = Index.restore(blob)
    index.reuse_removed = True
    assert index.remove(int(g.keys[entry])) == 1
    fresh = _fresh(1, d, "f32", 77)
    index.add(123456789, fresh[0])
    go = v2format.loads(index.save())
    assert go.size == n and go.keys[entry] == 123456789 and go.entry_slot == entry and go.max_level == top
    assert go.levels[entry] == top
    for level in range(top + 1):  # every row rebuilt by the INSERT search, which keeps the slot out of its own results
        assert entry not in go.neighbors[entry][level]
        assert len(go.neighbors[entry][level]) > 0 or not g.neighbors[entry][level]
    rep = structure_report(index.save())
    assert rep["n_problems"] == 0, rep["problems"]
    _assert_search_parity(index, queries, "entry reused")
    res = index.search(fresh, 1)
    assert int(res.keys[0, 0]) == 123456789


def test_prefilter_on_reused_rows():
    from usearch_b200.index import Index
    n, d, m = 4000, 768, 32
    base, queries = common.make_collection(n, d, "f32", 200)
    for metric in ("cos", "ip"):
        _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
        index = Index.restore(blob)
        index.reuse_removed = True
        victims = np.random.default_rng(2).choice(n, n // 5, replace=False).astype(np.uint64)
        index.remove(victims)
        index.add(np.arange(10**6, 10**6 + n // 5, dtype=np.uint64), _fresh(n // 5, d, "f32", 9))
        index.expansion_search = EF
        runs = []
        for pf in (1, 0):
            index.tune(prefilter=pf)
            r = index.search(queries, K, stats=True)
            runs.append((r.keys, r.distances, r.counts, index.last_computed, index.last_visited))
        common.assert_same_results(runs[0], runs[1], f"{metric} prefilter on/off")
        common.assert_same_results(_pinned_search(index.save(), queries), runs[0], f"{metric} reused rows")


def test_multi_index_reuse():
    from usearch_b200.index import Index
    n, d, m = 3000, 64, 16
    base, queries = common.make_collection(n, d, "f32", 200)
    keys = (np.arange(n) // 3).astype(np.uint64)  # three entries per key
    index = Index(ndim=d, metric="l2sq", dtype="f32", connectivity=m, multi=True)
    index.add(keys, base)
    assert index.count(5) == 3
    assert index.remove([5, 6]) == 6 and index.count(5) == 0
    index.reuse_removed = True
    capacity = index.capacity
    index.add(np.full(4, 99999, dtype=np.uint64), _fresh(4, d, "f32", 8))
    assert index.capacity == capacity and index.count(99999) == 4 and len(index) == n - 2
    rep = structure_report(index.save())
    assert rep["n_problems"] == 0, rep["problems"]
    _assert_search_parity(index, queries, "multi reuse")


def test_reuse_off_appends_and_reuse_on_without_removals_is_identical():
    from usearch_b200.index import Index
    n, d, m = 3000, 128, 16
    base, _ = common.make_collection(n, d, "f32", 1)
    fresh = _fresh(300, d, "f32", 31)
    _, blob = common.build_reference_blob(base, "cos", "f32", d, m, threads=16)
    index = Index.restore(blob)
    assert not index.reuse_removed
    index.remove(np.arange(100, dtype=np.uint64))
    capacity = index.capacity
    index.add(np.arange(10**6, 10**6 + 300, dtype=np.uint64), fresh)
    go = v2format.loads(index.save())
    assert np.array_equal(go.keys[n:], np.arange(10**6, 10**6 + 300, dtype=np.uint64))
    assert (go.keys[:n] == v2format.FREE_KEY).sum() == 100 and index.capacity > capacity
    blobs = []
    for reuse in (False, True):
        built = Index(ndim=d, metric="cos", dtype="f32", connectivity=m)
        built.reuse_removed = reuse
        built.add(np.arange(n, dtype=np.uint64), base)
        built.add(np.arange(n, n + 300, dtype=np.uint64), fresh)
        blobs.append(built.save())
    assert np.array_equal(blobs[0], blobs[1])
