"""f64 indexes on the GPU against tests/golden/f64_cases.npz, the reference's own results on f64 graphs it built
(tests/golden/make_golden_f64.py). The fixture's graphs are rebuilt from their seeds and checked against the SHA-256 of
the reference's files. Graphs that only exist here (built, edited or joined on the GPU) are held against the port of the
reference's search with the f64 pinned metric (tests/native/port_f64.c), which tests/test_f64_oracle.py holds equal to
the fixture and to the live reference."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

import common
import f64_reference as fr

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(common.ROOT, "tools"))
from build_check import structure_report  # noqa: E402

PLAN_ERROR = "Expansion or dimensionality too large for on-chip state"
CASES = ["cos_d768", "l2sq_d97", "ip_d24", "l2sq_d3200"]
KNOBS = {
    "default": {},
    "stage_sets=1": {"stage_sets": 1},
    "stage_sets=2": {"stage_sets": 2},
    "warps_per_sm=1": {"warps_per_sm": 1},
    "warps_per_sm=2": {"warps_per_sm": 2},
    "heap_head=2": {"heap_head": 2},
    "heap_head=16": {"heap_head": 16},
    "heap_head=64": {"heap_head": 64},
    "stage_sets=2,heap_head=2": {"stage_sets": 2, "heap_head": 2},
}
DEFAULT_KNOBS = {"stage_sets": 0, "warps_per_sm": 0, "prefilter": 1, "heap_head": 0}


@pytest.fixture(scope="module")
def fx():
    return fr.load_fixture()


def _restore(fx, name):
    from usearch_b200.index import Index
    blob, base = fr.case_blob(fx, name)
    return Index.restore(blob), base, fr.case_queries(fx, name)


def _want(fx, prefix):
    return tuple(fx[f"{prefix}/{t}"] for t in ("keys", "distances", "counts", "computed", "visited"))


def _search(index, q, k, allowed=None):
    got = index.search(q, k, stats=True) if allowed is None else index.filtered_search(q, k, allowed)
    return got.keys, got.distances, got.counts, index.last_computed, index.last_visited


def _searches(fx, name):
    out = []
    for key in fx:
        if key.startswith(f"{name}/ef") and key.endswith("_pinned/keys"):
            ef, k = key.split("/")[1].split("_")[:2]
            out.append((int(ef[2:]), int(k[1:])))
    return out


@pytest.mark.parametrize("name", CASES)
def test_graph_search_matches_reference(fx, name):
    index, _, q = _restore(fx, name)
    assert index.dtype == "f64"
    for ef, k in _searches(fx, name):
        index.expansion_search = ef
        common.assert_same_results(_want(fx, f"{name}/ef{ef}_k{k}_pinned"), _search(index, q, k), f"{name} ef {ef} k {k}")
        if k == 10:  # the reference's native SimSIMD f64 kernels: same labels
            assert np.array_equal(_search(index, q, k)[0], fx[f"{name}/ef{ef}_k{k}_native/keys"])


@pytest.mark.parametrize("name", ["cos_d768", "ip_d24"])
@pytest.mark.parametrize("knobs", list(KNOBS))
def test_every_launch_plan(fx, name, knobs):
    index, _, q = _restore(fx, name)
    index.expansion_search = 64
    index.tune(**{**DEFAULT_KNOBS, **KNOBS[knobs]})
    try:
        plan = index.launch_plan(10)
    except RuntimeError as e:  # a forced layout that does not fit: the search refuses it the same way
        assert str(e) == PLAN_ERROR and KNOBS[knobs], f"{name} [{knobs}]: {e}"
        with pytest.raises(RuntimeError, match=re.escape(PLAN_ERROR)):
            index.search(q, 10)
        return
    assert not plan["prefilter"] and plan["code_pass"] == 0, plan  # f64 rows have no int8 shadow
    common.assert_same_results(_want(fx, f"{name}/ef64_k10_pinned"), _search(index, q, 10), f"{name} [{knobs}]")


def test_3208_dims_refused_cleanly(fx):
    """3200 f64 dims (25,600 B rows, the f32 ceiling of 6400 dims) are served above; one 16-byte chunk more is refused"""
    from usearch_b200 import v2format
    from usearch_b200.index import Index
    blob, _ = fr.case_blob(fx, "l2sq_d3200")
    g = v2format.loads(blob)
    g.vectors = np.concatenate([np.asarray(g.vectors).reshape(g.size, -1), np.zeros((g.size, 64), np.uint8)], axis=1)
    g.dimensions = 3208
    index = Index.restore(v2format.dumps(g))
    q = np.zeros((4, 3208))
    with pytest.raises(RuntimeError, match=re.escape(PLAN_ERROR)):
        index.launch_plan(10)
    with pytest.raises(RuntimeError, match=re.escape(PLAN_ERROR)):
        index.search(q, 10)
    assert len(index) == g.size


@pytest.mark.parametrize("name", ["l2sq_d97", "ip_d24"])
def test_filtered_search(fx, name):
    """keys % 3 != 1 allowed; ip_d24 also has removed entries (every third key below 600)"""
    index, _, q = _restore(fx, name)
    index.expansion_search = 64
    allowed = np.arange(int(fx[f"{name}/n"]), dtype=np.uint64)
    allowed = allowed[allowed % 3 != 1]
    common.assert_same_results(_want(fx, f"{name}/filtered_ef64_k10"), _search(index, q, 10, allowed), f"{name} filtered")


def test_f32_queries(fx):
    name = "l2sq_d97"
    index, _, q = _restore(fx, name)
    index.expansion_search = 64
    common.assert_same_results(_want(fx, f"{name}/f32q_ef64_k10"), _search(index, q.astype(np.float32), 10), "f32 queries")


def test_compact_then_reuse(fx):
    """remove(keys, compact=True) leaves the lists the reference's remove + isolate leaves, and searches as it does; then
    adds with reuse_removed fill the removed slots, and the search on the edited file equals the port's"""
    from usearch_b200 import v2format
    name = "ip_d24"
    index, _, q = _restore(fx, name)
    index.expansion_search = 64
    sys.path.insert(0, common.GOLDEN)
    from make_golden_f64 import COMPACT_REMOVED
    index.remove(COMPACT_REMOVED, compact=True)
    blob, _ = fr.case_blob(fx, name)
    want_g = v2format.loads(np.concatenate([blob[: blob.size - fx[f"{name}/graph"].size], fx[f"{name}/compact/graph"]]))
    got_g = v2format.loads(index.save())
    assert got_g.neighbors == want_g.neighbors and np.array_equal(got_g.keys, want_g.keys)
    common.assert_same_results(_want(fx, f"{name}/compact/ef64_k10"), _search(index, q, 10), "after compact")
    index.reuse_removed = True
    fresh = fr.rows(77, 300, int(fx[f"{name}/d"]))
    index.add(np.arange(50_000, 50_300, dtype=np.uint64), fresh)
    saved = index.save()
    removed = 200 + len(COMPACT_REMOVED)
    assert v2format.loads(saved).size == int(fx[f"{name}/n"]) + 300 - removed  # every removed slot was reused
    assert structure_report(saved)["n_problems"] == 0
    port = fr.PortF64(saved, 64)
    common.assert_same_results(port.search(q, 10), _search(index, q, 10), "after reuse")
    common.assert_same_results(port.search(fresh[:32], 10), _search(index, fresh[:32], 10), "after reuse, own rows")


def test_usearch_distance(fx):
    """usearch_distance through the C ABI, metric(a, b) on two caller vectors, equals the pinned metric"""
    from usearch_b200.index import METRIC_KIND, SCALAR_KIND, load_library
    lib = load_library()
    for name in ("cos_d768", "l2sq_d97", "ip_d24"):
        _, base, _ = _restore(fx, name)
        pairs = fx[f"{name}/pairs"][:16]
        err = C.c_char_p()
        got = np.array([lib.usearch_distance(base[i].ctypes.data_as(C.c_void_p), base[j].ctypes.data_as(C.c_void_p),
                                             SCALAR_KIND["f64"], base.shape[1], METRIC_KIND[fx[f"{name}/metric"].item()],
                                             C.byref(err)) for i, j in pairs], dtype=np.float32)
        assert not err.value, err.value
        assert np.array_equal(got.view(np.uint32), fx[f"{name}/pairs_pinned"][:16].view(np.uint32)), name


@pytest.mark.parametrize("name", ["cos_d768", "l2sq_d97", "ip_d24"])
def test_exact_search(fx, name):
    from usearch_b200.index import exact_search
    index, base, q = _restore(fx, name)
    for k in (10, 300):
        if f"{name}/exact_k{k}/keys" not in fx:  # 768-d f64 rows do not fit the tiled stage that counts > 256 need
            with pytest.raises(RuntimeError, match="count > 256"):
                index.search(q, k, exact=True)
            continue
        got = index.search(q, k, exact=True)
        want = _want(fx, f"{name}/exact_k{k}")
        assert np.array_equal(got.keys, want[0]) and np.array_equal(got.counts, want[2])
        assert np.array_equal(got.distances.view(np.uint32), want[1].view(np.uint32))
        free = exact_search(base, q, k, metric=fx[f"{name}/metric"].item())
        wd, wk = fx[f"{name}/free_k{k}/distances"], fx[f"{name}/free_k{k}/keys"]
        assert np.array_equal(free.distances.view(np.uint32), wd.view(np.uint32))
        unique = np.ones_like(wd, dtype=bool)  # std::partial_sort leaves the order of equal distances unspecified
        unique[:, 1:] &= wd[:, 1:] != wd[:, :-1]
        unique[:, :-1] &= wd[:, :-1] != wd[:, 1:]
        assert np.array_equal(free.keys[unique], wk[unique])


@pytest.mark.parametrize("name", ["cos_d768", "l2sq_d97", "ip_d24"])
def test_cluster_every_level(fx, name):
    index, _, q = _restore(fx, name)
    for level in range(int(fx[f"{name}/max_level"]) + 2):
        keys, dist = index.cluster(q, level, stats=True)
        p = f"{name}/cluster_l{level}"
        assert np.array_equal(keys, fx[f"{p}/keys"]), level
        assert np.array_equal(dist.view(np.uint32), fx[f"{p}/distances"].view(np.uint32)), level
        assert np.array_equal(index.last_computed, fx[f"{p}/computed"]) and np.array_equal(index.last_visited, fx[f"{p}/visited"])


@pytest.mark.parametrize("name", ["cos_d768", "l2sq_d97", "ip_d24"])
def test_pairwise_distance(fx, name):
    index, _, _ = _restore(fx, name)
    pairs = fx[f"{name}/pairs"]
    got = index.pairwise_distance(pairs[:, 0].astype(np.uint64), pairs[:, 1].astype(np.uint64))
    assert np.array_equal(got.view(np.uint32), fx[f"{name}/pairs_pinned"].view(np.uint32))


def test_casts_into_and_out_of_f64(fx):
    from usearch_b200.index import Index
    d = 40
    for kind in ("f32", "f16", "i8", "b1"):
        index = Index(ndim=d, metric="l2sq", dtype="f64", connectivity=16)
        rows = fx[f"casts/in_{kind}"]
        index.add(np.arange(len(rows)), rows)
        stored = np.stack([index.get(i, dtype="f64") for i in range(len(rows))])
        assert np.array_equal(stored.view(np.uint64), fx[f"casts/in_{kind}_stored"].view(np.uint64)), kind
    index = Index(ndim=d, metric="l2sq", dtype="f64", connectivity=16)
    doubles = fx["casts/out_rows"]
    index.add(np.arange(len(doubles)), doubles)
    for kind in ("f32", "f16", "i8", "b1"):
        got = np.stack([index.get(i, dtype=kind) for i in range(len(doubles))])
        assert np.array_equal(got.view(np.uint8), fx[f"casts/out_{kind}"].view(np.uint8)), kind


@pytest.mark.parametrize("name", ["cos_d768", "l2sq_d97"])
def test_gpu_built_graph_quality(fx, name):
    """a graph linked on the GPU from the fixture's rows against the reference's graph of the same rows, both searched by
    the reference's search (which the GPU search equals bit for bit on the reference's file, above) with 1024 fresh queries:
    recall@10 at ef 64 at least the reference's minus 0.01, work per query within 8 %, and the saved file serves the same
    results after a reload"""
    from usearch_b200.index import Index
    ref_index, base, _ = _restore(fx, name)
    metric, d, m = fx[f"{name}/metric"].item(), int(fx[f"{name}/d"]), int(fx[f"{name}/m"])
    q = fr.rows(1000 + int(fx[f"{name}/seed"]), 1024, d)
    index = Index(ndim=d, metric=metric, dtype="f64", connectivity=m, expansion_add=128, expansion_search=64)
    index.add(np.arange(len(base)), base)
    got = _search(index, q, 10)
    ref_index.expansion_search = 64
    want = _search(ref_index, q, 10)
    truth = index.search(q, 10, exact=True).keys
    recall = lambda keys: np.mean([len(set(a) & set(b)) / 10 for a, b in zip(keys.tolist(), truth.tolist())])
    assert recall(got[0]) >= recall(want[0]) - 0.01, (recall(got[0]), recall(want[0]))
    assert abs(got[3].mean() - want[3].mean()) <= 0.08 * want[3].mean(), (got[3].mean(), want[3].mean())
    saved = index.save()
    rep = structure_report(saved)
    assert rep["n_problems"] == 0, rep["problems"]
    common.assert_same_results(fr.PortF64(saved, 64).search(q, 10), got, f"{name}: GPU-built graph, port vs GPU")
    again = Index.restore(saved)
    again.expansion_search = 64
    common.assert_same_results(got, _search(again, q, 10), f"{name}: GPU-built graph after save / restore")


@pytest.mark.parametrize("exact", [False, True], ids=["approximate", "exact"])
def test_join(fx, exact):
    """a reference-built graph with removed entries joined with a GPU-built one, against the reference's loop restated over
    the port's proposals and pinned metric (tests/join_reference.py)"""
    from usearch_b200.index import Index
    a, base, _ = _restore(fx, "ip_d24")
    a.expansion_search = 64
    b = Index(ndim=24, metric="ip", dtype="f64", connectivity=8, expansion_add=64, expansion_search=64)
    b.add(np.arange(10_000, 11_500, dtype=np.uint64), base[500:2000] + 0.05 * fr.rows(78, 1500, 24))
    want, want_stats = fr.port_join(a.save(), b.save(), 0, 64, exact)
    got = a.join(b, exact=exact)
    assert got == want, f"{sum(got.get(k) != v for k, v in want.items())} pairs differ of {len(want)}"
    assert a.last_join_stats == want_stats
