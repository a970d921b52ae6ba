"""The layer-0 prefilter of cos / ip f32 (a candidate whose int8-shadow lower bound reaches the radius is dropped without
reading its row) changes nothing observable: labels, distance bits, counts and both counters equal the pinned reference,
and equal the same index searched with the prefilter off. Every case also checks, through the kernel's counters, that
the prefilter ran and rejected candidates."""
import numpy as np
import pytest

import common
from oracle import bindings

pytestmark = pytest.mark.gpu


def _pinned(blob, q, k, ef):
    ref = bindings.RefIndex("parity")
    ref.view(blob)
    ref.pin_metric(True)
    ref.change_expansion_search(ef)
    return ref.search(q, k, threads=16)


def _search(index, q, k, prefilter=1, allowed=None):
    index.tune(prefilter=prefilter)
    index.profile_phases(True)
    got = index.search(q, k, stats=True) if allowed is None else index.filtered_search(q, k, allowed)
    phases = index.profile_phases(False)
    return (got.keys, got.distances, got.counts, index.last_computed, index.last_visited), phases


def _check(index, want, q, k, what, allowed=None):
    on, ph = _search(index, q, k, 1, allowed)
    common.assert_same_results(want, on, f"{what}: prefilter on vs pinned reference")
    assert ph["prefiltered"] > 0, f"{what}: the prefilter never ran"
    assert ph["survivors"] < ph["prefiltered"], f"{what}: the prefilter rejected nothing"
    off, ph_off = _search(index, q, k, 0, allowed)
    assert ph_off["prefiltered"] == 0
    common.assert_same_results(on, off, f"{what}: prefilter on vs off")
    return ph


@pytest.mark.parametrize("metric,n,d,m,ef,k,nq", [
    ("cos", 8000, 768, 32, 128, 10, 256),
    ("ip", 8000, 768, 32, 128, 10, 256),
    ("cos", 6000, 97, 13, 64, 7, 256),   # ragged: 388-byte rows, 112-byte codes
    ("ip", 6000, 97, 16, 64, 10, 256),
])
def test_prefilter_matches_pinned_reference(metric, n, d, m, ef, k, nq):
    from usearch_b200.index import Index
    base, q = common.make_collection(n, d, "f32", nq)
    _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    ph = _check(index, _pinned(blob, q, k, ef), q, k, f"{metric}/{d}")
    assert ph["survivors"] < 0.5 * ph["prefiltered"], ph


@pytest.mark.skipif(not common.have_reference(), reason="oracle/_ref not built")
def test_prefilter_filtered_search_with_removed_keys():
    from usearch_b200.index import Index
    n, d, m, ef, k = 8000, 256, 16, 96, 10
    base, q = common.make_collection(n, d, "f32", 256)
    ref, _ = common.build_reference_blob(base, "cos", "f32", d, m, threads=16, keys=np.arange(n, dtype=np.uint64) * 7 + 3)
    for key in range(3, 3 + 7 * 400, 7 * 4):
        ref.remove(key)
    blob = ref.save()
    ref.pin_metric(True)
    ref.change_expansion_search(ef)
    allowed = np.random.default_rng(5).permutation(n)[: n // 2].astype(np.uint64) * 7 + 3
    want = ref.filtered_search(q, k, allowed, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    _check(index, want, q, k, "filtered", allowed)


@pytest.mark.parametrize("metric", ["cos", "ip"])
def test_prefilter_after_add_many(metric):
    """Members added on the GPU get their shadow as they arrive (and on the capacity regrow): a loaded index grown by
    half again, then searched, equals the reference searching the saved result."""
    from usearch_b200.index import Index
    n0, n1, d, m, ef, k = 5000, 4000, 768, 16, 64, 10
    base, q = common.make_collection(n0 + n1, d, "f32", 256)
    _, blob = common.build_reference_blob(base[:n0], metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.add(np.arange(n0, n0 + n1, dtype=np.uint64), base[n0:])
    index.expansion_search = ef
    saved = index.save()
    # queries that are new members: their own shadow row decides their first hops
    _check(index, _pinned(saved, base[n0:n0 + 256], k, ef), base[n0:n0 + 256], k, f"{metric} grown, member queries")
    _check(index, _pinned(saved, q, k, ef), q, k, f"{metric} grown")


def _near_duplicate_rows(d=256):
    """300 clusters of 20 rows: each centre, a duplicate of it, and 18 copies with every element one ULP up or down; 256
    queries close to random centres."""
    rng = np.random.default_rng(7)
    centres, copies = 300, 20
    c = rng.standard_normal((centres, d), dtype=np.float32)
    base = np.repeat(c, copies, axis=0)
    up = rng.integers(0, 2, size=base.shape).astype(bool)  # every element one ULP up or down
    base = np.nextafter(base, np.where(up, np.inf, -np.inf).astype(np.float32)).astype(np.float32)
    base[::copies] = c  # one exact copy of each centre
    base[1::copies] = c  # and a duplicate of it
    q = (c[rng.integers(0, centres, 256)] + 1e-3 * rng.standard_normal((256, d), dtype=np.float32)).astype(np.float32)
    return base, q


@pytest.mark.parametrize("metric", ["cos", "ip"])
def test_prefilter_near_duplicate_rows(metric):
    """Clusters of rows one or a few ULPs apart (and exact duplicates): distances tie or differ in the last bits, where
    only an exact bound keeps the reference's choices."""
    from usearch_b200.index import Index
    d, m, ef, k = 256, 16, 64, 10
    base, q = _near_duplicate_rows(d)
    _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    _check(index, _pinned(blob, q, k, ef), q, k, f"{metric} near-duplicates")
