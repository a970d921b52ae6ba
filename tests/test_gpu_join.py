"""`Index.join` and `Index.pairwise_distance` on one GPU against the reference, bit for bit.

Graphs the reference builds deterministically are joined against the results of the reference's own
`index_dense_gt::join` (one thread, pinned metric) recorded by tests/golden/make_golden_join.py. Graphs that only exist
here (edited or built on the GPU) are joined against the reference's loop restated over the reference's own proposal
searches and pinned metric (tests/join_reference.py), which the CPU tests hold equal to the reference's join."""
import functools
import hashlib
import os
import sys

import numpy as np
import pytest

import common
import join_reference as jr
from oracle import bindings
from usearch_b200 import datagen, v2format
from usearch_b200.index import Index

pytestmark = pytest.mark.gpu

sys.path.insert(0, common.GOLDEN)
import make_golden_join as golden  # noqa: E402

GOLDEN = np.load(os.path.join(common.GOLDEN, "join_cases.npz"))


@functools.lru_cache(maxsize=1)
def _golden_cases():
    """rebuilt with the reference (pinned metric, one thread): the same files, checked by hash"""
    return golden.cases()


def _sha(blob):
    return hashlib.sha256(np.ascontiguousarray(blob, dtype=np.uint8).tobytes()).hexdigest()


@pytest.mark.parametrize("name", sorted({f.split("/")[0] for f in GOLDEN.files}))
def test_join_matches_reference_join(name):
    a_blob, b_blob, max_p, ef, exact = _golden_cases()[name]
    assert [_sha(a_blob), _sha(b_blob)] == GOLDEN[f"{name}/sha"].tolist(), "the reference rebuilt different graphs"
    ia, ib = _load(a_blob, ef), _load(b_blob, ef)
    got = ia.join(ib, max_proposals=max_p, exact=exact)
    want = dict(zip(GOLDEN[f"{name}/a_keys"].tolist(), GOLDEN[f"{name}/b_keys"].tolist()))
    assert got == want, f"{sum(got.get(k) != v for k, v in want.items())} pairs differ of {len(want)}"
    stats = GOLDEN[f"{name}/stats"].tolist()
    assert [ia.last_join_stats[k] for k in ("intersection_size", "engagements", "visited_members", "computed_distances")] == stats
    if name == "p_above_expansion":  # the reference went past the one batched search, so this join did too
        assert int(GOLDEN[f"{name}/deepest"][0]) > ef
    if name == "removed":
        free = int(v2format.FREE_KEY)
        assert free in got or free in got.values()
    if name.startswith("cos-f32-768-approx"):  # the prefilter gives the same bits when it is off
        ib.tune(prefilter=0)
        ia.tune(prefilter=0)
        assert ia.join(ib, max_proposals=max_p, exact=exact) == got



def _rows(n, d, scalar, seed, base=None, noise=0.05):
    if base is None:
        x = datagen.latent(n, d, seed=seed, rank=min(16, d))
    else:
        x = base[np.random.default_rng(seed).permutation(len(base))[:n]]
        x = x + noise * np.random.default_rng(seed + 1).standard_normal(x.shape).astype(np.float32)
    return datagen.to_scalar(np.ascontiguousarray(x, dtype=np.float32), scalar)


def _pair(metric, scalar, d, na, nb, seed=0, keys_b_offset=10_000):
    base = datagen.latent(max(na, nb), d, seed=seed + 100, rank=min(16, d))
    a = _rows(na, d, scalar, seed + 1, base)
    b = _rows(nb, d, scalar, seed + 2, base)
    _, a_blob = common.build_reference_blob(a, metric, scalar, d, 16, 64)
    _, b_blob = common.build_reference_blob(b, metric, scalar, d, 16, 64,
                                            keys=np.arange(nb, dtype=np.uint64) + keys_b_offset)
    return a_blob, b_blob


def _check(ia, ib, max_proposals=0, exact=False, what=""):
    expansion = max(ia.expansion_search, ib.expansion_search)
    want, want_stats = jr.reference_join(ia.save(), ib.save(), max_proposals, expansion, exact)
    got = ia.join(ib, max_proposals=max_proposals, exact=exact)
    assert got == want, f"{what}: {sum(got.get(k) != v for k, v in want.items())} pairs differ of {len(want)}"
    assert ia.last_join_stats == want_stats, what
    return got


def _load(blob, ef=64):
    ix = Index.restore(blob)
    ix.expansion_search = ef
    return ix


@pytest.mark.parametrize("compact", [False, True], ids=["plain", "compact"])
def test_join_with_removed_entries(compact):
    """removals made here, with and without erasing the links to them"""
    a_blob, b_blob = _pair("l2sq", "f32", 97, 300, 360, seed=5)
    ia, ib = _load(a_blob), _load(b_blob)
    ia.remove(np.arange(0, 300, 7, dtype=np.uint64), compact=compact)
    ib.remove(np.arange(10_000, 10_360, 5, dtype=np.uint64), compact=compact)
    got = _check(ia, ib, what="removed")
    free = int(v2format.FREE_KEY)
    # removed women are proposed to and removed men propose: their pairs carry the free key
    assert free in got or free in got.values()


def test_join_multi_index():
    d = 64
    base = datagen.latent(400, d, seed=9, rank=16)
    a = Index(ndim=d, metric="cos", dtype="f32", multi=True)
    a.add(np.arange(300, dtype=np.uint64) // 2, _rows(300, d, "f32", 10, base))
    b = Index(ndim=d, metric="cos", dtype="f32", multi=True)
    b.add(np.arange(350, dtype=np.uint64) // 3 + 1000, _rows(350, d, "f32", 11, base))
    _check(a, b, what="multi")


def test_join_gpu_built_and_prefilter_off():
    d = 768
    base = datagen.latent(600, d, seed=12, rank=16)
    a = Index(ndim=d, metric="cos", dtype="f32", connectivity=16)
    a.add(None, _rows(400, d, "f32", 13, base))
    b = Index(ndim=d, metric="cos", dtype="f32", connectivity=16)
    b.add(np.arange(500, dtype=np.uint64) + 5000, _rows(500, d, "f32", 14, base))
    got = _check(a, b, what="GPU-built")
    stats = dict(a.last_join_stats)
    b.tune(prefilter=0)
    assert a.join(b) == got and a.last_join_stats == stats


def test_pairwise_distance_matches_reference():
    d = 97
    rows = _rows(200, d, "f32", 15)
    for metric in ("cos", "ip", "l2sq"):
        _, blob = common.build_reference_blob(rows, metric, "f32", d, 16, 64)
        ix = _load(blob)
        ref = bindings.RefIndex("parity")
        ref.load(blob)
        ref.pin_metric(True)
        left = np.random.default_rng(1).integers(0, 200, 64).astype(np.uint64)
        right = np.random.default_rng(2).integers(0, 200, 64).astype(np.uint64)
        want = np.array([ref.distance(rows[l], rows[r]) for l, r in zip(left, right)], dtype=np.float32)
        got = ix.pairwise_distance(left, right)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), metric
        one = ix.pairwise_distance(int(left[0]), int(right[0]))
        assert np.float32(one).view(np.uint32) == want[0].view(np.uint32)
        # the batched kernel and usearch_distance give the same bits
        assert np.float32(one).view(np.uint32) == np.float32(_usearch_distance(rows[left[0]], rows[right[0]], metric, d)).view(np.uint32)
        # a missing key: aggregated_distances_t's default
        missing = ix.pairwise_distance(np.array([5, 10_000], dtype=np.uint64), np.array([10_001, 7], dtype=np.uint64))
        assert (missing == np.finfo(np.float32).max).all()


def _usearch_distance(a, b, metric, d):
    import ctypes as C
    from usearch_b200.index import METRIC_KIND, SCALAR_KIND, load_library
    lib = load_library()
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    err = C.c_char_p()
    v = lib.usearch_distance(a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), SCALAR_KIND["f32"], d, METRIC_KIND[metric],
                             C.byref(err))
    assert not err.value
    return v


def test_pairwise_distance_multi_left_key():
    """several vectors under BOTH keys: the minimum over every pair (the reference takes only the first left vector)"""
    d = 64
    rows = _rows(12, d, "f32", 17)
    ix = Index(ndim=d, metric="l2sq", dtype="f32", multi=True)
    ix.add(np.array([0, 0, 0, 1, 1, 1, 1] + list(range(2, 7)), dtype=np.uint64), rows)
    ref = bindings.RefIndex("parity", metric="l2sq", scalar="f32", dims=d)
    ref.pin_metric(True)
    want = min(ref.distance(rows[i], rows[j]) for i in range(0, 3) for j in range(3, 7))
    assert np.float32(ix.pairwise_distance(0, 1)).view(np.uint32) == np.float32(want).view(np.uint32)


def test_pairwise_distance_multi():
    d = 64
    rows = _rows(30, d, "f32", 16)
    ix = Index(ndim=d, metric="l2sq", dtype="f32", multi=True)
    keys = np.array([0] * 1 + [1] * 5 + list(range(2, 26)), dtype=np.uint64)
    ix.add(keys, rows)
    ref = bindings.RefIndex("parity", metric="l2sq", scalar="f32", dims=d)
    ref.pin_metric(True)
    # key 0 holds one vector, key 1 five: the minimum over the five pairs
    want = min(ref.distance(rows[0], rows[j]) for j in range(1, 6))
    got = ix.pairwise_distance(0, 1)
    assert np.float32(got).view(np.uint32) == np.float32(want).view(np.uint32)


def test_join_output_capacity_is_checked():
    """the C entry never writes past the caller's arrays: too small a capacity is an error"""
    import ctypes as C
    from usearch_b200.index import load_library
    a_blob, b_blob = _pair("cos", "f32", 64, 50, 60, seed=30)
    ia, ib = _load(a_blob), _load(b_blob)
    lib = load_library()
    small = 10
    a_keys = np.full(small + 1, 7, dtype=np.uint64)
    b_keys = np.full(small + 1, 7, dtype=np.uint64)
    err = C.c_char_p()
    n = lib.usearch_b200_join(ia._h, ib._h, 0, False, a_keys.ctypes.data_as(C.c_void_p), b_keys.ctypes.data_as(C.c_void_p), small,
                              None, C.byref(err))
    assert n == 0 and b"too small" in err.value
    assert (a_keys == 7).all() and (b_keys == 7).all()
    assert len(ia.join(ib)) == ia.last_join_stats["intersection_size"] > small


def test_join_phase_timings():
    a_blob, b_blob = _pair("cos", "f32", 97, 200, 260, seed=31)
    ia, ib = _load(a_blob), _load(b_blob)
    ia.join(ib)
    assert set(ia.last_join_ms) == {"search", "pair_distances", "replay"}
    assert ia.last_join_ms["search"] > 0 and ia.last_join_ms["pair_distances"] > 0 and ia.last_join_ms["replay"] >= 0


def test_join_refusals():
    a_blob, b_blob = _pair("cos", "f32", 64, 50, 60, seed=20)
    ia, ib = _load(a_blob), _load(b_blob)
    with pytest.raises(RuntimeError, match="Can't join with itself"):
        ia.join(ia)
    other = Index(ndim=64, metric="l2sq", dtype="f32")
    other.add(None, _rows(10, 64, "f32", 21))
    with pytest.raises(RuntimeError, match="different metrics"):
        ia.join(other)
    other_dims = Index(ndim=32, metric="cos", dtype="f32")
    other_dims.add(None, _rows(10, 32, "f32", 22))
    with pytest.raises(RuntimeError, match="dimensions"):
        ia.join(other_dims)
    other_kind = Index(ndim=64, metric="cos", dtype="f16")
    other_kind.add(None, _rows(10, 64, "f16", 23))
    with pytest.raises(RuntimeError, match="scalar kinds"):
        ia.join(other_kind)
    # different devices and sharded handles are refused too (frozen_index_t::join); neither can be set up on one GPU here
    with pytest.raises(RuntimeError, match="65535"):
        ia.join(ib, max_proposals=70_000)
    empty = Index(ndim=64, metric="cos", dtype="f32")
    assert ia.join(empty) == {} and empty.join(ia) == {}
