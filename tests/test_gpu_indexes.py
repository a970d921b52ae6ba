"""`Indexes`: several indexes on one GPU searched as one, against the reference's `Indexes.search` run on one thread.

The specification is the reference's fold: every shard's result, in merge order and in its stored order, goes into the
query's row through `search_result_t::merge_into` (index.hpp:2650-2670). `indexes_reference.merge_model` states that fold
literally: libstdc++'s `lower_bound` probe, then the shift. A CPU test holds the model, fed with the reference's own
per-shard searches, equal to the reference's own `Indexes` loop compiled at test time; the GPU tests hold the merge kernel
to the model on hand-made rows (NaN, signed zeros, infinities) and the whole `Indexes.search` to the model over the
reference's per-shard searches, on shards built by the reference and on the GPU."""
import os

import numpy as np
import pytest

import common
import indexes_reference as ir
from indexes_reference import SNAN_BITS, merge_model
from oracle import bindings

NQ = 500
EF = 64


# ---- shards built by the reference ------------------------------------------------------------------------------------

FAMILIES = {  # name: metric, scalar, shard sizes, d
    "cos_f32": ("cos", "f32", [2000, 2000, 2000, 2000], 64),
    "l2sq_i8": ("l2sq", "i8", [1500, 1200, 900], 48),
    "hamming_b1": ("hamming", "b1", [1500, 1500, 1500], 128),
}


def _reference_shards(family, seed=7):
    metric, scalar, sizes, d = FAMILIES[family]
    base, q = common.make_collection(sum(sizes), d, scalar, NQ, seed=seed)
    refs, blobs, start = [], [], 0
    for n in sizes:
        keys = np.arange(start, start + n, dtype=np.uint64)
        ref, blob = common.build_reference_blob(base[start:start + n], metric, scalar, d, 16, threads=8, keys=keys)
        ref.pin_metric(True)
        ref.change_expansion_search(EF)
        refs.append(ref)
        blobs.append(blob)
        start += n
    return refs, blobs, q, scalar


def _gpu_shards(blobs):
    from usearch_b200.index import Index
    shards = []
    for blob in blobs:
        index = Index.restore(blob)
        index.expansion_search = EF
        shards.append(index)
    return shards


def _gpu_result(indexes, q, k, exact=False):
    got = indexes.search(q, k, exact=exact)
    return got.keys, got.distances, got.counts, indexes.last_computed, indexes.last_visited


_CACHE = {}


def _family(family):
    if family not in _CACHE:
        _CACHE[family] = _reference_shards(family)
    return _CACHE[family]


needs_reference = pytest.mark.skipif(not common.have_reference(), reason="reference library not built")


# ---- CPU: the model is the reference's fold ---------------------------------------------------------------------------

needs_live = pytest.mark.skipif(not ir.live_available(), reason="reference sources absent: the live loop compiles from them")


@needs_live
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("exact", [False, True])
def test_model_matches_the_reference_loop(family, exact):
    """The model over the reference's per-shard searches equals the reference's own `Indexes` loop (`merge_into`), keys,
    distance bits, counts and both counters; also with the first shard a member twice."""
    refs, blobs, q, scalar = _family(family)
    q = q[:120]
    for k in (1, 10, 50):
        want = ir.live_search(blobs, list(range(len(blobs))), q, k, expansion=EF, query_scalar=scalar, exact=exact)
        common.assert_same_results(want, ir.reference_search(refs, q, k, query_scalar=scalar, exact=exact),
                                   f"model vs reference loop {family} k={k}")
    twice = ir.live_search(blobs[:1], [0, 0], q, 10, expansion=EF, query_scalar=scalar, exact=exact)
    common.assert_same_results(twice, ir.reference_search([refs[0], refs[0]], q, 10, query_scalar=scalar, exact=exact),
                               f"model vs reference loop {family}, one shard twice")


@needs_live
def test_model_matches_the_reference_loop_on_mixed_kinds():
    """An f32 and an f16 shard under f32 queries: each shard casts the queries for itself."""
    refs, blobs, q = _mixed_kind_shards()
    for exact in (False, True):
        want = ir.live_search(blobs, [0, 1], q, 10, expansion=EF, query_scalar="f32", exact=exact)
        common.assert_same_results(want, ir.reference_search(refs, q, 10, query_scalar="f32", exact=exact),
                                   f"model vs reference loop, f32 + f16 shards exact={exact}")


@needs_live
def test_model_matches_the_reference_loop_on_cross_shard_ties():
    """Three shards holding the same rows under different keys: every candidate ties across shards."""
    refs, blobs, q = _tie_shards()
    for exact in (False, True):
        for k in (3, 30):
            want = ir.live_search(blobs, [0, 1, 2], q, k, expansion=EF, exact=exact)
            common.assert_same_results(want, ir.reference_search(refs, q, k, exact=exact), f"ties exact={exact} k={k}")


def test_model_breaks_ties_towards_the_later_insertion():
    keys = np.array([[[1, 2, 3]], [[4, 5, 6]]], dtype=np.uint64)
    dists = np.array([[[0.5, 0.5, 1.0]], [[0.0, 0.5, 1.0]]], dtype=np.float32)
    k, d, c = merge_model(keys, dists, np.array([[3], [3]]), 4)
    assert k[0].tolist() == [4, 5, 2, 1] and d[0].tolist() == [0.0, 0.5, 0.5, 0.5] and c.tolist() == [4]


def test_model_follows_the_probe_with_nan():
    """With a NaN in the row, lower_bound's probe is not a count of smaller elements: the model must follow the probe."""
    nan = float("nan")
    keys = np.array([[[1, 2, 3, 4]]], dtype=np.uint64)
    dists = np.array([[[1.0, nan, 3.0, 0.5]]], dtype=np.float32)
    k, d, c = merge_model(keys, dists, np.array([[4]]), 4)
    # 1.0 -> [1.0]; NaN -> [NaN, 1.0]; 3.0 probes row[1] = 1.0 < 3 and lands at 2, where a count of smaller elements
    # would give 1; 0.5 probes row[1], then row[0] = NaN, and lands at 0
    assert c.tolist() == [4] and k[0].tolist() == [4, 2, 1, 3]


def test_empty_group_returns_empty_rows():
    from usearch_b200.index import Indexes
    group = Indexes()
    assert len(group) == 0
    got = group.search(np.ones((3, 8), dtype=np.float32), 4)
    assert got.counts.tolist() == [0, 0, 0] and (got.keys == 0).all()
    assert (got.distances.view(np.uint32) == SNAN_BITS).all()
    assert got.visited_members == 0 and got.computed_distances == 0
    assert len(group.search(np.ones(8, dtype=np.float32), 4)) == 0


# ---- GPU: the merge kernel on hand-made rows ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 7, 32, 33, 256])
def test_kernel_matches_the_model_on_hand_made_rows(k):
    from usearch_b200.index import merge_into
    rng = np.random.default_rng(k)
    S, nq = 5, 64
    pool = np.array([0.0, -0.0, 0.25, 0.5, 1.0, -1.0, np.inf, -np.inf, np.nan, 2.0], dtype=np.float32)
    dists = pool[rng.integers(0, pool.size, size=(S, nq, k))]
    # some rows sorted as a search returns them, some not: the fold must not assume either
    dists[:, : nq // 2] = np.sort(dists[:, : nq // 2], axis=2)
    keys = rng.integers(1, 1 << 40, size=(S, nq, k), dtype=np.uint64)
    counts = rng.integers(0, k + 1, size=(S, nq)).astype(np.uint32)
    counts[:, 0] = 0
    counts[:, 1] = k
    counts[0, 2] = k + 5  # clamped to k
    got = merge_into(keys, dists, counts)
    want = merge_model(keys, dists, np.minimum(counts, k), k)
    common.assert_same_results((got.keys, got.distances, got.counts), want, f"merge kernel k={k}")


# ---- GPU: Indexes.search against the reference -------------------------------------------------------------------------

@pytest.mark.gpu
@needs_reference
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("exact", [False, True])
def test_indexes_search_matches_the_reference(family, exact):
    from usearch_b200.index import Indexes
    refs, blobs, q, scalar = _family(family)
    shards = _gpu_shards(blobs)
    group = Indexes(shards)
    assert len(group) == sum(FAMILIES[family][2])
    for k in (1, 10, 50):
        want = ir.reference_search(refs, q, k, query_scalar=scalar, exact=exact)
        got = _gpu_result(group, q, k, exact)
        common.assert_same_results(want, got, f"{family} exact={exact} k={k}")
        res = group.search(q, k, exact=exact)
        assert res.computed_distances == int(want[3].sum()) and res.visited_members == int(want[4].sum())
    assert all(s.kernel_launches >= 1 for s in shards)


def _tie_shards(metric="l2sq", scalar="f32", n=600, d=16, copies=3):
    base, q = common.make_collection(n, d, scalar, 200, seed=11)
    refs, blobs = [], []
    for c in range(copies):
        ref, blob = common.build_reference_blob(base, metric, scalar, d, 16, threads=1,
                                                keys=np.arange(n, dtype=np.uint64) + 10000 * c)
        ref.pin_metric(True)
        ref.change_expansion_search(EF)
        refs.append(ref)
        blobs.append(blob)
    return refs, blobs, q


@pytest.mark.gpu
@needs_reference
@pytest.mark.parametrize("exact", [False, True])
def test_cross_shard_ties_put_the_later_shard_first(exact):
    from usearch_b200.index import Indexes
    refs, blobs, q = _tie_shards()
    group = Indexes(_gpu_shards(blobs))
    for k in (3, 10, 30):
        want = ir.reference_search(refs, q, k, exact=exact)
        got = _gpu_result(group, q, k, exact)
        common.assert_same_results(want, got, f"ties k={k}")
        # every member is present three times: runs of equal distances come out shard 2, shard 1, shard 0
        for row in range(q.shape[0]):
            bits = got[1][row, : int(got[2][row])].view(np.uint32)
            shard = got[0][row, : int(got[2][row])] // 10000
            for i in range(1, bits.size):
                if bits[i] == bits[i - 1]:
                    assert shard[i] <= shard[i - 1]


@pytest.mark.gpu
@needs_reference
def test_the_same_handle_twice():
    from usearch_b200.index import Indexes
    refs, blobs, q, scalar = _family("l2sq_i8")
    a = _gpu_shards(blobs[:1])[0]
    group = Indexes([a, a])
    assert len(group) == 2 * a.size
    for exact in (False, True):
        want = ir.reference_search([refs[0], refs[0]], q, 10, query_scalar=scalar, exact=exact)
        common.assert_same_results(want, _gpu_result(group, q, 10, exact), f"[a, a] exact={exact}")
        got = group.search(q, 10, exact=exact)
        assert (got.distances[:, 0].view(np.uint32) == got.distances[:, 1].view(np.uint32)).all()


@pytest.mark.gpu
@needs_reference
def test_edges_empty_small_removed_multi_and_gpu_built_shards():
    from usearch_b200.index import Index, Indexes
    metric, scalar, d = "cos", "f32", 32
    base, q = common.make_collection(3000, d, scalar, 300, seed=21)
    refs, gpu = [], []

    def add_shard(blob):
        ref = bindings.RefIndex("parity")
        ref.load(blob)
        ref.pin_metric(True)
        ref.change_expansion_search(EF)
        refs.append(ref)
        index = Index.restore(blob)
        index.expansion_search = EF
        gpu.append(index)

    # an empty shard
    empty = Index(ndim=d, metric=metric, dtype=scalar)
    gpu.append(empty)
    empty_ref = bindings.RefIndex("parity", metric=metric, scalar=scalar, dims=d)
    empty_ref.pin_metric(True)
    refs.append(empty_ref)
    # a reference-built shard
    _, blob = common.build_reference_blob(base[:1000], metric, scalar, d, 16, keys=np.arange(1000, dtype=np.uint64))
    add_shard(blob)
    # a shard smaller than k
    _, blob = common.build_reference_blob(base[1000:1005], metric, scalar, d, 16, keys=np.arange(1000, 1005, dtype=np.uint64))
    add_shard(blob)
    # a shard with removed entries
    ref, _ = common.build_reference_blob(base[1005:1800], metric, scalar, d, 16, keys=np.arange(1005, 1800, dtype=np.uint64))
    for key in range(1005, 1800, 7):
        ref.remove(key)
    add_shard(ref.save())
    # a GPU-built multi index: keys repeat
    multi = Index(ndim=d, metric=metric, dtype=scalar, connectivity=16, multi=True)
    multi.add(np.repeat(np.arange(2000, 2300, dtype=np.uint64), 2), base[1800:2400])
    add_shard(multi.save())
    # a GPU-built shard
    built = Index(ndim=d, metric=metric, dtype=scalar, connectivity=16)
    built.add(np.arange(2400, 3000, dtype=np.uint64), base[2400:3000])
    add_shard(built.save())

    group = Indexes(gpu)
    assert len(group) == sum(len(g) for g in gpu)
    for exact in (False, True):
        for k in (1, 10, 64):
            want = ir.reference_search(refs, q, k, exact=exact)
            common.assert_same_results(want, _gpu_result(group, q, k, exact), f"edges exact={exact} k={k}")
    # k greater than the total size: the empty shard and the 5-row shard
    small = Indexes([gpu[0], gpu[2]])
    total = len(small)
    for exact in (False, True):
        want = ir.reference_search([refs[0], refs[2]], q, total + 9, exact=exact)
        got = _gpu_result(small, q, total + 9, exact)
        common.assert_same_results(want, got, f"k > total exact={exact}")
        assert total == 5 and (got[2] == total).all()


def _mixed_kind_shards():
    base, q = common.make_collection(2000, 64, "f32", 300, seed=31)
    refs, blobs = [], []
    for i, scalar in enumerate(("f32", "f16")):
        part = base[i * 1000:(i + 1) * 1000]
        ref, blob = common.build_reference_blob(common.datagen.to_scalar(part, scalar), "cos", scalar, 64, 16,
                                                keys=np.arange(i * 1000, (i + 1) * 1000, dtype=np.uint64))
        ref.pin_metric(True)
        ref.change_expansion_search(EF)
        refs.append(ref)
        blobs.append(blob)
    return refs, blobs, q


@pytest.mark.gpu
@needs_reference
def test_mixed_scalar_kinds_with_f32_queries():
    from usearch_b200.index import Indexes
    refs, blobs, q = _mixed_kind_shards()
    group = Indexes(_gpu_shards(blobs))
    for exact in (False, True):
        want = ir.reference_search(refs, q, 10, query_scalar="f32", exact=exact)
        common.assert_same_results(want, _gpu_result(group, q, 10, exact), f"f32 + f16 shards exact={exact}")


@pytest.mark.gpu
def test_refusals():
    from usearch_b200.index import Index, Indexes
    blob = np.load(os.path.join(common.GOLDEN, "cos_f32_n2000_d64.npz"))["blob"]
    a, b = _gpu_shards([blob, blob])
    other = Index(ndim=32, metric="cos", dtype="f32")
    other.add(np.arange(10, dtype=np.uint64), np.random.default_rng(0).standard_normal((10, 32)).astype(np.float32))
    queries = np.random.default_rng(1).standard_normal((4, 64)).astype(np.float32)
    with pytest.raises(RuntimeError, match="different dimensions"):
        Indexes([a, other]).search(queries, 5)
    b.join_shards(0, 1, bytes(128))
    with pytest.raises(RuntimeError, match="sharded"):
        Indexes([a, b]).search(queries, 5)
    assert Indexes([a]).search(queries, 5).counts.tolist() == [5] * 4


@pytest.mark.gpu
@needs_reference
def test_paths_equal_indexes(tmp_path):
    from usearch_b200.index import Indexes
    _, blobs, q, _ = _family("hamming_b1")
    paths = []
    for i, blob in enumerate(blobs):
        path = tmp_path / f"shard{i}.usearch"
        blob.tofile(path)
        paths.append(str(path))
    by_path = Indexes(paths=paths)
    by_index = Indexes(indexes=_gpu_shards(blobs))
    assert len(by_path) == len(by_index)
    for shard in by_path._members:
        shard.expansion_search = EF
    for exact in (False, True):
        common.assert_same_results(_gpu_result(by_index, q, 10, exact), _gpu_result(by_path, q, 10, exact), f"paths exact={exact}")
    one = by_path.search(q[0], 10)
    assert len(one) == 10 and np.array_equal(one.keys, by_index.search(q, 10).keys[0])
