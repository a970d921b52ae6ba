"""Reading an index back out on the GPU: `get` for many keys, `index[keys]`, `keys`, `vectors`, `copy()` and the graph's
`stats`, held to the per-key `get` (itself held to the reference's casts) and to the model of the index's own saved file
(tests/surface_reference.py, held to the reference by tests/test_surface_reference.py)."""
import gc
import os
import subprocess

import numpy as np
import pytest

import common
import surface_reference as model
from usearch_b200.index import Index

pytestmark = pytest.mark.gpu

KINDS = ["f32", "f16", "bf16", "i8", "b1", "f64"]
GOLDEN = {"f32": "cos_f32_n2000_d64.npz", "i8": "ip_i8_n2000_d64.npz", "b1": "hamming_b1_n4000_d256.npz"}
METRIC = {"f32": "cos", "f16": "l2sq", "bf16": "ip", "i8": "cos", "b1": "hamming", "f64": "l2sq"}


def _vectors(n, d, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "b1":
        return np.packbits(rng.random((n, d)) > 0.5, axis=1)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[::7] *= 1e-3  # small values: the half kinds round them, i8 scales them
    return x.astype(np.float64) if kind == "f64" else x


def _built(kind, n=1500, d=40, multi=False, connectivity=16):
    index = Index(ndim=d, metric=METRIC[kind], dtype=kind, connectivity=connectivity, multi=multi)
    index.add(np.arange(n, dtype=np.uint64), _vectors(n, d, kind, seed=len(kind)))
    return index


def _golden(kind):
    return Index.restore(np.load(os.path.join(common.GOLDEN, GOLDEN[kind]))["blob"])


def _indexes(kind):
    yield "built", _built(kind)
    if kind in GOLDEN:
        yield "golden", _golden(kind)


def _stacked(index, keys, dtype):
    """the per-key path, a missing key's row zero"""
    cols = (index.ndim + 7) // 8 if dtype == "b1" else index.ndim
    np_t = {"f32": np.float32, "f64": np.float64, "f16": np.float16, "bf16": np.uint16, "i8": np.int8, "b1": np.uint8}[dtype]
    rows = [index.get(int(k), dtype) for k in keys]
    return np.stack([r if r is not None else np.zeros(cols, np_t) for r in rows]) if rows else np.zeros((0, cols), np_t)


@pytest.mark.parametrize("stored", KINDS)
def test_get_many_equals_per_key_get_for_every_kind(stored):
    for name, index in _indexes(stored):
        keys = np.asarray(index.keys)
        index.remove(keys[5:9])
        rng = np.random.default_rng(3)
        asked = np.concatenate([rng.choice(keys, 300), keys[[0, 0, 1]], keys[5:9], [10**12, 2**63 + 5]]).astype(np.uint64)
        for requested in KINDS:
            got = index.get(asked, requested)
            want = _stacked(index, asked, requested)
            assert got.dtype == want.dtype and got.shape == want.shape, (name, requested)
            assert got.tobytes() == want.tobytes(), (name, stored, requested)
        # any integer dtype and stride, NumPy dtypes, lists, an empty list, index[keys]
        strided = np.repeat(asked.astype(np.int64), 2)[::2]
        assert index.get(strided, index.dtype).tobytes() == index.get(asked).tobytes()
        assert index[list(asked[:5])].tobytes() == index.get(asked[:5]).tobytes()
        assert index.get([]).shape == (0, index.get(asked[:1]).shape[1])
        np_kind = {"f32": np.float32, "f64": np.float64, "f16": np.float16, "i8": np.int8, "b1": np.uint8}
        for kind, np_t in np_kind.items():
            assert index.get(asked[:20], np_t).tobytes() == index.get(asked[:20], kind).tobytes()


def test_get_many_crosses_chunks():
    index = _built("f32", n=3000, d=33)
    keys = np.random.default_rng(0).permutation(np.asarray(index.keys))
    whole = index.get(keys)
    for rows in (1, 7, 256, 2999):
        index.tune(get_chunk_rows=rows)
        for dtype in ("f32", "f16", "i8"):
            assert index.get(keys, dtype)[:50].tobytes() == _stacked(index, keys[:50], dtype).tobytes()
        assert index.get(keys).tobytes() == whole.tobytes()
    index.tune(get_chunk_rows=0)


def test_multi_index_returns_a_tuple_in_slot_order():
    index = Index(ndim=16, metric="l2sq", dtype="f32", multi=True)
    x = _vectors(900, 16, "f32", seed=1)
    keys = np.arange(900, dtype=np.uint64) % 300  # three entries per key, in slot order
    index.add(keys, x)
    got = index.get(np.array([5, 7, 5, 10**9], dtype=np.uint64))
    assert isinstance(got, tuple) and got[3] is None
    for out, key in zip(got[:3], (5, 7, 5)):
        assert np.array_equal(out, x[keys == key])
    assert np.array_equal(index.get(5, count=3), x[keys == 5])  # the scalar path is unchanged
    assert any(np.array_equal(index.get(5), row) for row in x[keys == 5])
    assert index.multi and len(index.keys) == 900
    vectors = index.vectors
    assert isinstance(vectors, tuple) and len(vectors) == 900


@pytest.mark.parametrize("kind", ["f32", "i8", "b1"])
def test_keys_and_vectors_equal_the_saved_file(kind):
    for _, index in _indexes(kind):
        index.remove(np.asarray(index.keys)[::5])
        g = model.parse(index.save())
        live = model.live_keys(g)
        keys = index.keys
        assert len(keys) == len(live) == len(index)
        assert np.array_equal(np.asarray(keys), live)
        assert keys[0] == live[0] and keys[-1] == live[-1] and keys[-len(live)] == live[0]
        assert np.array_equal(keys[3:40], live[3:40]) and np.array_equal(keys[40:3:-3], live[40:3:-3])
        assert np.array_equal(keys[np.array([9, 2, -1, 2])], live[[9, 2, -1, 2]])
        with pytest.raises(IndexError):
            keys[len(live)]
        assert list(keys) == live.tolist()
        vectors = index.vectors
        assert np.array_equal(vectors, index.get(np.asarray(keys)))
        assert vectors.view(np.uint8).reshape(len(live), -1).tobytes() == g.matrix[g.keys != model.FREE_KEY].tobytes()


def _assert_stats(index):
    g = model.parse(index.save())
    per, _ = model.levels_stats(g)
    assert [tuple(vars(s).values()) for s in index.levels_stats] == per
    assert tuple(vars(index.stats).values()) == model.stats(g)
    for level in range(len(per) + 1):
        assert tuple(vars(index.level_stats(level)).values()) == model.level_stats(g, level)
    assert index.nlevels == g.max_level + 1


@pytest.mark.parametrize("path", ["cos_f32_n2000_d64.npz", "ip_f32_n1500_d48_removed.npz", "hamming_b1_n4000_d256.npz",
                                  "ip_i8_n2000_d64.npz", "l2sq_f32_n2000_d33.npz", "tanimoto_b1_n2000_d96.npz"])
def test_stats_on_golden_graphs(path):
    blob = np.load(os.path.join(common.GOLDEN, path))["blob"]
    index = Index.restore(blob)
    g = model.parse(blob)
    assert tuple(vars(index.stats).values()) == model.stats(g)
    assert [tuple(vars(s).values()) for s in index.levels_stats] == model.levels_stats(g)[0]


def test_stats_on_built_removed_and_reused_graphs():
    index = _built("f32", n=4000, d=24)
    _assert_stats(index)
    index.remove(np.arange(0, 4000, 3, dtype=np.uint64))
    _assert_stats(index)
    index.remove(np.arange(1, 4000, 3, dtype=np.uint64), compact=True)
    assert index.last_pruned_edges > 0
    _assert_stats(index)
    index.reuse_removed = True
    index.add(np.arange(10**6, 10**6 + 500, dtype=np.uint64), _vectors(500, 24, "f32", seed=9))
    _assert_stats(index)
    empty = Index(ndim=8, metric="cos", dtype="f32")
    assert empty.levels_stats == [] and tuple(vars(empty.stats).values()) == (0, 0, 0, 0)


def _search_everything(index, queries):
    out = []
    plain = index.search(queries, 10, stats=True)
    out += [plain.keys, plain.distances.view(np.uint32), plain.counts, index.last_computed, index.last_visited]
    allowed = np.asarray(index.keys)[::2]
    filtered = index.filtered_search(queries, 10, allowed)
    out += [filtered.keys, filtered.distances.view(np.uint32), index.last_computed, index.last_visited]
    exact = index.search(queries, 10, exact=True)
    out += [exact.keys, exact.distances.view(np.uint32)]
    keys, dists = index.cluster(queries, level=1, stats=True)
    out += [keys, dists.view(np.uint32), index.last_computed, index.last_visited]
    return out


COPY_CASES = [("cos", "f32", 768, False), ("l2sq", "f16", 64, False), ("ip", "i8", 64, False), ("hamming", "b1", 256, False),
              ("l2sq", "f64", 48, False), ("cos", "f32", 32, True)]


@pytest.mark.parametrize("metric,kind,d,multi", COPY_CASES, ids=[f"{m}-{k}-{d}{'-multi' if u else ''}" for m, k, d, u in COPY_CASES])
def test_copy_is_an_identical_independent_index(metric, kind, d, multi):
    n = 2000
    index = Index(ndim=d, metric=metric, dtype=kind, connectivity=16, multi=multi)
    keys = np.arange(n, dtype=np.uint64) % (n // 2 if multi else n)
    index.add(keys, _vectors(n, d, kind, seed=d))
    index.remove(np.arange(0, 300, 7, dtype=np.uint64))
    index.reuse_removed = True
    index.tune(warps_per_sm=3)
    copy = index.copy()
    assert copy.save().tobytes() == index.save().tobytes()
    assert copy.reuse_removed and copy.multi == multi and copy.memory_usage == index.memory_usage
    assert copy.launch_plan(10) == index.launch_plan(10)
    queries = _vectors(64, d, kind, seed=99)
    for a, b in zip(_search_everything(index, queries), _search_everything(copy, queries)):
        assert np.array_equal(a, b)
    # the same edits on both keep them identical: reuse takes the same slots in the same order
    more = _vectors(200, d, kind, seed=5)
    for target in (index, copy):
        target.add(np.arange(10**6, 10**6 + 200, dtype=np.uint64), more)
        target.remove(np.arange(300, 400, dtype=np.uint64), compact=True)
        target.add(np.arange(2 * 10**6, 2 * 10**6 + 60, dtype=np.uint64), more[:60])
    saved = copy.save().tobytes()
    assert saved == index.save().tobytes()
    # independent: editing the original leaves the copy as it was, and the copy outlives it
    index.remove(np.arange(400, 600, dtype=np.uint64), compact=True)
    assert copy.save().tobytes() == saved
    del index
    gc.collect()
    assert copy.search(queries, 10).keys.shape == (64, 10)
    assert copy.save().tobytes() == saved


def test_copy_of_an_empty_index_and_reset():
    empty = Index(ndim=8, metric="l2sq", dtype="f32")
    copy = empty.copy()
    assert len(copy) == 0 and copy.ndim == 8
    copy.add(np.arange(10, dtype=np.uint64), _vectors(10, 8, "f32", seed=0))
    assert len(copy) == 10 and len(empty) == 0
    copy.reset()
    assert len(copy) == 0 and copy.memory_usage == 0 and copy.ndim == 8
    copy.add(np.arange(5, dtype=np.uint64), _vectors(5, 8, "f32", seed=0))
    assert len(copy) == 5


def test_copy_refuses_a_sharded_handle():
    import torch  # noqa: F401  (loads the NCCL library torch ships, which the sharded search binds at run time)
    from usearch_b200.index import shards_unique_id
    index = _built("f32", n=200, d=16)
    index.join_shards(0, 1, shards_unique_id())
    with pytest.raises(RuntimeError, match="sharded"):
        index.copy()


def test_ported_reference_flows():
    """The retrieval, duplicate, stats and save / load / copy scenarios of the reference's Python suite, restated."""
    d, n = 32, 500
    index = Index(ndim=d, metric="cos", dtype="f32")
    x = _vectors(n, d, "f32", seed=11)
    index.add(np.arange(n, dtype=np.uint64), x)
    # retrieval: every vector comes back under its key, one by one and all at once
    assert np.array_equal(index[42], x[42])
    assert np.array_equal(index.get(np.arange(n)), x)
    assert np.array_equal(index.vectors, x)
    assert sorted(index.keys) == list(range(n))
    # duplicates are refused on a plain index and kept on a multi one
    with pytest.raises(RuntimeError, match="Duplicate"):
        index.add(3, x[3])
    multi = Index(ndim=d, metric="cos", dtype="f32", multi=True)
    multi.add(np.array([1, 1, 2], dtype=np.uint64), x[:3])
    assert multi.count(1) == 2 and len(multi.get([1])[0]) == 2
    # stats
    assert index.stats.nodes == n and index.levels_stats[0].nodes == n and index.level_stats(0).max_edges == n * 32
    assert index.nlevels == len(index.levels_stats)
    # save / load / restore / copy all read back the same
    blob = index.save()
    for other in (Index.restore(blob), Index(ndim=d).load(blob), index.copy()):
        assert np.array_equal(other.vectors, x) and other.stats == index.stats
    del index[np.arange(10)]
    assert len(index) == n - 10 and not index.get(np.arange(12))[:10].any()
    index.reset()
    assert len(index) == 0 and index.ndim == d


def test_cpp_mirror_client(tmp_path):
    include, libdir = os.path.join(common.ROOT, "include"), os.path.join(common.ROOT, "usearch_b200")
    exe = str(tmp_path / "test_surface_mirror")
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Wextra", "-Werror", "-O1", f"-I{include}",
                    os.path.join(common.ROOT, "tests", "native", "test_surface_mirror.cpp"), "-o", exe, f"-L{libdir}",
                    "-lusearch_b200", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True)
    path = str(tmp_path / "golden.usearch")
    np.load(os.path.join(common.GOLDEN, "cos_f32_n2000_d64.npz"))["blob"].astype(np.uint8).tofile(path)
    out = subprocess.run([exe, path], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "SURFACE_MIRROR_OK" in out.stdout, out.stdout + out.stderr
