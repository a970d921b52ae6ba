"""Lookups by key from device memory: `count_device`, `get_device` and `filtered_search_device`, with keys and outputs
as torch CUDA tensors, held byte for byte to the host `count`, `get_many` and `filtered_search` of the same handle, on
golden and GPU-built graphs, after every kind of edit, and on a caller's stream."""
import ctypes as C
import os

import numpy as np
import pytest

import common
from usearch_b200.index import SCALAR_KIND, Index

pytestmark = pytest.mark.gpu

KINDS = ["f32", "f16", "bf16", "i8", "b1", "f64"]
METRIC = {"f32": "cos", "f16": "l2sq", "bf16": "ip", "i8": "cos", "b1": "hamming", "f64": "l2sq"}
BITS = {"f32": 32, "f64": 64, "f16": 16, "bf16": 16, "i8": 8, "b1": 1}
FREE_KEY = 2**64 - 1


def _torch():
    import torch
    return torch


def _on_device(array):
    torch = _torch()
    array = np.ascontiguousarray(array)
    if array.dtype == np.uint64:
        array = array.view(np.int64)
    return torch.from_numpy(array).cuda()


def _vectors(n, d, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "b1":
        return np.packbits(rng.random((n, d)) > 0.5, axis=1)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[::7] *= 1e-3
    return x.astype(np.float64) if kind == "f64" else x


def _built(kind, n=1200, d=37, multi=False):
    index = Index(ndim=d, metric=METRIC[kind], dtype=kind, multi=multi)
    keys = np.arange(n, dtype=np.uint64) % (n // 3) if multi else np.arange(n, dtype=np.uint64)
    index.add(keys, _vectors(n, d, kind, seed=len(kind)))
    return index


def _golden_indexes():
    for name in sorted(os.listdir(common.GOLDEN)):
        if not name.endswith(".npz"):
            continue
        z = np.load(os.path.join(common.GOLDEN, name))
        for field in z.files:
            if field == "blob":
                yield f"{name}:{field}", Index.restore(z[field])


def _row_bytes(index, kind):
    return (index.ndim * BITS[kind] + 7) // 8


def count_device(index, keys, stream=0):
    torch = _torch()
    d_keys = _on_device(keys.astype(np.uint64))
    counts = torch.full((len(keys),), -1, dtype=torch.int32, device="cuda")
    index.count_device(d_keys.data_ptr(), len(keys), counts.data_ptr(), stream=stream)
    return counts.cpu().numpy().view(np.uint32)


def get_device(index, keys, per_key, kind, stride=0, d_keys=None, stream=0):
    """rows [n, per_key, row bytes] and counts; the output starts as 0x5A so untouched rows would show"""
    torch = _torch()
    n, row = len(keys), _row_bytes(index, kind)
    stride = stride or row
    out = torch.full((max(n * per_key * stride, 1),), 0x5A, dtype=torch.uint8, device="cuda")
    counts = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda")
    if d_keys is None:
        d_keys = _on_device(keys.astype(np.uint64))
    index.get_device(d_keys.data_ptr(), n, out.data_ptr(), counts.data_ptr(), count=per_key, stride=stride, dtype=kind,
                     stream=stream)
    rows = out.cpu().numpy()[:n * per_key * stride].reshape(n, per_key, stride)
    return rows, counts.cpu().numpy()[:n].view(np.uint32)


def host_get_many(index, keys, per_key, kind):
    """usearch_b200_get_many placed into the device layout: key i's rows at [i, :counts[i]], the rest zero"""
    keys = np.ascontiguousarray(keys, dtype=np.uint64)
    n, row = len(keys), _row_bytes(index, kind)
    total = int(np.minimum(index.count(keys), per_key).sum()) if n else 0
    packed = np.zeros((max(total, 1), row), dtype=np.uint8)
    counts = np.zeros(n, dtype=np.uintp)
    err = C.c_char_p()
    got = index._lib.usearch_b200_get_many(index._h, keys.ctypes.data_as(C.c_void_p), n, C.c_size_t(per_key),
                                           packed.ctypes.data_as(C.c_void_p), row, SCALAR_KIND[kind],
                                           counts.ctypes.data_as(C.c_void_p), C.byref(err))
    assert not err.value, err.value
    assert got == total
    out = np.zeros((n, per_key, row), dtype=np.uint8)
    at = 0
    for i, c in enumerate(counts.astype(np.int64)):
        out[i, :c] = packed[at:at + c]
        at += c
    return out, counts.astype(np.uint32)


def _asked(index, rng, extra=()):
    keys = np.asarray(index.keys)
    asked = [rng.choice(keys, min(200, len(keys))) if len(keys) else np.zeros(0, np.uint64), keys[:3], keys[:3],
             [0, 10**12, FREE_KEY, 2**63 + 5], list(extra)]
    return np.concatenate([np.asarray(a, dtype=np.uint64) for a in asked])


def assert_lookups_match(index, keys, kinds=None, per_keys=(1,), removed=True):
    """count_device == count; get_device == get_many for every requested kind and per-key bound. A key's device rows are
    its lowest slots: with removals on the handle that is the host's full, sorted list cut to `per_key`."""
    counts = index.count(keys).astype(np.uint32)
    assert np.array_equal(count_device(index, keys), counts)
    for kind in kinds or [index.dtype]:
        full = int(counts.max()) if len(keys) and counts.max() else 1
        for per_key in per_keys:
            rows, got_counts = get_device(index, keys, per_key, kind)
            assert np.array_equal(got_counts, np.minimum(counts, per_key)), (kind, per_key)
            want, _ = host_get_many(index, keys, max(per_key, full), kind)
            assert rows.tobytes() == want[:, :per_key].tobytes(), (kind, per_key)
            if not removed or per_key >= full:
                want, want_counts = host_get_many(index, keys, per_key, kind)
                assert np.array_equal(want_counts, got_counts) and rows.tobytes() == want.tobytes(), (kind, per_key)


def test_golden_fixtures():
    rng = np.random.default_rng(0)
    for name, index in _golden_indexes():
        keys = _asked(index, rng)
        assert_lookups_match(index, keys, per_keys=(1, 3)), name


@pytest.mark.parametrize("stored", KINDS)
def test_every_stored_and_requested_kind(stored):
    rng = np.random.default_rng(1)
    index = _built(stored)  # 37 dimensions: b1 rows end inside a byte
    assert_lookups_match(index, _asked(index, rng), kinds=KINDS, removed=False)
    index.remove(np.arange(10, 40, dtype=np.uint64))
    assert_lookups_match(index, _asked(index, rng, extra=range(5, 45)), kinds=KINDS)


@pytest.mark.parametrize("multi", [False, True])
def test_built_indexes_through_remove_isolate_and_reuse(multi):
    rng = np.random.default_rng(2)
    index = _built("f32", n=1500, d=24, multi=multi)
    per_keys = (1, 2, 3, 5)
    assert_lookups_match(index, _asked(index, rng), per_keys=per_keys, removed=False)
    index.remove(np.arange(0, 500, 7, dtype=np.uint64))
    assert_lookups_match(index, _asked(index, rng, extra=range(0, 50)), per_keys=per_keys)
    index.remove(np.arange(1, 500, 11, dtype=np.uint64), compact=True)
    assert_lookups_match(index, _asked(index, rng, extra=range(0, 50)), per_keys=per_keys)
    index.reuse_removed = True
    index.add(np.arange(5000, 5100, dtype=np.uint64) % (5000 + 40 if multi else 10**9), _vectors(100, 24, "f32", 9))
    assert_lookups_match(index, _asked(index, rng, extra=range(5000, 5100)), per_keys=per_keys)


def test_multi_key_with_a_thousand_entries():
    index = Index(ndim=16, metric="l2sq", dtype="f32", multi=True)
    many = 10**6
    keys = np.where(np.arange(3000) % 3 == 0, many, np.arange(3000)).astype(np.uint64)
    index.add(keys, _vectors(3000, 16, "f32", 4))
    asked = np.array([many, 1, many, 2, 10**9, 0], dtype=np.uint64)
    assert index.count(many) == 1000
    assert_lookups_match(index, asked, kinds=["f32", "f16"], per_keys=(1, 7, 1000, 1003), removed=False)
    index.remove([many])
    index.reuse_removed = True
    index.add(np.full(600, many, dtype=np.uint64), _vectors(600, 16, "f32", 5))  # into removed slots, in the queue's order
    assert_lookups_match(index, asked, per_keys=(1, 7, 600, 700))


def test_empty_index_and_argument_checks():
    torch = _torch()
    index = Index(ndim=8, metric="l2sq", dtype="f32")
    keys = np.array([0, 1, FREE_KEY], dtype=np.uint64)
    assert count_device(index, keys).tolist() == [0, 0, 0]
    rows, counts = get_device(index, keys, 2, "f32")
    assert counts.tolist() == [0, 0, 0] and not rows.any()
    index.add(np.arange(10, dtype=np.uint64), _vectors(10, 8, "f32", 1))
    d_keys = _on_device(keys)
    out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(3, dtype=torch.int32, device="cuda")
    err = C.c_char_p()
    index._lib.usearch_b200_get_many_device(index._h, d_keys.data_ptr(), 3, 1, out.data_ptr(), 0, 99, counts.data_ptr(), None,
                                            C.byref(err))
    assert err.value == b"Unknown scalar kind!"
    with pytest.raises(RuntimeError, match="stride is smaller"):
        index.get_device(d_keys.data_ptr(), 3, out.data_ptr(), counts.data_ptr(), stride=16)
    index.get_device(d_keys.data_ptr(), 0, out.data_ptr(), counts.data_ptr())  # count == 0: nothing to do
    index.count_device(d_keys.data_ptr(), 0, counts.data_ptr())
    # a strided output: the bytes between rows stay untouched, for a cast and without one
    for kind in ("f32", "f16"):
        row = _row_bytes(index, kind)
        rows, counts = get_device(index, keys, 2, kind, stride=row + 16)
        want, _ = host_get_many(index, keys, 2, kind)
        assert rows[:, :, :row].tobytes() == want.tobytes() and (rows[:, :, row:] == 0x5A).all()


def test_memory_usage_counts_the_table_once_built():
    index = _built("f32", n=1000, d=16)
    before = index.memory_usage
    count_device(index, np.arange(5, dtype=np.uint64))
    assert index.memory_usage == before + 2048 * 16  # 1000 live entries: 2048 cells of 16 bytes
    assert index.copy().memory_usage == before
    index.clear()
    assert index.memory_usage == 0


def test_stale_tables_are_rebuilt():
    rng = np.random.default_rng(5)
    index = _built("f32", n=800, d=16)
    check = lambda ix, extra=(): assert_lookups_match(ix, _asked(ix, rng, extra=extra), per_keys=(1, 2))  # noqa: E731
    check(index)
    index.add(np.arange(800, 900, dtype=np.uint64), _vectors(100, 16, "f32", 6))
    check(index, range(790, 910))
    index.remove(np.arange(0, 50, dtype=np.uint64))
    check(index, range(0, 60))
    index.reuse_removed = True
    index.add(np.arange(10**6, 10**6 + 30, dtype=np.uint64), _vectors(30, 16, "f32", 7))
    check(index, range(10**6, 10**6 + 40))
    index.remove(np.arange(50, 90, dtype=np.uint64), compact=True)
    check(index, range(40, 100))
    assert index.rename(100, 7) == 1
    check(index, [7, 100])
    index.reserve(index.capacity * 4)  # a capacity regrow
    check(index)
    index.add(np.arange(2000, 2000 + index.capacity, dtype=np.uint64), _vectors(index.capacity, 16, "f32", 8))  # grows on add
    check(index, [2000, 2000 + 500])
    blob = index.save()
    index.load(blob)
    check(index)
    other = index.copy()
    index.remove(np.arange(100, 200, dtype=np.uint64))
    other.rename(150, 10**9)
    other.add(np.array([151 + 10**9], dtype=np.uint64), _vectors(1, 16, "f32", 9))
    check(index, [150, 10**9, 151 + 10**9])
    check(other, [150, 10**9, 151 + 10**9])
    assert count_device(index, np.array([150, 10**9], dtype=np.uint64)).tolist() == [0, 0]
    assert count_device(other, np.array([150, 10**9], dtype=np.uint64)).tolist() == [0, 1]
    index.clear()
    check(index)
    index.add(np.arange(10, dtype=np.uint64), _vectors(10, 16, "f32", 10))
    check(index, range(12))


def _filtered_device(index, queries, k, allowed):
    torch = _torch()
    nq = queries.shape[0]
    d_q = _on_device(queries)
    d_allowed = _on_device(np.asarray(allowed, dtype=np.uint64)) if len(allowed) else None
    keys = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    dists = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    counts, computed, visited = (torch.zeros(nq, dtype=torch.int32, device="cuda") for _ in range(3))
    index.filtered_search_device(d_q.data_ptr(), nq, queries.strides[0], k, d_allowed.data_ptr() if d_allowed is not None else 0,
                                 len(allowed), keys.data_ptr(), dists.data_ptr(), counts.data_ptr(), computed.data_ptr(),
                                 visited.data_ptr())
    return (keys.cpu().numpy().view(np.uint64), dists.cpu().numpy(), counts.cpu().numpy().view(np.uint32),
            computed.cpu().numpy().view(np.uint32), visited.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("metric,kind,d,multi", [("cos", "f32", 64, False), ("ip", "f32", 96, False), ("l2sq", "f32", 33, False),
                                                 ("l2sq", "i8", 40, False), ("hamming", "b1", 77, False),
                                                 ("l2sq", "f64", 24, False), ("l2sq", "f32", 20, True)])
def test_filtered_search_equals_the_host_path(metric, kind, d, multi):
    n, k, nq = 2000, 10, 48
    index = Index(ndim=d, metric=metric, dtype=kind, multi=multi)
    keys = np.arange(n, dtype=np.uint64) % (n // 2) if multi else np.arange(n, dtype=np.uint64)
    if kind == "i8":
        base = np.random.default_rng(3).integers(-100, 100, (n, d)).astype(np.int8)
        queries = np.random.default_rng(4).integers(-100, 100, (nq, d)).astype(np.int8)
    else:
        base, queries = _vectors(n, d, kind, 3), _vectors(nq, d, kind, 4)
    index.add(keys, base)
    index.remove(np.arange(0, 300, 3, dtype=np.uint64))
    if metric in ("cos", "ip"):
        assert index.launch_plan(k)["prefilter"]
    rng = np.random.default_rng(6)
    live = np.asarray(index.keys)
    sets = {"empty": [], "every": np.unique(live), "some": rng.choice(live, 300),
            "odd": np.concatenate([rng.choice(live, 50), rng.choice(live, 50),
                                   np.array([10**12, 2**63 + 1, FREE_KEY, 0, 3, 6, 9], dtype=np.uint64)])}
    for name, allowed in sets.items():
        allowed = np.asarray(allowed, dtype=np.uint64)
        want = index.filtered_search(queries, k, allowed)
        got = _filtered_device(index, queries, k, allowed)
        assert np.array_equal(got[2], want.counts.astype(np.uint32)), name
        for q in range(nq):
            c = int(want.counts[q])
            assert np.array_equal(got[0][q, :c], want.keys[q, :c]), name
            assert np.array_equal(got[1][q, :c].view(np.uint32), want.distances[q, :c].view(np.uint32)), name
        assert np.array_equal(got[3], index.last_computed.astype(np.uint32)), name
        assert np.array_equal(got[4], index.last_visited.astype(np.uint32)), name


def test_search_then_get_pipeline():
    torch = _torch()
    index = _built("f32", n=3000, d=48)
    index.remove(np.arange(0, 3000, 5, dtype=np.uint64))
    queries = _vectors(64, 48, "f32", 11)
    nq, k = 64, 10
    d_q = _on_device(queries)
    keys = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    dists = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    counts = torch.zeros(nq, dtype=torch.int32, device="cuda")
    index.search_device(d_q.data_ptr(), nq, queries.strides[0], k, keys.data_ptr(), dists.data_ptr(), counts.data_ptr())
    for kind in ("f32", "f16"):
        rows, found = get_device(index, np.zeros(nq * k, np.uint64), 1, kind, d_keys=keys.reshape(-1))
        host_keys = keys.cpu().numpy().view(np.uint64).reshape(-1)
        want = index.get(host_keys, kind).view(np.uint8).reshape(nq * k, 1, -1)
        valid = (np.arange(k)[None, :] < counts.cpu().numpy()[:, None]).reshape(-1)
        assert found[valid].tolist() == [1] * int(valid.sum())
        assert rows[valid].tobytes() == want[valid].tobytes()


def test_a_non_default_stream():
    torch = _torch()
    index = _built("f16", n=1000, d=32)
    stream = torch.cuda.Stream()
    base = _on_device(np.arange(0, 1200, 3, dtype=np.uint64))
    with torch.cuda.stream(stream):
        torch.cuda._sleep(20_000_000)  # the keys are written late on this stream
        keys = base * 1 + 1
        rows, counts = get_device(index, np.zeros(len(base), np.uint64), 2, "f32", d_keys=keys, stream=stream.cuda_stream)
        n_counts = torch.full((len(base),), -1, dtype=torch.int32, device="cuda")
        index.count_device(keys.data_ptr(), len(base), n_counts.data_ptr(), stream=stream.cuda_stream)
    stream.synchronize()
    host = np.arange(0, 1200, 3, dtype=np.uint64) + 1
    assert np.array_equal(n_counts.cpu().numpy().view(np.uint32), index.count(host).astype(np.uint32))
    want, want_counts = host_get_many(index, host, 2, "f32")
    assert np.array_equal(counts, want_counts) and rows.tobytes() == want.tobytes()
