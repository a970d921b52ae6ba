"""Grouped filtered search: a key set per query, one launch. Every row is held to `filtered_search` of the same handle with
that row's set (keys, distance bits, counts and both counters), and for f32 to the pinned reference's filtered search,
on golden and GPU-built graphs, through edits, rounds, scratch retries, the device entry and its refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest

import common
from usearch_b200.index import Index

pytestmark = pytest.mark.gpu

FREE_KEY = 2**64 - 1
GOLDEN = ["cos_f32_n2000_d64.npz", "l2sq_f32_n2000_d33.npz", "ip_f32_n1500_d48_removed.npz", "ip_i8_n2000_d64.npz",
          "hamming_b1_n4000_d256.npz", "tanimoto_b1_n2000_d96.npz"]


def _golden(name):
    z = np.load(os.path.join(common.GOLDEN, name))
    index = Index.restore(z["blob"])
    index.expansion_search = int(z["ef"])
    return index, z["blob"], z["queries"]


def _per_query(index, queries, k, sets, groups):
    """the rows of `filtered_search`, one query at a time, with its counters"""
    nq = len(queries)
    keys, dists = np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float32)
    counts, computed, visited = (np.zeros(nq, np.uint64) for _ in range(3))
    for i in range(nq):
        got = index.filtered_search(queries[i:i + 1], k, np.asarray(sets[groups[i]], dtype=np.uint64))
        keys[i], dists[i], counts[i] = got.keys[0], got.distances[0], got.counts[0]
        computed[i], visited[i] = index.last_computed[0], index.last_visited[0]
    return keys, dists, counts, computed, visited


def _grouped(index, queries, k, sets, groups):
    got = index.grouped_filtered_search(queries, k, sets, groups)
    return got.keys, got.distances, got.counts, index.last_computed.copy(), index.last_visited.copy()


def _assert_rows(want, got, what):
    """bit-for-bit, with the padding past each row's count ignored (the single-set host path leaves it as allocated)"""
    kw, dw, cw = want[0], want[1], want[2]
    kg, dg, cg = got[0], got[1], got[2]
    assert np.array_equal(cw.astype(np.uint64), cg.astype(np.uint64)), f"{what}: counts"
    for i in range(len(cw)):
        c = int(cw[i])
        assert np.array_equal(kw[i, :c], kg[i, :c]), f"{what}: keys of row {i}"
        assert np.array_equal(dw[i, :c].view(np.uint32), dg[i, :c].view(np.uint32)), f"{what}: distances of row {i}"
    assert np.array_equal(np.asarray(want[3], np.uint64), np.asarray(got[3], np.uint64)), f"{what}: computed_distances"
    assert np.array_equal(np.asarray(want[4], np.uint64), np.asarray(got[4], np.uint64)), f"{what}: visited_members"


def _mixed_sets(index, rng, extra=()):
    live = np.unique(np.asarray(index.keys))
    pick = lambda n: rng.choice(live, min(n, len(live)), replace=False)  # noqa: E731
    return [np.zeros(0, np.uint64), pick(1), pick(50), pick(max(len(live) * 3 // 4, 1)),
            np.concatenate([pick(20), pick(20), np.array([10**12, FREE_KEY, 2**63 + 7], np.uint64)]), *extra]


@pytest.mark.parametrize("name", GOLDEN)
def test_one_set_equals_filtered_search(name):
    index, _, queries = _golden(name)
    rng = np.random.default_rng(1)
    live = np.asarray(index.keys)
    allowed = rng.choice(live, len(live) // 3, replace=False)
    if name.startswith("cos_f32"):
        assert index.launch_plan(10)["prefilter"]
    groups = np.zeros(len(queries), np.uint32)
    want = index.filtered_search(queries, 10, allowed)
    want = (want.keys, want.distances, want.counts, index.last_computed.copy(), index.last_visited.copy())
    _assert_rows(want, _grouped(index, queries, 10, [allowed], groups), name)


@pytest.mark.parametrize("name", GOLDEN)
@pytest.mark.parametrize("shared", [True, False])
def test_a_set_per_query_and_shared_sets(name, shared):
    index, blob, queries = _golden(name)
    rng = np.random.default_rng(2)
    nq = len(queries)
    if shared:
        sets = _mixed_sets(index, rng)[:3]
        groups = rng.integers(0, 3, nq).astype(np.uint32)
    else:
        pool = _mixed_sets(index, rng)
        sets = [pool[i % len(pool)] if i % 3 else rng.choice(np.asarray(index.keys), 30) for i in range(nq)]
        groups = None
    g = np.arange(nq) if groups is None else groups
    got = _grouped(index, queries, 10, sets, groups)
    _assert_rows(_per_query(index, queries, 10, sets, g), got, name)
    if "_f32_" in name and common.have_reference():
        from oracle import bindings
        ref = bindings.RefIndex("parity")
        ref.load(blob)
        ref.pin_metric(True)
        ref.change_expansion_search(index.expansion_search)
        for s in np.unique(g):
            rows = np.nonzero(g == s)[0]
            want = ref.filtered_search(queries[rows].astype(np.float32), 10, np.asarray(sets[s], np.uint64))
            _assert_rows(want, tuple(np.asarray(x)[rows] for x in got), f"{name} vs reference, set {s}")
    if name.startswith("cos_f32"):
        index.tune(prefilter=0)
        _assert_rows(_per_query(index, queries, 10, sets, g), _grouped(index, queries, 10, sets, groups), name + " prefilter=0")
        index.tune(prefilter=1)


def test_edge_sets():
    index, _, queries = _golden("ip_f32_n1500_d48_removed.npz")
    live = np.asarray(index.keys)
    removed_keys = np.setdiff1d(np.arange(1500, dtype=np.uint64), live)
    sets = [np.repeat(live[:40], 3), np.array([10**15, 2**63, FREE_KEY], np.uint64), np.array([FREE_KEY], np.uint64),
            removed_keys, np.concatenate([removed_keys[:10], live[:5]]), live[:3], np.unique(live)]
    groups = np.arange(len(queries)) % len(sets)
    for k in (1, 10, 64):  # k above the size of some sets
        _assert_rows(_per_query(index, queries, k, sets, groups), _grouped(index, queries, k, sets, groups), f"k={k}")
    # every live key: the plain search's rows
    everything = _grouped(index, queries, 10, [np.unique(live)], np.zeros(len(queries), np.uint32))
    plain = index.search(queries, 10, stats=True)
    _assert_rows((plain.keys, plain.distances, plain.counts, index.last_computed, index.last_visited), everything, "every key")
    # no queries; one 1-D query
    empty = index.grouped_filtered_search(queries[:0], 10, [], None)
    assert empty.keys.shape == (0, 10)
    one = index.grouped_filtered_search(queries[0], 10, [live[:100]])
    ref = index.filtered_search(queries[0], 10, live[:100])
    assert np.array_equal(one.keys, ref.keys) and np.array_equal(one.distances.view(np.uint32), ref.distances.view(np.uint32))


def test_half_queries_into_an_f32_index():
    index, _, queries = _golden("l2sq_f32_n2000_d33.npz")
    rng = np.random.default_rng(3)
    sets = _mixed_sets(index, rng)
    groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
    q16 = queries.astype(np.float16)
    _assert_rows(_per_query(index, q16, 10, sets, groups), _grouped(index, q16, 10, sets, groups), "f16 queries")


def _built(n=3000, d=24, multi=False, seed=5):
    rng = np.random.default_rng(seed)
    index = Index(ndim=d, metric="l2sq", dtype="f32", multi=multi)
    keys = np.arange(n, dtype=np.uint64) % (n // 3) if multi else np.arange(n, dtype=np.uint64)
    index.add(keys, rng.standard_normal((n, d)).astype(np.float32))
    return index, rng.standard_normal((200, d)).astype(np.float32)


@pytest.mark.parametrize("multi", [False, True])
def test_gpu_built_graphs_and_removals(multi):
    index, queries = _built(multi=multi)
    rng = np.random.default_rng(6)
    check = lambda what: _assert_rows(  # noqa: E731
        _per_query(index, queries, 10, sets, groups), _grouped(index, queries, 10, sets, groups), what)
    sets = _mixed_sets(index, rng, extra=[np.arange(0, 40, dtype=np.uint64)])
    groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
    check("built")
    index.remove(np.arange(0, 300, 4, dtype=np.uint64))
    check("removed")
    index.remove(np.arange(1, 300, 9, dtype=np.uint64), compact=True)
    check("removed and compacted")


def test_rounds_equal_one_round():
    index, _, queries = _golden("cos_f32_n2000_d64.npz")
    rng = np.random.default_rng(7)
    sets = [rng.choice(np.asarray(index.keys), int(rng.integers(0, 800))) for _ in range(40)]
    groups = rng.integers(0, 40, len(queries)).astype(np.uint32)
    groups[:5] = 39  # the last round, and rounds without queries in between
    one = _grouped(index, queries, 10, sets, groups)
    launches = index.kernel_launches
    index.tune(group_bitmap_mb=0)  # one set per round
    many = _grouped(index, queries, 10, sets, groups)
    assert index.kernel_launches - launches > 2 * len(np.unique(groups))
    _assert_rows(one, many, "one set per round")
    _assert_rows(_per_query(index, queries, 10, sets, groups), many, "per query")


def test_scratch_retries_in_a_subprocess():
    """Undersized scratch makes queries overflow; each round retries exactly its own failed ids."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import numpy as np, common\n"
        "from test_gpu_grouped_filter import _golden, _grouped, _per_query, _assert_rows\n"
        "index, _, queries = _golden('cos_f32_n2000_d64.npz')\n"
        "rng = np.random.default_rng(8)\n"
        "sets = [rng.choice(np.asarray(index.keys), int(rng.integers(1, 1500))) for _ in range(6)]\n"
        "groups = rng.integers(0, 6, len(queries)).astype(np.uint32)\n"
        "want = _per_query(index, queries, 10, sets, groups)\n"
        "_assert_rows(want, _grouped(index, queries, 10, sets, groups), 'one round')\n"
        "before = index.kernel_launches\n"
        "index.tune(group_bitmap_mb=0)\n"
        "_assert_rows(want, _grouped(index, queries, 10, sets, groups), 'rounds')\n"
        "print('launches', index.kernel_launches - before)\n"
    ) % (common.ROOT, os.path.join(common.ROOT, "tests"))
    env = dict(os.environ, USEARCH_B200_VISITED="hash", USEARCH_B200_SCRATCH_SHRINK="64")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    # rounds of 6 sets: validation, sort (3) and per round a bitmap build, a search and at least one retry
    assert int(out.stdout.split("launches")[1].split()[0]) > 4 + 6 * 2, out.stdout


def _torch():
    import torch
    return torch


def _csr(sets):
    offsets = np.zeros(len(sets) + 1, np.uint64)
    offsets[1:] = np.cumsum([len(s) for s in sets])
    flat = np.concatenate([np.asarray(s, np.uint64) for s in sets]) if sets else np.zeros(0, np.uint64)
    return offsets, flat


def _device_call(index, queries, k, groups, offsets, flat, sets_count=None, stream=0, prepare=None):
    torch = _torch()
    nq = len(queries)
    d_q = torch.from_numpy(np.ascontiguousarray(queries)).cuda()
    d_groups = torch.from_numpy(np.asarray(groups, np.int64).astype(np.int32)).cuda()
    d_offsets = torch.from_numpy(offsets.view(np.int64)).cuda()
    d_keys_in = torch.from_numpy(np.ascontiguousarray(flat).view(np.int64)).cuda()
    keys = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    dists = torch.full((nq, k), 7, dtype=torch.float32, device="cuda")
    counts, computed, visited = (torch.full((nq,), 7, dtype=torch.int32, device="cuda") for _ in range(3))
    if prepare:
        d_groups, d_keys_in = prepare(d_groups, d_keys_in)
    index.grouped_filtered_search_device(d_q.data_ptr(), nq, queries.strides[0], k, d_groups.data_ptr(), d_offsets.data_ptr(),
                                         len(offsets) - 1 if sets_count is None else sets_count, d_keys_in.data_ptr(),
                                         keys.data_ptr(), dists.data_ptr(), counts.data_ptr(), computed.data_ptr(),
                                         visited.data_ptr(), stream=stream)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in (keys, dists, counts, computed, visited))


def _as_rows(raw):
    keys, dists, counts, computed, visited = raw
    return keys.view(np.uint64), dists, counts.view(np.uint32), computed.view(np.uint32), visited.view(np.uint32)


def test_device_entry_on_a_stream_after_a_kernel():
    torch = _torch()
    index, queries = _built(n=2500, d=32)
    rng = np.random.default_rng(9)
    sets = _mixed_sets(index, rng)
    groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
    offsets, flat = _csr(sets)
    want = _grouped(index, queries, 10, sets, groups)
    stream = torch.cuda.Stream()

    def late(d_groups, d_keys):  # the groups and keys are written by kernels queued on the caller's stream
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)
            g = d_groups * 1
            k = d_keys * 1
        return g, k
    got = _device_call(index, queries, 10, groups, offsets, flat, stream=stream.cuda_stream, prepare=late)
    _assert_rows(want, _as_rows(got), "device entry")


def test_device_entry_follows_edits():
    index, queries = _built(n=2000, d=16)
    rng = np.random.default_rng(10)

    def check(ix, what):
        sets = _mixed_sets(ix, rng, extra=[np.arange(0, 120, dtype=np.uint64), np.array([10**9, 10**9 + 1], np.uint64)])
        groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
        offsets, flat = _csr(sets)
        _assert_rows(_per_query(ix, queries, 10, sets, groups), _as_rows(_device_call(ix, queries, 10, groups, offsets, flat)), what)
    check(index, "built")
    index.add(np.arange(5000, 5100, dtype=np.uint64), rng.standard_normal((100, 16)).astype(np.float32))
    check(index, "add")
    index.remove(np.arange(0, 100, dtype=np.uint64))
    check(index, "remove")
    assert index.rename(150, 10**9) == 1
    check(index, "rename")
    other = index.copy()
    other.remove(np.arange(100, 200, dtype=np.uint64))
    check(other, "copy")
    check(index, "original")


def test_refusals_leave_outputs_untouched():
    index, queries = _built(n=1000, d=16)
    sets = [np.arange(10, dtype=np.uint64), np.arange(10, 20, dtype=np.uint64)]
    offsets, flat = _csr(sets)
    cases = {
        "out of range": (np.array([0, 2] * 100, np.uint32), offsets, None, "key set index is out of range"),
        "decreasing": (np.zeros(200, np.uint32), np.array([0, 10, 5], np.uint64), None, "offsets"),
        "not from 0": (np.zeros(200, np.uint32), np.array([3, 10, 20], np.uint64), None, "offsets"),
        "no sets": (np.zeros(200, np.uint32), offsets, 0, "at least one key set"),
    }
    for what, (groups, offs, count, message) in cases.items():
        with pytest.raises(RuntimeError, match=message):
            _device_call(index, queries, 10, groups, offs, flat, sets_count=count)
        torch = _torch()
        # the device entry raised before writing: run again into fresh outputs and look at them
        keys = torch.full((len(queries), 10), 7, dtype=torch.int64, device="cuda")
        counts = torch.full((len(queries),), 7, dtype=torch.int32, device="cuda")
        d_q = torch.from_numpy(queries).cuda()
        d_g = torch.from_numpy(groups.astype(np.int32)).cuda()
        d_o = torch.from_numpy(offs.view(np.int64)).cuda()
        d_k = torch.from_numpy(flat.view(np.int64)).cuda()
        with pytest.raises(RuntimeError, match=message):
            index.grouped_filtered_search_device(d_q.data_ptr(), len(queries), queries.strides[0], 10, d_g.data_ptr(), d_o.data_ptr(),
                                                 2 if count is None else count, d_k.data_ptr(), keys.data_ptr(), keys.data_ptr(),
                                                 counts.data_ptr())
        torch.cuda.synchronize()
        assert (keys.cpu().numpy() == 7).all() and (counts.cpu().numpy() == 7).all(), what
    # the host entry, through the C ABI with the Python checks bypassed
    import ctypes as C
    from usearch_b200.index import SCALAR_KIND
    keys = np.full((len(queries), 10), 7, np.uint64)
    for groups, offs in ((np.array([0, 2] * 100, np.uint32), offsets), (np.zeros(200, np.uint32), np.array([0, 10, 5], np.uint64))):
        err = C.c_char_p()
        index._lib.usearch_b200_grouped_filtered_search_many(
            index._h, queries.ctypes.data_as(C.c_void_p), len(queries), queries.strides[0], SCALAR_KIND["f32"], 10,
            groups.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), 2, flat.ctypes.data_as(C.c_void_p),
            keys.ctypes.data_as(C.c_void_p), keys.ctypes.data_as(C.c_void_p), None, None, None, C.byref(err))
        assert err.value and (keys == 7).all()


def test_empty_index_and_memory_usage():
    index = Index(ndim=16, metric="l2sq", dtype="f32")
    queries = np.ones((3, 16), np.float32)
    got = index.grouped_filtered_search(queries, 4, [[1, 2], []], [0, 1, 1])
    assert got.counts.tolist() == [0, 0, 0] and not got.keys.any() and index.last_computed.tolist() == [0, 0, 0]
    index, queries = _built(n=1000, d=16)
    before = index.memory_usage
    index.grouped_filtered_search(queries, 10, [np.arange(5, dtype=np.uint64)] * 3, np.arange(len(queries)) % 3)
    assert index.memory_usage >= before + 3 * ((1000 + 31) // 32) * 4
    assert index.copy().memory_usage <= before
    index.clear()
    assert index.memory_usage == 0
