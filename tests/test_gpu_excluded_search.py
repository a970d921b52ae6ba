"""Excluded search: `excluded_search` and `grouped_excluded_search`, graph and exact, and the device entry. Query i searches
the live entries whose key is NOT in its set.

Every row is held to code that already exists:
- `grouped_filtered_search` of the same handle with the complement allowed set (every live key not in the set): keys,
  distance bits, counts and both counters, graph and exact;
- for f32 graphs, the pinned reference's `filtered_search` with the complement;
- for the exact form, the unmodified `search(exact=True)` of a fresh index holding only the non-excluded live entries in
  slot order (the tie order, larger slot first, is kept);
- plain `search` / `search(exact=True)` for an empty set.
"""
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


def _live(index):
    return np.unique(np.asarray(index.keys))


def _complement(index, excluded):
    return np.setdiff1d(_live(index), np.asarray(excluded, np.uint64))


def _counters(index):
    return index.last_computed.copy(), index.last_visited.copy()


def _excluded(index, queries, k, sets, groups=None, exact=False):
    got = index.grouped_excluded_search(queries, k, sets, groups, exact=exact)
    return (np.asarray(got.keys), np.asarray(got.distances), np.asarray(got.counts, np.uint64), *_counters(index))


def _allowed(index, queries, k, sets, groups=None, exact=False):
    """the same rows through grouped filtered search with the complement of every set"""
    got = index.grouped_filtered_search(queries, k, [_complement(index, s) for s in sets], groups, exact=exact)
    return (np.asarray(got.keys), np.asarray(got.distances), np.asarray(got.counts, np.uint64), *_counters(index))


def _assert_rows(want, got, what, padding=False):
    """bit for bit up to each row's count (and past it with `padding`), counts and both counters"""
    assert np.array_equal(np.asarray(want[2], np.uint64), np.asarray(got[2], np.uint64)), f"{what}: counts"
    for i in range(len(want[2])):
        c = want[0].shape[1] if padding else int(want[2][i])
        assert np.array_equal(want[0][i, :c], got[0][i, :c]), f"{what}: keys of row {i}"
        assert np.array_equal(want[1][i, :c].view(np.uint32), got[1][i, :c].view(np.uint32)), f"{what}: distances of row {i}"
    if len(want) > 3 and len(got) > 3:
        assert np.array_equal(np.asarray(want[3], np.uint64), np.asarray(got[3], np.uint64)), f"{what}: computed_distances"
        assert np.array_equal(np.asarray(want[4], np.uint64), np.asarray(got[4], np.uint64)), f"{what}: visited_members"


def _fresh_exact(index, metric, queries, k, excluded):
    """search(exact=True) of a fresh index holding the live entries outside `excluded`, in slot order"""
    keys = np.asarray(index.keys)
    keep = keys[~np.isin(keys, np.asarray(excluded, np.uint64))]
    fresh = Index(ndim=index.ndim, metric=metric, dtype=index._dtype)
    fresh.reuse_removed = False
    if len(keep):
        fresh.add(keep, index.get(keep))
    got = fresh.search(queries, k, exact=True)
    return np.asarray(got.keys), np.asarray(got.distances), np.asarray(got.counts, np.uint64)


def _mixed_sets(index, rng):
    live = _live(index)
    pick = lambda n: rng.choice(live, min(n, len(live)), replace=False)  # noqa: E731
    return [np.zeros(0, np.uint64), pick(1), pick(50), pick(max(len(live) * 3 // 4, 1)),
            np.concatenate([pick(20), pick(20), np.array([10**12, FREE_KEY, 2**63 + 7], np.uint64)])]


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_rows_equal_the_complement(name):
    index, blob, queries = _golden(name)
    rng = np.random.default_rng(21)
    nq = len(queries)
    if name.startswith("cos_f32"):
        assert index.launch_plan(10)["prefilter"]
    shared = _mixed_sets(index, rng)[:3] + [_mixed_sets(index, rng)[4]]
    shared_groups = rng.integers(0, len(shared), nq).astype(np.uint32)
    pool = _mixed_sets(index, rng)
    per_query = [pool[i % len(pool)] if i % 3 else rng.choice(_live(index), 30) for i in range(nq)]
    for sets, groups, what in ((shared, shared_groups, "shared sets"), (per_query, None, "a set per query")):
        g = np.arange(nq) if groups is None else groups
        graph = _excluded(index, queries, 10, sets, groups)
        _assert_rows(_allowed(index, queries, 10, sets, groups), graph, f"{name} graph, {what}")
        exact = _excluded(index, queries, 10, sets, groups, exact=True)
        _assert_rows(_allowed(index, queries, 10, sets, groups, exact=True), exact, f"{name} exact, {what}", padding=True)
        if "_f32_" in name and common.have_reference():
            from oracle import bindings
            ref = bindings.RefIndex("parity")
            ref.load(blob)
            ref.pin_metric(True)
            ref.change_expansion_search(index.expansion_search)
            for s in np.unique(g)[:40]:
                rows = np.nonzero(g == s)[0]
                want = ref.filtered_search(queries[rows].astype(np.float32), 10, _complement(index, sets[s]))
                _assert_rows(want, tuple(np.asarray(x)[rows] for x in graph), f"{name} vs reference, set {s}")
    # the exact form against a fresh index of the entries left, at counts on both sides of the register merge
    for k in (1, 10, 257):
        got = _excluded(index, queries, k, shared, shared_groups, exact=True)
        for s in range(len(shared)):
            rows = np.nonzero(shared_groups == s)[0]
            want = _fresh_exact(index, name.split("_")[0], queries[rows], k, shared[s])
            _assert_rows(want, tuple(x[rows] for x in got[:3]), f"{name} fresh index k={k} set {s}", padding=True)
            assert (got[3][rows] == len(_complement(index, shared[s]))).all(), f"{name}: computed of set {s}"
            assert not got[4][rows].any()
    # prefilter off: the same rows
    if name.startswith("cos_f32"):
        index.tune(prefilter=0)
        _assert_rows(_allowed(index, queries, 10, shared, shared_groups), _excluded(index, queries, 10, shared, shared_groups),
                     name + " prefilter=0")
        index.tune(prefilter=1)


@pytest.mark.parametrize("name", ["cos_f32_n2000_d64.npz", "ip_f32_n1500_d48_removed.npz", "hamming_b1_n4000_d256.npz"])
def test_empty_set_is_plain_search_and_every_key_leaves_nothing(name):
    index, _, queries = _golden(name)
    nq = len(queries)
    plain = index.search(queries, 10, stats=True)
    want = (plain.keys, plain.distances, plain.counts, *_counters(index))
    _assert_rows(want, _excluded(index, queries, 10, [[]], np.zeros(nq, np.uint32)), f"{name}: empty set")
    one = index.excluded_search(queries, 10, [])
    _assert_rows(want, (one.keys, one.distances, one.counts, *_counters(index)), f"{name}: empty set, one-set entry")
    plain = index.search(queries, 10, exact=True)
    got = _excluded(index, queries, 10, [[]], np.zeros(nq, np.uint32), exact=True)
    _assert_rows((plain.keys, plain.distances, plain.counts), got[:3], f"{name}: empty set, exact", padding=True)
    assert (got[3] == len(index)).all() and not got[4].any()
    for exact in (False, True):
        got = index.excluded_search(queries, 10, _live(index), exact=exact)
        assert not np.asarray(got.counts).any(), f"{name}: every live key excluded, exact={exact}"
        if exact:  # padded as search(exact=True) pads: key 0 and a signalling NaN
            assert not np.asarray(got.keys).any() and (np.asarray(got.distances).view(np.uint32) == 0x7FA00000).all()
            assert not index.last_computed.any()


def test_edge_sets_shapes_and_half_queries():
    index, _, queries = _golden("ip_f32_n1500_d48_removed.npz")
    live = _live(index)
    removed_keys = np.setdiff1d(np.arange(1500, dtype=np.uint64), live)
    assert len(removed_keys)
    sets = [np.repeat(live[:40], 3), np.array([10**15, 2**63, FREE_KEY], np.uint64), np.array([FREE_KEY], np.uint64),
            removed_keys, np.concatenate([removed_keys[:10], live[:5]]), live[:3], live[5:]]
    groups = (np.arange(len(queries)) % len(sets)).astype(np.uint32)
    for k in (1, 10, 64):
        _assert_rows(_allowed(index, queries, k, sets, groups), _excluded(index, queries, k, sets, groups), f"graph k={k}")
        _assert_rows(_allowed(index, queries, k, sets, groups, exact=True), _excluded(index, queries, k, sets, groups, exact=True),
                     f"exact k={k}", padding=True)
    # a set of only absent, free or removed keys changes nothing
    for s in (1, 2, 3):
        rows = np.nonzero(groups == s)[0]
        plain = index.search(queries[rows], 10, stats=True)
        _assert_rows((plain.keys, plain.distances, plain.counts, *_counters(index)),
                     _excluded(index, queries[rows], 10, [sets[s]], np.zeros(len(rows), np.uint32)), f"set {s} changes nothing")
    # f16 queries into an f32 index
    q16 = queries.astype(np.float16)
    for exact in (False, True):
        _assert_rows(_allowed(index, q16, 10, sets, groups, exact), _excluded(index, q16, 10, sets, groups, exact), f"f16 exact={exact}")
    # one 1-D query, and no queries
    for exact in (False, True):
        one = index.excluded_search(queries[0], 10, live[:100], exact=exact)
        ref = index.filtered_search(queries[0], 10, live[100:], exact=exact)
        assert np.array_equal(one.keys, ref.keys) and np.array_equal(one.distances.view(np.uint32), ref.distances.view(np.uint32))
        assert index.excluded_search(queries[:0], 10, live[:3], exact=exact).keys.shape == (0, 10)
        assert index.grouped_excluded_search(queries[:0], 10, [], None, exact=exact).keys.shape == (0, 10)


def test_gpu_built_multi_index_counts_slots():
    rng = np.random.default_rng(22)
    n, d = 3000, 20
    rows = rng.standard_normal((n, d)).astype(np.float32)
    keys = (np.arange(n) % 700).astype(np.uint64)
    keys[:400] = 5  # one key with hundreds of entries
    index = Index(ndim=d, metric="l2sq", dtype="f32", multi=True)
    index.add(keys, rows)
    queries = rng.standard_normal((70, d)).astype(np.float32)
    sets = [np.array([5], np.uint64), np.array([5, 5, 6, 10**9], np.uint64), np.arange(0, 700, 3, dtype=np.uint64), np.zeros(0, np.uint64)]
    groups = (np.arange(len(queries)) % len(sets)).astype(np.uint32)
    _assert_rows(_allowed(index, queries, 10, sets, groups), _excluded(index, queries, 10, sets, groups), "multi graph")
    for k in (10, 300):
        got = _excluded(index, queries, k, sets, groups, exact=True)
        _assert_rows(_allowed(index, queries, k, sets, groups, exact=True), got, f"multi exact k={k}", padding=True)
        for s in range(len(sets)):
            sel = np.nonzero(groups == s)[0]
            keep = ~np.isin(keys, sets[s])
            fresh = Index(ndim=d, metric="l2sq", dtype="f32", multi=True)
            fresh.add(keys[keep], rows[keep])
            want = fresh.search(queries[sel], k, exact=True)
            _assert_rows((want.keys, want.distances, np.asarray(want.counts, np.uint64)), tuple(x[sel] for x in got[:3]),
                         f"multi fresh k={k} set {s}", padding=True)
            assert (got[3][sel] == keep.sum()).all(), f"computed of set {s}: the live entries less the excluded slots"


def test_buckets_on_both_sides_of_256_equal_one_bucket_at_a_time():
    index, _, queries = _golden("l2sq_f32_n2000_d33.npz")
    rng = np.random.default_rng(23)
    live = _live(index)
    sizes = [0, 3, 40, 200, 250, 600, 1500]  # k + e from 11 to past 1024
    sets = [rng.choice(live, s, replace=False) for s in sizes]
    groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
    for k in (10, 250):
        got = _excluded(index, queries, k, sets, groups, exact=True)
        _assert_rows(_allowed(index, queries, k, sets, groups, exact=True), got, f"k={k}", padding=True)
        for s in range(len(sets)):  # each set alone: one bucket per call
            rows = np.nonzero(groups == s)[0]
            alone = _excluded(index, queries[rows], k, [sets[s]], np.zeros(len(rows), np.uint32), exact=True)
            _assert_rows(alone, tuple(x[rows] for x in got), f"k={k} set {s} alone", padding=True)


def test_rounds_equal_one_round():
    index, _, queries = _golden("cos_f32_n2000_d64.npz")
    rng = np.random.default_rng(24)
    sets = [rng.choice(_live(index), int(rng.integers(0, 800))) for _ in range(40)]
    groups = rng.integers(0, 40, len(queries)).astype(np.uint32)
    groups[:5] = 39
    one = _excluded(index, queries, 10, sets, groups)
    launches = index.kernel_launches
    index.tune(group_bitmap_mb=0)  # one set per round
    many = _excluded(index, queries, 10, sets, groups)
    assert index.kernel_launches - launches > 2 * len(np.unique(groups))
    _assert_rows(one, many, "one set per round")
    _assert_rows(_allowed(index, queries, 10, sets, groups), many, "complement, one set per round")


def test_scratch_retries_in_a_subprocess():
    """Undersized scratch makes queries overflow; every round retries its own failed ids."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import numpy as np\n"
        "from test_gpu_excluded_search import _golden, _excluded, _allowed, _assert_rows, _live\n"
        "index, _, queries = _golden('cos_f32_n2000_d64.npz')\n"
        "rng = np.random.default_rng(25)\n"
        "sets = [rng.choice(_live(index), int(rng.integers(1, 1500))) for _ in range(6)]\n"
        "groups = rng.integers(0, 6, len(queries)).astype(np.uint32)\n"
        "want = _allowed(index, queries, 10, sets, groups)\n"
        "_assert_rows(want, _excluded(index, queries, 10, sets, groups), 'one round')\n"
        "before = index.kernel_launches\n"
        "index.tune(group_bitmap_mb=0)\n"
        "_assert_rows(want, _excluded(index, queries, 10, sets, groups), 'rounds')\n"
        "print('launches', index.kernel_launches - before)\n"
    ) % (common.ROOT, os.path.join(common.ROOT, "tests"))
    env = dict(os.environ, USEARCH_B200_VISITED="hash", USEARCH_B200_SCRATCH_SHRINK="64")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    # validation, sort (3) and per round a row build, a search and at least one retry
    assert int(out.stdout.split("launches")[1].split()[0]) > 4 + 6 * 2, out.stdout


def _torch():
    import torch
    return torch


def _csr(sets):
    offsets = np.zeros(len(sets) + 1, np.uint64)
    offsets[1:] = np.cumsum([len(s) for s in sets])
    flat = np.concatenate([np.asarray(s, np.uint64) for s in sets]) if sets else np.zeros(0, np.uint64)
    return offsets, flat


def _device_call(index, queries, k, groups, sets, exact, stream=0, prepare=None):
    torch = _torch()
    nq = len(queries)
    offsets, flat = _csr(sets)
    d_q = torch.from_numpy(np.ascontiguousarray(queries)).cuda()
    d_groups = torch.from_numpy(np.asarray(groups, np.int64).astype(np.int32)).cuda() if groups is not None else None
    d_offsets = torch.from_numpy(offsets.view(np.int64)).cuda()
    d_keys_in = torch.from_numpy(np.ascontiguousarray(flat).view(np.int64)).cuda()
    keys = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    dists = torch.full((nq, k), 7, dtype=torch.float32, device="cuda")
    counts, computed, visited = (torch.full((nq,), 7, dtype=torch.int32, device="cuda") for _ in range(3))
    if prepare:
        d_groups, d_keys_in = prepare(d_groups, d_keys_in)
    index.grouped_excluded_search_device(d_q.data_ptr(), nq, queries.strides[0], k, d_groups.data_ptr() if d_groups is not None else 0,
                                         d_offsets.data_ptr(), len(sets), d_keys_in.data_ptr(), keys.data_ptr(), dists.data_ptr(),
                                         counts.data_ptr(), computed.data_ptr(), 0 if exact else visited.data_ptr(), stream=stream,
                                         exact=exact)
    torch.cuda.synchronize()
    keys, dists, counts, computed, visited = (t.cpu().numpy() for t in (keys, dists, counts, computed, visited))
    visited = np.zeros_like(visited) if exact else visited
    return keys.view(np.uint64), dists, counts.view(np.uint32), computed.view(np.uint32), visited.view(np.uint32)


def _built(n=2500, d=32, seed=26):
    rng = np.random.default_rng(seed)
    index = Index(ndim=d, metric="l2sq", dtype="f32")
    index.add(np.arange(n, dtype=np.uint64), rng.standard_normal((n, d)).astype(np.float32))
    return index, rng.standard_normal((200, d)).astype(np.float32)


@pytest.mark.parametrize("exact", [False, True])
def test_device_entry_on_a_stream_after_a_kernel(exact):
    torch = _torch()
    index, queries = _built()
    rng = np.random.default_rng(27)
    sets = _mixed_sets(index, rng)
    groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
    want = _excluded(index, queries, 10, sets, groups, exact)
    stream = torch.cuda.Stream()

    def late(d_groups, d_keys):  # the groups and keys are written by kernels queued on the caller's stream
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)
            g = d_groups * 1
            k = d_keys * 1
        return g, k
    got = _device_call(index, queries, 10, groups, sets, exact, stream=stream.cuda_stream, prepare=late)
    _assert_rows(want, got, f"device entry exact={exact}", padding=exact)
    # one set without groups
    one = index.excluded_search(queries, 10, sets[3], exact=exact)
    got = _device_call(index, queries, 10, None, [sets[3]], exact)
    _assert_rows((one.keys, one.distances, one.counts, *_counters(index)), got, f"device one set exact={exact}", padding=exact)


def test_device_entries_follow_edits():
    index, queries = _built(n=2000, d=16)
    rng = np.random.default_rng(28)

    def check(ix, what):
        sets = _mixed_sets(ix, rng) + [np.arange(0, 120, dtype=np.uint64), np.array([10**9, 10**9 + 1], np.uint64)]
        groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
        for exact in (False, True):
            _assert_rows(_allowed(ix, queries, 10, sets, groups, exact), _device_call(ix, queries, 10, groups, sets, exact),
                         f"{what} exact={exact}")
    check(index, "built")
    index.add(np.arange(5000, 5100, dtype=np.uint64), rng.standard_normal((100, 16)).astype(np.float32))
    check(index, "add")
    index.remove(np.arange(0, 100, dtype=np.uint64))
    check(index, "remove")
    index.remove(np.arange(100, 160, 3, dtype=np.uint64), compact=True)
    check(index, "remove and compact")
    assert index.rename(170, 10**9) == 1
    check(index, "rename")
    other = index.copy()
    other.remove(np.arange(200, 300, dtype=np.uint64))
    check(other, "copy")
    check(index, "original")


def test_refusals_leave_outputs_untouched():
    import ctypes as C
    torch = _torch()
    index, _, queries = _golden("l2sq_f32_n2000_d33.npz")
    nq, k = 6, 5
    q = np.ascontiguousarray(queries[:nq])
    lib = index._lib

    def host(entry, groups, offsets, sets_count, flat, count=k):
        keys = np.full((nq, count), 7, np.uint64)
        dists = np.full((nq, count), 3.0, np.float32)
        counts, computed, visited = (np.full(nq, 9, np.uint64) for _ in range(3))
        err = C.c_char_p()
        extra = [] if "exact" in entry else [visited.ctypes.data_as(C.c_void_p)]
        getattr(lib, entry)(index._h, q.ctypes.data_as(C.c_void_p), nq, q.strides[0], 1, count,
                            None if groups is None else groups.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                            sets_count, flat.ctypes.data_as(C.c_void_p), keys.ctypes.data_as(C.c_void_p),
                            dists.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p),
                            computed.ctypes.data_as(C.c_void_p), *extra, C.byref(err))
        assert err.value, f"{entry}: not refused"
        assert (keys == 7).all() and (dists == 3.0).all() and (counts == 9).all() and (computed == 9).all() and (visited == 9).all()
        return err.value.decode()

    def device(exact, groups, offsets, sets_count, flat, message, ix=index, qq=q, count=k):
        keys = torch.full((nq, count), 7, dtype=torch.int64, device="cuda")
        dists = torch.full((nq, count), 3.0, dtype=torch.float32, device="cuda")
        counts, computed, visited = (torch.full((nq,), 9, dtype=torch.int32, device="cuda") for _ in range(3))
        dq = torch.as_tensor(qq).cuda()
        dg = torch.as_tensor(groups.view(np.int32)).cuda() if groups is not None else None
        do = torch.as_tensor(offsets.view(np.int64)).cuda()
        df = torch.as_tensor(flat.view(np.int64)).cuda() if flat.size else torch.zeros(1, dtype=torch.int64, device="cuda")
        with pytest.raises(RuntimeError, match=message):
            ix.grouped_excluded_search_device(dq.data_ptr(), nq, qq.strides[0], count, dg.data_ptr() if dg is not None else 0,
                                              do.data_ptr(), sets_count, df.data_ptr(), keys.data_ptr(), dists.data_ptr(),
                                              counts.data_ptr(), computed.data_ptr(), 0 if exact else visited.data_ptr(), exact=exact)
        torch.cuda.synchronize()
        assert (keys == 7).all() and (dists == 3.0).all() and (counts == 9).all() and (computed == 9).all() and (visited == 9).all()

    flat = np.arange(10, dtype=np.uint64)
    good_offsets = np.array([0, 4, 10], np.uint64)
    cases = [(np.array([0, 1, 2, 0, 1, 0], np.uint32), good_offsets, 2, "out of range"),
             (np.zeros(nq, np.uint32), np.array([1, 4, 10], np.uint64), 2, "start at 0"),
             (np.zeros(nq, np.uint32), np.array([0, 6, 4], np.uint64), 2, "never decrease"),
             (np.zeros(nq, np.uint32), np.array([0], np.uint64), 0, "at least one key set"),
             (None, good_offsets, 2, "exactly one key set")]
    entries = [("usearch_b200_grouped_excluded_search_many", False), ("usearch_b200_grouped_excluded_exact_search_many", True)]
    for entry, exact in entries:
        for groups, offsets, sets_count, message in cases:
            assert message in host(entry, groups, offsets, sets_count, flat)
            device(exact, groups, offsets, sets_count, flat, message)
    # count > 256 on f32 rows past the tiled exact stage: exact search's own refusal, here reached through k + e
    rng = np.random.default_rng(29)
    d = 4096
    big = Index.restore(__import__("float_exact_reference").blob("f32", rng.standard_normal((400, d)).astype(np.float32), "cos", d))
    assert np.array_equal(np.asarray(big.keys), np.arange(400))
    bq = rng.standard_normal((nq, d)).astype(np.float32)
    small, large = np.arange(0, 40, dtype=np.uint64), np.arange(0, 300, dtype=np.uint64)
    got = big.excluded_search(bq, 10, small, exact=True)  # k + e <= 256 is served
    want = big.filtered_search(bq, 10, np.arange(40, 400, dtype=np.uint64), exact=True)
    assert np.array_equal(got.keys, want.keys) and np.array_equal(got.distances.view(np.uint32), want.distances.view(np.uint32))
    with pytest.raises(RuntimeError, match="count > 256 needs vectors that fit the tiled stage"):
        big.excluded_search(bq, 10, large, exact=True)
    device(True, None, np.array([0, 300], np.uint64), 1, large, "count > 256", ix=big, qq=bq)
    # a sharded handle holds one shard of its index: every entry refuses it, even with good arguments
    index.join_shards(0, 1, bytes(128))
    for entry, exact in entries:
        assert "sharded handle" in host(entry, np.zeros(nq, np.uint32), good_offsets, 2, flat)
        device(exact, np.zeros(nq, np.uint32), good_offsets, 2, flat, "sharded handle")
        device(exact, None, good_offsets[:2], 1, flat, "sharded handle")


def test_empty_index_and_memory_usage():
    index = Index(ndim=16, metric="l2sq", dtype="f32")
    queries = np.ones((3, 16), np.float32)
    for exact in (False, True):
        got = index.grouped_excluded_search(queries, 4, [[1, 2], []], [0, 1, 1], exact=exact)
        assert got.counts.tolist() == [0, 0, 0] and not got.keys.any() and index.last_computed.tolist() == [0, 0, 0]
    index, queries = _built(n=1000, d=16)
    before = index.memory_usage
    index.grouped_excluded_search(queries, 10, [np.arange(5, dtype=np.uint64)] * 3, np.arange(len(queries)) % 3)
    assert index.memory_usage >= before + 3 * ((1000 + 31) // 32) * 4
    index.clear()
    assert index.memory_usage == 0
