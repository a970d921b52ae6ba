"""Exact filtered search: `filtered_search(..., exact=True)` and `grouped_filtered_search(..., exact=True)` scan exactly the
live entries whose key is in the query's set (the reference's search_exact_ with the predicate).

Every expectation comes from code that already exists:
- the pinned port's exact search (tests/float_exact_reference.py, tests/i8_exact_reference.py) with the slots outside the
  set treated as removed, which is what a failing predicate is to search_exact_;
- an independent GPU path: the allowed live entries copied, in slot order, into a fresh index and searched with the
  unmodified `search(exact=True)`. Slot order is kept, so the tie order (larger slot first) is the same;
- `search(exact=True)` itself for a set holding every live key, and the single-set call for each row of a grouped one.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import common
from usearch_b200.index import Index

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FREE_KEY = 2**64 - 1
GOLDEN = ["cos_f32_n2000_d64.npz", "l2sq_f32_n2000_d33.npz", "ip_f32_n1500_d48_removed.npz", "ip_i8_n2000_d64.npz",
          "hamming_b1_n4000_d256.npz", "tanimoto_b1_n2000_d96.npz"]


def _golden(name):
    z = np.load(os.path.join(common.GOLDEN, name))
    index = Index.restore(z["blob"])
    return index, name.split("_")[0], z["queries"]


def _rows(got):
    return np.asarray(got.keys), np.asarray(got.distances), np.asarray(got.counts, np.uint64)


def _exact(index, queries, k, sets, groups=None):
    got = index.grouped_filtered_search(queries, k, sets, groups, exact=True)
    assert not np.asarray(index.last_visited).any()
    return (*_rows(got), index.last_computed.copy())


def _same(want, got, what):
    """keys, distance bits and counts, padding included"""
    assert np.array_equal(np.asarray(want[2], np.uint64), np.asarray(got[2], np.uint64)), f"{what}: counts"
    bad = np.argwhere((want[0] != got[0]) | (want[1].view(np.uint32) != got[1].view(np.uint32)))
    assert bad.size == 0, f"{what}: {bad.shape[0]} positions differ, first (query, position) {bad[:3].tolist()}"


def _fresh_exact(kind, metric, d, keys, rows, queries, k, multi=False):
    """the unmodified exact search of a fresh index holding exactly (keys, rows), in this order"""
    fresh = Index(ndim=d, metric=metric, dtype=kind, multi=multi)
    fresh.reuse_removed = False
    if len(keys):
        fresh.add(np.asarray(keys, np.uint64), rows)
    return _rows(fresh.search(queries, k, exact=True))


def _independent(index, kind, metric, queries, k, allowed):
    """a plain index: its live entries in slot order whose key is allowed, searched by a fresh index"""
    live = np.asarray(index.keys)
    keep = live[np.isin(live, np.asarray(allowed, np.uint64))]
    rows = index.get(keep) if len(keep) else None
    return _fresh_exact(kind, metric, index.ndim, keep, rows, queries, k), len(keep)


def _mixed_sets(live, rng):
    pick = lambda n: rng.choice(live, min(n, len(live)), replace=False)  # noqa: E731
    return [np.zeros(0, np.uint64), pick(1), pick(50), pick(max(len(live) * 3 // 4, 1)), np.unique(live),
            np.concatenate([pick(20), pick(20), np.array([10**12, FREE_KEY, 2**63 + 7], np.uint64)])]


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_sets_equal_a_fresh_index_of_the_set(name):
    index, metric, queries = _golden(name)
    kind = index._dtype
    rng = np.random.default_rng(11)
    live = np.asarray(index.keys)
    sets = _mixed_sets(live, rng)
    groups = rng.integers(0, len(sets), len(queries)).astype(np.uint32)
    for k in (1, 10, 257):
        got = _exact(index, queries, k, sets, groups)
        for s in np.unique(groups):
            rows = np.nonzero(groups == s)[0]
            want, size = _independent(index, kind, metric, queries[rows], k, sets[s])
            _same(want, tuple(x[rows] for x in got[:3]), f"{name} k={k} set {s}")
            assert (got[3][rows] == size).all(), f"{name}: computed_distances of set {s}"
    # a set per query, and the single-set call for every row
    per_query = [rng.choice(live, int(rng.integers(0, 300))) for _ in range(len(queries))]
    grouped = _exact(index, queries, 10, per_query)
    for i in range(0, len(queries), max(1, len(queries) // 12)):
        one = index.filtered_search(queries[i], 10, per_query[i], exact=True)
        n = len(one.keys)
        assert n == grouped[2][i] and np.array_equal(one.keys, grouped[0][i, :n])
        assert np.array_equal(one.distances.view(np.uint32), grouped[1][i, :n].view(np.uint32))
        assert index.last_computed[0] == grouped[3][i]
    # every live key: search(exact=True) bit for bit
    _same(_rows(index.search(queries, 10, exact=True)), _exact(index, queries, 10, [live], np.zeros(len(queries), np.uint32)),
          f"{name}: every live key")


def _tie_rows(rng, n, d, kind="f32"):
    """rows drawn from a small pool, so exact duplicates fall on every tile and segment boundary of any list"""
    pool = rng.integers(-16, 17, (40, d)) / 8.0
    rows = pool[rng.integers(0, len(pool), n)]
    rows[::7] += rng.integers(-1, 2, (len(rows[::7]), d)) / 64.0
    return rows.astype(np.float64 if kind == "f64" else np.float32)


@pytest.mark.parametrize("metric", ["l2sq", "ip", "cos"])
def test_f32_against_the_pinned_port(metric):
    import float_exact_reference as F
    rng = np.random.default_rng(12)
    n, d = 1500, 24
    rows = _tie_rows(rng, n, d)
    queries = np.concatenate([rows[:3], _tie_rows(rng, 37, d)])
    index = Index.restore(F.blob("f32", rows, metric, d))
    removed = np.zeros(n, bool)
    removed[rng.choice(n, 100, replace=False)] = True
    index.remove(np.nonzero(removed)[0].astype(np.uint64))
    allowed = np.zeros(n, bool)
    allowed[rng.choice(n, 700, replace=False)] = True
    allowed_keys = np.concatenate([np.nonzero(allowed)[0], np.nonzero(removed)[0][:10]]).astype(np.uint64)  # removed keys too
    for k in (1, 10, 24, 25, 256, 257, 700, 1000):
        want = F.pinned_search("f32", metric, rows, queries, k, d, removed=removed | ~allowed)
        got = _exact(index, queries, k, [allowed_keys], np.zeros(len(queries), np.uint32))
        _same(want, got[:3], f"{metric} k={k}")
        assert (got[3] == (allowed & ~removed).sum()).all()
        assert not F.check_topk("f32", metric, rows, queries, d, k, *got[:3], removed=removed | ~allowed)


def test_i8_against_the_numpy_statement():
    import i8_exact_reference as R
    rng = np.random.default_rng(13)
    n, d = 2000, 64
    rows = rng.integers(-8, 9, (n, d)).astype(np.int8)
    rows[1::9] = rows[0::9][: len(rows[1::9])]  # duplicates
    queries = rng.integers(-8, 9, (150, d)).astype(np.int8)
    for metric in ("ip", "l2sq", "cos"):
        index = Index(ndim=d, metric=metric, dtype="i8")
        index.add(np.arange(n, dtype=np.uint64), rows)
        index.remove(np.arange(0, n, 13, dtype=np.uint64))
        removed = np.zeros(n, bool)
        removed[::13] = True
        sets = [np.arange(0, 1000, dtype=np.uint64), rng.choice(n, 60).astype(np.uint64), np.arange(n, dtype=np.uint64)]
        groups = rng.integers(0, 3, len(queries)).astype(np.uint32)
        for k in (1, 10, 25, 256, 300):
            got = _exact(index, queries, k, sets, groups)
            for s in range(3):
                sel = np.nonzero(groups == s)[0]
                outside = ~np.isin(np.arange(n), sets[s])
                want = R.search(metric, rows, queries[sel], k, removed=removed | outside)
                _same(want, tuple(x[sel] for x in got[:3]), f"i8 {metric} k={k} set {s}")


@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_gpu_built_multi_index(kind):
    rng = np.random.default_rng(14)
    n, d = 3000, 20
    rows = _tie_rows(rng, n, d, kind)
    keys = (np.arange(n) % 700).astype(np.uint64)
    keys[:400] = 5  # one key with hundreds of entries
    index = Index(ndim=d, metric="l2sq", dtype=kind, multi=True)
    index.add(keys, rows)
    queries = _tie_rows(rng, 70, d, kind)
    sets = [np.array([5], np.uint64), np.array([5, 5, 6, 10**9], np.uint64), np.arange(0, 700, 3, dtype=np.uint64)]
    groups = (np.arange(len(queries)) % 3).astype(np.uint32)
    for k in (10, 300):
        got = _exact(index, queries, k, sets, groups)
        for s in range(3):
            sel = np.nonzero(groups == s)[0]
            keep = np.isin(keys, sets[s])
            want = _fresh_exact(kind, "l2sq", d, keys[keep], rows[keep], queries[sel], k, multi=True)
            _same(want, tuple(x[sel] for x in got[:3]), f"{kind} multi k={k} set {s}")
            assert (got[3][sel] == keep.sum()).all()


def test_shapes_query_counts_half_queries_and_rows_read_in_place():
    rng = np.random.default_rng(15)
    index, metric, queries = _golden("l2sq_f32_n2000_d33.npz")
    live = np.asarray(index.keys)
    allowed = rng.choice(live, 900, replace=False)
    for nq in (1, 3, 4, 5, 7, 8, 9, 31, 32, 33, 127, 128, 129, 300):
        q = queries[np.arange(nq) % len(queries)]
        want, _ = _independent(index, "f32", metric, q, 10, allowed)
        _same(want, _exact(index, q, 10, [allowed], np.zeros(nq, np.uint32))[:3], f"nq={nq}")
    # a batch equals its slices
    many = _exact(index, queries, 10, [allowed, live[:100]], (np.arange(len(queries)) % 2).astype(np.uint32))
    for lo in range(0, len(queries), 17):
        hi = min(lo + 17, len(queries))
        part = _exact(index, queries[lo:hi], 10, [allowed, live[:100]], (np.arange(lo, hi) % 2).astype(np.uint32))
        _same(tuple(x[lo:hi] for x in many[:3]), part[:3], f"slice {lo}")
    # f16 queries into an f32 index: cast as search(exact=True) casts them
    q16 = queries.astype(np.float16)
    want, _ = _independent(index, "f32", metric, q16, 10, allowed)
    _same(want, _exact(index, q16, 10, [allowed], np.zeros(len(q16), np.uint32))[:3], "f16 queries")
    # 4096-d f32 rows fit neither the tiled nor the staged scan: the listed scan reads them in place
    d = 4096
    big = Index.restore(__import__("float_exact_reference").blob("f32", _tie_rows(rng, 400, d), "cos", d))
    bq = _tie_rows(rng, 20, d)
    sub = np.arange(3, 400, 3, dtype=np.uint64)
    want, _ = _independent(big, "f32", "cos", bq, 10, sub)
    _same(want, _exact(big, bq, 10, [sub], np.zeros(20, np.uint32))[:3], "4096-d in place")


def test_empty_cases():
    index, _, queries = _golden("cos_f32_n2000_d64.npz")
    assert index.grouped_filtered_search(queries[:0], 10, [], None, exact=True).keys.shape == (0, 10)
    got = _exact(index, queries, 10, [np.zeros(0, np.uint64), np.array([FREE_KEY], np.uint64)],
                 (np.arange(len(queries)) % 2).astype(np.uint32))
    assert not got[2].any() and not got[0].any() and not got[3].any()
    assert (got[1].view(np.uint32) == 0x7FA00000).all()
    empty = Index(ndim=64, metric="cos", dtype="f32")
    got = empty.filtered_search(queries, 5, [1, 2], exact=True)
    assert not np.asarray(got.counts).any() and (got.distances.view(np.uint32) == 0x7FA00000).all()


def _boundary_ties(metric, rng, L=1024):
    """(rows, q, allowed): list position p is slot 2p + 1 (the odd keys are allowed). Exact duplicates of `a` straddle
    every multiple of 8 positions, and a row `b` one ulp farther (confirmed by the pinned metric) follows each pair. The
    near tie is built as in float_exact_reference.edge_cases; every other row points away from q."""
    import float_exact_reference as F
    d = 21
    j = (d - 1) % 16
    q = rng.standard_normal(d)
    q[-1] = 1e-3 if metric == "l2sq" else 1.0
    q[j] = 4.0
    if metric == "cos":
        q[0] = 0.0
    q = F.to_f64("f32", F.to_kind("f32", q[None]), d)[0]
    a = (q if metric == "l2sq" else 0) + 0.05 * rng.standard_normal(d)
    a[j], a[-1] = 8.0, 0.0
    if metric == "cos":
        a[j], a[0] = 1.0, 8.0
    a = F.to_f64("f32", F.to_kind("f32", a[None]), d)[0]
    a, b = F.near_tie("f32", metric, q, a, rng)
    rows = (-3 * q[None] + 0.1 * rng.standard_normal((2 * L, d))).astype(np.float32)
    for m in range(1, L // 8):
        p = 8 * m
        rows[2 * (p - 1) + 1] = rows[2 * p + 1] = a
        rows[2 * (p + 1) + 1] = b
    return rows, q.astype(np.float32), np.arange(1, 2 * L, 2, dtype=np.uint64)


def _boundary_expectation(metric, rows, q, k, L=1024):
    import float_exact_reference as F
    outside = np.ones(2 * L, bool)
    outside[1::2] = False
    want = F.pinned_search("f32", metric, rows, q[None], k, rows.shape[1], removed=outside)
    # the expectation itself: the 254 copies of `a` lead, larger slot first, then the 127 copies of `b`
    ties = np.array(sorted({2 * (8 * m + j) + 1 for m in range(1, L // 8) for j in (-1, 0)}, reverse=True), np.uint64)
    n = min(k, 254)
    assert np.array_equal(np.asarray(want[0])[0, :n], ties[:n])
    if k > 254:
        bs = np.arange(2 * (8 * 127 + 1) + 1, 0, -16, dtype=np.uint64)[:127]
        assert np.array_equal(np.asarray(want[0])[0, 254:min(k, 381)], bs[:min(k, 381) - 254])
    return want


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_ties_on_every_tile_and_segment_boundary_of_a_list(metric):
    """Tiles (8 rows for the scan, 16 for the tiled scan) and segments (a multiple of the tile: ceil(1024 / S) rounded up,
    S = 8 for this launch) all start or end inside a tie, so the partial lists of neighbouring segments hold tied entries
    that only the slot order separates."""
    rows, q, allowed = _boundary_ties(metric, np.random.default_rng(18))
    index = Index.restore(__import__("float_exact_reference").blob("f32", rows, metric, rows.shape[1]))
    queries = np.repeat(q[None], 40, 0)
    for k in (1, 2, 253, 254, 255, 256, 300, 400):
        want = _boundary_expectation(metric, rows, q, k)
        got = _exact(index, queries, k, [allowed], np.zeros(len(queries), np.uint32))
        _same(tuple(np.repeat(x, len(queries), 0) for x in want), got[:3], f"{metric} ties k={k}")


_CHOICE = r"""
import sys, hashlib; sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as np
from test_gpu_exact_filter import _golden, _exact
h = hashlib.sha256()
for name in sys.argv[1:]:
    index, _, queries = _golden(name)
    rng = np.random.default_rng(16)
    live = np.asarray(index.keys)
    sets = [rng.choice(live, 700, replace=False), live[:40], live]
    groups = rng.integers(0, 3, len(queries)).astype(np.uint32)
    for k in (1, 10, 24, 25, 256):
        for x in _exact(index, queries, k, sets, groups):
            h.update(np.ascontiguousarray(x).tobytes())
print("DIGEST", h.hexdigest())
"""


def _digest(choice, names):
    env = dict(os.environ)
    env.pop("USEARCH_B200_EXACT", None)
    if choice:
        env["USEARCH_B200_EXACT"] = choice
    out = subprocess.run([sys.executable, "-c", _CHOICE % (common.ROOT, HERE), *names], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout.split("DIGEST")[1].split()[0]


def test_every_kernel_choice_gives_the_same_bits():
    """USEARCH_B200_EXACT is read once per process: one subprocess per choice. wgmma cannot follow a list, so a filtered
    call under it runs the mma.sync kernel."""
    floats = ["l2sq_f32_n2000_d33.npz", "tanimoto_b1_n2000_d96.npz"]
    base = _digest(None, floats)
    for choice in ("scan", "tiled"):
        assert _digest(choice, floats) == base, choice
    ints = ["ip_i8_n2000_d64.npz"]
    base = _digest(None, ints)
    for choice in ("scan", "tiled", "imma", "wgmma"):
        assert _digest(choice, ints) == base, choice


def _torch():
    return pytest.importorskip("torch")


def _device_call(index, queries, k, flat, offsets, groups, stream=None):
    torch = _torch()
    nq = len(queries)
    q = torch.as_tensor(np.ascontiguousarray(queries)).cuda()
    keys = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    dists = torch.full((nq, k), 3.0, dtype=torch.float32, device="cuda")
    counts = torch.full((nq,), 9, dtype=torch.int32, device="cuda")
    computed = torch.full((nq,), 9, dtype=torch.int32, device="cuda")
    index.grouped_filtered_search_device(q.data_ptr(), nq, q.stride(0) * q.element_size(), k,
                                         groups.data_ptr() if groups is not None else 0, offsets.data_ptr(), offsets.numel() - 1,
                                         flat.data_ptr(), keys.data_ptr(), dists.data_ptr(), counts.data_ptr(), computed.data_ptr(),
                                         stream=stream or 0, exact=True)
    return (keys.cpu().numpy().view(np.uint64), dists.cpu().numpy(), counts.cpu().numpy().astype(np.uint64),
            computed.cpu().numpy().astype(np.uint64))


def _csr(sets):
    torch = _torch()
    offsets = np.zeros(len(sets) + 1, np.int64)
    offsets[1:] = np.cumsum([len(s) for s in sets])
    flat = np.concatenate([np.asarray(s, np.uint64) for s in sets]).view(np.int64) if sets else np.zeros(0, np.int64)
    return torch.as_tensor(flat).cuda(), torch.as_tensor(offsets).cuda()


def test_device_entry_equals_host_on_a_side_stream_and_after_edits():
    torch = _torch()
    rng = np.random.default_rng(17)
    d, n = 16, 2500
    rows = _tie_rows(rng, n, d)
    index = Index(ndim=d, metric="cos", dtype="f32")
    index.add(np.arange(n, dtype=np.uint64), rows)
    queries = _tie_rows(rng, 90, d)
    sets = [np.arange(0, 2500, 2, dtype=np.uint64), rng.choice(n, 40).astype(np.uint64), np.arange(100, dtype=np.uint64)]
    groups_np = rng.integers(0, 3, len(queries)).astype(np.uint32)

    def check(what, idx=index):
        host = _exact(idx, queries, 10, sets, groups_np)
        flat, offsets = _csr(sets)
        dev = _device_call(idx, queries, 10, flat, offsets, torch.as_tensor(groups_np.view(np.int32)).cuda())
        _same(host[:3], dev[:3], what)
        assert np.array_equal(host[3], dev[3]), what

    check("built")
    # a non-default stream, after a kernel on it writes the groups and the set keys
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        g = torch.zeros(len(queries), dtype=torch.int32, device="cuda")
        g += torch.as_tensor(groups_np.view(np.int32)).cuda()
        flat, offsets = _csr(sets)
        flat = flat * 1  # written on this stream
    dev = _device_call(index, queries, 10, flat, offsets, g, stream=side.cuda_stream)
    _same(_exact(index, queries, 10, sets, groups_np)[:3], dev[:3], "side stream")
    # one set and no groups: every query uses set 0
    flat1, offsets1 = _csr(sets[:1])
    _same(_exact(index, queries, 10, sets[:1], np.zeros(len(queries), np.uint32))[:3],
          _device_call(index, queries, 10, flat1, offsets1, None)[:3], "groups NULL")
    index.add(np.arange(n, n + 200, dtype=np.uint64), _tie_rows(rng, 200, d))
    sets[2] = np.arange(n - 50, n + 150, dtype=np.uint64)
    check("after add")
    index.remove(np.arange(0, 2500, 10, dtype=np.uint64))
    check("after remove")
    index.remove(np.arange(1, 2500, 30, dtype=np.uint64), compact=True)
    check("after remove with compact")
    index.rename(4, 10**10)
    sets[1] = np.concatenate([sets[1], np.array([10**10], np.uint64)])
    check("after rename")
    copy = index.copy()
    copy.remove(np.arange(2, 500, 2, dtype=np.uint64))
    check("copy after its own edit", copy)
    check("the original after the copy's edit")
    # the free-function path: `filtered_search_device` with exact
    q = torch.as_tensor(queries).cuda()
    allowed = torch.as_tensor(sets[0].view(np.int64)).cuda()
    keys = torch.zeros((len(queries), 10), dtype=torch.int64, device="cuda")
    dists = torch.zeros((len(queries), 10), dtype=torch.float32, device="cuda")
    counts = torch.zeros(len(queries), dtype=torch.int32, device="cuda")
    index.filtered_search_device(q.data_ptr(), len(queries), d * 4, 10, allowed.data_ptr(), allowed.numel(), keys.data_ptr(),
                                 dists.data_ptr(), counts.data_ptr(), exact=True)
    want = index.filtered_search(queries, 10, sets[0], exact=True)
    _same(_rows(want), (keys.cpu().numpy().view(np.uint64), dists.cpu().numpy(), counts.cpu().numpy().astype(np.uint64)), "device one set")


def test_refusals_leave_outputs_untouched():
    import ctypes as C
    torch = _torch()
    index, _, queries = _golden("l2sq_f32_n2000_d33.npz")
    nq, k = 6, 5
    q = np.ascontiguousarray(queries[:nq])
    lib = index._lib

    def host(groups, offsets, sets_count, flat):
        keys = np.full((nq, k), 7, np.uint64)
        dists = np.full((nq, k), 3.0, np.float32)
        counts = np.full(nq, 9, np.uint64)
        computed = np.full(nq, 9, np.uint64)
        err = C.c_char_p()
        lib.usearch_b200_grouped_filtered_exact_search_many(
            index._h, q.ctypes.data_as(C.c_void_p), nq, q.strides[0], 1, k,
            None if groups is None else groups.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), sets_count,
            flat.ctypes.data_as(C.c_void_p), keys.ctypes.data_as(C.c_void_p), dists.ctypes.data_as(C.c_void_p),
            counts.ctypes.data_as(C.c_void_p), computed.ctypes.data_as(C.c_void_p), C.byref(err))
        assert err.value, "not refused"
        assert (keys == 7).all() and (dists == 3.0).all() and (counts == 9).all() and (computed == 9).all()
        return err.value.decode()

    flat = np.arange(10, dtype=np.uint64)
    good_offsets = np.array([0, 4, 10], np.uint64)
    cases = [(np.array([0, 1, 2, 0, 1, 0], np.uint32), good_offsets, 2, "out of range"),
             (np.zeros(nq, np.uint32), np.array([1, 4, 10], np.uint64), 2, "start at 0"),
             (np.zeros(nq, np.uint32), np.array([0, 6, 4], np.uint64), 2, "never decrease"),
             (np.zeros(nq, np.uint32), np.array([0], np.uint64), 0, "at least one key set"),
             (None, good_offsets, 2, "exactly one key set")]

    def check(groups, offsets, sets_count, message):
        assert message in host(groups, offsets, sets_count, flat)
        keys = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
        dists = torch.full((nq, k), 3.0, dtype=torch.float32, device="cuda")
        counts = torch.full((nq,), 9, dtype=torch.int32, device="cuda")
        dq = torch.as_tensor(q).cuda()
        dg = torch.as_tensor(groups.view(np.int32)).cuda() if groups is not None else None
        do = torch.as_tensor(offsets.view(np.int64)).cuda() if offsets.size else torch.zeros(1, dtype=torch.int64, device="cuda")
        df = torch.as_tensor(flat.view(np.int64)).cuda()
        with pytest.raises(RuntimeError, match=message):
            index.grouped_filtered_search_device(dq.data_ptr(), nq, q.strides[0], k, dg.data_ptr() if dg is not None else 0,
                                                 do.data_ptr(), sets_count, df.data_ptr(), keys.data_ptr(), dists.data_ptr(),
                                                 counts.data_ptr(), exact=True)
        assert (keys == 7).all() and (dists == 3.0).all() and (counts == 9).all()

    for case in cases:
        check(*case)
    # a sharded handle holds one shard of its index: both entries refuse it, even with good arguments (a world of one
    # shard needs no communicator)
    index.join_shards(0, 1, bytes(128))
    check(np.zeros(nq, np.uint32), good_offsets, 2, "sharded handle")
    check(None, good_offsets[:2], 1, "sharded handle")
