"""The graph search on NaN, infinite, zero, subnormal and saturated distances, against the pinned reference.

Each family mixes edge rows (and queries of the same kinds) among latent rows, builds the graph with the reference,
and hands the same file to the pinned reference and to `Index.restore`. Every family runs under the default plan, a
heap head of 2 entries (the serial pop over the HBM tail), one warp per SM (pop_warp over large heads) and one or two
stage sets, at ef 64 (register `top`) and ef 300 (shared-memory `top`) with k in {1, 10, ef}. `filtered_search`,
`grouped_filtered_search`, `cluster` and `Indexes.search` run on the edge rows as well, and the builder's INSERT search
is held to the host model on edge rows. Every returned (query, key, distance) is also held to the float64 statement of
the metric."""
import numpy as np
import pytest

import common
import float_exact_reference as fx
import i8_exact_reference as i8x
import indexes_reference as ir
from oracle import bindings
from test_gpu_build_model import Build
from usearch_b200 import datagen

pytestmark = pytest.mark.gpu

PLAN_ERROR = "Expansion or dimensionality too large for on-chip state"
DEFAULT_KNOBS = {"stage_sets": 0, "warps_per_sm": 0, "prefilter": 1, "heap_head": 0}
SNAN_BITS = 0x7FA00000
FLT_MAX = float(np.finfo(np.float32).max)
F16_MAX, BF16_MAX = 65504.0, float(np.uint32(0x7F7F0000).view(np.float32))

# name: kind, metric, d, edge kinds of rows and queries
FAMILIES = {
    "l2sq_f32_32": ("f32", "l2sq", 32, ("nan", "huge", "zero", "subnormal", "dup")),
    "l2sq_f32_128": ("f32", "l2sq", 128, ("nan", "huge", "zero", "subnormal", "dup")),
    "ip_f32_128": ("f32", "ip", 128, ("nan", "mixed", "dup")),
    "ip_f32_97": ("f32", "ip", 97, ("nan", "mixed", "dup")),
    "cos_f32_128": ("f32", "cos", 128, ("nan", "zero", "subnormal", "dup")),
    "cos_f32_97": ("f32", "cos", 97, ("nan", "zero", "subnormal", "dup")),
    **{f"{m}_{k}_{d}": (k, m, d, ("inf", "nan", "maxfin", "zero")) for k in ("f16", "bf16") for m in ("l2sq", "ip", "cos")
       for d in (24, 256)},
    **{f"{m}_i8_{d}": ("i8", m, d, ("sat", "zero")) for m in ("l2sq", "ip", "cos") for d in (64, 1024)},
    **{f"{m}_b1_256": ("b1", m, 256, ("zeros", "ones")) for m in ("hamming", "tanimoto", "sorensen")},
}
# cos clamps an undefined value to 0 (`r > 0 ? r : 0`), so only l2sq, ip and sorensen return NaN
NAN_FAMILIES = {name for name, (kind, metric, d, edges) in FAMILIES.items()
                if metric in ("l2sq", "ip", "sorensen") and ("nan" in edges or "mixed" in edges or metric == "sorensen")}
PLANS = {
    "default": {},
    "heap_head=2": {"heap_head": 2},
    "warps_per_sm=1": {"warps_per_sm": 1},
    "stage_sets=1": {"stage_sets": 1},
    "stage_sets=2": {"stage_sets": 2},
}
N, NQ, M = 3000, 96, 16


# ---- edge rows --------------------------------------------------------------------------------------------------------

def _edge(kind, edge, d, rng):
    """one row of the edge kind, as float64 values (i8: integers, b1: 0 / 1)"""
    sign = rng.choice([-1.0, 1.0], d)
    if edge == "nan":
        x = rng.standard_normal(d)
        x[rng.choice(d, 1 + rng.integers(3), replace=False)] = np.nan
        return x
    if edge == "huge":  # l2sq: squares near 1e38..1e40, their sums past f32
        return sign * rng.uniform(1e19, 1e20, d)
    if edge == "mixed":  # ip: +-1e20 of mixed sign: products of +-1e40 overflow to +inf in some accumulators, -inf in others
        return sign * 1e20
    if edge in ("zero", "zeros"):
        return np.zeros(d)
    if edge == "ones":
        return np.ones(d)
    if edge == "subnormal":  # f32: below 2^-126
        return sign * rng.uniform(1, 8, d) * 2.0 ** -140
    if edge == "inf":
        x = rng.standard_normal(d)
        x[rng.choice(d, 1 + rng.integers(2), replace=False)] = rng.choice([-np.inf, np.inf])
        return x
    if edge == "maxfin":
        x = rng.standard_normal(d)
        top = F16_MAX if kind == "f16" else BF16_MAX
        x[rng.choice(d, 1 + rng.integers(3), replace=False)] = top * rng.choice([-1.0, 1.0])
        return x
    if edge == "sat":
        pick = rng.integers(4)
        return [np.full(d, -128.0), np.full(d, 127.0), np.full(d, -127.0), sign * 127.0][pick]
    raise ValueError(edge)


def _to_kind(kind, x):
    if kind == "i8":
        return np.asarray(x, np.int8)
    return fx.to_kind(kind, x)


def make_family(name, seed=11):
    """(rows, queries) in the family's stored kind: about a tenth of the rows and a third of the queries are edges"""
    kind, metric, d, edges = FAMILIES[name]
    rng = np.random.default_rng(seed)
    lat = datagen.latent(N + NQ, d, seed=seed, rank=min(16, d)).astype(np.float64)
    if kind == "i8":
        lat = datagen.to_scalar(lat.astype(np.float32), "i8").astype(np.float64)
    elif kind == "b1":
        lat = (lat > 0).astype(np.float64)
    rows, queries = lat[:N].copy(), lat[N:].copy()
    per_row, per_query = max(8, N // (10 * len(edges))), max(2, NQ // (3 * len(edges)))
    spots = rng.permutation(N)
    qspots = rng.permutation(NQ)
    for e, edge in enumerate(edges):
        for i in spots[e * per_row:(e + 1) * per_row]:
            if edge == "dup":
                rows[i] = rows[spots[-1 - (i % 7)]]
            else:
                rows[i] = _edge(kind, edge, d, rng)
        for i in qspots[e * per_query:(e + 1) * per_query]:
            queries[i] = rows[spots[-1 - (i % 7)]] if edge == "dup" else _edge(kind, edge, d, rng)
    with np.errstate(over="ignore", invalid="ignore"):
        return _to_kind(kind, rows), _to_kind(kind, queries)


# ---- the comparer -----------------------------------------------------------------------------------------------------

def assert_same_results(want, got, what):
    """(keys, distances, counts, computed, visited) equal bit for bit, with one exception: at a position below the
    count, a NaN distance matches a NaN of any payload. The reference on x86 returns 0xFFC00000 or a propagated payload,
    the GPU 0x7FFFFFFF; NaN payloads carry no meaning here, where a NaN sits and under which key does. Padding past the
    count stays exact: key 0 and the signalling-NaN bits 0x7FA00000."""
    wk, wd, wc = want[0], np.asarray(want[1], np.float32), np.asarray(want[2], np.uint64)
    gk, gd, gc = got[0], np.asarray(got[1], np.float32), np.asarray(got[2], np.uint64)
    assert np.array_equal(wc, gc), f"{what}: counts differ for {np.count_nonzero(wc != gc)} queries"
    bad = np.nonzero((wk != gk).any(axis=1))[0]
    assert bad.size == 0, f"{what}: labels differ for {bad.size} queries, first {bad[:5]}"
    below = np.arange(wd.shape[1])[None, :] < wc[:, None].astype(np.int64)
    both_nan = np.isnan(wd) & np.isnan(gd) & below
    diff = (wd.view(np.uint32) != gd.view(np.uint32)) & ~both_nan
    assert not diff.any(), f"{what}: distance bits differ at {np.argwhere(diff)[:5].tolist()}"
    assert (gd.view(np.uint32)[~below] == SNAN_BITS).all(), f"{what}: padding is not the signalling NaN"
    if len(want) > 3 and want[3] is not None:
        assert np.array_equal(np.asarray(want[3], np.uint64), np.asarray(got[3], np.uint64)), f"{what}: computed_distances differ"
        assert np.array_equal(np.asarray(want[4], np.uint64), np.asarray(got[4], np.uint64)), f"{what}: visited_members differ"


def _prefix(want, k):
    """the reference's result at k <= ef is the first k of its result at k = ef: the same `top`, dumped shorter"""
    keys, dists, counts, computed, visited = want
    return keys[:, :k], dists[:, :k], np.minimum(counts, k), computed, visited


# ---- the float64 statement --------------------------------------------------------------------------------------------

def _statement(kind, metric, rows, queries, d):
    """(distance, bound, regime) [nq, n] in float64. regime 0: the evaluation neither overflows nor underflows, so the
    distance must lie within `bound` (or be +-inf where the statement passes f32's range); 1: the accumulation can
    overflow or the norms underflow in the kernel's precision, so only the pinned pair is the judge; NaN statements
    require NaN."""
    if kind == "i8":
        ab, a2, b2 = i8x.triples(queries, rows)
        return i8x.distances(metric, ab, a2, b2).astype(np.float64), np.zeros(ab.shape), np.zeros(ab.shape, np.int8)
    with np.errstate(all="ignore"):
        dist, bound = fx.statement(kind, metric, rows, queries, d)
        if kind == "b1":
            return dist, bound, np.zeros(dist.shape, np.int8)
        a, b = fx.to_f64(kind, queries, d), fx.to_f64(kind, rows, d)
        top, tiny = 2.0 ** 126, 2.0 ** -100
        finite_a, finite_b = np.isfinite(a).all(1), np.isfinite(b).all(1)
        if metric == "l2sq":
            dist = np.stack([((a[i][None, :] - b) ** 2).sum(1) for i in range(a.shape[0])])
            s = dist
            # a term that underflows loses at most the smallest subnormal
            bound = np.nan_to_num(bound, nan=0.0, posinf=np.inf) + (d + 16) * 2.0 ** -149
        else:
            s = np.abs(np.nan_to_num(a)) @ np.abs(np.nan_to_num(b)).T
        regime = (~(finite_a[:, None] & finite_b[None, :]) | (s > top)).astype(np.int8)
        if metric == "cos":  # a norm that underflows to zero in the kernel's precision but not in the statement's
            a2, b2 = (a * a).sum(1), (b * b).sum(1)
            small = lambda x: (x > 0) & (x < tiny)  # noqa: E731
            regime |= (small(a2)[:, None] | small(b2)[None, :]).astype(np.int8)
            regime |= ((np.abs(a).max(1) < 2.0 ** -60)[:, None] & (a2 > 0)[:, None]).astype(np.int8)
            regime |= ((np.abs(b).max(1) < 2.0 ** -60)[None, :] & (b2 > 0)[None, :]).astype(np.int8)
            # the reference clamps with `r > 0 ? r : 0`: an undefined cosine is 0, never NaN
            undefined = np.isnan(dist)
            dist, bound = np.where(undefined, 0.0, dist), np.where(undefined, 0.0, bound)
            regime[undefined] = 0
    return dist, bound, regime


def held_to_statement(fam, rows, queries, keys, dists, counts, pinned):
    """every returned (query, key, distance): bits equal to the pinned metric of that pair (class for NaN), and the
    float64 statement: NaN where it is undefined, +-inf where it passes f32's range, within its bound elsewhere.
    Returns the number of pairs held to a bound, so that a caller can require some."""
    kind, metric, d, _ = FAMILIES[fam]
    dist, bound, regime = _statement(kind, metric, rows, queries, d)
    with np.errstate(invalid="ignore"):
        return _held(fam, dist, bound, regime, keys, dists, counts, pinned)


def _held(fam, dist, bound, regime, keys, dists, counts, pinned):
    checked = 0
    problems = []
    for i in range(keys.shape[0]):
        c = int(counts[i])
        ks = keys[i, :c].astype(np.int64)
        got = dists[i, :c]
        p = pinned[i, ks]
        same = (p.view(np.uint32) == got.view(np.uint32)) | (np.isnan(p) & np.isnan(got))
        if not same.all():
            problems.append(f"query {i}: key {ks[~same][0]} distance {got[~same][0]!r}, pinned {p[~same][0]!r}")
        st, bd, rg = dist[i, ks], bound[i, ks], regime[i, ks]
        g = got.astype(np.float64)
        undefined = np.isnan(st)
        if (undefined & ~np.isnan(g)).any():
            problems.append(f"query {i}: a number where the statement is undefined")
        plain = (rg == 0) & ~undefined
        over = plain & (np.abs(st) - bd > FLT_MAX)
        if (over & ~(np.isinf(g) & (np.sign(g) == np.sign(st)))).any():
            problems.append(f"query {i}: a finite distance where the statement passes f32's range")
        inside = plain & (np.abs(st) + bd < FLT_MAX)
        off = inside & ~(np.abs(g - st) <= bd)
        if off.any():
            j = int(np.argmax(off))
            problems.append(f"query {i}: key {ks[j]} distance {g[j]!r}, statement {st[j]!r} +- {bd[j]:.3g}")
        checked += int(inside.sum() + over.sum())
    assert not problems, f"{fam}: {len(problems)} problems, first: {problems[:3]}"
    return checked


def pinned_matrix(fam, rows, queries):
    kind, metric, d, _ = FAMILIES[fam]
    if kind == "i8":
        return i8x.distances(metric, *i8x.triples(queries, rows))
    with np.errstate(all="ignore"):
        return fx.pinned_matrix(kind, metric, rows, queries, d)


# ---- fixtures ---------------------------------------------------------------------------------------------------------

def _pinned_ref(blob, ef):
    ref = bindings.RefIndex("parity")
    ref.view(blob)
    ref.pin_metric(True)
    ref.change_expansion_search(ef)
    return ref


@pytest.fixture(scope="module")
def family():
    """per family, once: rows, queries, the reference-built graph, the pinned reference's results at ef 64 and 300"""
    from usearch_b200.index import Index
    cache = {}

    def get(name):
        if name not in cache:
            kind, metric, d, _ = FAMILIES[name]
            rows, queries = make_family(name)
            ref, blob = common.build_reference_blob(rows, metric, kind, d, M, threads=16)
            want = {ef: _pinned_ref(blob, ef).search(queries, ef, threads=16) for ef in (64, 300)}
            cache.clear()  # one family at a time: the handles hold device memory
            cache[name] = (rows, queries, blob, want, Index.restore(blob))
        return cache[name]

    yield get
    cache.clear()


def _search(index, q, k, knobs, ef, prefilter=1):
    index.tune(**{**DEFAULT_KNOBS, "prefilter": prefilter, **knobs})
    index.expansion_search = ef
    index.profile_phases(True)
    got = index.search(q, k, stats=True)
    phases = index.profile_phases(False)
    return (got.keys, got.distances, got.counts, index.last_computed, index.last_visited), phases


def _has_shadow(name):
    kind, metric = FAMILIES[name][:2]
    return kind == "f32" and metric in ("cos", "ip")


CASES = [(name, plan, pf) for name in FAMILIES for plan in PLANS for pf in ((1, 0) if _has_shadow(name) else (1,))]


@pytest.mark.parametrize("name,plan,prefilter", CASES)
def test_search_matches_pinned_reference(family, name, plan, prefilter):
    rows, queries, blob, want, index = family(name)
    forced = PLANS[plan]
    what = f"{name} [{plan}, prefilter={prefilter}]"
    index.tune(**{**DEFAULT_KNOBS, "prefilter": prefilter, **forced})
    for ef in (64, 300):
        index.expansion_search = ef
        try:
            lp = index.launch_plan(ef)
        except RuntimeError as e:  # a forced layout that does not fit is refused, never run differently
            assert str(e) == PLAN_ERROR and forced, f"{what}: {e}"
            continue
        saw_heap = 0
        for k in (1, 10, ef):
            got, ph = _search(index, queries, k, forced, ef, prefilter)
            assert_same_results(_prefix(want[ef], k), got, f"{what} ef={ef} k={k}")
            saw_heap = max(saw_heap, ph["max_heap"])
            if not (prefilter and _has_shadow(name)):
                assert ph["prefiltered"] == 0, what
        if "heap_head" in forced:
            assert lp["heap_smem_cap"] == 2 and saw_heap > 2, f"{what}: the heap never reached its HBM tail"
        if "warps_per_sm" in forced:
            assert lp["warps_per_sm_target"] <= 1, f"{what}: {lp}"
        if "stage_sets" in forced and lp["stage_bytes"]:
            assert lp["stage_sets"] == forced["stage_sets"], f"{what}: {lp}"
    if plan == "default" and prefilter == 1:
        keys, dists, counts = want[300][:3]
        if name in NAN_FAMILIES:
            below = np.arange(300)[None, :] < counts[:, None].astype(np.int64)
            assert (np.isnan(dists) & below).any(), f"{name}: no NaN distance reached `top`"
        checked = held_to_statement(name, rows, queries, keys, dists, counts, pinned_matrix(name, rows, queries))
        assert checked > 0, f"{name}: no pair was held to the float64 statement"


F32_FAMILIES = [name for name in FAMILIES if FAMILIES[name][0] == "f32"]


@pytest.mark.parametrize("plan", ["default", "heap_head=2"])
@pytest.mark.parametrize("name", F32_FAMILIES)
def test_filtered_and_grouped_search(family, name, plan):
    rows, queries, blob, _, index = family(name)
    k, ef = 10, 64
    keys = np.arange(N, dtype=np.uint64)
    half = np.random.default_rng(3).permutation(N)[: N // 2].astype(np.uint64)
    other = np.setdiff1d(keys, half)
    ref = _pinned_ref(blob, ef)
    want = ref.filtered_search(queries, k, half, threads=16)
    index.tune(**{**DEFAULT_KNOBS, **PLANS[plan]})
    index.expansion_search = ef
    got = index.filtered_search(queries, k, half)
    assert_same_results(want, (got.keys, got.distances, got.counts, index.last_computed, index.last_visited),
                        f"{name} filtered [{plan}]")
    groups = (np.arange(NQ) % 2).astype(np.uint32)
    per_set = [want, ref.filtered_search(queries, k, other, threads=16)]
    want_g = tuple(np.where((groups == 1)[:, None] if np.ndim(per_set[0][j]) == 2 else groups == 1, per_set[1][j], per_set[0][j])
                   for j in range(5))
    got = index.grouped_filtered_search(queries, k, [half, other], groups)
    assert_same_results(want_g, (got.keys, got.distances, got.counts, index.last_computed, index.last_visited),
                        f"{name} grouped [{plan}]")


@pytest.mark.parametrize("name", list(FAMILIES))
def test_cluster_matches_pinned_reference(family, name):
    rows, queries, blob, _, index = family(name)
    index.tune(**DEFAULT_KNOBS)
    wk, wd, wc, wv = _pinned_ref(blob, 64).cluster(queries, 1)
    gk, gd = index.cluster(queries, 1, stats=True)
    assert np.array_equal(wk, gk), f"{name}: cluster keys differ"
    assert np.array_equal(wd.view(np.uint32), gd.view(np.uint32)) or \
        ((wd.view(np.uint32) == gd.view(np.uint32)) | (np.isnan(wd) & np.isnan(gd))).all(), f"{name}: cluster distances"
    assert np.array_equal(wc, index.last_computed) and np.array_equal(wv, index.last_visited), f"{name}: cluster counters"


@pytest.mark.parametrize("name", ["l2sq_f32_128", "ip_f32_97", "cos_f16_256", "ip_bf16_24", "l2sq_i8_1024",
                                  "sorensen_b1_256"])
def test_indexes_over_two_shards(name):
    from usearch_b200.index import Index, Indexes
    kind, metric, d, _ = FAMILIES[name]
    rows, queries = make_family(name)
    k, ef, cut = 10, 64, N // 2
    blobs, refs = [], []
    for lo, hi in ((0, cut), (cut, N)):
        ref = bindings.RefIndex("parity", metric=metric, scalar=kind, dims=d, connectivity=M, expansion_add=128,
                                expansion_search=64)
        ref.add(np.arange(lo, hi, dtype=np.uint64), rows[lo:hi], threads=16)
        blobs.append(ref.save())
        refs.append(_pinned_ref(blobs[-1], ef))
    want = ir.reference_search(refs, queries, k, query_scalar=kind)
    members = [Index.restore(b) for b in blobs]
    for member in members:
        member.expansion_search = ef
    ix = Indexes(members)
    got = ix.search(queries, k)
    assert_same_results(want, (got.keys, got.distances, got.counts, ix.last_computed, ix.last_visited), f"{name} Indexes")


# ---- the builder on edge rows -----------------------------------------------------------------------------------------

def _build_rows(kind, metric, d, edges, n=2500, seed=5):
    rng = np.random.default_rng(seed)
    lat = datagen.latent(n, d, seed=seed, rank=min(16, d)).astype(np.float64)
    if kind == "i8":
        lat = datagen.to_scalar(lat.astype(np.float32), "i8").astype(np.float64)
    elif kind == "b1":
        lat = (lat > 0).astype(np.float64)
    spots = rng.permutation(n)
    per = n // (8 * len(edges))
    for e, edge in enumerate(edges):
        for i in spots[e * per:(e + 1) * per]:
            if edge == "zero-dup":  # zero rows, and duplicates of them
                lat[i] = 0.0
            else:
                lat[i] = _edge(kind, edge, d, rng)
    with np.errstate(over="ignore", invalid="ignore"):
        return _to_kind(kind, lat)


BUILD_CASES = {
    "zero-rows-f32-l2sq": ("f32", "l2sq", 32, ("zero-dup",)),
    "zero-rows-f32-cos": ("f32", "cos", 64, ("zero-dup",)),
    "subnormal-f32-cos": ("f32", "cos", 64, ("subnormal",)),
    "subnormal-f32-l2sq": ("f32", "l2sq", 32, ("subnormal",)),
    "overflow-f32-l2sq": ("f32", "l2sq", 32, ("huge",)),
    "saturated-i8-l2sq": ("i8", "l2sq", 1024, ("sat", "zero")),
    "saturated-i8-cos": ("i8", "cos", 64, ("sat", "zero")),
    "zeros-b1-hamming": ("b1", "hamming", 256, ("zeros",)),
    "zeros-b1-tanimoto": ("b1", "tanimoto", 256, ("zeros",)),
    "nan-f32-l2sq": ("f32", "l2sq", 32, ("nan",)),
    "inf-f16-l2sq": ("f16", "l2sq", 24, ("inf",)),
}


@pytest.mark.parametrize("name", list(BUILD_CASES))
def test_build_on_edge_rows_equals_the_model(name):
    kind, metric, d, edges = BUILD_CASES[name]
    rows = _build_rows(kind, metric, d, edges)
    b = Build(metric, kind, d)
    half = len(rows) // 2
    b.add(np.arange(half, dtype=np.uint64), rows[:half])
    b.add(np.arange(half, len(rows), dtype=np.uint64), rows[half:])
    assert b.total()["reverse_refines"] > 0, f"{name}: {b.total()}"
