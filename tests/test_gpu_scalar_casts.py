"""The scalar casts on the GPU, on the edge tables of scalar_cast_edges.py: the device casts of `add` and the casts of
`get` against scalar_casts.h's host casts (which tests/test_scalar_casts.py pins to the reference's own cast_gt over
every f32 pattern, and which are checked here against that cast_gt too where the reference sources are present), and
the query casts of every search entry against the reference searching with queries it cast itself.

NaN is compared as stored bytes only (add, get): in a search its distances order differently in the two result
containers, which is a separate question from the cast."""
import numpy as np
import pytest

import cast_reference as cr
import common
import indexes_reference as ir
import scalar_cast_edges as edges
from oracle import bindings

pytestmark = pytest.mark.gpu
needs_reference = pytest.mark.skipif(not common.have_reference(), reason="oracle/_ref not built")

METRIC = {"f16": "cos", "bf16": "cos", "i8": "cos", "b1": "hamming"}
KINDS = ("f64", "f32", "f16", "bf16", "i8", "b1")


def _f16_bits(n: int, d: int, seed: int) -> np.ndarray:
    """raw f16 rows: a quarter with the exponent all ones (the reference decodes those as finite 2^16 .. 2^17), a quarter
    zeros and subnormals, the rest any pattern"""
    w = np.random.default_rng(seed).integers(0, 1 << 16, size=(n, d), dtype=np.uint32).astype(np.uint16)
    w[::4] |= 0x7C00
    w[1::4] &= ~np.uint16(0x7C00)
    return w


def _source_rows(n: int, d: int, kind: str, seed: int) -> np.ndarray:
    """n rows in `kind` (f32, f64 or f16): edge rows, rows of exact f16 ties and rows of exact bf16 ties"""
    if kind == "f16":
        return _f16_bits(n, d, seed).view(np.float16)
    third = n // 3
    rows = np.concatenate([edges.edge_rows(third, d, seed), edges.tie_rows(third, d, "f16", seed),
                           edges.tie_rows(n - 2 * third, d, "bf16", seed)])
    if kind == "f32":
        return rows
    with np.errstate(invalid="ignore"):
        wide = rows.astype(np.float64)
    wide[:, ::3] *= 1 + 2.0 ** -40  # just off the f32 grid: narrowed to f32 before a half cast
    wide[::5, 1] = 1e39  # beyond the f32 range
    wide[1::7, 2] = 1e-320  # below it: > 0 for b1
    return wide


def _stored_matrix(blob: np.ndarray) -> np.ndarray:
    rows, cols = (int(v) for v in np.frombuffer(np.ascontiguousarray(blob[:8]).tobytes(), dtype=np.uint32))
    return np.asarray(blob[8:8 + rows * cols]).reshape(rows, cols)


def _first_difference(want: np.ndarray, got: np.ndarray, src: np.ndarray) -> str:
    r, c = (int(v) for v in np.argwhere(want != got)[0])
    raw = np.ascontiguousarray(src[r]).view(np.uint8)
    return f"row {r} byte {c}: source row bytes {raw[:32].tobytes().hex()}..., reference {want[r, c]:02x}, ours {got[r, c]:02x}"


ADD_CASES = [(to, src, d) for to in ("f16", "bf16", "i8", "b1") for src in ("f32", "f64", "f16") for d in (97, 768)
             if not (to == "b1" and d == 97)]  # b1 at a ragged width: see the test


@pytest.mark.parametrize("to,src,d", ADD_CASES)
def test_device_add_stores_what_the_reference_stores(to, src, d):
    """`add` of f32, f64 or f16 rows into an f16 / bf16 / i8 / b1 index casts them on the device (one thread per element,
    one per row for i8: 600 rows span several blocks of both kernels). The stored vector bytes of `save()` must equal
    cast_gt<src, to> of the same rows, which is what the reference's add_ stores (index_dense.hpp:2010-2018). A b1 index
    of a ragged width is left out: the reference ORs the last partial byte into its reused per-thread cast buffer, so a
    bit set by one row stays set in the rows that thread casts after it."""
    from usearch_b200.index import Index
    n = 600
    rows = _source_rows(n, d, src, seed=d + len(to))
    want = cr.host_cast(rows, src, to, d)
    if cr.reference_available():
        cr.assert_same_casts(cr.ref_cast(rows, src, to, d), want, rows, src, to, d, "host casts vs the reference")
    index = Index(ndim=d, metric=METRIC[to], dtype=to, connectivity=16)
    index.add(np.arange(n, dtype=np.uint64), rows)
    got = _stored_matrix(index.save())
    cr.assert_same_casts(want, got, rows, src, to, d, "device add")


def _bf16_nearest_even(x: np.ndarray) -> np.ndarray:
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def _tie_index(kind: str, d: int):
    n, m, ef = 3000, 16, 64
    base, _ = common.make_collection(n, d, kind, 8, seed=d)
    ref, blob = common.build_reference_blob(base, "cos", kind, d, m, threads=16)
    ref.pin_metric(True)
    ref.change_expansion_search(ef)
    return ref, blob, n, ef


@needs_reference
@pytest.mark.parametrize("kind,d", [("f16", 97), ("f16", 768), ("bf16", 97), ("bf16", 768)])
def test_tie_queries_search_like_the_reference(kind, d):
    """f32 queries whose every element is an exact tie of the index's half kind (finite): the device cast of every search
    entry -- graph search, filtered, exact, cluster, and an `Indexes` holding the index -- against the reference
    searching with the same f32 queries, cast by its own cast_gt. Labels, distance bits, counts and both counters."""
    from usearch_b200.index import Index, Indexes
    ref, blob, n, ef = _tie_index(kind, d)
    q = edges.tie_rows(300, d, kind, seed=d)
    q_cast = ir._cast_queries(ref, q, "f32")  # the reference's own cast of every row
    ieee = q.astype(np.float16).view(np.uint16) if kind == "f16" else _bf16_nearest_even(q)
    assert (q_cast.view(np.uint16) != ieee).mean() > 0.3, "the queries must be ties an IEEE cast rounds differently"
    index = Index.restore(blob)
    index.expansion_search = ef
    k = 10

    want = ref.filtered_search(q, k, np.arange(n, dtype=np.uint64), threads=16)  # every key allowed: search_(f32 const*)
    got = index.search(q, k, stats=True)
    common.assert_same_results(want, (got.keys, got.distances, got.counts, index.last_computed, index.last_visited),
                               f"search f32 -> {kind}")

    allowed = np.random.default_rng(d).permutation(n)[: n // 3].astype(np.uint64)
    want = ref.filtered_search(q, k, allowed, threads=16)
    got = index.filtered_search(q, k, allowed)
    common.assert_same_results(want, (got.keys, got.distances, got.counts, index.last_computed, index.last_visited),
                               f"filtered f32 -> {kind}")

    want = ref.search(q_cast, k, threads=16, exact=True)
    got = index.search(q, k, exact=True)
    common.assert_same_results(want[:3], (got.keys, got.distances, got.counts), f"exact f32 -> {kind}")

    for level in (0, 1, 2):
        wk, wd, wc, wv = ref.cluster(q_cast, level)
        gk, gd = index.cluster(q, level, stats=True)
        assert np.array_equal(wk, gk) and np.array_equal(wd.view(np.uint32), gd.view(np.uint32)), f"cluster {level}"
        assert np.array_equal(wc, index.last_computed) and np.array_equal(wv, index.last_visited), f"cluster {level}"

    group = Indexes([index])
    for exact in (False, True):
        want = ir.reference_search([ref], q, k, query_scalar="f32", exact=exact)
        got = group.search(q, k, exact=exact)
        common.assert_same_results(want, (got.keys, got.distances, got.counts, group.last_computed, group.last_visited),
                                   f"Indexes f32 -> {kind} exact={exact}")


def _raw_rows(kind: str, n: int, d: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    if kind == "f16":
        return _f16_bits(n, d, seed).view(np.float16)
    if kind == "bf16":
        w = rng.integers(0, 1 << 16, size=(n, d), dtype=np.uint32).astype(np.uint16)
        w[::4] |= 0x7F80  # inf and NaN patterns
        w[1::4] &= ~np.uint16(0x7F80)  # zeros and subnormals
        return w
    if kind == "i8":
        return rng.integers(-128, 128, size=(n, d), dtype=np.int16).astype(np.int8)
    return rng.integers(0, 256, size=(n, bindings.bytes_per_vector(d, "b1")), dtype=np.uint8)


@needs_reference
@pytest.mark.parametrize("kind", ["f16", "bf16", "i8", "b1"])
@pytest.mark.parametrize("d", [97, 768])
def test_get_casts_like_the_reference(kind, d):
    """`get(key, dtype=k)` out of a reference-built index whose rows hold raw edge bytes (f16 / bf16 inf and NaN patterns,
    subnormals, i8 -128, packed bits), into every kind: equal to cast_gt<kind, k> of the stored rows, what the
    reference's get_ returns (index_dense.hpp:2121-2150)"""
    from usearch_b200.index import Index
    n = 64
    rows = _raw_rows(kind, n, d, seed=d)
    ref = bindings.RefIndex("parity", metric=METRIC[kind], scalar=kind, dims=d, connectivity=16)
    ref.add(np.arange(n, dtype=np.uint64), rows, threads=1)
    blob = ref.save()
    stored = _stored_matrix(blob)
    index = Index.restore(blob)
    for to in KINDS:
        want = cr.host_cast(stored, kind, to, d)
        if cr.reference_available():
            cr.assert_same_casts(cr.ref_cast(stored, kind, to, d), want, stored, kind, to, d, "host casts vs the reference")
        got = np.stack([np.ascontiguousarray(index.get(key, dtype=to)).view(np.uint8) for key in range(n)])
        cr.assert_same_casts(want, got, stored, kind, to, d, "get")
