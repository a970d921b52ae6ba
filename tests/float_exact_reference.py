"""Edge inputs for the f32, f16, bf16, f64 and b1 exact-search scans (usearch_b200/csrc/exact_kernel.cu), the pinned
expectation of each, and an independent float64 statement of every metric.

The scans cut the dataset into tiles (16 rows for LPV 4 and b1, 32 for halves) and segments (a whole number of tiles
scanned by one CTA, merged afterwards), keep k-best lists in registers up to 256 and in global memory above, and run
QT queries per warp, QPC per CTA. The cases put exact ties, one-ulp near ties and removed slots on those boundaries,
and use counts, query counts and row lengths on both sides of every limit.

Expected results come from the plain-C port (oracle/hnsw_oracle.c, tests/native/port_f64.c for f64), built from this
repository: `pinned_matrix` reads every distance of a set of rows from its exact search, in either argument order, and
the keyed top-k of tests/i8_exact_reference.py orders them. `check_topk` then holds any result to the float64
statement of the metric within a stated rounding bound, so a mistake shared by the port and a kernel cannot pass.

NaN distances are left out on purpose (sorensen of two empty fingerprints, inf / NaN inputs, overflowing sums): with a
NaN in its list the reference's answer depends on insertion order, which no segmented scan can reproduce."""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from i8_exact_reference import PAD_BITS, top_k, unique_mask  # noqa: E402,F401  (the keyed top-k is kind-independent)

KINDS = ("f32", "f16", "bf16", "f64", "b1")
METRICS = {"f32": ("l2sq", "ip", "cos"), "f16": ("l2sq", "ip", "cos"), "bf16": ("l2sq", "ip", "cos"),
           "f64": ("l2sq", "ip", "cos"), "b1": ("hamming", "tanimoto", "sorensen")}
LPV = {"f32": 4, "f64": 4, "f16": 1, "bf16": 1, "b1": 2}
SMEM = 227 * 1024


def tile_rows(kind):
    """rows per tile of the tiled scan (32 / LPV lane groups x VT rows each)"""
    lpv = LPV[kind]
    return (32 // lpv) * (2 if lpv == 4 else 1)


def qt(kind):
    return 4 if LPV[kind] == 4 else 8


def qpc(kind):
    return 8 * qt(kind)


# ---- the shared-memory plan of exact_search_device -------------------------------------------------------------------

def vec_stride(kind, d):
    bpv = (d + 7) // 8 if kind == "b1" else d * {"f32": 4, "f64": 8, "f16": 2, "bf16": 2}[kind]
    return (bpv + 15) // 16 * 16


def _smem(kind, d, queries, rows):
    vs = vec_stride(kind, d)
    stage = (vs + 127) // 128 * 128 + 16 * LPV[kind]
    return (queries * vs + 16 + 127) // 128 * 128 + 2 * rows * stage


def tiled_fits(kind, d):
    return _smem(kind, d, qpc(kind), tile_rows(kind)) <= SMEM


def staged_fits(kind, d):
    """whether the one-query-per-warp scan stages 8 queries and 2 x 32 / LPV rows; longer rows are read in place"""
    return _smem(kind, d, 8, 32 // LPV[kind]) <= SMEM


def limit(fits, kind):
    """the largest length (dims, or bits for b1) that fits"""
    step = 8 if kind == "b1" else 1
    d = step
    while fits(kind, d + step):
        d += step
    return d


# ---- kinds --------------------------------------------------------------------------------------------------------

def to_kind(kind, x):
    """float64 [m, d] (b1: 0 / 1) -> the stored rows of `kind` (bf16 as uint16 words, b1 packed bytes)"""
    x = np.asarray(x)
    if kind == "f64":
        return np.ascontiguousarray(x, np.float64)
    if kind == "f32":
        return np.ascontiguousarray(x, np.float32)
    if kind == "f16":
        return np.ascontiguousarray(x, np.float16)
    if kind == "bf16":
        b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
        return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    assert kind == "b1"
    return np.packbits(np.asarray(x, np.uint8) != 0, axis=1)


def to_f64(kind, rows, d):
    """the stored rows as float64 (b1: int64 bits of the first d)"""
    if kind == "bf16":
        return (rows.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    if kind == "b1":
        return np.unpackbits(rows, axis=1)[:, :d].astype(np.int64)
    return rows.astype(np.float64)


def dims_of(kind, rows, d=None):
    return d if d is not None else (rows.shape[1] * 8 if kind == "b1" else rows.shape[1])


# ---- the port: pinned distances in either order ----------------------------------------------------------------------

def blob(kind, rows, metric, d):
    from tools.exact_bench import linkless_blob
    return linkless_blob(rows, metric, kind, d)


def port(kind, image):
    if kind == "f64":
        import f64_reference
        return f64_reference.PortF64(image)
    from oracle import bindings
    return bindings.PortIndex(image)


def pinned_matrix(kind, metric, rows, queries, d, swap=False, chunk=256):
    """f32 [nq, n]: the port's metric(query, row), or metric(row, query) with `swap` (the free exact search's order)"""
    stored, probe = (queries, rows) if swap else (rows, queries)
    out = np.zeros((probe.shape[0], stored.shape[0]), np.float32)
    for lo in range(0, stored.shape[0], chunk):
        part = np.ascontiguousarray(stored[lo:lo + chunk])
        keys, dist, counts = port(kind, blob(kind, part, metric, d)).search(probe, part.shape[0], exact=True)[:3]
        assert (counts == part.shape[0]).all()
        np.put_along_axis(out[:, lo:lo + part.shape[0]], keys.astype(np.int64), dist, axis=1)
    return out.T.copy() if swap else out


def pinned_search(kind, metric, rows, queries, k, d, removed=None, swap=False):
    """(keys, distances, counts) of the port's exact search: index mode, or the free function's order with `swap`"""
    return top_k(pinned_matrix(kind, metric, rows, queries, d, swap), k, removed)


# ---- the float64 statement ------------------------------------------------------------------------------------------

U32 = 2.0 ** -24


def statement(kind, metric, rows, queries, d):
    """(distance [nq, n] float64, bound [nq, n]): the metric in float64 (b1 in exact integers) and a bound on how far a
    correctly rounded evaluation in the kernels' precision can land from it: gamma_n of the sum of |terms| for the
    accumulations (n = d plus the reduction tree), plus one f32 rounding per operation of the normalisation."""
    a, b = to_f64(kind, queries, d), to_f64(kind, rows, d)
    if kind == "b1":
        both = a @ b.T
        na, nb = a.sum(1)[:, None], b.sum(1)[None, :]
        union = na + nb - both
        if metric == "hamming":
            return (union - both).astype(np.float64), np.zeros(both.shape)
        if metric == "tanimoto":
            dist = np.where(union > 0, 1 - both / np.maximum(union, 1), 1.0)
        else:
            assert metric == "sorensen"
            dist = 1 - 2 * both / (na + nb)
        return dist, 4 * U32 * (1 + np.abs(dist))
    u = 2.0 ** -53 if kind == "f64" else U32
    n = d + 16
    g = n * u / (1 - n * u)
    if metric == "l2sq":
        dist = np.zeros((a.shape[0], b.shape[0]))
        for i in range(a.shape[0]):
            dist[i] = ((a[i][None, :] - b) ** 2).sum(1)
        return dist, (g + 4 * u) * dist + 2 * U32 * dist
    dot, s = a @ b.T, np.abs(a) @ np.abs(b).T
    if metric == "ip":
        dist = 1 - dot
        return dist, g * s + 2 * U32 * (np.abs(dot) + np.abs(dist))
    assert metric == "cos"
    a2, b2 = (a * a).sum(1)[:, None], (b * b).sum(1)[None, :]
    norm = np.sqrt(a2 * b2)
    with np.errstate(divide="ignore", invalid="ignore"):
        dist = np.maximum(0.0, 1 - dot / norm)
        bound = 3 * g * s / norm + 4 * U32
    dist = np.where(dot == 0, 1.0, dist)
    zero = (a2 == 0) & (b2 == 0)
    dist = np.where(zero, 0.0, dist)
    bound = np.where((a2 == 0) | (b2 == 0), 0.0, bound)
    return dist, bound


def check_topk(kind, metric, rows, queries, d, k, keys, dists, counts, removed=None, swap=False):
    """problems (strings) of one result against the float64 statement: counts, padding, no removed or repeated labels,
    ascending distances, each distance within the bound of its label's statement, and no row left out that is surely
    closer than a reported one. The statement is symmetric, so `swap` changes nothing here."""
    del swap
    dist, bound = statement(kind, metric, rows, queries, d)
    n = rows.shape[0]
    live = np.ones(n, bool) if removed is None else ~np.asarray(removed, bool)
    want_count = min(k, int(live.sum()))
    out = []
    for i in range(queries.shape[0]):
        c = int(counts[i])
        if c != want_count:
            out.append(f"query {i}: count {c}, want {want_count}")
            continue
        ks, ds = keys[i, :c].astype(np.int64), dists[i, :c].astype(np.float64)
        pad = dists[i, c:].view(np.uint32)
        if (pad != PAD_BITS).any() or (keys[i, c:] != 0).any():
            out.append(f"query {i}: padding past {c} is not key 0 / 0x{int(PAD_BITS):08x}")
        if (ks >= n).any() or not live[ks[ks < n]].all() or np.unique(ks).size != c:
            out.append(f"query {i}: removed, unknown or repeated labels")
            continue
        if (np.diff(ds) < 0).any() or np.isnan(ds).any():
            out.append(f"query {i}: distances not ascending")
        off = np.abs(ds - dist[i, ks]) > bound[i, ks]
        if off.any():
            j = int(np.argmax(off))
            out.append(f"query {i}: slot {ks[j]} reported {ds[j]!r}, float64 statement {dist[i, ks[j]]!r} +- {bound[i, ks[j]]:.3g}")
        rest = live.copy()
        rest[ks] = False
        if c and rest.any():
            worst = (dist[i, ks] - bound[i, ks]).max()
            closer = np.nonzero(dist[i, rest] + bound[i, rest] < worst)[0]
            if closer.size:
                out.append(f"query {i}: {closer.size} rows left out are closer than a reported one")
    return out


# ---- edge inputs ----------------------------------------------------------------------------------------------------

def _grid(rng, shape, kind):
    """values exact in every kind and in every sum the cases form: multiples of 1/8 in [-2, 2] (b1: random bits)"""
    if kind == "b1":
        return (rng.random(shape) < 0.5).astype(np.float64)
    return rng.integers(-16, 17, shape) / 8.0


def _gauss(rng, shape, kind):
    if kind == "b1":
        return (rng.random(shape) < 0.3).astype(np.float64)
    return rng.standard_normal(shape)


def _case(kind, name, metrics, rows64, queries64, ks, d, removed=(), free=True, index=True, batches=False):
    return dict(kind=kind, name=name, metrics=tuple(metrics), rows=to_kind(kind, rows64), queries=to_kind(kind, queries64),
                d=d, ks=tuple(ks), removed=tuple(sorted(set(removed))), free=free, index=index, batches=batches)


def ragged_dims(kind):
    """lengths whose rows end in a partial 16-byte chunk (b1: partial bytes and words)"""
    return {"f32": (1, 2, 3, 37, 66, 99), "f64": (1, 3, 37), "f16": (9, 10, 11, 12, 13, 14, 15),
            "bf16": (9, 10, 11, 12, 13, 14, 15), "b1": (1, 63, 65, 127, 129, 200)}[kind]


def long_dims(kind):
    """lengths past the staged scan: read in place (f32 8192 goes through the free function only)"""
    return {"f32": (4096, 6400), "f64": (2048,), "f16": (2048, 4096), "bf16": (2048, 4096), "b1": ()}[kind]


def boundary_dims(kind):
    """one length on each side of the tiled stage's limit and of the staged scan's"""
    step = 8 if kind == "b1" else 1
    t, s = limit(tiled_fits, kind), limit(staged_fits, kind)
    return (t, t + step, s, s + step)


def near_tie(kind, metric, q, a, rng, tries=60, width=512):
    """(a, b): rows whose pinned distances from q are consecutive f32 values, b the farther. b moves a's last coordinate
    over a fine grid; where the sums' rounding leaves only even steps from this a, a's first coordinate is nudged and
    the sweep repeated. The port's metric confirms the gap."""
    d = q.size
    qs = to_kind(kind, q[None])
    for t in range(tries):
        if t and t % 12 == 0:
            a = a.copy()
            a[0] += 0.01 * rng.standard_normal()
            a = to_f64(kind, to_kind(kind, a[None]), d)[0]
        da = pinned_matrix(kind, metric, to_kind(kind, a[None]), qs, d)[0, 0]
        target = np.nextafter(da, np.float32(np.inf)).view(np.uint32)
        scale = float(np.spacing(da)) * 2.0 ** (t % 12 - 4) / max(abs(q[-1]), 1e-3)
        cand = np.repeat(a[None], width, 0)
        cand[:, -1] = a[-1] + scale * rng.uniform(-64, 64, width)
        stored = to_kind(kind, cand)
        dist = pinned_matrix(kind, metric, stored, qs, d)[0]
        hit = np.nonzero(dist.view(np.uint32) == target)[0]
        if hit.size:
            return a, to_f64(kind, stored[hit[:1]], d)[0]
    raise AssertionError(f"no one-ulp near tie found for {kind}/{metric}")


def edge_cases(kind, big=True):
    """the edge inputs of one kind as dicts: kind, name, metrics, rows, queries (stored kind), d, ks, removed slots,
    and whether the case runs in index mode, through the free function, and in sliced batches"""
    rng = np.random.default_rng({"f32": 1, "f16": 2, "bf16": 3, "f64": 4, "b1": 5}[kind])
    metrics = METRICS[kind]
    tv, out = tile_rows(kind), []
    # 1. tiles: exact duplicates (and, for l2sq, mirror pairs q0 +- delta) across every tile boundary, removed slots on
    #    the first and last slot of a tile, one whole removed tile, a short last tile; every count edge
    d = ragged_dims(kind)[2]
    n = 45 * 16 + 3
    rows = _grid(rng, (n, d), kind)
    queries = _grid(rng, (qt(kind) + 1, d), kind)
    delta = _grid(rng, (1, d), kind)[0]
    for b in range(tv, n, tv):
        if kind != "b1" and (b // tv) % 3 == 0:
            rows[b - 1], rows[b] = queries[0] + delta, queries[0] - delta
        else:
            rows[b] = rows[b - 1]
    removed = [tv, 2 * tv - 1, *range(3 * tv, 4 * tv), n - 1]
    ks = (1, 31, 32, 33, 255, 256, 257, 700, n - 1, n)
    if kind == "b1":  # no empty fingerprints under sorensen (0 / 0)
        rows[rows.sum(1) == 0, 0] = 1
        queries[queries.sum(1) == 0, 0] = 1
    out.append(_case(kind, "tiles", metrics, rows, queries, ks + (n + 5,), d, removed=removed, free=False))
    out.append(_case(kind, "tiles_free", metrics, rows, queries, ks, d, index=False))
    # 2. segments: few queries over many rows, so that the planner cuts many segments; duplicates on every tile boundary
    n = 20011 if big else 2011
    d = 8 if kind != "b1" else 64
    rows = _grid(rng, (n, d), kind)
    rows[tv::tv] = rows[tv - 1:n - 1:tv]
    if kind == "b1":
        rows[rows.sum(1) == 0, 0] = 1
    queries = _grid(rng, (7, d), kind)
    if kind == "b1":
        queries[queries.sum(1) == 0, 0] = 1
    out.append(_case(kind, "segments", metrics, rows, queries, (1, 33, 257), d, removed=[tv, 5 * tv - 1, n - 1]))
    # 3. one batch of several hundred queries, also searched in slices of 1, QT +- 1, 7, 9 and QPC +- 1 queries
    n, d = 700, ragged_dims(kind)[1]
    rows = _gauss(rng, (n, d), kind)
    rows[tv * 3] = rows[tv * 3 - 1]
    queries = _gauss(rng, (300, d), kind)
    if kind == "b1":
        rows[rows.sum(1) == 0, 0] = 1
        queries[queries.sum(1) == 0, 0] = 1
    out.append(_case(kind, "batch", metrics, rows, queries, (1, 10, 257), d, batches=True))
    # 4. lengths: ragged tails, both sides of both stage limits, past the staged scan
    for d in ragged_dims(kind) + boundary_dims(kind) + long_dims(kind):
        n = 300 if d in boundary_dims(kind)[:2] else 40
        rows = _gauss(rng, (n, d), kind)
        rows[16] = rows[15]
        queries = _gauss(rng, (9, d), kind)
        if kind == "b1":
            rows[rows.sum(1) == 0, 0] = 1
            queries[queries.sum(1) == 0, 0] = 1
        ks = (1, 10, 257) if n == 300 else (1, 10)
        out.append(_case(kind, f"d{d}", metrics, rows, queries, ks, d))
    if kind == "f32":
        out.append(_case(kind, "d8192", metrics, _gauss(rng, (40, 8192), kind), _gauss(rng, (9, 8192), kind), (1, 10), 8192,
                         index=False))
    if kind == "b1":  # 5. empty fingerprints: hamming counts bits, tanimoto's empty union is 1
        d = 96
        rows = _gauss(rng, (3 * tv + 5, d), kind)
        rows[[0, tv - 1, tv, 3 * tv + 4]] = 0
        queries = np.vstack([np.zeros((2, d)), _gauss(rng, (3, d), kind)])
        out.append(_case(kind, "empty", ("hamming", "tanimoto"), rows, queries, (1, 4, 10), d))
        return out
    # 5. cos at zero: zero rows on tile edges and zero queries (0 / 0 -> 0, a zero product -> 1)
    d = 24
    rows = _gauss(rng, (3 * tv + 5, d), kind)
    rows[[0, tv - 1, tv, 3 * tv + 4]] = 0
    queries = np.vstack([np.zeros((2, d)), _gauss(rng, (3, d), kind)])
    out.append(_case(kind, "zeros", metrics, rows, queries, (1, 4, 10), d))
    # 6. one-ulp near ties across the first tile boundary, one case per metric
    d = 21
    for metric in metrics:
        rows = 0.3 * _gauss(rng, (3 * tv + 5, d), kind)
        queries = _gauss(rng, (5, d), kind)
        # the last coordinate is moved: small, so that its steps stay below one ulp; coordinate j shares its accumulator
        # and dominates the sum, so that each step of the moved term survives the reduction tree
        j = (d - 1) % 16
        queries[0, -1] = 1e-3 if metric == "l2sq" else 1.0
        queries[0, j] = 4.0
        q = to_f64(kind, to_kind(kind, queries[:1]), d)[0]
        a = (q if metric == "l2sq" else 0) + 0.05 * _gauss(rng, (d,), kind)
        a[j], a[-1] = (7.0 if metric == "ip" else 8.0), 0.0  # ip: 1 - dot in the binade of dot
        if metric == "cos":  # a small cosine: the dot product's ulp stays below the distance's
            a[j], a[0], q[0] = 1.0, 8.0, 0.0
            queries[0, 0] = 0.0
        a = to_f64(kind, to_kind(kind, a[None]), d)[0]
        rows[tv - 1], rows[tv] = near_tie(kind, metric, q, a, rng)
        out.append(_case(kind, f"near_tie_{metric}", (metric,), rows, queries, (1, 2, 3, 10), d))
    # 7. cos through the free function, the queries' scaled copies among rows whose norms span orders of magnitude: for
    #    a parallel pair 1 - (ab ra) rb is a few f64 ulps, which the f32 result keeps, so metric(row, query) and
    #    metric(query, row) differ in their bits. Small integers times 3-bit multipliers: every sum is exact in every kind
    d, nq = 16, 9
    queries = rng.integers(-4, 5, (nq, d)).astype(np.float64)
    queries[:, 0] = rng.choice([-3.0, -1.0, 1.0, 3.0], nq)
    scales = np.array([3, 5, 7, 80, 96, 7 / 64, 3 / 32, 5 / 128])
    copies = (scales[:, None, None] * queries[None]).reshape(-1, d)
    span = 2.0 if kind == "f16" else 4.0
    other = _gauss(rng, (600, d), kind) * 10.0 ** rng.uniform(-span, span, (600, 1))
    out.append(_case(kind, "swap_scales", ("cos",), np.vstack([copies, other]), queries, (1, 10, 257), d, index=False))
    return out
