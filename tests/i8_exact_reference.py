"""Exact search over i8 vectors in numpy, the plain statement the GPU scans are held to.

The three i8 metrics are functions of the integer triple (ab, a2, b2) = (sum a*b, sum a*a, sum b*b), formed here in int64,
then rounded to f32 exactly as the kernels (usearch_b200/csrc/exact_i8.h) and the pinned reference metrics
(oracle/metrics_pinned.h) state them:
    ip    1 - f32(ab)
    l2sq  f32(a2 + b2 - 2 ab)
    cos   0 if a2 == b2 == 0; 1 if ab == 0; else max(0, 1 - (f32(ab) * ra) * rb), ra = 1 / sqrt(f32(a2)) of the FIRST
          operand: metric(query, stored) for an index, metric(stored, query) for the free exact search (`swap`)
The k best of a row are ordered by distance ascending, then slot DESCENDING (what a run of sorted inserts in slot order
converges to); removed slots are skipped; rows with fewer than k members are padded with key 0 and the signalling-NaN
bits 0x7FA00000."""
from __future__ import annotations

import numpy as np

PAD_BITS = np.uint32(0x7FA00000)


def triples(queries: np.ndarray, rows: np.ndarray):
    """(ab [nq, n], a2 [nq], b2 [n]) in int64"""
    q = np.asarray(queries, dtype=np.int8).astype(np.int64)
    r = np.asarray(rows, dtype=np.int8).astype(np.int64)
    return q @ r.T, (q * q).sum(axis=1), (r * r).sum(axis=1)


def distances(metric: str, ab: np.ndarray, a2: np.ndarray, b2: np.ndarray, swap: bool = False) -> np.ndarray:
    """f32 distances [nq, n] of query rows (a2) against stored rows (b2)"""
    one = np.float32(1)
    if metric == "ip":
        return one - ab.astype(np.float32)
    if metric == "l2sq":
        return (a2[:, None] + b2[None, :] - 2 * ab).astype(np.float32)
    assert metric == "cos", metric
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        qr = one / np.sqrt(a2.astype(np.float32))
        vr = one / np.sqrt(b2.astype(np.float32))
        abf = ab.astype(np.float32)
        p = (abf * vr[None, :]) * qr[:, None] if swap else (abf * qr[:, None]) * vr[None, :]
        r = one - p
    r = np.where(r > 0, r, np.float32(0)).astype(np.float32)
    r = np.where(ab == 0, one, r)
    return np.where((a2[:, None] == 0) & (b2[None, :] == 0), np.float32(0), r).astype(np.float32)


def top_k(dist: np.ndarray, k: int, removed: np.ndarray | None = None, keys: np.ndarray | None = None):
    """(keys [nq, k] u64, distances [nq, k] f32, counts [nq]) under (distance ascending, slot descending)"""
    nq, n = dist.shape
    slots = np.arange(n)
    live = np.ones(n, bool) if removed is None else ~np.asarray(removed, bool)
    keys = slots.astype(np.uint64) if keys is None else np.asarray(keys, np.uint64)
    out_k = np.zeros((nq, k), np.uint64)
    out_d = np.full((nq, k), PAD_BITS, np.uint32).view(np.float32)
    counts = np.zeros(nq, np.uint64)
    for i in range(nq):
        cand = slots[live]
        order = cand[np.lexsort((-cand, dist[i, cand]))][:k]
        out_k[i, :order.size] = keys[order]
        out_d[i, :order.size] = dist[i, order]
        counts[i] = order.size
    return out_k, out_d, counts


def search(metric: str, rows: np.ndarray, queries: np.ndarray, k: int, removed: np.ndarray | None = None, swap: bool = False,
           keys: np.ndarray | None = None):
    """index-mode exact search (swap=False) or the free one's order (swap=True, keys = row numbers)"""
    ab, a2, b2 = triples(queries, rows)
    return top_k(distances(metric, ab, a2, b2, swap), k, removed, keys)


def unique_mask(sorted_d: np.ndarray, k: int) -> np.ndarray:
    """positions < k whose distance differs from both neighbours in a row sorted ascending (k + 1 columns when known)"""
    d = sorted_d
    u = np.ones((d.shape[0], k), bool)
    u[:, 1:] &= d[:, 1:k] != d[:, :k - 1]
    u[:, :-1] &= d[:, :k - 1] != d[:, 1:k]
    if d.shape[1] > k:
        u[:, -1] &= d[:, k - 1] != d[:, k]
    return u


# ---- edge inputs: where the scans' numerics and tiles go wrong (the numpy reference above is pinned to the live
# reference on every one of them, and the GPU scans are held to it) ----

TIE_D = 128


def tie_pair():
    """(query, W, C) of d = 128: q = 127 x 63 then 1; W and C both lie at cos distance 0.9999571 from q (the same f32
    bits), with ab = 33 and 43. A k-best list holding W must take C when C has the larger slot."""
    q = np.zeros(TIE_D, np.int8)
    q[:63], q[63] = 127, 1
    w = np.zeros(TIE_D, np.int8)
    w[63], w[64:100], w[100:102] = 33, 127, 18
    c = np.zeros(TIE_D, np.int8)
    c[63], c[64:125], c[125], c[126] = 43, 127, 23, 51
    return q, w, c


def _case(name, metrics, rows, queries, ks, removed=()):
    return dict(name=name, metrics=tuple(metrics), rows=np.ascontiguousarray(rows, np.int8),
                queries=np.ascontiguousarray(queries, np.int8), ks=tuple(ks), removed=tuple(removed))


def edge_cases(big: bool = True):
    """the edge inputs as dicts: name, metrics, rows [n, d] i8, queries [nq, d] i8, ks, removed slots"""
    rng = np.random.default_rng(2024)
    out = []
    # 1. the constructed tie: W at slot 0, 255 zero rows, C at 256 (the second 256-vector tile), and the mirror image
    q, w, c = tie_pair()
    rows = np.zeros((257, TIE_D), np.int8)
    rows[0], rows[256] = w, c
    mirror = rows[::-1].copy()
    other = rng.integers(-128, 128, (3, TIE_D)).astype(np.int8)
    out.append(_case("tie_wc", ["cos"], rows, np.vstack([q, other, q]), [1, 24]))
    out.append(_case("tie_cw", ["cos"], mirror, np.vstack([q, other]), [1, 24]))
    # 2. near-orthogonal cos rows drawn from a small pool: exact ties at distances in (0.999, 1.001) and at 1 (ab = 0),
    #    copies spread over every 256-vector tile and, with n ~ 16k, over several segments
    n = 16389 if big else 1100
    pool = np.zeros((48, TIE_D), np.int8)
    pool[:, 64:] = rng.integers(-127, 128, (48, 64))
    for i in range(48):
        j = rng.choice(64, size=i % 3, replace=False)
        pool[i, j] = rng.choice([-2, -1, 1, 2], size=j.size)
    rows = pool[rng.integers(0, 48, n)]
    rows[[0, 255, 256, n - 1]] = pool[0]
    queries = np.zeros((130, TIE_D), np.int8)
    queries[:, :64] = rng.choice(np.array([-127, 127], np.int8), (130, 64))
    out.append(_case("cos_ties", ["cos"], rows, queries, [1, 24, 25]))
    out.append(_case("cos_ties_removed", ["cos"], rows, queries[:9], [24], removed=[0, 255, 256, n - 1]))
    # 3. saturated rows: sums past 2^24 at d = 1040 and 4096 (ab up to 128^2 d = 2^26)
    for d in (1040, 4096):
        alt = np.where(np.arange(d) % 2 == 0, 127, -128).astype(np.int8)
        half = np.where(np.arange(d) < d // 2, -128, 127).astype(np.int8)
        sat = np.stack([np.full(d, -128), np.full(d, 127), np.full(d, -127), alt, -alt.astype(np.int16).clip(-128, 127), half,
                        -half.astype(np.int16).clip(-128, 127)]).astype(np.int8)
        rows = np.vstack([sat, rng.integers(-128, 128, (40, d)), sat, np.where(rng.random((40, d)) < 0.5, -128, 127)]).astype(np.int8)
        rows[60:62, :7] = 0  # one unit-scale step below the saturated sums
        queries = np.vstack([sat, rows[50:53]])
        out.append(_case(f"saturated_d{d}", ["ip", "l2sq", "cos"], rows, queries, [1, 24, 25]))
    # 4. zero rows and zero queries (cos 0/0 -> 0, ab = 0 -> 1; ip -> 1)
    rows = rng.integers(-128, 128, (300, 16)).astype(np.int8)
    rows[[0, 7, 255, 256, 299]] = 0
    queries = np.vstack([np.zeros((2, 16), np.int8), rows[1:4]])
    out.append(_case("zeros", ["cos", "ip", "l2sq"], rows, queries, [1, 24, 25]))
    # 5. duplicates, negated and scaled copies: cos 0 (clamped) and 2
    base = rng.integers(-40, 41, (40, 129)).astype(np.int8)
    rows = np.vstack([base, base, -base, 2 * base, 3 * base, -3 * base, base[:20]])[rng.permutation(260)]
    rows = np.vstack([rows, base[:3]]).astype(np.int8)
    out.append(_case("copies", ["cos", "ip", "l2sq"], rows, np.vstack([base[:5], -base[5:8], 3 * base[8:10]]), [1, 24, 25, 256, 257]))
    # 6. ragged shapes around the 128-query and 256-vector tiles, full range [-128, 127], removed slots at tile edges
    shapes = [(1, 1, 1), (255, 127, 15), (256, 128, 16), (257, 129, 17), (257, 1, 128), (256, 129, 129), (255, 128, 1),
              (1, 129, 16), (257, 127, 129), (256, 1, 17)]
    for n, nq, d in shapes:
        rows = rng.integers(-128, 128, (n, d)).astype(np.int8)
        if n > 2:
            rows[n // 2] = rows[1]  # a duplicate: ties everywhere it is near
        queries = rng.integers(-128, 128, (nq, d)).astype(np.int8)
        removed = sorted({s for s in (0, 255, 256, n - 1) if s < n and n > 1})
        out.append(_case(f"shape_n{n}_nq{nq}_d{d}", ["cos", "ip", "l2sq"], rows, queries, [1, 24, 25, 256, 257],
                         removed=removed if (n + nq + d) % 2 else ()))
    return out
