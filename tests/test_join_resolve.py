"""The host replay of `join` (usearch_b200/csrc/join_resolve.h), built natively, against the reference's own
`index_dense_gt::join` run on one thread with the pinned metric (tests/native/ref_join_driver.cpp), and against the
reference's loop restated in Python, both fed with the reference's own proposals (tests/join_reference.py). No GPU.

Also checks, on the reference itself, the observation the GPU join rests on: for i <= expansion, proposal i is row i of a
single search with count min(P, expansion), counters included (exact search: for every i)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import common
import join_reference as jr
from oracle import bindings
from usearch_b200 import datagen, v2format

pytestmark = pytest.mark.skipif(not (common.have_reference() and jr.live_available()), reason="reference sources unavailable")

_u32p, _u64p, _f32p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("join_resolve") / "libjoin_resolve.so")
    subprocess.run(["g++", "-std=c++11", "-O1", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC",
                    "-I", os.path.join(common.ROOT, "usearch_b200", "csrc"),
                    os.path.join(common.ROOT, "tests", "native", "join_resolve_shim.cpp"), "-o", out], check=True)
    lib = C.CDLL(out)
    lib.join_replay_columns.restype = C.c_char_p
    lib.join_replay_columns.argtypes = [C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, _u32p, _f32p, _f32p, _u64p, _u64p, _u32p,
                                        C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    return lib


def _blob(rows, metric, scalar, d, m=16, keys=None, remove=()):
    ref = bindings.RefIndex("parity", metric=metric, scalar=scalar, dims=d, connectivity=m, expansion_add=64, expansion_search=64)
    ref.pin_metric(True)
    ref.add(np.arange(len(rows), dtype=np.uint64) if keys is None else keys, rows, threads=1)
    for key in remove:
        ref.remove(int(key))
    return ref.save()


def _multi(blob, divisor):
    """the same graph as a multi index: slot s holds key s // divisor"""
    g = v2format.loads(blob)
    live = g.keys != v2format.FREE_KEY
    g.keys = np.where(live, g.keys // np.uint64(divisor), g.keys)
    g.multi = True
    return v2format.dumps(g)


def _native(shim, men, women, max_proposals, columns):
    ncols = max(columns)
    stack = lambda j, t: np.ascontiguousarray(np.stack([np.asarray(columns[i][j]) for i in range(1, ncols + 1)]), dtype=t)
    woman, dist, back = stack(0, np.uint32), stack(1, np.float32), stack(2, np.float32)
    comp, vis = stack(3, np.uint64), stack(4, np.uint64)
    m2w = np.zeros(men, dtype=np.uint32)
    stats = (C.c_size_t * 4)()
    asked = C.c_size_t(0)
    err = shim.join_replay_columns(men, women, max_proposals, ncols, woman.ctypes.data_as(_u32p), dist.ctypes.data_as(_f32p),
                                   back.ctypes.data_as(_f32p), comp.ctypes.data_as(_u64p), vis.ctypes.data_as(_u64p),
                                   m2w.ctypes.data_as(_u32p), stats, C.byref(asked))
    assert err is None, err
    return m2w, list(stats), asked.value


def _rows(n, d, scalar, seed, noise=0.0, base=None):
    if base is None:
        x = datagen.latent(n, d, seed=seed, rank=min(16, d))
    else:
        x = base[np.random.default_rng(seed).permutation(len(base))[:n]]
        x = x + noise * np.random.default_rng(seed + 1).standard_normal(x.shape).astype(np.float32)
    return datagen.to_scalar(np.ascontiguousarray(x, dtype=np.float32), scalar)


def _case(name):
    """(a rows, b rows, metric, scalar, d, max_proposals, expansion, exact)"""
    d = 32
    base = datagen.latent(500, d, seed=7, rank=12)
    if name == "men_fewer":
        return _rows(300, d, "f32", 1, 0.05, base), _rows(500, d, "f32", 2, 0.05, base), "cos", "f32", d, 0, 64, False
    if name == "swap":
        return _rows(500, d, "f32", 3, 0.05, base), _rows(300, d, "f32", 4, 0.05, base), "cos", "f32", d, 0, 64, False
    if name in ("p1", "p3"):
        return (_rows(300, d, "f32", 5, 0.1, base), _rows(400, d, "f32", 6, 0.1, base), "l2sq", "f32", d,
                1 if name == "p1" else 3, 64, False)
    if name == "p_above_expansion":
        return _rows(200, d, "f32", 8, 0.1, base), _rows(260, d, "f32", 9, 0.1, base), "ip", "f32", d, 12, 8, False
    if name == "exact":
        return _rows(200, d, "f32", 10, 0.05, base), _rows(300, d, "f32", 11, 0.05, base), "cos", "f32", d, 0, 64, True
    if name == "ties":
        # near-duplicate rows: hamming on 64 bits gives many equal distances; duplicated women make whole rows tie
        men = _rows(250, 64, "b1", 12)
        women = np.concatenate([men[:150], men[:150], _rows(100, 64, "b1", 13)])
        return men, women, "hamming", "b1", 64, 6, 64, False
    if name in ("removed", "multi"):
        return _rows(300, d, "f32", 14, 0.05, base), _rows(340, d, "f32", 15, 0.05, base), "l2sq", "f32", d, 0, 64, False
    raise KeyError(name)


CASES = ["men_fewer", "swap", "p1", "p3", "p_above_expansion", "exact", "ties", "removed", "multi"]


@pytest.mark.parametrize("name", CASES)
def test_replay_matches_reference_loop(shim, name):
    a, b, metric, scalar, d, max_p, ef, exact = _case(name)
    if name == "removed":  # removed men propose, removed women are proposed to; their pairs carry the free key
        a_blob = _blob(a, metric, scalar, d, remove=range(0, len(a), 7))
        b_blob = _blob(b, metric, scalar, d, keys=np.arange(len(b), dtype=np.uint64) + 1000, remove=range(1000, 1000 + len(b), 5))
    else:
        a_blob, b_blob = _blob(a, metric, scalar, d), _blob(b, metric, scalar, d, keys=np.arange(len(b), dtype=np.uint64) + 1000)
    if name == "multi":  # repeated keys on both sides: the last write of the export walk wins
        a_blob, b_blob = _multi(a_blob, 2), _multi(b_blob, 3)
    swapped = len(b) < len(a)
    men_blob, women_blob = (b_blob, a_blob) if swapped else (a_blob, b_blob)
    men, women = min(len(a), len(b)), max(len(a), len(b))
    P = jr.default_proposals(men, max_p)
    columns = jr.reference_columns(men_blob, women_blob, P, ef, exact)
    want_m2w, want_eng, want_vis, want_comp = jr.replay(men, women, P, columns)
    got_m2w, stats, asked = _native(shim, men, women, max_p, columns)
    assert got_m2w.tolist() == want_m2w
    assert stats == [sum(w != jr.MISSING for w in want_m2w), want_eng, want_vis, want_comp]
    assert asked <= P
    if name == "ties":  # first proposals collide on equal distances, so the strict `>` and the re-push order decide
        first_woman, first_dist = np.asarray(columns[1][0]), np.asarray(columns[1][1])
        assert len(set(first_woman.tolist())) < men
        assert len(set(zip(first_woman.tolist(), first_dist.tolist()))) < men
    if name == "p_above_expansion":  # the replay asked for columns beyond the one batched search
        assert asked > ef
    # the reference's own join, one thread, pinned metric: counters, and the mapping built from the replay's pairs
    live, live_stats = jr.live_join(a_blob, b_blob, max_p, ef, exact)
    assert live_stats == dict(intersection_size=stats[0], engagements=stats[1], visited_members=stats[2], computed_distances=stats[3])
    restated, restated_stats = jr.reference_join(a_blob, b_blob, max_p, ef, exact)
    assert restated == live and restated_stats == live_stats
    if name == "removed":
        assert int(v2format.FREE_KEY) in live or int(v2format.FREE_KEY) in live.values()


@pytest.mark.parametrize("exact", [False, True])
def test_proposals_are_prefixes_of_one_search(exact):
    """proposal i == row i of one search with count min(P, expansion), with the same counters (the batching the GPU uses)"""
    d, ef = 32, 16
    a = _rows(200, d, "f32", 20)
    b = _rows(300, d, "f32", 21)
    b_blob = _blob(b, "cos", "f32", d)
    g = v2format.loads(b_blob)
    g.keys = np.arange(g.size, dtype=np.uint64)
    ref = bindings.RefIndex("parity")
    ref.load(v2format.dumps(g))
    ref.pin_metric(True)
    ref.change_expansion_search(ef)
    K = ef
    keys, dist, counts, comp, vis = ref.search(a, K, threads=4, exact=exact)
    for i in (1, 2, 5, K):
        ki, di, ci, compi, visi = ref.search(a, i, threads=4, exact=exact)
        assert np.array_equal(ki, keys[:, :i]) and np.array_equal(di.view(np.uint32), dist[:, :i].view(np.uint32))
        assert np.array_equal(ci, np.minimum(counts, i))
        assert np.array_equal(compi, comp) and np.array_equal(visi, vis)
