"""The reference's `join` (index.hpp:4345-4543) as its one-thread run makes it, restated in Python over the reference's
own proposals, for the join tests.

Proposal i of man m is `women.search(men_values[m], i)` of the reference: here the pinned reference searches the women's
saved graph re-keyed so that keys are slots and nothing is removed (which is index_gt::search without a predicate), with
count i for every i, not just once. The husband's distance is the reference's metric with the woman's row first."""
from __future__ import annotations

import math

import numpy as np

from oracle import bindings
from usearch_b200 import v2format

MISSING = 0xFFFFFFFF


def _slot_keyed(blob):
    g = v2format.loads(blob)
    keys = g.keys.copy()
    g.keys = np.arange(g.size, dtype=np.uint64)
    g.multi = False
    return g, keys, v2format.dumps(g)


def default_proposals(men: int, max_proposals: int = 0) -> int:
    if max_proposals == 0:
        max_proposals = int(math.log(men) + 1)
    return min(max_proposals, men)


def reference_columns(men_blob, women_blob, proposals: int, expansion: int, exact: bool):
    """column i (1-based) -> (woman slot, metric(man, woman), metric(woman, man), computed, visited), one entry per man"""
    men_g, _, _ = _slot_keyed(men_blob)
    women_g, _, women_blob_slots = _slot_keyed(women_blob)
    ref = bindings.RefIndex("parity")
    ref.load(women_blob_slots)
    ref.pin_metric(True)
    ref.change_expansion_search(expansion)
    rows = np.ascontiguousarray(men_g.vectors)
    wrows = women_g.vectors
    columns = {}
    for i in range(1, proposals + 1):
        keys, dist, counts, computed, visited = ref.search(rows, i, threads=8, exact=exact)
        last = np.minimum(counts.astype(np.int64), i) - 1
        assert (last >= 0).all()
        woman = keys[np.arange(len(rows)), last].astype(np.int64)
        distance = dist[np.arange(len(rows)), last]
        from_woman = np.array([ref.distance(wrows[w], rows[m]) for m, w in enumerate(woman)], dtype=np.float32)
        columns[i] = (woman, distance, from_woman, computed.astype(np.uint64), visited.astype(np.uint64))
    return columns


def replay(men: int, women: int, proposals: int, columns):
    """the FIFO of index.hpp:4412-4511 on one thread: (man_to_woman, engagements, visited, computed)"""
    from collections import deque
    man_to_woman = [MISSING] * men
    woman_to_man = [MISSING] * women
    counts = [0] * men
    free = deque(range(men))
    engagements = visited = computed = 0
    while free:
        m = free.popleft()
        if counts[m] >= proposals:
            continue
        counts[m] += 1
        woman, distance, _, comp, vis = columns[counts[m]]
        visited += int(vis[m])
        computed += int(comp[m])
        w = int(woman[m])
        h = woman_to_man[w]
        if h == MISSING:
            man_to_woman[m], woman_to_man[w] = w, m
            engagements += 1
        else:
            # women_metric(women_values[w], men_values[h]) > match.distance
            from_husband = columns[counts[h]][2][h]
            if np.float32(from_husband) > np.float32(distance[m]):
                man_to_woman[h] = MISSING
                man_to_woman[m], woman_to_man[w] = w, m
                engagements += 1
                free.append(h)
            else:
                free.append(m)
    return man_to_woman, engagements, visited, computed


def reference_join(a_blob, b_blob, max_proposals: int = 0, expansion: int = 64, exact: bool = False):
    """(a_to_b dict, stats dict) of the reference's one-thread join of a with b"""
    a_n, b_n = v2format.loads(a_blob).size, v2format.loads(b_blob).size
    swapped = b_n < a_n
    men_blob, women_blob = (b_blob, a_blob) if swapped else (a_blob, b_blob)
    men_keys = v2format.loads(men_blob).keys
    women_keys = v2format.loads(women_blob).keys
    men, women = len(men_keys), len(women_keys)
    stats = {"intersection_size": 0, "engagements": 0, "visited_members": 0, "computed_distances": 0}
    if men == 0:
        return {}, stats
    proposals = default_proposals(men, max_proposals)
    columns = reference_columns(men_blob, women_blob, proposals, expansion, exact)
    man_to_woman, engagements, visited, computed = replay(men, women, proposals, columns)
    a_to_b = {}
    for m in range(men):
        w = man_to_woman[m]
        if w == MISSING:
            continue
        stats["intersection_size"] += 1
        mk, wk = int(men_keys[m]), int(women_keys[w])
        if swapped:
            a_to_b[wk] = mk
        else:
            a_to_b[mk] = wk
    stats.update(engagements=engagements, visited_members=visited, computed_distances=computed)
    return a_to_b, stats


# ---- the reference's own join, compiled at test time where the reference sources are (never on the GPU machines) ----

_live = {}


def live_available() -> bool:
    from oracle import build as oracle_build
    return oracle_build.reference_available()


def _live_lib(flavour: str):
    """tests/native/ref_join_driver.cpp against the reference headers, linked with the oracle's SimSIMD object of the
    same flavour, built once per process into a temporary directory"""
    if flavour in _live:
        return _live[flavour]
    import ctypes as C
    import os
    import subprocess
    import tempfile
    from oracle import build as oracle_build
    oracle_build.build_reference(flavour)
    ref, here = oracle_build.REF, oracle_build.HERE
    simsimd = os.path.join(oracle_build.REF_OUT, f"simsimd_{flavour}.o")
    opt = ["-O2", "-ffp-contract=off", "-march=x86-64-v3"] if flavour == "parity" else ["-O3", "-ffast-math", "-march=native"]
    out = os.path.join(tempfile.mkdtemp(prefix="ref_join_"), f"libref_join_{flavour}.so")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["g++", "-std=c++17", *opt, "-fPIC", "-shared", "-w", "-DUSEARCH_USE_SIMSIMD=1", "-DUSEARCH_USE_FP16LIB=0",
                    "-DUSEARCH_USE_OPENMP=0", "-DSIMSIMD_NATIVE_F16=0", "-DSIMSIMD_NATIVE_BF16=0", "-DSIMSIMD_DYNAMIC_DISPATCH=1",
                    f"-I{ref}/include", f"-I{ref}/simsimd/include", f"-I{ref}/fp16/include", f"-I{here}",
                    os.path.join(root, "tests", "native", "ref_join_driver.cpp"), simsimd, "-o", out, "-lpthread", "-lm"],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    u64p = C.POINTER(C.c_uint64)
    lib.ref_join_blobs.restype = C.c_char_p
    lib.ref_join_blobs.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_size_t,
                                   C.c_int, u64p, u64p, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    _live[flavour] = lib
    return lib


def live_join(a_blob, b_blob, max_proposals: int = 0, expansion: int = 64, exact: bool = False, threads: int = 1,
              flavour: str = "parity"):
    """(a_to_b dict, stats dict) of the reference's `index_dense_gt::join` itself: `parity` with the pinned metric (the
    bits this library reproduces), `perf` with its native metric and production flags"""
    import ctypes as C
    lib = _live_lib(flavour)
    a = np.ascontiguousarray(a_blob, dtype=np.uint8)
    b = np.ascontiguousarray(b_blob, dtype=np.uint8)
    n = max(int(a[:4].view(np.uint32)[0]), 1)  # the slots of `a` (the matrix head): an upper bound on its pairs
    a_keys = np.zeros(n, dtype=np.uint64)
    b_keys = np.zeros(n, dtype=np.uint64)
    pairs = C.c_size_t(0)
    stats = (C.c_size_t * 4)()
    u64p = C.POINTER(C.c_uint64)
    err = lib.ref_join_blobs(a.ctypes.data_as(C.c_void_p), a.size, b.ctypes.data_as(C.c_void_p), b.size, max_proposals, expansion,
                             int(exact), threads, int(flavour == "parity"), a_keys.ctypes.data_as(u64p), b_keys.ctypes.data_as(u64p),
                             C.byref(pairs), stats)
    if err:
        raise RuntimeError(err.decode())
    k = pairs.value
    a_to_b = dict(zip(a_keys[:k].tolist(), b_keys[:k].tolist()))
    return a_to_b, dict(zip(("intersection_size", "engagements", "visited_members", "computed_distances"), (int(x) for x in stats)))
