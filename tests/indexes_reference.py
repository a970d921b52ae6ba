"""The reference's `Indexes.search` run on one thread, stated two ways for the `Indexes` tests.

* :func:`merge_model` is the fold of `search_result_t::merge_into` (index.hpp:2650-2670) written out literally:
  libstdc++'s `lower_bound` probe, then the shift. :func:`reference_search` feeds it the reference's own per-shard
  searches (the oracle's `RefIndex`, pinned metric; queries cast by the reference's own casts where a shard's scalar kind
  differs). It needs only the built oracle, so it also runs on the GPU machines.
* :func:`live_search` is the reference's own loop (python/lib.cpp:350-390: `index_dense_gt::search` and `merge_into`,
  members in order), compiled at test time from tests/native/ref_indexes_driver.cpp against the reference headers where
  they lie. A CPU test holds :func:`reference_search` equal to it.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import bindings

SNAN_BITS = 0x7FA00000


def _lower_bound(row, n, d):
    """std::lower_bound(row, row + n, d) with libstdc++'s probe sequence (halve `len`, test `*mid < d`)."""
    first, length = 0, n
    while length > 0:
        half = length >> 1
        mid = first + half
        if row[mid] < d:
            first = mid + 1
            length -= half + 1
        else:
            length = half
    return first


def merge_model(keys, dists, counts, k):
    """merge_into of shard 0's rows, then shard 1's, ... into empty rows: keys / dists [S, nq, >= k], counts [S, nq].
    Returns (keys [nq, k] u64, distances [nq, k] f32, counts [nq] u64) with dump_to's padding past the counts."""
    S, nq = counts.shape
    out_k = np.zeros((nq, k), dtype=np.uint64)
    out_d = np.full((nq, k), np.uint32(SNAN_BITS)).view(np.float32)
    out_c = np.zeros(nq, dtype=np.uint64)
    for q in range(nq):
        row_k = [0] * k
        row_d = [0.0] * k
        merged = 0
        for s in range(S):
            for i in range(min(int(counts[s, q]), k)):
                key, d = int(keys[s, q, i]), float(dists[s, q, i])
                offset = _lower_bound(row_d, merged, d)
                if offset == k:
                    continue
                worse = merged - offset - (1 if merged == k else 0)
                row_k[offset + 1:offset + 1 + worse] = row_k[offset:offset + worse]
                row_d[offset + 1:offset + 1 + worse] = row_d[offset:offset + worse]
                row_k[offset], row_d[offset] = key, d
                merged += merged != k
        out_k[q, :merged] = row_k[:merged]
        out_d[q, :merged] = np.asarray(row_d[:merged], dtype=np.float32)
        out_c[q] = merged
    return out_k, out_d, out_c


def _cast_queries(ref: bindings.RefIndex, queries: np.ndarray, query_scalar: str) -> np.ndarray:
    """The queries as the shard's `index_dense_gt::search` sees them: f32 rows go through the reference's own cast into
    the shard's scalar kind (index_dense.hpp:2057-2064); rows already in that kind are used as they are."""
    scalar = {v: k for k, v in bindings.SCALAR.items()}[ref.lib.ref_scalar_kind(ref.h)]
    if scalar == query_scalar:
        return queries
    if query_scalar != "f32":
        raise ValueError("only f32 queries are cast here")
    dims = ref.dims
    out = np.zeros((queries.shape[0], bindings.bytes_per_vector(dims, scalar)), dtype=np.uint8)
    rows = np.ascontiguousarray(queries, dtype=np.float32)
    for i in range(rows.shape[0]):
        ref.lib.ref_cast_from_f32(bindings.SCALAR[scalar], rows[i].ctypes.data_as(C.POINTER(C.c_float)), dims,
                                  out[i].ctypes.data_as(C.c_void_p))
    return out


def reference_search(refs: list, queries: np.ndarray, k: int, *, query_scalar: str = "f32", exact: bool = False):
    """(keys [nq,k], distances, counts, computed, visited) of `Indexes(refs).search` on one thread: the reference's own
    per-shard searches folded by :func:`merge_model`; counters summed over shards."""
    queries = np.ascontiguousarray(queries)
    nq = queries.shape[0]
    if not refs:
        keys, dists, counts = merge_model(np.zeros((0, nq, k), np.uint64), np.zeros((0, nq, k), np.float32),
                                          np.zeros((0, nq), np.uint64), k)
        return keys, dists, counts, np.zeros(nq, np.uint64), np.zeros(nq, np.uint64)
    per_shard = [ref.search(_cast_queries(ref, queries, query_scalar), k, threads=1, exact=exact) for ref in refs]
    keys, dists, counts = merge_model(np.stack([p[0] for p in per_shard]), np.stack([p[1] for p in per_shard]),
                                      np.stack([p[2] for p in per_shard]), k)
    return keys, dists, counts, sum(p[3] for p in per_shard), sum(p[4] for p in per_shard)


_live = {}


def live_available() -> bool:
    from oracle import build as oracle_build
    return oracle_build.reference_available()


def _live_lib():
    """tests/native/ref_indexes_driver.cpp against the reference headers, linked with the oracle's SimSIMD object of the
    parity flavour, built once per process into a temporary directory"""
    if "lib" in _live:
        return _live["lib"]
    import subprocess
    import tempfile
    from oracle import build as oracle_build
    oracle_build.build_reference("parity")
    ref, here = oracle_build.REF, oracle_build.HERE
    simsimd = os.path.join(oracle_build.REF_OUT, "simsimd_parity.o")
    out = os.path.join(tempfile.mkdtemp(prefix="ref_indexes_"), "libref_indexes.so")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-march=x86-64-v3", "-fPIC", "-shared", "-w",
                    "-DUSEARCH_USE_SIMSIMD=1", "-DUSEARCH_USE_FP16LIB=0", "-DUSEARCH_USE_OPENMP=0", "-DSIMSIMD_NATIVE_F16=0",
                    "-DSIMSIMD_NATIVE_BF16=0", "-DSIMSIMD_DYNAMIC_DISPATCH=1", f"-I{ref}/include", f"-I{ref}/simsimd/include",
                    f"-I{ref}/fp16/include", f"-I{here}", os.path.join(root, "tests", "native", "ref_indexes_driver.cpp"),
                    simsimd, "-o", out, "-lpthread", "-lm"], check=True, capture_output=True)
    lib = C.CDLL(out)
    u64p = C.POINTER(C.c_uint64)
    lib.ref_indexes_search_blobs.restype = C.c_char_p
    lib.ref_indexes_search_blobs.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_size_t, C.POINTER(C.c_size_t),
                                             C.c_size_t, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int,
                                             C.c_size_t, C.c_int, u64p, C.POINTER(C.c_float), u64p, u64p, u64p]
    _live["lib"] = lib
    return lib


def live_search(blobs: list, order: list, queries: np.ndarray, k: int, *, expansion: int = 64, query_scalar: str = "f32",
                exact: bool = False):
    """The reference's own `Indexes.search` loop on one thread over members blobs[order[0]], blobs[order[1]], ...
    (pinned metric, expansion_search = `expansion`): (keys, distances, counts, computed, visited)."""
    lib = _live_lib()
    blobs = [np.ascontiguousarray(b, dtype=np.uint8) for b in blobs]
    ptrs = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
    lengths = (C.c_size_t * len(blobs))(*[b.size for b in blobs])
    members = (C.c_size_t * max(len(order), 1))(*order)
    queries = np.ascontiguousarray(queries)
    nq = queries.shape[0]
    keys = np.zeros((nq, k), dtype=np.uint64)
    dists = np.zeros((nq, k), dtype=np.float32)
    counts, computed, visited = (np.zeros(nq, dtype=np.uint64) for _ in range(3))
    u64p = C.POINTER(C.c_uint64)
    err = lib.ref_indexes_search_blobs(ptrs, lengths, len(blobs), members, len(order), expansion, 1,
                                       queries.ctypes.data_as(C.c_void_p), nq, queries.strides[0], bindings.SCALAR[query_scalar],
                                       k, int(exact), keys.ctypes.data_as(u64p), dists.ctypes.data_as(C.POINTER(C.c_float)),
                                       counts.ctypes.data_as(u64p), computed.ctypes.data_as(u64p), visited.ctypes.data_as(u64p))
    if err:
        raise RuntimeError(err.decode())
    return keys, dists, counts, computed, visited
