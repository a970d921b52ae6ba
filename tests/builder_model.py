"""The GPU builder's batch schedule restated on the host (tests/native/builder_model.c), and `draw_level`.

`BuilderModel` starts from an empty graph or from a v2 blob and runs `add` as usearch_b200/csrc/builder.cu does
(DESIGN.md §3.5): the same batches, the same tasks, the same INSERT searches over the graph as it stood before each batch,
the same refine_ and the same reverse step, with the pinned metrics. Its lists are what a GPU build must produce, list
for list. It needs only oracle/ and tests/native/, so it runs wherever the repository is."""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMPTY = 0xFFFFFFFF
# batches, tasks and (level, neighbour) runs; reverse refines (on level 0 alone as well), runs cut to 256 - listed
# arrivals, candidate lists cut to 256, forward refines with fewer candidates than M, reverse sorts that met equal
# distances, reused members, arrivals dropped because the list already held them
COUNTERS = ("batches", "tasks", "reverse_runs", "reverse_refines", "reverse_refines_base", "room_cuts", "candidate_cuts",
            "short_refines", "sort_ties", "reused", "held_arrivals")
METRIC = {"ip": ord("i"), "cos": ord("c"), "l2sq": ord("e"), "hamming": ord("b"), "tanimoto": ord("t"),
          "sorensen": ord("s"), "jaccard": ord("j")}
SCALAR = {"b1": 1, "bf16": 4, "f64": 10, "f32": 11, "f16": 12, "i8": 23}

_vp, _u32p, _u64p, _f32p = C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
_lib = []


def lib():
    """tests/native/builder_model.c, compiled once per process"""
    if _lib:
        return _lib[0]
    out = os.path.join(tempfile.mkdtemp(prefix="builder_model_"), "libbuilder_model.so")
    subprocess.run(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", os.path.join(ROOT, "oracle"),
                    "-I", os.path.join(ROOT, "tests", "native"), os.path.join(ROOT, "tests", "native", "builder_model.c"),
                    "-o", out, "-lm", "-lpthread"], check=True, capture_output=True)
    L = C.CDLL(out)
    L.bm_new.restype = _vp
    L.bm_new.argtypes = [C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t]
    L.bm_open.restype = _vp
    L.bm_open.argtypes = [_vp, C.c_size_t, C.POINTER(C.c_char_p)]
    L.bm_free.argtypes = [_vp]
    L.bm_add.restype = C.c_int
    L.bm_add.argtypes = [_vp, _u64p, _vp, C.c_size_t, C.c_size_t, _vp, _u32p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t]
    L.bm_candidates.restype = C.c_long
    L.bm_candidates.argtypes = [_vp, _vp, C.c_uint32, C.c_size_t, C.c_size_t, _u32p, _f32p]
    for name in ("bm_size", "bm_connectivity", "bm_connectivity_base", "bm_entry", "bm_upper_rows"):
        getattr(L, name).restype = C.c_size_t
        getattr(L, name).argtypes = [_vp]
    L.bm_max_level.restype = C.c_long
    L.bm_max_level.argtypes = [_vp]
    L.bm_export.argtypes = [_vp, _vp, _u64p, _u32p, _u32p]
    L.bm_vectors.argtypes = [_vp, _vp]
    L.bm_batches.argtypes = [_vp, _vp, _vp]
    L.bm_counters.argtypes = [_vp, _u64p]
    L.bm_distance.restype = C.c_float
    L.bm_distance.argtypes = [_vp, C.c_uint32, C.c_uint32]
    _lib.append(L)
    return L


def _p(a, t=_vp):
    return a.ctypes.data_as(t)


def draw_level(slot: int, connectivity: int, seed: int = 0) -> int:
    """frozen_index_t::draw_level: the splitmix64 finaliser of (slot ^ seed * K), u = ((bits >> 11) + 1) / 2^53 in (0, 1],
    level = min(-ln u / ln M, 30), truncated"""
    mask = (1 << 64) - 1
    x = (slot ^ (seed * 0xD6E8FEB86659FD93)) & mask
    x = (x + 0x9E3779B97F4A7C15) & mask
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & mask
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & mask
    x ^= x >> 31
    u = (float(x >> 11) + 1.0) * (1.0 / 9007199254740992.0)
    r = -math.log(u) * (1.0 / math.log(connectivity))
    return int(min(r, 30.0))


def draw_levels(first: int, count: int, connectivity: int, seed: int = 0) -> np.ndarray:
    return np.array([draw_level(s, connectivity, seed) for s in range(first, first + count)], dtype=np.int16)


class BuilderModel:
    """The graph after `add`, as the GPU builder must leave it. Start from a saved file (`blob`) or from nothing."""

    def __init__(self, blob=None, *, metric: str = "", scalar: str = "", dims: int = 0, connectivity: int = 16,
                 connectivity_base: int = 0):
        self.L = lib()
        if blob is not None:
            blob = np.ascontiguousarray(blob, dtype=np.uint8)
            err = C.c_char_p()
            self.h = self.L.bm_open(_p(blob), blob.size, C.byref(err))
            if not self.h:
                raise RuntimeError(err.value.decode())
        else:
            self.h = self.L.bm_new(METRIC[metric], SCALAR[scalar], dims, connectivity, connectivity_base or 2 * connectivity)
            if not self.h:
                raise RuntimeError(f"no builder model for {metric} / {scalar}")

    def __del__(self):
        if getattr(self, "h", None):
            self.L.bm_free(self.h)
            self.h = None

    size = property(lambda s: s.L.bm_size(s.h))
    connectivity = property(lambda s: s.L.bm_connectivity(s.h))
    connectivity_base = property(lambda s: s.L.bm_connectivity_base(s.h))
    entry_slot = property(lambda s: s.L.bm_entry(s.h))
    max_level = property(lambda s: s.L.bm_max_level(s.h))

    def add(self, keys, rows: np.ndarray, levels, *, reuse=(), expansion_add: int = 128, batch: int = 32768, ratio: int = 32):
        """`rows` in the stored scalar kind; the first min(len, len(reuse)) go into the slots `reuse` (the free queue, oldest
        first), the others are appended with `levels`"""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        rows = np.ascontiguousarray(rows)
        reuse = np.ascontiguousarray(reuse, dtype=np.uint32)
        appended = len(keys) - min(len(keys), len(reuse))
        levels = np.ascontiguousarray(levels, dtype=np.int16)
        assert levels.size == appended, (levels.size, appended)
        rc = self.L.bm_add(self.h, _p(keys, _u64p), _p(rows), len(keys), rows.strides[0], _p(levels), _p(reuse, _u32p),
                           reuse.size, expansion_add, batch, ratio)
        assert rc == 0, f"bm_add failed ({rc})"

    def candidates(self, row: np.ndarray, level: int, ef: int, self_slot: int = EMPTY):
        """the candidate slots and distances of one INSERT task over the current graph"""
        row = np.ascontiguousarray(row)
        slots, dists = np.zeros(ef, np.uint32), np.zeros(ef, np.float32)
        n = self.L.bm_candidates(self.h, _p(row), self_slot, level, ef, _p(slots, _u32p), _p(dists, _f32p))
        assert n >= 0
        return slots[:n], dists[:n]

    def counters(self) -> dict:
        out = np.zeros(len(COUNTERS), np.uint64)
        self.L.bm_counters(self.h, _p(out, _u64p))
        return {k: int(v) for k, v in zip(COUNTERS, out)}

    def batches(self):
        """per slot: the batch (numbered from 0 over the model's life) that linked it, and the last one that wrote one
        of its rows; -1 for slots of the starting graph that no batch touched"""
        linked, written = np.zeros(self.size, np.int32), np.zeros(self.size, np.int32)
        self.L.bm_batches(self.h, _p(linked), _p(written))
        return linked, written

    def distance(self, a: int, b: int) -> float:
        """the pinned metric between two stored slots, `a` as the query"""
        return float(self.L.bm_distance(self.h, a, b))

    def neighbors(self):
        """(levels, keys, [slot][level] -> list of slots), the shape of v2format.Graph.neighbors"""
        n, m, m0 = self.size, self.connectivity, self.connectivity_base
        levels, keys = np.zeros(n, np.int16), np.zeros(n, np.uint64)
        rows0 = np.zeros((n, m0), np.uint32)
        upper = np.zeros((max(self.L.bm_upper_rows(self.h), 1), m), np.uint32)
        self.L.bm_export(self.h, _p(levels), _p(keys, _u64p), _p(rows0, _u32p), _p(upper, _u32p))
        out, u = [], 0
        for s in range(n):
            per = [rows0[s][rows0[s] != EMPTY].tolist()]
            for _ in range(int(levels[s])):
                per.append(upper[u][upper[u] != EMPTY].tolist())
                u += 1
            out.append(per)
        return levels, keys, out

    def graph(self, metric: str, scalar: str, dims: int):
        """the model's graph as a v2format.Graph (save it with v2format.dumps)"""
        from usearch_b200 import v2format
        levels, keys, lists = self.neighbors()
        bpv = (dims * v2format.SCALAR_BITS[scalar] + 7) // 8
        vectors = np.zeros((self.size, bpv), np.uint8)
        self.L.bm_vectors(self.h, _p(vectors))
        return v2format.Graph(metric, scalar, dims, self.connectivity, self.connectivity_base, vectors, keys, levels, lists,
                              int(self.max_level), int(self.entry_slot))
