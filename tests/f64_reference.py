"""The reference's f64 index (tests/native/ref_f64_driver.cpp), compiled at test time where the reference sources are,
and the f64 fixture (tests/golden/f64_cases.npz) it produced.

The fixture keeps its vectors as seeds: every row and query is `numpy.random.default_rng(seed).standard_normal`, which
gives the same doubles on every platform. NumPy does not promise that stream across its versions (NEP 19); it has not
changed since NumPy 1.17, and should it ever change, `case_blob` fails on the SHA-256 of the reference's file, which it
checks for every rebuilt graph, rather than let a test compare different data.

`PortF64` is the plain-C port of the search (oracle/hnsw_oracle.c) with the f64 pinned metric: it needs no reference
sources, so the GPU tests hold graphs that only exist on the GPU against it."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "f64_cases.npz")
METRIC = {"ip": ord("i"), "cos": ord("c"), "l2sq": ord("e")}
KIND = {"b1": 1, "bf16": 4, "f64": 10, "f32": 11, "f16": 12, "i8": 23}

_u64p, _f32p = C.POINTER(C.c_uint64), C.POINTER(C.c_float)


def rows(seed: int, n: int, d: int) -> np.ndarray:
    return np.random.default_rng(seed).standard_normal((n, d))


# ---- the fixture ---------------------------------------------------------------------------------------------------

def load_fixture() -> dict:
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def case_names(fx: dict) -> list[str]:
    return [str(s) for s in fx["cases"]]


def case_blob(fx: dict, name: str) -> tuple[np.ndarray, np.ndarray]:
    """(blob, base rows) of one fixture case; the blob is the reference's saved file, byte for byte"""
    n, d = int(fx[f"{name}/n"]), int(fx[f"{name}/d"])
    base = rows(int(fx[f"{name}/seed"]), n, d)
    head = np.array([n, d * 8], dtype=np.uint32).view(np.uint8)
    blob = np.concatenate([head, base.view(np.uint8).ravel(), fx[f"{name}/graph"]])
    assert hashlib.sha256(blob.tobytes()).hexdigest() == str(fx[f"{name}/sha256"]), \
        f"{name}: the rows rebuilt from the seed differ from the reference's file (has numpy's default_rng stream changed?)"
    return blob, base


def case_queries(fx: dict, name: str) -> np.ndarray:
    return rows(int(fx[f"{name}/seed"]) + 1, int(fx[f"{name}/nq"]), int(fx[f"{name}/d"]))


# ---- the live reference --------------------------------------------------------------------------------------------

def available() -> bool:
    from oracle import build as oracle_build
    return oracle_build.reference_available()


_libs: dict = {}


def lib(flavour: str = "parity"):
    if flavour in _libs:
        return _libs[flavour]
    from oracle import build as oracle_build
    oracle_build.build_reference(flavour)
    ref = oracle_build.REF
    simsimd = os.path.join(oracle_build.REF_OUT, f"simsimd_{flavour}.o")
    opt = ["-O2", "-ffp-contract=off", "-march=x86-64-v3"] if flavour == "parity" else ["-O3", "-ffast-math", "-march=native"]
    out = os.path.join(tempfile.mkdtemp(prefix="ref_f64_"), f"libref_f64_{flavour}.so")
    subprocess.run(["g++", "-std=c++17", *opt, "-fPIC", "-shared", "-w", "-DUSEARCH_USE_SIMSIMD=1", "-DUSEARCH_USE_FP16LIB=0",
                    "-DUSEARCH_USE_OPENMP=0", "-DSIMSIMD_NATIVE_F16=0", "-DSIMSIMD_NATIVE_BF16=0", "-DSIMSIMD_DYNAMIC_DISPATCH=1",
                    f"-I{ref}/include", f"-I{ref}/simsimd/include", f"-I{ref}/fp16/include", f"-I{os.path.join(ROOT, 'tests', 'native')}",
                    os.path.join(ROOT, "tests", "native", "ref_f64_driver.cpp"), simsimd, "-o", out, "-lpthread", "-lm"],
                   check=True, capture_output=True)
    L = C.CDLL(out)
    L.f64_make.restype = C.c_void_p
    L.f64_make.argtypes = [C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t]
    L.f64_free.argtypes = [C.c_void_p]
    L.f64_isa_name.restype = C.c_char_p
    L.f64_isa_name.argtypes = [C.c_void_p]
    for name in ("f64_size", "f64_serialized_length"):
        getattr(L, name).restype = C.c_size_t
        getattr(L, name).argtypes = [C.c_void_p]
    L.f64_change_expansion_search.argtypes = [C.c_void_p, C.c_size_t]
    L.f64_pin.argtypes = [C.c_void_p, C.c_int]
    L.f64_add.restype = C.c_size_t
    L.f64_add.argtypes = [C.c_void_p, _u64p, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t]
    L.f64_remove.restype = C.c_size_t
    L.f64_remove.argtypes = [C.c_void_p, C.c_uint64]
    L.f64_isolate.argtypes = [C.c_void_p]
    L.f64_save.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.f64_view.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.f64_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, _u64p, C.c_size_t,
                             _u64p, _f32p, _u64p, _u64p, _u64p]
    L.f64_cluster.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, _u64p, _f32p, _u64p, _u64p]
    L.f64_get.restype = C.c_size_t
    L.f64_get.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    L.f64_exact_search.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_size_t, C.c_size_t, C.c_int, _u64p, _f32p]
    L.f64_distance.restype = C.c_float
    L.f64_distance.argtypes = [C.c_int, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    _libs[flavour] = L
    return L


def _p(a, t=C.c_void_p):
    return a.ctypes.data_as(t)


class RefF64:
    """index_dense_gt<u64, u32> over f64 rows; `pin(True)` swaps the metric for tests/native/f64_pinned.h"""

    def __init__(self, metric: str, d: int, connectivity: int = 16, expansion_add: int = 128, expansion_search: int = 64,
                 flavour: str = "parity"):
        self.L = lib(flavour)
        self.d = d
        self.h = self.L.f64_make(METRIC[metric], d, connectivity, expansion_add, expansion_search)
        assert self.h, "f64_make failed"
        self._keep = None

    def __del__(self):
        if getattr(self, "h", None):
            self.L.f64_free(self.h)
            self.h = None

    isa_name = property(lambda s: s.L.f64_isa_name(s.h).decode())
    size = property(lambda s: s.L.f64_size(s.h))

    def pin(self, pinned: bool = True):
        assert self.L.f64_pin(self.h, int(pinned)) == 0

    def change_expansion_search(self, ef: int):
        self.L.f64_change_expansion_search(self.h, ef)

    def add(self, keys, vectors: np.ndarray, kind: str = "f64", threads: int = 1) -> int:
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        vectors = np.ascontiguousarray(vectors)
        return self.L.f64_add(self.h, _p(keys, _u64p), _p(vectors), KIND[kind], len(keys), vectors.strides[0], threads)

    def remove(self, key: int) -> int:
        return self.L.f64_remove(self.h, int(key))

    def isolate(self):
        self.L.f64_isolate(self.h)

    def save(self) -> np.ndarray:
        n = self.L.f64_serialized_length(self.h)
        buf = np.empty(n, dtype=np.uint8)
        assert self.L.f64_save(self.h, _p(buf), n) == 0
        return buf

    def view(self, blob: np.ndarray):
        self._keep = np.ascontiguousarray(blob, dtype=np.uint8)
        assert self.L.f64_view(self.h, _p(self._keep), self._keep.size) == 0

    def search(self, queries: np.ndarray, k: int, *, kind: str = "f64", exact: bool = False, allowed=None):
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        keys, dist = np.zeros((nq, k), dtype=np.uint64), np.zeros((nq, k), dtype=np.float32)
        counts, computed, visited = (np.zeros(nq, dtype=np.uint64) for _ in range(3))
        al = None if allowed is None else np.sort(np.ascontiguousarray(allowed, dtype=np.uint64))
        rc = self.L.f64_search(self.h, _p(queries), KIND[kind], nq, queries.strides[0], k, int(exact),
                               None if al is None else _p(al, _u64p), 0 if al is None else al.size,
                               _p(keys, _u64p), _p(dist, _f32p), _p(counts, _u64p), _p(computed, _u64p), _p(visited, _u64p))
        assert rc == 0, rc
        return keys, dist, counts, computed, visited

    def cluster(self, queries: np.ndarray, level: int):
        queries = np.ascontiguousarray(queries, dtype=np.float64)
        nq = queries.shape[0]
        keys, dist = np.zeros(nq, dtype=np.uint64), np.zeros(nq, dtype=np.float32)
        computed, visited = np.zeros(nq, dtype=np.uint64), np.zeros(nq, dtype=np.uint64)
        assert self.L.f64_cluster(self.h, _p(queries), nq, level, _p(keys, _u64p), _p(dist, _f32p), _p(computed, _u64p),
                                  _p(visited, _u64p)) == 0
        return keys, dist, computed, visited

    def get(self, key: int, kind: str) -> np.ndarray:
        cols = (self.d + 7) // 8 if kind == "b1" else self.d
        t = {"f64": np.float64, "f32": np.float32, "f16": np.float16, "bf16": np.uint16, "i8": np.int8, "b1": np.uint8}[kind]
        out = np.zeros(cols, dtype=t)
        assert self.L.f64_get(self.h, int(key), KIND[kind], _p(out)) == 1
        return out


# ---- the port over f64 graphs (no reference sources needed) ---------------------------------------------------------

_port = []


def port_lib():
    """tests/native/port_f64.c (oracle/hnsw_oracle.c with the f64 pinned metric), built once per process"""
    if _port:
        return _port[0]
    out = os.path.join(tempfile.mkdtemp(prefix="port_f64_"), "libport_f64.so")
    subprocess.run(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", os.path.join(ROOT, "oracle"),
                    "-I", os.path.join(ROOT, "tests", "native"), os.path.join(ROOT, "tests", "native", "port_f64.c"), "-o", out,
                    "-lm", "-lpthread"], check=True, capture_output=True)
    L = C.CDLL(out)
    L.oracle_open_f64.restype = C.c_void_p
    L.oracle_open_f64.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_char_p)]
    L.oracle_close_f64.argtypes = [C.c_void_p]
    L.oracle_change_expansion_search.argtypes = [C.c_void_p, C.c_size_t]
    L.oracle_distance.restype = C.c_float
    L.oracle_distance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.oracle_search_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int,
                                     _u64p, _f32p, _u64p, _u64p, _u64p]
    L.oracle_cluster_many.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, _u64p, _f32p, _u64p, _u64p]
    _port.append(L)
    return L


class PortF64:
    """the port's search, exact search, cluster and distance over a saved f64 graph"""

    def __init__(self, blob: np.ndarray, expansion_search: int = 64):
        self.L = port_lib()
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        err = C.c_char_p()
        self.h = self.L.oracle_open_f64(_p(blob), blob.size, C.byref(err))
        if not self.h:
            raise RuntimeError(err.value.decode())
        self.L.oracle_change_expansion_search(self.h, expansion_search)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.oracle_close_f64(self.h)
            self.h = None

    def change_expansion_search(self, ef: int):
        self.L.oracle_change_expansion_search(self.h, ef)

    def distance(self, a: np.ndarray, b: np.ndarray) -> float:
        a = np.ascontiguousarray(a, dtype=np.float64)
        b = np.ascontiguousarray(b, dtype=np.float64)
        return float(self.L.oracle_distance(self.h, _p(a), _p(b)))

    def search(self, queries: np.ndarray, k: int, *, exact: bool = False, threads: int = 8):
        queries = np.ascontiguousarray(queries, dtype=np.float64)
        nq = queries.shape[0]
        keys, dist = np.zeros((nq, k), dtype=np.uint64), np.zeros((nq, k), dtype=np.float32)
        counts, computed, visited = (np.zeros(nq, dtype=np.uint64) for _ in range(3))
        self.L.oracle_search_many(self.h, _p(queries), nq, queries.strides[0], k, threads, int(exact), _p(keys, _u64p),
                                  _p(dist, _f32p), _p(counts, _u64p), _p(computed, _u64p), _p(visited, _u64p))
        return keys, dist, counts, computed, visited

    def cluster(self, queries: np.ndarray, level: int):
        queries = np.ascontiguousarray(queries, dtype=np.float64)
        nq = queries.shape[0]
        keys, dist = np.zeros(nq, dtype=np.uint64), np.zeros(nq, dtype=np.float32)
        computed, visited = np.zeros(nq, dtype=np.uint64), np.zeros(nq, dtype=np.uint64)
        self.L.oracle_cluster_many(self.h, _p(queries), nq, queries.strides[0], level, _p(keys, _u64p), _p(dist, _f32p),
                                   _p(computed, _u64p), _p(visited, _u64p))
        return keys, dist, computed, visited


def exact_search(dataset: np.ndarray, queries: np.ndarray, k: int, metric: str, pinned: bool = True, flavour: str = "parity"):
    L = lib(flavour)
    dataset = np.ascontiguousarray(dataset, dtype=np.float64)
    queries = np.ascontiguousarray(queries, dtype=np.float64)
    nq, d = queries.shape
    keys, dist = np.zeros((nq, k), dtype=np.uint64), np.zeros((nq, k), dtype=np.float32)
    assert L.f64_exact_search(_p(dataset), dataset.shape[0], _p(queries), nq, METRIC[metric], d, k, int(pinned),
                              _p(keys, _u64p), _p(dist, _f32p)) == 0
    return keys, dist


def distance(metric: str, a: np.ndarray, b: np.ndarray, pinned: bool = True, flavour: str = "parity") -> float:
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    return float(lib(flavour).f64_distance(METRIC[metric], a.size, int(pinned), _p(a), _p(b)))


def port_join(a_blob, b_blob, max_proposals: int = 0, expansion: int = 64, exact: bool = False):
    """tests/join_reference.py's restatement of the reference's one-thread join, fed with the port's f64 searches and
    pinned metric instead of the live reference's: (a_to_b dict, stats dict)"""
    import join_reference as jr
    from usearch_b200 import v2format
    a_n, b_n = v2format.loads(a_blob).size, v2format.loads(b_blob).size
    swapped = b_n < a_n
    men_blob, women_blob = (b_blob, a_blob) if swapped else (a_blob, b_blob)
    men_g, men_keys, _ = jr._slot_keyed(men_blob)
    women_g, women_keys, women_slots = jr._slot_keyed(women_blob)
    men, women = len(men_keys), len(women_keys)
    stats = {"intersection_size": 0, "engagements": 0, "visited_members": 0, "computed_distances": 0}
    if men == 0:
        return {}, stats
    proposals = jr.default_proposals(men, max_proposals)
    port = PortF64(women_slots, expansion)
    rows_m = np.ascontiguousarray(men_g.vectors).view(np.float64).reshape(men, -1)
    rows_w = np.ascontiguousarray(women_g.vectors).view(np.float64).reshape(women, -1)
    columns = {}
    for i in range(1, proposals + 1):
        keys, dist, counts, computed, visited = port.search(rows_m, i, exact=exact)
        last = np.minimum(counts.astype(np.int64), i) - 1
        woman = keys[np.arange(men), last].astype(np.int64)
        from_woman = np.array([port.distance(rows_w[w], rows_m[m]) for m, w in enumerate(woman)], dtype=np.float32)
        columns[i] = (woman, dist[np.arange(men), last], from_woman, computed, visited)
    man_to_woman, engagements, visited, computed = jr.replay(men, women, proposals, columns)
    a_to_b = {}
    for m in range(men):
        w = man_to_woman[m]
        if w == jr.MISSING:
            continue
        stats["intersection_size"] += 1
        mk, wk = int(men_keys[m]), int(women_keys[w])
        if swapped:
            a_to_b[wk] = mk
        else:
            a_to_b[mk] = wk
    stats.update(engagements=engagements, visited_members=visited, computed_distances=computed)
    return a_to_b, stats
