"""CPU tests of the index-surface model (tests/surface_reference.py) against the reference itself: its three `stats`
functions, `export_keys` (as a set: the reference lists keys in hash-table order, the model in slot order) and `get`,
on the committed golden graphs and on graphs the reference builds with multi keys, removals, isolate and slot reuse.
The reference is compiled at test time from tests/native/ref_surface_driver.cpp where its sources lie; else these skip.
Also: the new calls of `Index` raise without a device instead of answering from the host."""
import ctypes as C
import glob
import os
import subprocess
import tempfile

import numpy as np
import pytest

import common
import surface_reference as model

_lib = {}


def _driver():
    from oracle import build as oracle_build
    if not oracle_build.reference_available():
        pytest.skip("the reference's sources are not present")
    if "lib" in _lib:
        return _lib["lib"]
    ref = oracle_build.REF
    out = os.path.join(tempfile.mkdtemp(prefix="ref_surface_"), "libref_surface.so")
    proc = subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-DUSEARCH_USE_SIMSIMD=0",
                           "-DUSEARCH_USE_FP16LIB=1", "-DUSEARCH_USE_OPENMP=0", f"-I{ref}/include", f"-I{ref}/fp16/include",
                           os.path.join(common.ROOT, "tests", "native", "ref_surface_driver.cpp"), "-o", out, "-lpthread", "-lm"],
                          capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-2000:]
    lib = C.CDLL(out)
    sz = C.POINTER(C.c_size_t)
    lib.ref_surface_scenario.restype = C.c_char_p
    lib.ref_surface_scenario.argtypes = [C.c_int, C.c_size_t, C.c_size_t, C.POINTER(C.POINTER(C.c_uint8)), sz]
    lib.ref_surface_free.argtypes = [C.c_void_p]
    lib.ref_surface_describe.restype = C.c_char_p
    lib.ref_surface_describe.argtypes = [C.c_void_p, C.c_size_t, sz, sz, sz, sz, sz, C.c_size_t, C.c_void_p, C.c_size_t, sz]
    lib.ref_surface_get.restype = C.c_char_p
    lib.ref_surface_get.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    _lib["lib"] = lib
    return lib


def _scenario(which: int, n: int = 600, dims: int = 24) -> np.ndarray:
    lib = _driver()
    ptr, length = C.POINTER(C.c_uint8)(), C.c_size_t()
    err = lib.ref_surface_scenario(which, n, dims, C.byref(ptr), C.byref(length))
    assert err is None, err
    blob = np.ctypeslib.as_array(ptr, shape=(length.value,)).copy()
    lib.ref_surface_free(ptr)
    return blob


def _describe(blob: np.ndarray):
    lib = _driver()
    cap = 64
    top = C.c_size_t()
    total, per_total = np.zeros(4, np.uintp), np.zeros(4, np.uintp)
    level4, per4 = np.zeros((cap, 4), np.uintp), np.zeros((cap, 4), np.uintp)
    g = model.parse(blob)
    keys = np.zeros(max(len(g.keys), 1), np.uint64)
    nkeys = C.c_size_t()
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_size_t))  # noqa: E731
    err = lib.ref_surface_describe(blob.ctypes.data, blob.size, C.byref(top), p(total), p(level4), p(per4), p(per_total), cap,
                                   keys.ctypes.data, keys.size, C.byref(nkeys))
    assert err is None, err
    t = top.value
    as_tuples = lambda a: [tuple(int(x) for x in row) for row in a]  # noqa: E731
    return dict(total=tuple(int(x) for x in total), level=as_tuples(level4[:t + 2]), per=as_tuples(per4[:t + 1]),
                per_total=tuple(int(x) for x in per_total), keys=keys[:nkeys.value], max_level=t)


def _reference_rows(blob: np.ndarray, keys: np.ndarray):
    g = model.parse(blob)
    rows = np.zeros((len(g.keys) + 1, g.matrix.shape[1]), np.uint8)
    counts = np.zeros(keys.size, np.uintp)
    keys = np.ascontiguousarray(keys, np.uint64)
    err = _driver().ref_surface_get(blob.ctypes.data, blob.size, keys.ctypes.data, keys.size, rows.ctypes.data, rows.shape[0],
                                    counts.ctypes.data)
    assert err is None, err
    return rows, counts


def _check(blob: np.ndarray):
    want = _describe(blob)
    g = model.parse(blob)
    assert model.stats(g) == want["total"]
    for level in range(want["max_level"] + 2):
        assert model.level_stats(g, level) == want["level"][level], level
    per, per_total = model.levels_stats(g)
    assert per == want["per"] and per_total == want["per_total"]
    live = model.live_keys(g)
    assert sorted(live.tolist()) == sorted(want["keys"].tolist())
    unique = np.unique(live)
    rows, counts = _reference_rows(blob, unique)
    at = 0
    for key, c in zip(unique, counts):
        mine = model.rows_of(g, key)
        assert mine.shape[0] == int(c)
        # a multi key's rows come back in the reference's lookup order: compare them as a multiset
        assert sorted(map(bytes, mine)) == sorted(map(bytes, rows[at:at + int(c)]))
        at += int(c)
    return g


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(common.GOLDEN, "*_n*_d*.npz"))), ids=os.path.basename)
def test_model_matches_the_reference_on_golden_graphs(path):
    _check(np.load(path)["blob"])


@pytest.mark.parametrize("which,name", [(0, "multi"), (1, "removed"), (2, "removed_isolated"), (3, "reused")])
def test_model_matches_the_reference_on_edited_graphs(which, name):
    g = _check(_scenario(which))
    if name == "multi":
        assert g.multi and len(np.unique(model.live_keys(g))) < len(model.live_keys(g))
    if name.startswith("removed"):
        assert (g.keys == model.FREE_KEY).sum() == 200
    if name == "reused":
        assert (g.keys == model.FREE_KEY).sum() == 50 and ((g.keys >= 1000000) & (g.keys != model.FREE_KEY)).sum() == 150


def test_isolate_prunes_what_the_model_counts():
    before, after = model.parse(_scenario(1)), model.parse(_scenario(2))
    assert model.stats(after)[1] < model.stats(before)[1]
    assert model.stats(after)[0] == model.stats(before)[0]  # removed members still count as nodes


def test_new_calls_raise_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    from usearch_b200.index import Index
    index = Index(ndim=16, metric="cos", dtype="f32")
    assert len(index.keys) == 0 and index.multi is False and index.nlevels == 1
    for call in (lambda: index.get([1, 2]), lambda: index.get(np.array([1], np.int32), dtype=np.float16),
                 lambda: index[[1, 2]], lambda: list(index.keys), lambda: np.asarray(index.keys), lambda: index.vectors,
                 lambda: index.copy(), lambda: index.stats, lambda: index.levels_stats, lambda: index.level_stats(0)):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            call()
    index.reset()  # releases nothing and keeps the configuration
    assert index.ndim == 16
    with pytest.raises(ValueError, match="Unsupported dtype"):
        index.get([1], dtype=np.int64)
