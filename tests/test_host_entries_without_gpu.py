"""The C search entries on host buffers, called through ctypes past the Python checks, on an index without members: each
answers with padded empty rows and returns a total of 0, with or without `counts`, and the grouped entries refuse
malformed key sets with their own messages, in their own order, before writing any output: the allowed and excluded sets,
graph and exact, through the one host body they share. None of this needs a device."""
import ctypes as C

import numpy as np
import pytest

import common  # noqa: F401  (the repository on sys.path)

NQ, K, DIM = 3, 4, 8
SNAN_BITS = 0x7FA00000
FILTER = C.CFUNCTYPE(C.c_int, C.c_uint64, C.c_void_p)
NO_SETS = "A batch of queries needs at least one key set"
BAD_GROUP = "A query's key set index is out of range"
BAD_OFFSETS = "Key set offsets must start at 0 and never decrease"
NO_GROUPS = "Without a set index per query, there must be exactly one key set"


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def lib():
    from usearch_b200.index import LIB_PATH, load_library
    load_library()
    lib = C.CDLL(LIB_PATH)  # function objects of its own: the argument types set here stay out of the package's
    err, p, n = C.POINTER(C.c_char_p), C.c_void_p, C.c_size_t
    lib.usearch_init.restype = p
    lib.usearch_free.argtypes = [p, err]
    for name in ("usearch_b200_filtered_search_many", "usearch_filtered_search", "usearch_b200_grouped_filtered_search_many",
                 "usearch_b200_grouped_filtered_exact_search_many", "usearch_b200_grouped_excluded_search_many",
                 "usearch_b200_grouped_excluded_exact_search_many", "usearch_b200_exact_search_many"):
        getattr(lib, name).restype = n
    lib.usearch_b200_filtered_search_many.argtypes = [p, p, n, n, C.c_int, n, p, n, p, p, p, p, p, err]
    lib.usearch_filtered_search.argtypes = [p, p, C.c_int, n, FILTER, p, p, p, err]
    lib.usearch_b200_grouped_filtered_search_many.argtypes = [p, p, n, n, C.c_int, n, p, p, n, p, p, p, p, p, p, err]
    lib.usearch_b200_grouped_filtered_exact_search_many.argtypes = [p, p, n, n, C.c_int, n, p, p, n, p, p, p, p, p, err]
    lib.usearch_b200_grouped_excluded_search_many.argtypes = lib.usearch_b200_grouped_filtered_search_many.argtypes
    lib.usearch_b200_grouped_excluded_exact_search_many.argtypes = lib.usearch_b200_grouped_filtered_exact_search_many.argtypes
    lib.usearch_b200_exact_search_many.argtypes = [p, p, n, n, C.c_int, n, p, p, p, err]
    return lib


@pytest.fixture
def index(lib):
    from usearch_b200.index import METRIC_KIND, SCALAR_KIND, _InitOptions
    opts = _InitOptions(METRIC_KIND["l2sq"], None, SCALAR_KIND["f32"], DIM, 16, 128, 64, False)
    err = C.c_char_p()
    handle = lib.usearch_init(C.byref(opts), C.byref(err))
    assert handle and err.value is None
    yield C.c_void_p(handle)
    lib.usearch_free(handle, None)


QUERIES = np.ones((NQ, DIM), np.float32)
F32 = 1  # usearch_scalar_f32_k
KEEP_ALL = FILTER(lambda key, state: 1)


def _grouped(lib, index, excluded, exact, groups, offsets, set_keys):
    """the grouped entry of the mode, as call(keys, dists, counts, computed, visited, error)"""
    def call(keys, dists, counts, computed, visited, error):
        head = (index, QUERIES.ctypes.data, NQ, DIM * 4, F32, K, _ptr(groups), _ptr(offsets), len(offsets) - 1, _ptr(set_keys),
                _ptr(keys), _ptr(dists), _ptr(counts), _ptr(computed))
        form = "excluded" if excluded else "filtered"
        if exact:
            return getattr(lib, f"usearch_b200_grouped_{form}_exact_search_many")(*head, error)
        return getattr(lib, f"usearch_b200_grouped_{form}_search_many")(*head, _ptr(visited), error)
    return call


def _entry(lib, index, name):
    """(queries, counters the entry writes, call(keys, dists, counts, computed, visited, error))"""
    sets = (np.array([0, 1, 0], np.uint32), np.array([0, 2, 3], np.uint64), np.array([1, 2, 3], np.uint64))
    allowed = np.array([1, 2, 3], np.uint64)
    if name == "filtered_search_many":
        return NQ, ("computed", "visited"), lambda k, d, c, cm, v, e: lib.usearch_b200_filtered_search_many(
            index, QUERIES.ctypes.data, NQ, DIM * 4, F32, K, _ptr(allowed), len(allowed), _ptr(k), _ptr(d), _ptr(c), _ptr(cm),
            _ptr(v), e)
    if name == "filtered_search":
        return 1, (), lambda k, d, c, cm, v, e: lib.usearch_filtered_search(index, QUERIES.ctypes.data, F32, K, KEEP_ALL, None,
                                                                            _ptr(k), _ptr(d), e)
    if name == "grouped_filtered_search_many":
        return NQ, ("computed", "visited"), _grouped(lib, index, False, False, *sets)
    if name == "grouped_filtered_exact_search_many":
        return NQ, ("computed",), _grouped(lib, index, False, True, *sets)
    if name == "grouped_excluded_search_many":
        return NQ, ("computed", "visited"), _grouped(lib, index, True, False, *sets)
    if name == "grouped_excluded_exact_search_many":
        return NQ, ("computed",), _grouped(lib, index, True, True, *sets)
    assert name == "exact_search_many"
    return NQ, (), lambda k, d, c, cm, v, e: lib.usearch_b200_exact_search_many(index, QUERIES.ctypes.data, NQ, DIM * 4, F32, K,
                                                                                _ptr(k), _ptr(d), _ptr(c), e)


ENTRIES = ["filtered_search_many", "filtered_search", "grouped_filtered_search_many", "grouped_filtered_exact_search_many",
           "exact_search_many", "grouped_excluded_search_many", "grouped_excluded_exact_search_many"]


@pytest.mark.parametrize("with_counts", [True, False])
@pytest.mark.parametrize("name", ENTRIES)
def test_an_index_without_members_answers_padded_rows_and_a_zero_total(lib, index, name, with_counts):
    nq, counters, call = _entry(lib, index, name)
    keys, dists = np.full((nq, K), 7, np.uint64), np.zeros((nq, K), np.float32)
    counts = np.full(nq, 9, np.uintp) if with_counts else None
    computed, visited = np.full(nq, 9, np.uint64), np.full(nq, 9, np.uint64)
    err = C.c_char_p()
    total = call(keys, dists, counts, computed, visited, C.byref(err))
    assert err.value is None and total == 0
    assert (keys == 0).all() and (dists.view(np.uint32) == SNAN_BITS).all()
    if with_counts and name != "filtered_search":
        assert (counts == 0).all()
    assert (computed == 0).all() == ("computed" in counters)
    assert (visited == 0).all() == ("visited" in counters)


# the allowed forms keep the ids "False" / "True" (exact) they had before the excluded forms joined
@pytest.mark.parametrize("excluded,exact", [(False, False), (False, True), (True, False), (True, True)],
                         ids=["False", "True", "excluded-False", "excluded-True"])
@pytest.mark.parametrize("groups,offsets,message", [
    ([0, 1, 0], [1, 2, 3], BAD_OFFSETS),    # offsets not starting at 0
    ([0, 1, 0], [0, 2, 1], BAD_OFFSETS),    # offsets decreasing
    ([0, 2, 0], [0, 2, 3], BAD_GROUP),      # a set index past the last set
    ([0, 5, 0], [1, 2, 3], BAD_OFFSETS),    # the offsets are checked before the set indices
    (None, [0, 2, 3], NO_GROUPS),           # no set indices, two sets
    (None, [1, 2, 0], NO_GROUPS),           # ... checked before the offsets
    ([0, 0, 0], [0], NO_SETS),              # zero sets
    (None, [0], NO_SETS),                   # ... checked first
])
def test_grouped_entries_refuse_malformed_sets_before_writing(lib, index, excluded, exact, groups, offsets, message):
    groups = None if groups is None else np.array(groups, np.uint32)
    call = _grouped(lib, index, excluded, exact, groups, np.array(offsets, np.uint64), np.array([1, 2, 3], np.uint64))
    keys, dists = np.full((NQ, K), 7, np.uint64), np.zeros((NQ, K), np.float32)
    counts, computed, visited = np.full(NQ, 9, np.uintp), np.full(NQ, 9, np.uint64), np.full(NQ, 9, np.uint64)
    err = C.c_char_p()
    assert call(keys, dists, counts, computed, visited, C.byref(err)) == 0
    assert err.value is not None and err.value.decode() == message
    assert (keys == 7).all() and (dists == 0).all() and (counts == 9).all() and (computed == 9).all() and (visited == 9).all()
