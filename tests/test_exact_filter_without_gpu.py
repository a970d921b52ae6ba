"""Exact filtered search without a GPU: the entries are exported and declared, a C++11 client of the mirror (the set-based
forms and the reference's predicate overload) compiles, and the Python argument checks raise before the library is
called."""
import os
import re
import subprocess

import numpy as np
import pytest

import common

NATIVE = os.path.join(common.ROOT, "tests", "native")
ENTRIES = ["usearch_b200_grouped_filtered_exact_search_many", "usearch_b200_grouped_filtered_exact_search_many_device"]


def test_entries_are_exported_and_declared():
    from usearch_b200.index import EXPORTED_SYMBOLS, load_library
    lib = load_library()
    header = open(os.path.join(common.ROOT, "include", "usearch_b200.h")).read()
    for name in ENTRIES:
        assert name in EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\b%s\(" % name, header), name
    mirror = open(os.path.join(common.ROOT, "include", "usearch_b200.hpp")).read()
    for name in ("grouped_filtered_exact_search", "grouped_filtered_exact_search_device"):
        assert re.search(r"\b%s\(" % name, mirror), name
    assert re.search(r"search_result_t filtered_search\(scalar_at const\* vector, std::size_t wanted, predicate_at&& predicate", mirror)


def test_cpp_mirror_client_compiles(tmp_path):
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Wextra", "-Werror", "-Wno-unused-variable", "-O1", "-I",
                    os.path.join(common.ROOT, "include"), "-c", os.path.join(NATIVE, "test_exact_filter_client.cpp"), "-o",
                    str(tmp_path / "client.o")], check=True, capture_output=True)


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"the library was called: {name}")


def _index():
    from usearch_b200.index import Index
    index = Index(ndim=8, metric="l2sq", dtype="f32")
    index._lib = _NoLibrary()
    return index


@pytest.mark.parametrize("key_sets,groups,message", [
    ([[1, 2]] * 3, None, "one set per query"),
    ([[1, 2], [3]], [0, 1], "one set index per query"),
    ([[1, 2], [3]], [[0, 1, 1, 0]], "one set index per query"),
    ([[1, 2], [3]], [0, 1, 2, 0], "out of range"),
    ([[1, 2], [3]], [0, -1, 1, 0], "out of range"),
    ([1, 2, 3, 4], None, "not of keys"),
])
def test_grouped_argument_checks_come_first(key_sets, groups, message):
    with pytest.raises(ValueError, match=message):
        _index().grouped_filtered_search(np.zeros((4, 8), np.float32), 10, key_sets, groups, exact=True)


def test_single_set_argument_checks_come_first():
    index = _index()
    for not_a_set in ([[1, 2], [3, 4]], 5, np.uint64(5), np.array(5, np.uint64)):
        with pytest.raises(ValueError, match="flat sequence of keys"):
            index.filtered_search(np.zeros((4, 8), np.float32), 10, not_a_set, exact=True)
    with pytest.raises(ValueError, match="no visited_members"):
        index.filtered_search_device(1, 1, 32, 10, 1, 1, 1, 1, 1, 0, 1, exact=True)
    with pytest.raises(ValueError, match="no visited_members"):
        index.grouped_filtered_search_device(1, 1, 32, 10, 0, 1, 1, 1, 1, 1, 1, 0, 1, exact=True)
