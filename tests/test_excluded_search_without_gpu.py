"""Excluded search without a GPU: the entries are exported and declared, a C++11 client of the mirror compiles, and the
Python argument checks raise before the library is called."""
import os
import re
import subprocess

import numpy as np
import pytest

import common

NATIVE = os.path.join(common.ROOT, "tests", "native")
ENTRIES = ["usearch_b200_grouped_excluded_search_many", "usearch_b200_grouped_excluded_search_many_device",
           "usearch_b200_grouped_excluded_exact_search_many", "usearch_b200_grouped_excluded_exact_search_many_device"]


def test_entries_are_exported_and_declared():
    from usearch_b200.index import EXPORTED_SYMBOLS, load_library
    lib = load_library()
    header = open(os.path.join(common.ROOT, "include", "usearch_b200.h")).read()
    for name in ENTRIES:
        assert name in EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\b%s\(" % name, header), name
    mirror = open(os.path.join(common.ROOT, "include", "usearch_b200.hpp")).read()
    for name in ("grouped_excluded_search", "grouped_excluded_search_device", "grouped_excluded_exact_search",
                 "grouped_excluded_exact_search_device"):
        assert re.search(r"\b%s\(" % name, mirror), name


def test_cpp_mirror_client_compiles(tmp_path):
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Wextra", "-Werror", "-Wno-unused-variable", "-O1", "-I",
                    os.path.join(common.ROOT, "include"), "-c", os.path.join(NATIVE, "test_excluded_search_client.cpp"), "-o",
                    str(tmp_path / "client.o")], check=True, capture_output=True)


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"the library was called: {name}")


def _index():
    from usearch_b200.index import Index
    index = Index(ndim=8, metric="l2sq", dtype="f32")
    index._lib = _NoLibrary()
    return index


@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("key_sets,groups,message", [
    ([[1, 2]] * 3, None, "one set per query"),
    ([[1, 2], [3]], [0, 1], "one set index per query"),
    ([[1, 2], [3]], [[0, 1, 1, 0]], "one set index per query"),
    ([[1, 2], [3]], [0, 1, 2, 0], "out of range"),
    ([[1, 2], [3]], [0, -1, 1, 0], "out of range"),
    ([1, 2, 3, 4], None, "not of keys"),
])
def test_grouped_argument_checks_come_first(key_sets, groups, message, exact):
    with pytest.raises(ValueError, match=message):
        _index().grouped_excluded_search(np.zeros((4, 8), np.float32), 10, key_sets, groups, exact=exact)


@pytest.mark.parametrize("exact", [False, True])
def test_single_set_and_device_argument_checks_come_first(exact):
    index = _index()
    for not_a_set in ([[1, 2], [3, 4]], 5, np.uint64(5), np.array(5, np.uint64)):
        with pytest.raises(ValueError, match="flat sequence of keys"):
            index.excluded_search(np.zeros((4, 8), np.float32), 10, not_a_set, exact=exact)
    with pytest.raises(ValueError, match="matrix or a vector"):
        index.grouped_excluded_search(np.zeros((2, 2, 8), np.float32), 10, [[1]] * 2, exact=exact)
    with pytest.raises(ValueError, match="no visited_members"):
        index.grouped_excluded_search_device(1, 1, 32, 10, 0, 1, 1, 1, 1, 1, 1, 0, 1, exact=True)
