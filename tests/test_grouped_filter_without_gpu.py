"""Grouped filtered search without a GPU: the entries are exported and declared, a C++11 client of the mirror compiles,
and the Python argument checks raise before the library is called."""
import os
import re
import subprocess

import numpy as np
import pytest

import common

NATIVE = os.path.join(common.ROOT, "tests", "native")
ENTRIES = ["usearch_b200_grouped_filtered_search_many", "usearch_b200_grouped_filtered_search_many_device"]


def test_entries_are_exported_and_declared():
    from usearch_b200.index import EXPORTED_SYMBOLS, load_library
    lib = load_library()
    header = open(os.path.join(common.ROOT, "include", "usearch_b200.h")).read()
    for name in ENTRIES:
        assert name in EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\b%s\(" % name, header), name


def test_cpp_mirror_client_compiles(tmp_path):
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(common.ROOT, "include"), "-c",
                    os.path.join(NATIVE, "test_grouped_filter_client.cpp"), "-o", str(tmp_path / "client.o")],
                   check=True, capture_output=True)


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"the library was called: {name}")


@pytest.mark.parametrize("key_sets,groups,message", [
    ([[1, 2]] * 3, None, "one set per query"),                 # groups=None needs len(key_sets) == nq
    ([[1, 2], [3]], [0, 1], "one set index per query"),        # groups shorter than the batch
    ([[1, 2], [3]], [[0, 1, 1, 0]], "one set index per query"),
    ([[1, 2], [3]], [0, 1, 2, 0], "out of range"),
    ([[1, 2], [3]], [0, -1, 1, 0], "out of range"),
    ([1, 2, 3, 4], None, "not of keys"),                        # a flat key list is not a list of sets
])
def test_argument_checks_come_first(key_sets, groups, message):
    from usearch_b200.index import Index
    index = Index(ndim=8, metric="l2sq", dtype="f32")
    index._lib = _NoLibrary()
    with pytest.raises(ValueError, match=message):
        index.grouped_filtered_search(np.zeros((4, 8), np.float32), 10, key_sets, groups)
