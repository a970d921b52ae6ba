"""CPU tests of the lookups by key from device memory: the key -> slot table's insert and probe run natively on the
host against the host map, the three entries are exported and report a missing device without touching their pointers,
and a C++11 client of the header mirror compiles."""
import os
import subprocess

import pytest

import common

NATIVE = os.path.join(common.ROOT, "tests", "native")
CSRC = os.path.join(common.ROOT, "usearch_b200", "csrc")
ENTRIES = ["usearch_b200_count_many_device", "usearch_b200_get_many_device", "usearch_b200_filtered_search_many_device"]


def test_device_key_table_native(tmp_path):
    """Shuffled insert orders (a 1000-entry multi key, removed slots) find the slots the host map finds; sizing and load
    factor as documented."""
    exe = tmp_path / "device_keys"
    subprocess.run(["g++", "-std=c++11", "-O1", "-Wall", "-Wextra", "-Werror", "-I", CSRC,
                    os.path.join(NATIVE, "test_device_keys.cpp"), "-o", str(exe)], check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert "DEVICE_KEYS_OK" in out


def test_cpp_mirror_device_lookups_compile(tmp_path):
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Wextra", "-Werror", "-O1", "-I", os.path.join(common.ROOT, "include"), "-c",
                    os.path.join(NATIVE, "test_device_lookup_client.cpp"), "-o", str(tmp_path / "client.o")],
                   check=True, capture_output=True)


def test_entries_are_exported():
    from usearch_b200.index import EXPORTED_SYMBOLS, load_library
    lib = load_library()
    for name in ENTRIES:
        assert name in EXPORTED_SYMBOLS and hasattr(lib, name)


def _have_device():
    import torch
    return torch.cuda.is_available()


def test_each_entry_reports_a_missing_device():
    if _have_device():
        pytest.skip("a CUDA device is present")
    from usearch_b200.index import Index
    index = Index(ndim=16, metric="l2sq", dtype="f32")
    calls = [lambda: index.count_device(0, 4, 0),
             lambda: index.get_device(0, 4, 0, 0, count=2, dtype="f16"),
             lambda: index.filtered_search_device(0, 4, 64, 10, 0, 3, 0, 0, 0)]
    for call in calls:
        with pytest.raises(RuntimeError, match="No CUDA device"):
            call()
