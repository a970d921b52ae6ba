"""The chunked free exact search without a GPU: the device entry is exported and declared, a C++11 client of the mirror
compiles, the Python argument errors come before any library call, and without a device both entries fail loudly."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import common

NATIVE = os.path.join(common.ROOT, "tests", "native")


def test_entry_is_exported_and_declared():
    from usearch_b200.index import EXPORTED_SYMBOLS, load_library
    lib = load_library()
    header = open(os.path.join(common.ROOT, "include", "usearch_b200.h")).read()
    assert "usearch_b200_exact_search_device" in EXPORTED_SYMBOLS and hasattr(lib, "usearch_b200_exact_search_device")
    assert re.search(r"\busearch_b200_exact_search_device\(void const\* dataset, size_t dataset_size, size_t dataset_stride", header)
    assert re.search(r"\busearch_exact_search\(", header)
    mirror = open(os.path.join(common.ROOT, "include", "usearch_b200.hpp")).read()
    for name in ("exact_search", "exact_search_device"):
        assert re.search(r"\berror_t %s\(" % name, mirror), name


def test_cpp_mirror_client_compiles(tmp_path):
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Wextra", "-Werror", "-Wno-unused-variable", "-O1", "-I",
                    os.path.join(common.ROOT, "include"), "-c", os.path.join(NATIVE, "test_exact_chunked_client.cpp"), "-o",
                    str(tmp_path / "client.o")], check=True, capture_output=True)


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError(f"the library was called: {name}")


@pytest.fixture
def no_library(monkeypatch):
    import usearch_b200.index as m
    monkeypatch.setattr(m, "_lib", _NoLibrary())
    return m


def test_host_argument_checks_come_first(no_library):
    m = no_library
    rows = np.zeros((10, 8), np.float32)
    with pytest.raises(ValueError, match="matrix"):
        m.exact_search(np.zeros(8, np.float32), rows, 3)
    with pytest.raises(ValueError, match="dimensions differ"):
        m.exact_search(rows, np.zeros((2, 9), np.float32), 3)
    with pytest.raises(ValueError, match="negative"):
        m.exact_search(rows, rows, -1)
    with pytest.raises(ValueError, match="negative"):
        m.exact_search(rows, rows, 3, threads=-2)
    with pytest.raises(ValueError, match="matrix"):
        m.search(np.zeros((2, 3, 8), np.float32), rows, 3, exact=True)
    with pytest.raises(ValueError, match="dimensions differ"):
        m.search(rows, np.zeros(9, np.float32), 3, exact=True)
    with pytest.raises(ValueError, match="Unknown metric"):
        m.search(rows, rows, 3, "nope", exact=True)


@pytest.mark.parametrize("kwargs,message", [
    (dict(n=-1), "n must not be negative"),
    (dict(count=-3), "count must not be negative"),
    (dict(dataset_stride=-4), "dataset_stride must not be negative"),
    (dict(dtype="f128"), "Unknown dtype"),
    (dict(metric="nope"), "Unknown metric"),
])
def test_device_argument_checks_come_first(no_library, kwargs, message):
    args = dict(dataset_ptr=1, n=10, dataset_stride=32, queries_ptr=1, nq=2, queries_stride=32, ndim=8, count=3, keys_ptr=1,
                distances_ptr=1)
    extra = {k: kwargs.pop(k) for k in ("dtype", "metric") if k in kwargs}
    args.update(kwargs)
    with pytest.raises(ValueError, match=message):
        no_library.exact_search_device(**args, **extra)


def test_without_a_device_both_entries_fail_loudly():
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import numpy as np\n"
            "from usearch_b200.index import exact_search, exact_search_device\n"
            "rows = np.ones((64, 16), np.float32)\n"
            "for call in (lambda: exact_search(rows, rows[:4], 3), lambda: exact_search_device(1, 64, 64, 1, 4, 64, 16, 3, 1, 1)):\n"
            "    try:\n"
            "        call()\n"
            "        print('SERVED')\n"
            "    except RuntimeError as e:\n"
            "        print('REFUSED', e)\n") % common.ROOT
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    lines = out.stdout.strip().splitlines()
    assert lines == ["REFUSED No CUDA device: the GPU search backend has no CPU fallback"] * 2, out.stdout
