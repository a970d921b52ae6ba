"""CPU tests of the boundary: the shared library loads, exports every symbol the header declares,
and — with no GPU in this container — fails loudly instead of falling back to a CPU path."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import common

HEADER = os.path.join(common.ROOT, "include", "usearch_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = set(re.findall(r"\b(usearch_[a-z0-9_]+)\s*\(", text))
    return sorted(n for n in names if not n.endswith("_t"))  # drop the function-pointer typedef


def test_library_exports_every_declared_symbol():
    from usearch_b200 import build
    from usearch_b200.index import EXPORTED_SYMBOLS, load_library
    build.build()
    lib = load_library()
    declared = declared_symbols()
    assert len(declared) >= 38 + 8
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/usearch_b200.h but not exported"
    assert sorted(EXPORTED_SYMBOLS) == declared
    reference_abi = [s for s in declared if not s.startswith("usearch_b200_") and s != "usearch_search_many"]
    assert len(reference_abi) == 38  # c/usearch.h:116-481


def test_no_product_code_touches_the_oracle():
    """The product package must never import, include, link or load anything under oracle/."""
    pkg = os.path.join(common.ROOT, "usearch_b200")
    usage = re.compile(r"(^\s*(from|import)\s+oracle\b)|(#\s*include\s*[\"<][^\">]*oracle)|liboracle|libusearch_ref|oracle\.bindings"
                       r"|oracle/(?!metrics_pinned\.h\))", re.M)
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                hit = usage.search(text)
                assert not hit, f"{f} uses the oracle: {hit.group(0)!r}"
    build_text = open(os.path.join(pkg, "build.py")).read()
    assert "oracle" not in build_text


def test_init_and_metadata_without_gpu():
    from usearch_b200.index import Index, load_library
    lib = load_library()
    assert lib.usearch_version().decode().startswith("2.21.0")
    g = np.load(os.path.join(common.GOLDEN, "cos_f32_n2000_d64.npz"))
    meta = Index.metadata(g["blob"])
    assert meta == {"metric": "cos", "dtype": "f32", "ndim": 64, "multi": False}
    with pytest.raises(RuntimeError, match="Magic header mismatch"):
        Index.metadata(np.zeros(200, dtype=np.uint8))
    index = Index(ndim=64, metric="cos", dtype="f32", connectivity=16, expansion_search=77)
    assert index.ndim == 64 and index.connectivity == 16 and index.expansion_search == 77 and index.size == 0
    assert index.hardware_acceleration == "sm_90a"
    import torch
    if not torch.cuda.is_available():  # mutation needs the device just like search does: no CPU fallback
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            index.add(1, np.zeros(64, dtype=np.float32))
        assert not index.contains(1) and index.count(1) == 0 and index.get(1) is None
    with pytest.raises(RuntimeError):  # unsupported pair must be refused at init (c/lib.cpp:164-167)
        Index(ndim=64, metric="haversine", dtype="f32")


def test_tune_knobs_and_launch_plan_of_an_empty_index():
    """Every documented knob is accepted, an unknown one is refused, and an index without members has no plan to read."""
    from usearch_b200.index import Index
    index = Index(ndim=8, metric="cos", dtype="f32")
    index.tune(stage_sets=2, warps_per_sm=1, prefilter=0, heap_head=2)
    index.tune(stage_sets=0, warps_per_sm=0, prefilter=1, heap_head=0)
    with pytest.raises(ValueError, match="unknown knob"):
        index.tune(heap_tail=2)
    with pytest.raises(RuntimeError, match="no CPU fallback|no launch plan"):
        index.launch_plan(4)


def test_load_fails_loudly_without_cuda_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from usearch_b200.index import Index
    g = np.load(os.path.join(common.GOLDEN, "cos_f32_n2000_d64.npz"))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        Index.restore(g["blob"])


def test_searching_an_empty_index_returns_no_matches_without_a_device():
    """index_gt::search on an empty index: zero matches, padded rows, no error (index.hpp:3036-3037) — answered on the host,
    so this also runs on a box without a GPU and exercises every search entry of the C ABI."""
    from usearch_b200.index import Index
    index = Index(ndim=8, metric="cos", dtype="f32")
    q = np.ones((3, 8), dtype=np.float32)
    for res in (index.search(q, 4), index.search(q, 4, stats=True), index.search(q, 4, exact=True)):
        assert res.counts.tolist() == [0, 0, 0] and (res.keys == 0).all() and np.isnan(res.distances).all()
        assert (res.distances.view(np.uint32) == 0x7FA00000).all()   # the signalling NaN of dump_to
    assert len(index.search(q[0], 4)) == 0
    assert len(index.search(q[0].astype(np.float64), 4)) == 0
    with pytest.raises(RuntimeError, match="No clusters"):
        index.cluster(q, 1)
    assert not index.contains(1) and index.count(1) == 0 and index.get(1) is None and index.remove(1) == 0 and index.rename(1, 2) == 0
