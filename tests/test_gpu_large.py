"""Large-index check: a vector slab beyond 4 GiB, so every byte offset on the device and in the loader must be
64-bit (skipped when the host has less than 32 GB free, USEARCH_B200_LARGE=0 disables). The graph is synthetic (random links over three levels) — the traversal
does not need a navigable graph to be compared decision for decision with the oracle."""
import os

import numpy as np
import pytest

import common
from oracle import bindings

pytestmark = pytest.mark.gpu

M, M0 = 4, 8


def synthetic_blob(n: int, d: int, seed: int = 7):
    """v2 image: slots [0, n2) on level 2, [n2, n1) on level 1, the rest on level 0; entry slot 0."""
    from usearch_b200 import v2format
    rng = np.random.default_rng(seed)
    n2, n1 = max(n // 4096, 2), max(n // 64, 4)
    vectors = rng.integers(-127, 128, size=(n, d), dtype=np.int8)
    empty = v2format.dumps(v2format.Graph(metric="l2sq", scalar="i8", dimensions=d, connectivity=M, connectivity_base=M0,
                                          vectors=np.zeros((0, d), np.uint8), keys=np.zeros(0, np.uint64),
                                          levels=np.zeros(0, np.int16)))
    head = bytearray(empty[8:8 + 64].tobytes())
    head[17:25] = np.uint64(n).tobytes()
    levels = np.zeros(n, np.int16)
    levels[:n1] = 1
    levels[:n2] = 2
    tapes = []
    for level, lo, hi in ((2, 0, n2), (1, n2, n1), (0, n1, n)):
        fields = [("key", "<u8"), ("level", "<i2"), ("cnt0", "<u4"), ("nb0", "<u4", (M0,))]
        for l in range(1, level + 1):
            fields += [(f"cnt{l}", "<u4"), (f"nb{l}", "<u4", (M,))]
        t = np.zeros(hi - lo, dtype=np.dtype(fields, align=False))
        t["key"] = np.arange(lo, hi, dtype=np.uint64) * 3 + 1
        t["level"] = level
        t["cnt0"] = M0
        t["nb0"] = rng.integers(0, n, size=(hi - lo, M0), dtype=np.uint32)
        for l in range(1, level + 1):
            pool = n2 if l == 2 else n1   # members that exist on level l
            t[f"cnt{l}"] = M
            t[f"nb{l}"] = rng.integers(0, pool, size=(hi - lo, M), dtype=np.uint32)
        tapes.append(t.tobytes())
    parts = [np.array([n, d], dtype=np.uint32).tobytes(), vectors.tobytes(), bytes(head),
             np.array([n, M, M0, 2, 0], dtype=np.uint64).tobytes(), levels.tobytes()] + tapes
    return np.frombuffer(b"".join(parts), dtype=np.uint8), vectors


def _enough_host_memory() -> bool:
    try:
        import psutil
        return psutil.virtual_memory().available > 32 * 2 ** 30
    except Exception:
        return False


@pytest.mark.skipif(os.environ.get("USEARCH_B200_LARGE") == "0" or not _enough_host_memory(),
                    reason="needs about 15 GB of host memory")
def test_slab_beyond_4gib():
    from usearch_b200.index import Index
    n, d = 4_600_000, 1024                      # 4.71e9 bytes of vectors
    blob, vectors = synthetic_blob(n, d)
    assert vectors.nbytes > 2 ** 32
    rng = np.random.default_rng(11)
    # queries near members of the far end of the slab, so that the best matches live beyond the 4 GiB mark
    picks = rng.integers(n - 200_000, n, size=256)
    q = np.clip(vectors[picks].astype(np.int16) + rng.integers(-3, 4, size=(256, d)), -127, 127).astype(np.int8)
    index = Index.restore(blob)
    assert index.size == n and index.max_level == 2
    port = bindings.PortIndex(blob, 64)
    index.expansion_search = 64
    want = port.search(q, 10, threads=16)
    got = index.search(q, 10, stats=True)
    common.assert_same_results(want, (got.keys, got.distances, got.counts, index.last_computed, index.last_visited), "large graph search")
    # brute force finds the perturbed members themselves (keys = 3 * slot + 1), all beyond the 4 GiB mark
    exact = index.search(q[:64], 5, exact=True)
    assert np.array_equal(exact.keys[:, 0], picks[:64].astype(np.uint64) * 3 + 1)
    want_exact = port.search(q[:4], 5, threads=4, exact=True)
    assert np.array_equal(exact.keys[:4], want_exact[0]) and np.array_equal(exact.distances[:4], want_exact[1])
    # members of every level through the descent-only entry point
    for level in (1, 2):
        wk, wd, wc, wv = port.cluster(q[:64], level)
        gk, gd = index.cluster(q[:64], level, stats=True)
        assert np.array_equal(gk, wk) and np.array_equal(gd, wd) and np.array_equal(index.last_computed, wc)
