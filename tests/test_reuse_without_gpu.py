"""CPU tests of removal and slot reuse: an empty index answers batched removes and lookups without touching a device,
and the reuse switch round-trips."""
import numpy as np

import common  # noqa: F401  (puts the repository on sys.path)


def test_batched_remove_and_lookups_on_an_empty_index():
    from usearch_b200.index import Index
    index = Index(ndim=16, metric="cos", dtype="f32")
    assert index.remove([1, 2, 3]) == 0
    assert index.remove(7, compact=True) == 0 and index.last_pruned_edges == 0
    assert index.remove(np.arange(5, dtype=np.uint64), compact=True) == 0
    assert index.remove([]) == 0
    assert index.contains([1, 2]).tolist() == [False, False]
    assert index.count([1, 2, 3]).tolist() == [0, 0, 0]
    assert index.count(np.array([], dtype=np.uint64)).shape == (0,)
    assert index.contains(1) is False and index.count(1) == 0


def test_reuse_removed_round_trips():
    from usearch_b200.index import Index
    index = Index(ndim=16, metric="l2sq", dtype="f32")
    assert index.reuse_removed is False
    index.reuse_removed = True
    assert index.reuse_removed is True
    index.clear()
    assert index.reuse_removed is True  # a per-handle setting, like the expansion factors
    index.reuse_removed = False
    assert index.reuse_removed is False
