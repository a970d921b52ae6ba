"""The scratch of the key-set searches is all counted by `memory_usage` and all freed by `clear`: the sort buffers of
grouped search in rounds included, not only the bitmap rows."""
import numpy as np
import pytest

from usearch_b200.index import Index

pytestmark = pytest.mark.gpu


def test_rounds_scratch_is_counted_and_cleared():
    rng = np.random.default_rng(11)
    index = Index(ndim=16, metric="l2sq", dtype="f32")
    index.add(np.arange(1000, dtype=np.uint64), rng.standard_normal((1000, 16)).astype(np.float32))
    queries = rng.standard_normal((200, 16)).astype(np.float32)
    sets = [rng.choice(1000, 50, replace=False).astype(np.uint64) for _ in range(3)]
    groups = np.arange(len(queries)) % 3
    one_round = index.grouped_filtered_search(queries, 10, sets, groups)  # builds the key table and the rows
    before = index.memory_usage
    index.tune(group_bitmap_mb=0)  # one set per round: the queries sorted by set
    rounds = index.grouped_filtered_search(queries, 10, sets, groups)
    assert np.array_equal(rounds.keys, one_round.keys)
    assert index.memory_usage >= before + 12 * len(queries)  # query ids, their order and their sorted sets, u32 each
    index.clear()
    assert index.memory_usage == 0
