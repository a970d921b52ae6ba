"""The layer-0 hop of the prefiltered f32 cos / ip search, against the pinned reference (labels, distance bits, counts and
both counters):
- heaps that grow past 1024 entries on rows one ULP apart and exact duplicates, so that their pops go through the
  warp-wide `pop_warp` between 512 and 1024 entries and through the serial pop beyond, in shared memory and through the
  HBM tail, all with max_heap_gt's tie order;
- the plan the prefilter gets at 768-d (one resident warp per SM given up for a heap head of at least 512 entries), and
  at a ragged 97-d, where the head is already that large;
- odd numbers of 32-byte k-steps in the tensor-core dot products (their two accumulator chains end unevenly)."""
import numpy as np
import pytest

import common
from test_gpu_prefilter import _check, _pinned

pytestmark = pytest.mark.gpu

DEFAULT_KNOBS = {"stage_sets": 0, "warps_per_sm": 0, "prefilter": 1, "heap_head": 0}


def _tune(index, **knobs):
    index.tune(**{**DEFAULT_KNOBS, **knobs})


def _near_duplicate_clusters(d, centres, copies, seed):
    """`centres` clusters of `copies` rows: each centre, a duplicate of it, and copies with every element one ULP up or
    down; 256 queries close to random centres."""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centres, d), dtype=np.float32)
    base = np.repeat(c, copies, axis=0)
    up = rng.integers(0, 2, size=base.shape).astype(bool)
    base = np.nextafter(base, np.where(up, np.inf, -np.inf).astype(np.float32)).astype(np.float32)
    base[::copies] = c
    base[1::copies] = c
    q = (c[rng.integers(0, centres, 256)] + 1e-3 * rng.standard_normal((256, d), dtype=np.float32)).astype(np.float32)
    return base, q


@pytest.fixture(scope="module")
def large_heaps():
    """ef = 2000 on 20000 near-duplicate rows: `next` takes every fresh candidate until `top` holds 2000 entries."""
    out = {}

    def get(metric):
        if metric not in out:
            from usearch_b200.index import Index
            d, m, ef, k = 128, 16, 2000, 10
            base, q = _near_duplicate_clusters(d, 1000, 20, seed=11)
            _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
            index = Index.restore(blob)
            index.expansion_search = ef
            out[metric] = (index, q, k, _pinned(blob, q, k, ef))
        return out[metric]

    yield get
    out.clear()


@pytest.mark.parametrize("metric", ["cos", "ip"])
@pytest.mark.parametrize("knobs", [{"warps_per_sm": 1}, {"warps_per_sm": 1, "heap_head": 1024}, {"warps_per_sm": 1, "heap_head": 700}],
                         ids=["head=all", "head=1024", "head=700"])
def test_heaps_past_the_warp_pop_keep_tie_order(large_heaps, metric, knobs):
    index, q, k, want = large_heaps(metric)
    _tune(index, **knobs)
    plan = index.launch_plan(k)
    ph = _check(index, want, q, k, f"{metric} near-duplicates, ef 2000, {knobs}")
    assert ph["max_heap"] > 1024, f"the heap stayed at {ph['max_heap']} entries"
    if "heap_head" in knobs:  # pops past the head walk the HBM tail
        assert plan["heap_smem_cap"] == knobs["heap_head"], plan
    else:  # the whole heap in shared memory: the serial pop above 1024 entries stays there
        assert plan["heap_smem_cap"] > ph["max_heap"], (plan, ph["max_heap"])


@pytest.mark.parametrize("metric,n,d,m,ef,k", [
    ("cos", 8000, 768, 32, 128, 10),
    ("ip", 6000, 97, 13, 64, 7),
    ("cos", 6000, 96, 16, 64, 10),  # 3 k-steps: an odd count
    ("ip", 6000, 224, 16, 64, 10),  # 7 k-steps
])
def test_prefilter_plan_and_kstep_counts(metric, n, d, m, ef, k):
    from usearch_b200.index import Index
    base, q = common.make_collection(n, d, "f32", 256)
    _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    _tune(index)
    plan = index.launch_plan(k)
    assert plan["prefilter"], plan
    assert plan["qsplit_len"] == ((d + 15) // 16 * 16 + 31) // 32 * 32, plan  # 32-byte k-steps over the code stride
    assert plan["heap_smem_cap"] >= 512, plan
    if d == 768:  # 200 entries at 7 warps per SM: the planner gives one up
        assert plan["warps_per_sm_target"] == 6, plan
    _check(index, _pinned(blob, q, k, ef), q, k, f"{metric}/{d}")
    _tune(index, warps_per_sm=7)  # the plan without the trade, same results
    _check(index, _pinned(blob, q, k, ef), q, k, f"{metric}/{d}, 7 warps per SM")
