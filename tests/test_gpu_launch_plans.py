"""The launch plan never changes a result. `frozen_index_t::plan()` picks stage sets, resident warps, the shared-memory
head of the candidate heap and the prefilter's layout from the shape; the tuning knobs force the other choices. Every
plan must return exactly what the pinned reference returns on the same graph: labels, distance bits, counts and both
counters. The kernel counters and `Index.launch_plan` show that each forced path ran: the heap's HBM tail and its serial
pop, pop_warp's fallback above 512 entries, prefilter passes of 64 codes, and the prefilter's fallback at the largest f32
dimensionalities. The builder, which searches through the same planner, must produce the same bytes under any plan."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import common
from test_gpu_prefilter import _check, _near_duplicate_rows, _pinned

pytestmark = pytest.mark.gpu

PLAN_ERROR = "Expansion or dimensionality too large for on-chip state"
DEFAULT_KNOBS = {"stage_sets": 0, "warps_per_sm": 0, "prefilter": 1, "heap_head": 0}
SMEM_CTA_MAX = 227 * 1024

# name: metric, scalar, n, d, M, ef, k, nq
SHAPES = {
    "cos_f32_768": ("cos", "f32", 4000, 768, 32, 128, 10, 256),   # two code passes per hop; 64 codes with two sets
    "ip_f32_97": ("ip", "f32", 4000, 97, 13, 64, 10, 256),        # ragged code_stride, one partial tile
    "cos_f32_64": ("cos", "f32", 4000, 64, 40, 64, 10, 256),      # smallest STAGED f32, M0 = 80: three code passes
    "ip_f32_4096": ("ip", "f32", 2000, 4096, 16, 64, 10, 256),    # 1 warp per SM, 128 k-steps
    "l2sq_f32_128_ef1000": ("l2sq", "f32", 8000, 128, 16, 1000, 10, 256),  # heaps above 512 entries in shared memory
    "cos_f16_768": ("cos", "f16", 4000, 768, 32, 128, 10, 256),   # WORD metrics
    "ip_bf16_256": ("ip", "bf16", 4000, 256, 16, 64, 10, 256),
    "ip_i8_1024": ("ip", "i8", 4000, 1024, 16, 64, 10, 256),      # 16-warp kernel
    "hamming_b1_256": ("hamming", "b1", 6000, 256, 64, 64, 10, 256),  # DIRECT, WIDE rows, ties everywhere
    "l2sq_f32_32": ("l2sq", "f32", 4000, 32, 16, 64, 10, 256),    # DIRECT f32
}

KNOBS = {
    "default": {},
    "stage_sets=1": {"stage_sets": 1},
    "stage_sets=2": {"stage_sets": 2},
    "warps_per_sm=1": {"warps_per_sm": 1},  # heap head up to 4096 entries
    "warps_per_sm=2": {"warps_per_sm": 2},
    "heap_head=2": {"heap_head": 2},
    "heap_head=16": {"heap_head": 16},
    "heap_head=64": {"heap_head": 64},
    "stage_sets=2,heap_head=2": {"stage_sets": 2, "heap_head": 2},
}


def _has_shadow(shape):
    metric, scalar = SHAPES[shape][:2]
    return scalar == "f32" and metric in ("cos", "ip")


CASES = [(shape, name, pf) for shape in SHAPES for name in KNOBS for pf in ((1, 0) if _has_shadow(shape) else (1,))]


@pytest.fixture(scope="module")
def prepared():
    """Per shape, once: the reference-built graph, the pinned reference's results, and the index loaded from it."""
    from usearch_b200.index import Index
    cache = {}

    def get(shape):
        if shape not in cache:
            metric, scalar, n, d, m, ef, k, nq = SHAPES[shape]
            base, q = common.make_collection(n, d, scalar, nq)
            _, blob = common.build_reference_blob(base, metric, scalar, d, m, threads=16)
            index = Index.restore(blob)
            index.expansion_search = ef
            cache[shape] = (index, q, k, _pinned(blob, q, k, ef))
        return cache[shape]

    yield get
    cache.clear()


def _tune(index, **knobs):
    index.tune(**{**DEFAULT_KNOBS, **knobs})


def _search(index, q, k, allowed=None):
    index.profile_phases(True)
    got = index.search(q, k, stats=True) if allowed is None else index.filtered_search(q, k, allowed)
    phases = index.profile_phases(False)
    return (got.keys, got.distances, got.counts, index.last_computed, index.last_visited), phases


def _assert_plan_invariants(plan, what):
    assert plan["heap_smem_cap"] >= 2 and plan["heap_smem_cap"] % 2 == 0, f"{what}: {plan}"
    assert plan["smem_per_warp"] <= SMEM_CTA_MAX, f"{what}: {plan}"
    if plan["prefilter"]:
        assert plan["code_pass"] % 16 == 0 and 16 <= plan["code_pass"] <= 64, f"{what}: {plan}"
        assert plan["code_pass"] * plan["code_smem_stride"] <= plan["stage_bytes"], f"{what}: {plan}"
        assert plan["code_smem_stride"] % 32 == 16, f"{what}: {plan}"
        assert plan["qsplit_len"] % 32 == 0 and plan["qsplit_len"] > 0, f"{what}: {plan}"
    else:  # nothing of the prefilter's layout is reserved when it cannot run
        assert plan["code_pass"] == 0 and plan["qsplit_len"] == 0, f"{what}: {plan}"


@pytest.mark.parametrize("shape,knobs,prefilter", CASES)
def test_every_plan_matches_pinned_reference(prepared, shape, knobs, prefilter):
    index, q, k, want = prepared(shape)
    what = f"{shape} [{knobs}, prefilter={prefilter}]"
    forced = KNOBS[knobs]
    _tune(index, prefilter=prefilter, **forced)
    try:
        plan = index.launch_plan(k)
    except RuntimeError as e:  # a forced layout that does not fit: the search must refuse it the same way
        assert str(e) == PLAN_ERROR, f"{what}: {e}"
        assert forced, f"{what}: the default plan does not fit"
        with pytest.raises(RuntimeError, match=re.escape(str(e))):
            index.search(q, k, stats=True)
        return
    _assert_plan_invariants(plan, what)
    got, ph = _search(index, q, k)
    common.assert_same_results(want, got, what)
    if plan["prefilter"]:
        assert prefilter and _has_shadow(shape)
        assert ph["prefiltered"] > 0, f"{what}: the prefilter never ran"
    else:
        assert ph["prefiltered"] == 0, f"{what}: the readout says the prefilter is off, the kernel ran it"
        if _has_shadow(shape) and prefilter:  # only the largest f32 shapes fall back; these all have room
            pytest.fail(f"{what}: the prefilter is off although it fits: {plan}")
    if "heap_head" in forced:
        assert plan["heap_smem_cap"] == max(2, forced["heap_head"] & ~1), f"{what}: {plan}"
        assert ph["max_heap"] > plan["heap_smem_cap"], f"{what}: the heap never reached its HBM tail ({ph['max_heap']})"
    if "warps_per_sm" in forced:
        assert plan["warps_per_sm_target"] <= forced["warps_per_sm"], f"{what}: {plan}"
    if "stage_sets" in forced and plan["stage_bytes"]:
        assert plan["stage_sets"] == forced["stage_sets"], f"{what}: {plan}"
    if shape == "cos_f32_768" and forced.get("stage_sets") == 2 and prefilter:
        assert plan["code_pass"] == 64, f"{what}: {plan}"
        assert ph["survivors"] < ph["prefiltered"], f"{what}: the prefilter rejected nothing"
    if shape == "l2sq_f32_128_ef1000" and not forced:  # pop_warp gives way to the serial pop inside shared memory
        assert plan["heap_smem_cap"] > 512, f"{what}: {plan}"
        assert ph["max_heap"] > 512, f"{what}: the heap stayed at {ph['max_heap']} entries"


def test_a_forced_layout_that_does_not_fit_is_refused(prepared):
    """Two stage sets of 4096-d f32 rows need more shared memory than a CTA may have: both the readout and the search
    raise the planner's error, and the handle still serves searches once the knob is back."""
    index, q, k, want = prepared("ip_f32_4096")
    _tune(index, stage_sets=2)
    with pytest.raises(RuntimeError, match=re.escape(PLAN_ERROR)):
        index.launch_plan(k)
    with pytest.raises(RuntimeError, match=re.escape(PLAN_ERROR)):
        index.search(q, k)
    _tune(index)
    got, _ = _search(index, q, k)
    common.assert_same_results(want, got, "ip_f32_4096 after a refused plan")


@pytest.mark.parametrize("metric", ["cos", "ip"])
def test_heap_tail_keeps_tie_order_on_near_duplicates(metric):
    """Rows one ULP apart and exact duplicates, with a heap head of 2 entries: the serial pop through the HBM tail must
    keep max_heap_gt's tie order."""
    from usearch_b200.index import Index
    d, m, ef, k = 256, 16, 64, 10
    base, q = _near_duplicate_rows(d)
    _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    _tune(index, heap_head=2)
    assert index.launch_plan(k)["heap_smem_cap"] == 2
    ph = _check(index, _pinned(blob, q, k, ef), q, k, f"{metric} near-duplicates, heap head 2")
    assert ph["max_heap"] > 2


@pytest.mark.parametrize("knobs", [{"stage_sets": 2}, {"heap_head": 2}], ids=["stage_sets=2", "heap_head=2"])
def test_filtered_search_with_removed_keys_under_forced_plans(knobs):
    from usearch_b200.index import Index
    n, d, m, ef, k = 8000, 256, 16, 96, 10
    base, q = common.make_collection(n, d, "f32", 256)
    ref, _ = common.build_reference_blob(base, "cos", "f32", d, m, threads=16, keys=np.arange(n, dtype=np.uint64) * 7 + 3)
    for key in range(3, 3 + 7 * 400, 7 * 4):
        ref.remove(key)
    blob = ref.save()
    ref.pin_metric(True)
    ref.change_expansion_search(ef)
    allowed = np.random.default_rng(5).permutation(n)[: n // 2].astype(np.uint64) * 7 + 3
    want = ref.filtered_search(q, k, allowed, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    _tune(index, **knobs)
    plan = index.launch_plan(k)
    for name, value in knobs.items():
        assert plan["heap_smem_cap" if name == "heap_head" else name] == value, plan
    ph = _check(index, want, q, k, f"filtered {knobs}", allowed)
    if "heap_head" in knobs:
        assert ph["max_heap"] > 2


def test_heap_overflow_retry_in_bitmap_mode():
    """A heap head of 2 entries and a 64x undersized HBM tail: with bitmap `visits`, which cannot overflow, the heap
    does, and the overflowed queries are run again with larger tails until they fit."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import numpy as np, common\n"
        "from oracle import bindings\n"
        "from usearch_b200.index import Index\n"
        "base, q = common.make_collection(20000, 64, 'f32', 4096, iid=True)\n"
        "ref, blob = common.build_reference_blob(base, 'l2sq', 'f32', 64, 16, threads=16)\n"
        "want = bindings.PortIndex(blob, 64).search(q, 10, threads=16)\n"
        "index = Index.restore(blob); index.expansion_search = 64\n"
        "plan = index.launch_plan(10)\n"
        "assert plan['visits'] == 'bitmap' and plan['heap_smem_cap'] == 2 and plan['heap_spill_cap'] == 16, plan\n"
        "got = index.search(q, 10, stats=True)\n"
        "common.assert_same_results(want, (got.keys, got.distances, got.counts, index.last_computed, index.last_visited), 'retry')\n"
        "print('launches', index.kernel_launches)\n"
    ) % (common.ROOT, os.path.join(common.ROOT, "tests"))
    env = dict(os.environ, USEARCH_B200_VISITED="bitmap", USEARCH_B200_SCRATCH_SHRINK="64", USEARCH_B200_HEAP_HEAD="2")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    launches = int(out.stdout.split("launches")[1].split()[0])
    assert launches >= 2, "expected at least one retry launch after a heap overflow: " + out.stdout


@pytest.mark.parametrize("metric,scalar,d", [("cos", "f32", 768), ("ip", "i8", 256), ("hamming", "b1", 256)])
def test_build_does_not_depend_on_the_plan(metric, scalar, d):
    """The builder's INSERT search runs under the same planner: two builds under the default knobs and one under
    {stage_sets=2, warps_per_sm=1, heap_head=2} must serialise to the same bytes."""
    from usearch_b200.index import Index
    base, _ = common.make_collection(3000, d, scalar, 1)

    def build(**knobs):
        index = Index(ndim=d, metric=metric, dtype=scalar, connectivity=16, expansion_add=128)
        _tune(index, **knobs)
        index.add(np.arange(len(base), dtype=np.uint64), base)
        return index.save()

    first, second = build(), build()
    assert first.size == second.size and np.array_equal(first, second), "two builds under the default plan differ"
    forced = build(stage_sets=2, warps_per_sm=1, heap_head=2)
    assert forced.size == first.size and np.array_equal(forced, first), "the build depends on the launch plan"


def _large(metric, n, d, nq=64, m=16, ef=64):
    from usearch_b200.index import Index
    base, q = common.make_collection(n, d, "f32", nq)
    _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    return index, blob, q


@pytest.mark.parametrize("metric", ["cos", "ip"])
def test_f32_6144_dims_search_and_add(metric):
    """Above 6048 dims the prefilter's shared memory does not fit next to two 8-slot stage sets' worth of rows: the
    search goes without the prefilter instead of failing, and so does the builder, which never reserves it."""
    n0, n1, d, ef, k = 2000, 500, 6144, 64, 10
    base, q = common.make_collection(n0 + n1, d, "f32", 64)
    _, blob = common.build_reference_blob(base[:n0], metric, "f32", d, 16, threads=16)
    from usearch_b200.index import Index
    index = Index.restore(blob)
    index.expansion_search = ef
    got, ph = _search(index, q, k)
    common.assert_same_results(_pinned(blob, q, k, ef), got, f"{metric}/{d}")
    assert ph["prefiltered"] == 0
    index.add(np.arange(n0, n0 + n1, dtype=np.uint64), base[n0:])
    saved = index.save()
    got, _ = _search(index, q, k)
    common.assert_same_results(_pinned(saved, q, k, ef), got, f"{metric}/{d} grown")
    plan = index.launch_plan(k)
    assert not plan["prefilter"] and plan["qsplit_len"] == 0, plan


def test_f32_6048_dims_keeps_the_prefilter():
    index, blob, q = _large("cos", 2000, 6048)
    k = 10
    plan = index.launch_plan(k)
    assert plan["prefilter"], plan
    _assert_plan_invariants(plan, "cos/6048")
    got, ph = _search(index, q, k)
    common.assert_same_results(_pinned(blob, q, k, 64), got, "cos/6048")
    assert ph["prefiltered"] > 0


def test_f32_6400_dims_is_served():
    index, blob, q = _large("l2sq", 2000, 6400)
    k = 10
    _assert_plan_invariants(index.launch_plan(k), "l2sq/6400")
    got, _ = _search(index, q, k)
    common.assert_same_results(_pinned(blob, q, k, 64), got, "l2sq/6400")


@pytest.mark.parametrize("metric", ["l2sq", "cos"])
def test_f32_6416_dims_is_refused_cleanly(metric):
    """One 16-byte chunk more than 6400 f32 dims: the stage area alone no longer fits, so the search raises."""
    index, _, q = _large(metric, 300, 6416, nq=4)
    with pytest.raises(RuntimeError, match=re.escape(PLAN_ERROR)):
        index.launch_plan(10)
    with pytest.raises(RuntimeError, match=re.escape(PLAN_ERROR)):
        index.search(q, 10)
    assert index.size == 300
