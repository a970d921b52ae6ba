"""The prefilter's code passes at every shape they take: one pass of 1, 2, 3 or 4 tiles of 16 candidates (a 64-candidate
code pass, which the plan gives 128-d codes when two stage sets are forced), and hops with more candidates than one code
pass holds (the default 32-candidate pass). Labels, distance bits, counts and both counters equal the pinned reference,
with the prefilter on and off."""
import numpy as np
import pytest

import common
from oracle import bindings

pytestmark = pytest.mark.gpu


def _pinned(blob, q, k, ef):
    ref = bindings.RefIndex("parity")
    ref.view(blob)
    ref.pin_metric(True)
    ref.change_expansion_search(ef)
    return ref.search(q, k, threads=16)


def _run(index, q, k, prefilter, stage_sets):
    index.tune(prefilter=prefilter, stage_sets=stage_sets)
    index.profile_phases(True)
    got = index.search(q, k, stats=True)
    phases = index.profile_phases(False)
    return (got.keys, got.distances, got.counts, index.last_computed, index.last_visited), phases


def _index(metric, base, d, m, ef):
    from usearch_b200.index import Index
    _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    return index, blob


@pytest.mark.parametrize("metric", ["cos", "ip"])
@pytest.mark.parametrize("stage_sets,code_pass", [(2, 64), (1, 32)])
def test_code_passes_match_pinned_reference(metric, stage_sets, code_pass):
    d, m, ef, k = 128, 32, 96, 10
    base, q = common.make_collection(6000, d, "f32", 256, iid=True)
    index, blob = _index(metric, base, d, m, ef)
    want = _pinned(blob, q, k, ef)
    on, ph = _run(index, q, k, 1, stage_sets)
    plan = index.launch_plan(k)
    assert plan["prefilter"] and plan["code_pass"] == code_pass, plan
    common.assert_same_results(want, on, f"{metric}, {code_pass}-candidate code passes, prefilter on")
    assert ph["prefiltered"] > 0 and ph["survivors"] < ph["prefiltered"], ph
    per_hop = ph["prefiltered"] / ph["prefiltered_hops"]
    if code_pass == 64:  # passes of several tiles: more than one tile's worth of candidates per hop on average
        assert per_hop > 16, ph
    else:  # some hops hold more candidates than one pass
        assert ph["code_passes_per_prefiltered_hop"] > 1.0, ph
    off, ph_off = _run(index, q, k, 0, stage_sets)
    assert ph_off["prefiltered"] == 0 and ph_off["prefiltered_hops"] == 0
    common.assert_same_results(want, off, f"{metric}, prefilter off")


@pytest.mark.parametrize("metric", ["cos", "ip"])
def test_wide_code_passes_near_duplicate_rows(metric):
    """Rows one ULP apart and exact duplicates, through 64-candidate code passes: dots and distances that tie or differ
    in the last bits."""
    d, m, ef, k = 128, 32, 64, 10
    rng = np.random.default_rng(11)
    centres, copies = 300, 20
    c = rng.standard_normal((centres, d), dtype=np.float32)
    base = np.repeat(c, copies, axis=0)
    up = rng.integers(0, 2, size=base.shape).astype(bool)
    base = np.nextafter(base, np.where(up, np.inf, -np.inf).astype(np.float32)).astype(np.float32)
    base[::copies] = c
    base[1::copies] = c
    q = (c[rng.integers(0, centres, 256)] + 1e-3 * rng.standard_normal((256, d), dtype=np.float32)).astype(np.float32)
    index, blob = _index(metric, base, d, m, ef)
    want = _pinned(blob, q, k, ef)
    on, ph = _run(index, q, k, 1, 2)
    assert index.launch_plan(k)["code_pass"] == 64
    common.assert_same_results(want, on, f"{metric} near-duplicates, prefilter on")
    assert ph["prefiltered"] > 0, ph
    off, _ = _run(index, q, k, 0, 2)
    common.assert_same_results(want, off, f"{metric} near-duplicates, prefilter off")


def test_phase_counters_keep_their_first_sixteen_words():
    """usearch_b200_profile_phases keeps its 16-word buffer; the longer readout extends it with the same first words."""
    import ctypes as C
    d, m, ef, k = 128, 16, 64, 10
    base, q = common.make_collection(3000, d, "f32", 128)
    index, _ = _index("cos", base, d, m, ef)
    index.profile_phases(True)
    index.search(q, k)
    short = np.full(17, 7, dtype=np.uint64)  # one word past the 16: left alone
    index._lib.usearch_b200_profile_phases(index._h, 1, short.ctypes.data_as(C.c_void_p))
    assert short[16] == 7 and short[7] == len(q), short
    index.search(q, k)
    full = np.zeros(24, dtype=np.uint64)
    kept = index._lib.usearch_b200_profile_phases_n(index._h, 0, full.ctypes.data_as(C.c_void_p), full.size)
    assert kept == 21 and full[7] == len(q) and (full[21:] == 0).all(), full
    assert full[18] > 0 and full[17] >= full[18], full  # prefiltered hops, at least one code pass each
