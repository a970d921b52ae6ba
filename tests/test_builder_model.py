"""The host model of the GPU builder's batch schedule (tests/builder_model.py), pinned on its own so that a failure of
tests/test_gpu_build_model.py points at the GPU: its INSERT search is the port's layer-0 search, its graphs are clean, and
they are as good as the reference's own build by the reference's search (the DESIGN.md §3.5 bar)."""
import os
import sys

import numpy as np
import pytest

import common
from builder_model import BuilderModel, draw_levels
from oracle import bindings
from usearch_b200 import v2format

sys.path.insert(0, os.path.join(common.ROOT, "tools"))
from build_check import exact_truth, hamming_truth, recall, structure_report  # noqa: E402

FAMILIES = [("l2sq", "f32", 32), ("ip", "f32", 97), ("cos", "f32", 64), ("cos", "f16", 48), ("l2sq", "bf16", 40),
            ("ip", "i8", 64), ("cos", "i8", 48), ("hamming", "b1", 128), ("tanimoto", "b1", 96), ("l2sq", "f64", 24),
            ("cos", "f64", 33)]


def rows_of(n, d, scalar, seed=42, nq=0):
    if scalar == "f64":
        base, q = common.make_collection(n, d, "f32", max(nq, 1), seed=seed)
        return base.astype(np.float64), q.astype(np.float64)
    return common.make_collection(n, d, scalar, max(nq, 1), seed=seed)


def model_build(metric, scalar, base, m=16, expansion_add=128, batch=32768, ratio=32, cuts=()):
    """the model's graph of `base` (keys = slots), added in calls that start at the rows in `cuts`"""
    n, d = base.shape[0], base.shape[1] * (8 if scalar == "b1" else 1)
    model = BuilderModel(metric=metric, scalar=scalar, dims=d, connectivity=m)
    bounds = [0, *cuts, n]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        model.add(np.arange(lo, hi, dtype=np.uint64), base[lo:hi], draw_levels(lo, hi - lo, m), expansion_add=expansion_add,
                  batch=batch, ratio=ratio)
    return model, v2format.dumps(model.graph(metric, scalar, d))


@pytest.mark.parametrize("metric,scalar,d", FAMILIES, ids=[f"{m}-{s}-{d}" for m, s, d in FAMILIES])
def test_level0_candidates_are_the_port_search(metric, scalar, d):
    """search_to_insert_ with no predicate and search_to_find_in_base_ run the same loop: on a graph without removed
    entries the model's level-0 candidates are the port's search results (keys == slots here), bit for bit"""
    n, ef = 1500, 40
    base, queries = rows_of(n, d, scalar, nq=60)
    model, blob = model_build(metric, scalar, base)
    if scalar == "f64":
        from f64_reference import PortF64
        port = PortF64(blob, ef)
        keys, dist, counts, _, _ = port.search(queries, ef)
    else:
        port = bindings.PortIndex(blob, ef)
        keys, dist, counts, _, _ = port.search(queries, ef, threads=4)
    for i, q in enumerate(queries):
        slots, dists = model.candidates(q, 0, ef)
        c = int(counts[i])
        assert len(slots) == c, (i, len(slots), c)
        assert np.array_equal(slots.astype(np.uint64), keys[i, :c]), i
        assert np.array_equal(dists.view(np.uint32), dist[i, :c].view(np.uint32)), i


HUB_SCATTERED = 1500


def hub_rows(n, d, spread=1e-3, seed=3):
    """HUB_SCATTERED scattered rows, then n - HUB_SCATTERED rows in a tight cluster around row 0, the farthest first.
    Added in two calls with a batch ratio of 1, the cluster is one batch in which every member picks row 0 first: far
    more than 256 - M0 arrivals for one neighbour."""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, d)).astype(np.float32)
    noise = spread * rng.standard_normal((n - HUB_SCATTERED, d)).astype(np.float32)
    base[HUB_SCATTERED:] = base[0] + noise[np.argsort(-np.linalg.norm(noise, axis=1), kind="stable")]
    return base


STRUCTURE_CASES = {
    # name: (metric, scalar, n, d, m, expansion_add, batch, ratio, data, counter the case is written for)
    "default": ("l2sq", "f32", 3000, 32, 16, 128, 32768, 32, "latent", "reverse_refines"),
    "hub": ("l2sq", "f32", 2300, 16, 16, 128, 32768, 1, "hub", "room_cuts"),
    "ef300": ("cos", "f32", 2000, 24, 16, 300, 32768, 32, "latent", "candidate_cuts"),
    "ef8": ("ip", "f32", 1500, 24, 16, 8, 32768, 32, "latent", "short_refines"),
    "m4": ("l2sq", "f32", 1500, 16, 4, 64, 32768, 32, "latent", "reverse_refines"),
    "m40": ("l2sq", "f32", 3000, 16, 40, 128, 32768, 4, "latent", "reverse_refines_base"),
    "duplicates": ("l2sq", "f32", 2000, 16, 16, 128, 32768, 32, "duplicates", "reverse_refines"),
    "batch7": ("hamming", "b1", 1500, 128, 16, 128, 7, 32, "latent", "reverse_refines"),
}


def structure_case_rows(name):
    metric, scalar, n, d, *_, data, _ = STRUCTURE_CASES[name]
    if data == "hub":
        return hub_rows(n, d)
    base, _ = rows_of(n, d, scalar)
    if data == "duplicates":
        base[n // 2:n // 2 + 200] = base[:200]
        base[-50:] = base[7]
    return base


@pytest.mark.parametrize("name", list(STRUCTURE_CASES))
def test_model_graphs_are_clean_and_reach_their_path(name):
    metric, scalar, n, d, m, ea, batch, ratio, _, counter = STRUCTURE_CASES[name]
    cuts = (HUB_SCATTERED,) if name == "hub" else ()
    model, blob = model_build(metric, scalar, structure_case_rows(name), m=m, expansion_add=ea, batch=batch, ratio=ratio,
                              cuts=cuts)
    rep = structure_report(blob)
    assert rep["n_problems"] == 0, rep["problems"]
    assert rep["min_degree0"] > 0
    assert model.counters()[counter] > 0, model.counters()


def test_model_reuse_of_removed_slots():
    """a loaded graph with removed entries (keys set to the free key), their slots reused: the rebuilt rows hold no self
    links and no repeats, and a reused slot keeps its level"""
    n, d = 2000, 32
    base, _ = rows_of(n, d, "f32")
    fresh, _ = rows_of(300, d, "f32", seed=7)
    _, blob = model_build("l2sq", "f32", base)
    g = v2format.loads(blob)
    victims = np.random.default_rng(1).choice(n, 200, replace=False).astype(np.uint32)
    g.keys[victims] = v2format.FREE_KEY
    model = BuilderModel(v2format.dumps(g))
    model.add(np.arange(10**6, 10**6 + 300, dtype=np.uint64), fresh, draw_levels(n, 100, 16), reuse=victims)
    after = model.graph("l2sq", "f32", d)
    rep = structure_report(v2format.dumps(after))
    assert rep["n_problems"] == 0, rep["problems"]
    assert np.array_equal(after.levels[:n], g.levels)
    assert np.array_equal(after.keys[victims], np.arange(10**6, 10**6 + 200, dtype=np.uint64))
    assert np.array_equal(after.vectors[victims].view(np.float32), fresh[:200])


BAR_CASES = [("cos", "f32", 4000, 64, 16), ("l2sq", "f32", 3000, 48, 16), ("hamming", "b1", 4000, 256, 32)]


@pytest.mark.skipif(not common.have_reference(), reason="needs the reference library (oracle/_ref)")
@pytest.mark.parametrize("metric,scalar,n,d,m", BAR_CASES, ids=[f"{c[0]}-{c[1]}" for c in BAR_CASES])
def test_model_graph_meets_the_build_bar(metric, scalar, n, d, m):
    """recall of the reference's search on the model's graph >= on the reference's own graph - 0.01, work within 8 %"""
    base, queries = rows_of(n, d, scalar, nq=300)
    _, model_blob = model_build(metric, scalar, base, m=m)
    _, ref_blob = common.build_reference_blob(base, metric, scalar, d, m, threads=8)
    truth = hamming_truth(base, queries, 10) if scalar == "b1" else exact_truth(base, queries, metric, 10)
    got = {}
    for label, blob in (("ref", ref_blob), ("model", model_blob)):
        searcher = bindings.RefIndex("parity")
        searcher.load(blob)
        searcher.change_expansion_search(64)
        k, _, _, comp, _ = searcher.search(queries, 10, threads=8)
        got[label] = (recall(k, truth), float(comp.mean()))
    assert got["model"][0] >= got["ref"][0] - 0.01, got
    assert abs(got["model"][1] - got["ref"][1]) <= 0.08 * got["ref"][1], got
