"""GPU-built graphs (`Index.add`, csrc/builder.cu) held to the host model of the builder's batch schedule
(tests/builder_model.py), list for list, on every level.

From its code the GPU build is deterministic: levels are a function of the slot, batch boundaries follow a fixed rule,
the INSERT searches read only the graph as it stood before the batch, every forward task writes only its member's rows,
the pair sort is stable, and every reverse run writes only its own (level, neighbour) row. So each case below adds rows
on the GPU, saves, runs the model from the same starting graph with the levels of the saved file, and requires every
list in stored order, the entry point and the top level to be equal, and the levels to be `draw_level`'s. Each case
also requires the model's counter of the path it was written for to be non-zero.

The batch knobs (USEARCH_B200_BUILD_BATCH / _RATIO) are read once per process, so the cases that set them run in a
subprocess."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import common
from builder_model import BuilderModel, draw_levels
from usearch_b200 import v2format

pytestmark = pytest.mark.gpu

BATCH, RATIO = 32768, 32  # the builder's defaults


def _rows(n, d, scalar, seed=42):
    """rows in the stored scalar kind, so that `add` copies them unchanged"""
    if scalar == "f64":
        return common.make_collection(n, d, "f32", 1, seed=seed)[0].astype(np.float64)
    return common.make_collection(n, d, scalar, 1, seed=seed)[0]


def _hub_rows(scattered, clustered, d, spread=1e-3, seed=3):
    """`scattered` rows, then `clustered` rows in a tight cluster around row 0, the farthest from it first: every
    member of the cluster picks row 0 first, and the arrival at the end of row 0's cut run is the closest one that
    makes the cut, so it is kept by the reverse refine, and the cut decides the row"""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((scattered + clustered, d)).astype(np.float32)
    noise = spread * rng.standard_normal((clustered, d)).astype(np.float32)
    base[scattered:] = base[0] + noise[np.argsort(-np.linalg.norm(noise, axis=1), kind="stable")]
    return base


class Build:
    """one Index and the model, fed the same calls"""

    def __init__(self, metric, scalar, d, m=16, expansion_add=128, start=None):
        from usearch_b200.index import Index
        self.metric, self.scalar, self.d, self.m, self.ea = metric, scalar, d, m, expansion_add
        self.batch = int(os.environ.get("USEARCH_B200_BUILD_BATCH", BATCH))
        self.ratio = int(os.environ.get("USEARCH_B200_BUILD_RATIO", RATIO))
        if start is None:
            self.index = Index(ndim=d, metric=metric, dtype=scalar, connectivity=m, expansion_add=expansion_add)
            self.model = BuilderModel(metric=metric, scalar=scalar, dims=d, connectivity=m)
            self.own_levels_from = 0
        else:
            self.index = Index.restore(start)
            self.index.expansion_add = expansion_add
            self.model = BuilderModel(self.index.save())
            self.own_levels_from = self.model.size  # the file's own levels are the reference's
        self.free = []  # the queue of removed slots, oldest first
        self.counters = {}
        self.adds = 0

    def _restart_model(self):
        for k, v in self.model.counters().items():
            self.counters[k] = self.counters.get(k, 0) + v
        self.model = BuilderModel(self.index.save())

    def total(self) -> dict:
        return {k: v + self.counters.get(k, 0) for k, v in self.model.counters().items()}

    def remove(self, keys, compact):
        """removal is not the builder's: the model restarts from the saved file"""
        _, slot_keys, _ = self.model.neighbors()
        where = {int(k): s for s, k in enumerate(slot_keys)}
        assert self.index.remove(keys, compact=compact) == len(keys)
        self.free += [where[int(k)] for k in keys]
        self._restart_model()

    def add(self, keys, rows):
        keys = np.asarray(keys, dtype=np.uint64)
        first = self.model.size
        reuse = self.free[:len(keys)] if self.index.reuse_removed else []
        self.free = self.free[len(reuse):]
        appended = len(keys) - len(reuse)
        self.index.add(keys, rows)
        blob = self.index.save()
        g = v2format.loads(blob)
        what = f"{self.metric}/{self.scalar} d={self.d} M={self.m} ef={self.ea}, add call {self.adds}"
        self.adds += 1
        assert g.size == first + appended, what
        new_slots = np.concatenate([np.asarray(reuse, dtype=np.int64), np.arange(first, first + appended)])
        assert np.array_equal(g.vectors[new_slots], np.ascontiguousarray(rows).view(np.uint8).reshape(len(keys), -1)), what
        assert np.array_equal(g.keys[new_slots], keys), what
        self.model.add(keys, rows, g.levels[first:], reuse=reuse, expansion_add=self.ea, batch=self.batch, ratio=self.ratio)
        lo = max(first, self.own_levels_from)
        assert np.array_equal(g.levels[lo:], draw_levels(lo, g.size - lo, self.m)), f"{what}: levels"
        assert_same_graph(self.model, g, what)
        return blob


def assert_same_graph(model, g, what):
    levels, _, lists = model.neighbors()
    assert np.array_equal(g.levels, levels), f"{what}: levels differ"
    assert (g.entry_slot, g.max_level) == (model.entry_slot, model.max_level), \
        f"{what}: entry / top level: GPU {(g.entry_slot, g.max_level)}, model {(model.entry_slot, model.max_level)}"
    bad = [s for s in range(g.size) if g.neighbors[s] != lists[s]]
    if not bad:
        return
    linked_in, written_in = model.batches()
    s = bad[0]
    level = next(lv for lv in range(len(lists[s])) if g.neighbors[s][lv] != lists[s][lv])
    role = "member" if linked_in[s] == written_in[s] and linked_in[s] >= 0 else "centre"

    def show(lst):
        return ", ".join(f"{t}:{model.distance(s, t):.9g}" for t in lst)

    raise AssertionError(
        f"{what}: {len(bad)} slots differ; first: slot {s} ({role}, linked in model batch {linked_in[s]}, last written in "
        f"batch {written_in[s]}), level {level}\n  GPU   [{len(g.neighbors[s][level])}] {show(g.neighbors[s][level])}\n"
        f"  model [{len(lists[s][level])}] {show(lists[s][level])}\n  (entries as slot:pinned distance from slot {s})")


# ---- the cases ------------------------------------------------------------------------------------------------------

def _one_call(metric, scalar, n, d, m=16, expansion_add=128, rows=None):
    b = Build(metric, scalar, d, m, expansion_add)
    b.add(np.arange(n, dtype=np.uint64), _rows(n, d, scalar) if rows is None else rows)
    return b.total()


def _duplicates():
    n, d = 3000, 32
    rows = _rows(n, d, "f32")
    rows[n // 2:n // 2 + 300] = rows[:300]
    rows[-60:] = rows[7]
    return _one_call("l2sq", "f32", n, d, rows=rows)


def _hub():
    scattered, clustered, d = 1500, 800, 16
    rows = _hub_rows(scattered, clustered, d)
    b = Build("l2sq", "f32", d)
    b.add(np.arange(scattered, dtype=np.uint64), rows[:scattered])
    b.add(np.arange(scattered, scattered + clustered, dtype=np.uint64), rows[scattered:])
    return b.total()


def _uneven():
    d = 64
    rows = _rows(4013, d, "f32")
    b = Build("cos", "f32", d)
    at = 0
    for size in (1, 2, 97, 1500, 13, 2400):
        b.add(np.arange(at, at + size, dtype=np.uint64), rows[at:at + size])
        at += size
    return b.total()


def _grow_loaded():
    n0, d = 3000, 64
    rows = _rows(n0 + 2000, d, "f32")
    _, blob = common.build_reference_blob(rows[:n0], "cos", "f32", d, 16, threads=8)
    b = Build("cos", "f32", d, start=blob)
    b.add(np.arange(n0, n0 + 1500, dtype=np.uint64), rows[n0:n0 + 1500])
    b.add(np.arange(n0 + 1500, n0 + 2000, dtype=np.uint64), rows[n0 + 1500:])
    return b.total()


def _reuse(metric, scalar, compact):
    n, d = 3000, 64
    rows = _rows(n, d, scalar)
    b = Build(metric, scalar, d)
    b.add(np.arange(n, dtype=np.uint64), rows)
    g = v2format.loads(b.index.save())
    victims = np.random.default_rng(4).choice(n, 300, replace=False).astype(np.uint64)
    victims = np.unique(np.append(victims, g.keys[g.entry_slot]))
    np.random.default_rng(5).shuffle(victims)
    b.remove(victims, compact)
    b.index.reuse_removed = True
    fresh = _rows(len(victims) + 40, d, scalar, seed=77)
    keys = np.arange(10**6, 10**6 + len(fresh), dtype=np.uint64)
    b.add(keys[:100], fresh[:100])  # reused slots only
    b.add(keys[100:], fresh[100:])  # the rest of the queue, then appended rows
    return b.total()


# name: (run, counter the case is written for, environment)
CASES = {
    "l2sq-f32-32": (lambda: _one_call("l2sq", "f32", 4000, 32), "reverse_refines", {}),
    "cos-f32-768": (lambda: _one_call("cos", "f32", 1500, 768), "reverse_refines", {}),
    "ip-f32-97": (lambda: _one_call("ip", "f32", 3000, 97), "reverse_refines", {}),
    "cos-f16-256": (lambda: _one_call("cos", "f16", 3000, 256), "reverse_refines", {}),
    "l2sq-bf16-100": (lambda: _one_call("l2sq", "bf16", 3000, 100), "reverse_refines", {}),
    "ip-i8-64": (lambda: _one_call("ip", "i8", 3000, 64), "reverse_refines", {}),
    "cos-i8-96": (lambda: _one_call("cos", "i8", 3000, 96), "reverse_refines", {}),
    "hamming-b1-256": (lambda: _one_call("hamming", "b1", 3000, 256), "sort_ties", {}),
    "tanimoto-b1-192": (lambda: _one_call("tanimoto", "b1", 3000, 192), "reverse_refines", {}),
    "l2sq-f64-48": (lambda: _one_call("l2sq", "f64", 3000, 48), "reverse_refines", {}),
    "cos-f64-64": (lambda: _one_call("cos", "f64", 3000, 64), "reverse_refines", {}),
    "batch-1": (lambda: _one_call("cos", "f32", 1200, 48), "reverse_refines", {"USEARCH_B200_BUILD_BATCH": "1"}),
    "batch-7": (lambda: _one_call("ip", "i8", 2000, 64), "reverse_refines", {"USEARCH_B200_BUILD_BATCH": "7"}),
    "ratio-4": (lambda: _one_call("l2sq", "f32", 5000, 32), "reverse_refines", {"USEARCH_B200_BUILD_RATIO": "4"}),
    "hub": (_hub, "room_cuts", {"USEARCH_B200_BUILD_RATIO": "1"}),
    "duplicates": (_duplicates, "sort_ties", {}),
    "expansion-300": (lambda: _one_call("cos", "f32", 3000, 24, expansion_add=300), "candidate_cuts", {}),
    "expansion-8": (lambda: _one_call("ip", "f32", 2000, 24, expansion_add=8), "short_refines", {}),
    "m-4": (lambda: _one_call("l2sq", "f32", 2000, 16, m=4, expansion_add=64), "reverse_refines", {}),
    "m-40": (lambda: _one_call("l2sq", "f32", 4000, 16, m=40), "reverse_refines_base", {}),
    "uneven-adds": (_uneven, "reverse_refines", {}),
    "grow-loaded": (_grow_loaded, "reverse_refines", {}),
    "reuse": (lambda: _reuse("l2sq", "f32", False), "held_arrivals", {}),
    "reuse-compact": (lambda: _reuse("cos", "f16", True), "reused", {}),
}


def run_case(name):
    run, counter, _ = CASES[name]
    counters = run()
    assert counters[counter] > 0, f"{name}: the model never took the path the case is for ({counter}): {counters}"
    return counters


@pytest.mark.parametrize("name", list(CASES))
def test_gpu_build_equals_the_model(name):
    env = CASES[name][2]
    if not env:
        run_case(name)
        return
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import json, test_gpu_build_model as t\n"
            "print('MODEL_OK ' + json.dumps(t.run_case(%r)))\n") % (common.ROOT, os.path.join(common.ROOT, "tests"), name)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "MODEL_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-4000:]
    json.loads(out.stdout.split("MODEL_OK ", 1)[1].splitlines()[0])


def test_the_same_input_builds_the_same_file():
    """two builds of the same rows by two handles: byte-identical saved files"""
    from usearch_b200.index import Index
    n, d = 3000, 96
    rows = _rows(n, d, "f32")
    blobs = []
    for _ in range(2):
        index = Index(ndim=d, metric="cos", dtype="f32", connectivity=16)
        index.add(np.arange(1000, dtype=np.uint64), rows[:1000])
        index.add(np.arange(1000, n, dtype=np.uint64), rows[1000:])
        blobs.append(index.save())
    assert np.array_equal(blobs[0], blobs[1])
