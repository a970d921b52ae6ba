"""Writes tests/golden/join_cases.npz: the reference's own `index_dense_gt::join` (one thread, pinned metric,
tests/native/ref_join_driver.cpp) on graphs the reference builds deterministically (pinned metric, one thread), for
tests/test_gpu_join.py, which runs where the reference sources are not. Per case: the a -> b mapping, the four counters,
and the SHA-256 of both saved graphs so that the GPU test knows it rebuilt the same files.

    python tests/golden/make_golden_join.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import join_reference as jr  # noqa: E402
from oracle import bindings  # noqa: E402
from usearch_b200 import datagen, v2format  # noqa: E402

METRIC_CASES = [("cos", "f32", 768), ("cos", "f32", 97), ("ip", "f32", 97), ("l2sq", "f32", 97), ("cos", "f16", 64),
                ("ip", "i8", 64), ("hamming", "b1", 256)]
B_KEYS = 10_000


def rows(n, d, scalar, seed, base, noise=0.05):
    x = base[np.random.default_rng(seed).permutation(len(base))[:n]]
    x = x + noise * np.random.default_rng(seed + 1).standard_normal(x.shape).astype(np.float32)
    return datagen.to_scalar(np.ascontiguousarray(x, dtype=np.float32), scalar)


def build(x, metric, scalar, d, keys, remove=()):
    """deterministic: pinned metric, one thread"""
    ref = bindings.RefIndex("parity", metric=metric, scalar=scalar, dims=d, connectivity=16, expansion_add=64, expansion_search=64)
    ref.pin_metric(True)
    ref.add(keys, x, threads=1)
    for key in remove:
        ref.remove(int(key))
    return ref.save()


def as_multi(blob, divisor):
    g = v2format.loads(blob)
    live = g.keys != v2format.FREE_KEY
    g.keys = np.where(live, g.keys // np.uint64(divisor), g.keys)
    g.multi = True
    return v2format.dumps(g)


def cases():
    """name -> (a blob, b blob, max_proposals, expansion, exact)"""
    out = {}
    for metric, scalar, d in METRIC_CASES:
        base = datagen.latent(420, d, seed=100, rank=min(16, d))
        a = build(rows(300, d, scalar, 1, base), metric, scalar, d, np.arange(300, dtype=np.uint64))
        b = build(rows(420, d, scalar, 2, base), metric, scalar, d, np.arange(420, dtype=np.uint64) + B_KEYS)
        for exact in (False, True):
            tag = f"{metric}-{scalar}-{d}-{'exact' if exact else 'approx'}"
            out[f"{tag}-men_fewer"] = (a, b, 0, 64, exact)
            out[f"{tag}-swap"] = (b, a, 0, 64, exact)
    d = 64
    # near-duplicates: hamming ties make men collide, so proposals run past an expansion of 4
    men = datagen.to_scalar(datagen.latent(250, d, seed=12, rank=16), "b1")
    women = np.concatenate([men[:150], men[:150], datagen.to_scalar(datagen.latent(100, d, seed=13, rank=16), "b1")])
    out["p_above_expansion"] = (build(men, "hamming", "b1", d, np.arange(250, dtype=np.uint64)),
                                build(women, "hamming", "b1", d, np.arange(400, dtype=np.uint64) + B_KEYS), 12, 4, False)
    base = datagen.latent(360, 97, seed=5, rank=16)
    out["removed"] = (build(rows(300, 97, "f32", 6, base), "l2sq", "f32", 97, np.arange(300, dtype=np.uint64), remove=range(0, 300, 7)),
                      build(rows(360, 97, "f32", 7, base), "l2sq", "f32", 97, np.arange(360, dtype=np.uint64) + B_KEYS,
                            remove=range(B_KEYS, B_KEYS + 360, 5)), 0, 64, False)
    a = build(rows(300, 64, "f32", 8, base[:, :64].copy()), "cos", "f32", 64, np.arange(300, dtype=np.uint64))
    b = build(rows(350, 64, "f32", 9, base[:, :64].copy()), "cos", "f32", 64, np.arange(350, dtype=np.uint64) + B_KEYS)
    out["multi"] = (as_multi(a, 2), as_multi(b, 3), 0, 64, False)
    return out


def sha(blob) -> str:
    return hashlib.sha256(np.ascontiguousarray(blob, dtype=np.uint8).tobytes()).hexdigest()


def main():
    arrays = {}
    for name, (a, b, max_p, ef, exact) in cases().items():
        a_to_b, stats = jr.live_join(a, b, max_p, ef, exact)
        items = sorted(a_to_b.items())
        arrays[f"{name}/a_keys"] = np.array([k for k, _ in items], dtype=np.uint64)
        arrays[f"{name}/b_keys"] = np.array([v for _, v in items], dtype=np.uint64)
        arrays[f"{name}/stats"] = np.array([stats[k] for k in ("intersection_size", "engagements", "visited_members",
                                                               "computed_distances")], dtype=np.uint64)
        arrays[f"{name}/sha"] = np.array([sha(a), sha(b)])
        if name == "p_above_expansion":  # the deepest proposal the reference loop reached (restated over its searches)
            g_men = v2format.loads(a).size
            cols = jr.reference_columns(a, b, 12, 4, False)
            arrays[f"{name}/deepest"] = np.array([_deepest(g_men, v2format.loads(b).size, 12, cols)], dtype=np.uint64)
        print(name, stats)
    np.savez_compressed(os.path.join(HERE, "join_cases.npz"), **arrays)


def _deepest(men, women, proposals, columns):
    deepest = [0]
    def counting(i):
        deepest[0] = max(deepest[0], i)
        return columns[i]
    class Cols(dict):
        def __getitem__(self, i):
            return counting(i)
    jr.replay(men, women, proposals, Cols(columns))
    return deepest[0]


if __name__ == "__main__":
    main()
