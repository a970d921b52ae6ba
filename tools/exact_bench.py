"""Dev tool: wall-clock of the exact-search paths (not a bench line).
usage: exact_bench.py n d nq [scalar] [metric]"""
import sys, time
import numpy as np
sys.path.insert(0, ".")
from usearch_b200.index import Index, exact_search
from usearch_b200 import datagen, v2format


def linkless_blob(base: np.ndarray, metric: str, scalar: str, d: int) -> np.ndarray:
    """A v2 image whose graph has no edges (exact search never touches them); vectorised, unlike v2format.dumps."""
    n, bpv = base.shape[0], base.view(np.uint8).reshape(base.shape[0], -1).shape[1]
    g = v2format.Graph(metric=metric, scalar=scalar, dimensions=d, connectivity=2, connectivity_base=4,
                       vectors=np.zeros((0, bpv), np.uint8), keys=np.zeros(0, np.uint64), levels=np.zeros(0, np.int16))
    empty = v2format.dumps(g)
    head = bytearray(empty[8:8 + 64].tobytes())
    head[17:25] = np.uint64(n).tobytes()
    tape = np.zeros(n, dtype=np.dtype([("key", "<u8"), ("level", "<i2"), ("cnt", "<u4"), ("nb", "<u4", (4,))], align=False))
    tape["key"] = np.arange(n, dtype=np.uint64)
    parts = [np.array([n, bpv], dtype=np.uint32).tobytes(), base.view(np.uint8).tobytes(), bytes(head),
             np.array([n, 2, 4, 0, 0], dtype=np.uint64).tobytes(), np.zeros(n, np.int16).tobytes(), tape.tobytes()]
    return np.frombuffer(b"".join(parts), dtype=np.uint8)


def main():
    n, d, nq, k = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), 10
    scalar = sys.argv[4] if len(sys.argv) > 4 else "f32"
    metric = sys.argv[5] if len(sys.argv) > 5 else "cos"
    base = datagen.to_scalar(datagen.latent(n, d, seed=1, rank=16), scalar)
    q = datagen.to_scalar(datagen.latent(nq, d, seed=2, rank=16), scalar)
    index = Index.restore(linkless_blob(base, metric, scalar, d))
    for rep in range(4):
        t = time.perf_counter()
        m = index.search(q, k, exact=True)
        dt = time.perf_counter() - t
    pairs = n * nq
    print(f"index.search(exact) n={n} d={d} nq={nq} {scalar}/{metric}: {dt*1e3:.1f} ms, {nq/dt:.0f} q/s, "
          f"{pairs*d/dt/1e12:.2f} T multiply-adds/s")
    t = time.perf_counter()
    f = exact_search(base, q, k, metric=metric, dtype=scalar)
    dt = time.perf_counter() - t
    print(f"exact_search (free, incl. H2D of {base.nbytes/1e9:.2f} GB): {dt*1e3:.1f} ms; distances equal: "
          f"{np.array_equal(f.distances.view(np.uint32), m.distances.view(np.uint32))}")


if __name__ == "__main__":
    main()
