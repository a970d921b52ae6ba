"""Pure-Python model of what an index reports about itself, read from its v2 blob with its own parser: the three `stats`
functions of `index_gt` (index.hpp:3133-3225, quirks included), the live keys and each key's stored rows.

Layout (index_dense.hpp:994-1062, index.hpp:3276-3317): [u32 rows, u32 bytes per row][matrix][64-byte head][40-byte
graph header: size, M, M0, max_level, entry][i16 level per node][per node: u64 key, i16 level, {u32 count, u32[M0]},
level x {u32 count, u32[M]}]. A node's tape is a 10-byte head (key and level) and its lists."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

FREE_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)
HEAD_BYTES = 10


@dataclass
class Graph:
    keys: np.ndarray      # [n] u64, slot order
    levels: np.ndarray    # [n] i16
    matrix: np.ndarray    # [n, bytes per row] u8
    edges: list           # edges[slot][level] = the list's stored count
    m: int
    m0: int
    max_level: int
    multi: bool


def parse(blob) -> Graph:
    b = np.ascontiguousarray(blob, dtype=np.uint8).tobytes()
    rows, cols = np.frombuffer(b, np.uint32, 2, 0)
    rows, cols = int(rows), int(cols)
    at = 8
    matrix = np.frombuffer(b, np.uint8, rows * cols, at).reshape(rows, cols)
    at += rows * cols
    assert b[at:at + 7] == b"usearch", "not a v2 index"
    multi = b[at + 41] != 0
    at += 64
    n, m, m0, max_level, _entry = (int(x) for x in np.frombuffer(b, np.uint64, 5, at))
    at += 40
    levels = np.frombuffer(b, np.int16, n, at).copy()
    at += 2 * n
    keys = np.zeros(n, np.uint64)
    edges = []
    for s in range(n):
        keys[s] = np.frombuffer(b, np.uint64, 1, at)[0]
        level = int(np.frombuffer(b, np.int16, 1, at + 8)[0])
        at += HEAD_BYTES
        counts = [int(np.frombuffer(b, np.uint32, 1, at)[0])]
        at += 4 + 4 * m0
        for _ in range(level):
            counts.append(int(np.frombuffer(b, np.uint32, 1, at)[0]))
            at += 4 + 4 * m
        edges.append(counts)
    return Graph(keys, levels, matrix, edges, m, m0, max_level if n else 0, multi)


def _stats(nodes, edges, max_edges, allocated):
    return (int(nodes), int(edges), int(max_edges), int(allocated))


def stats(g: Graph):
    """stats(): every node once; max_edges = sum(level M + M0); allocated = the node tapes"""
    nb, nb0 = 4 + 4 * g.m, 4 + 4 * g.m0
    n = len(g.keys)
    lv = g.levels.astype(np.int64)
    return _stats(n, sum(sum(e) for e in g.edges), int((lv * g.m + g.m0).sum()), int((HEAD_BYTES + nb0 + lv * nb).sum()))


def level_stats(g: Graph, level: int):
    """stats(level): nodes on `level` and above; the 10-byte head counted at every level"""
    nb = 4 + 4 * g.m if level else 4 + 4 * g.m0
    members = [s for s in range(len(g.keys)) if g.levels[s] >= level]
    nodes = len(members)
    return _stats(nodes, sum(g.edges[s][level] for s in members), nodes * (g.m if level else g.m0), nodes * (HEAD_BYTES + nb))


def levels_stats(g: Graph):
    """stats(per_level, max_level): (per level, their sum); the head counted on level 0 only. Empty index: ([], zeros)."""
    if not len(g.keys):
        return [], _stats(0, 0, 0, 0)
    nb, nb0 = 4 + 4 * g.m, 4 + 4 * g.m0
    per = []
    for level in range(g.max_level + 1):
        members = [s for s in range(len(g.keys)) if g.levels[s] >= level]
        nodes = len(members)
        per.append(_stats(nodes, sum(g.edges[s][level] for s in members), nodes * (g.m if level else g.m0),
                          nodes * (nb if level else nb0 + HEAD_BYTES)))
    return per, tuple(int(sum(p[i] for p in per)) for i in range(4))


def live_keys(g: Graph) -> np.ndarray:
    """every key != the free key, in slot order (one per entry of a multi index)"""
    return g.keys[g.keys != FREE_KEY]


def rows_of(g: Graph, key) -> np.ndarray:
    """the stored rows under `key`, in slot order: [count, bytes per row] u8"""
    return g.matrix[g.keys == np.uint64(key)] if np.uint64(key) != FREE_KEY else g.matrix[:0]
