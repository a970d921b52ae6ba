"""The prefilter multiplies the int8 codes with a two-level int8 split of the query on the tensor cores. Queries whose
elements span a huge dynamic range (q1 saturates on a few elements, q2 carries the rest, or both levels lose the tiny
ones to the residual bound) must still give the pinned reference's labels, distance bits, counts and counters, with
the prefilter on and off."""
import numpy as np
import pytest

import common
from test_gpu_prefilter import _check, _pinned

pytestmark = pytest.mark.gpu


def _extreme_queries(q, rng):
    q = q.copy()
    nq, d = q.shape
    scale = np.float32(2.0) ** rng.integers(-40, 40, size=(nq, d)).astype(np.float32)
    q[: nq // 4] *= scale[: nq // 4]  # every element at its own magnitude, 2^-40 .. 2^39
    spikes = rng.integers(0, d, size=nq // 4)
    q[nq // 4: nq // 2] *= np.float32(1e-6)  # tiny elements, one huge one
    q[np.arange(nq // 4, nq // 2), spikes] = np.float32(1e6)
    q[nq // 2: 3 * nq // 4] = np.round(q[nq // 2: 3 * nq // 4] * 64) / 64  # on a coarse grid: sa2 is often 0
    sub = q[3 * nq // 4:]
    sub[:, ::3] *= np.float32(2.0 ** -135)  # a third of the elements subnormal
    return q.astype(np.float32)


@pytest.mark.parametrize("metric,d", [("cos", 768), ("ip", 768), ("cos", 97)])
def test_prefilter_extreme_dynamic_range_queries(metric, d):
    from usearch_b200.index import Index
    n, m, ef, k, nq = 6000, 16, 64, 10, 256
    base, q = common.make_collection(n, d, "f32", nq)
    q = _extreme_queries(q, np.random.default_rng(11))
    _, blob = common.build_reference_blob(base, metric, "f32", d, m, threads=16)
    index = Index.restore(blob)
    index.expansion_search = ef
    _check(index, _pinned(blob, q, k, ef), q, k, f"{metric}/{d} extreme queries")
