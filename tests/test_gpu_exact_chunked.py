"""The free exact search (`exact_search`, `usearch_exact_search`) scanned in chunks of rows, and its device entry.

USEARCH_B200_EXACT_CHUNK_ROWS forces the rows per chunk and USEARCH_B200_EXACT the scan kernel; both are read once per
process, so every (kernel, chunk rows) pair runs in a subprocess (`run_worker`) that dumps its results, and the test
holds them to the same worker's one-chunk run: keys, distance bits and counts, refusals included. Every dataset puts
exact duplicates and one-ulp near ties on both sides of every boundary the forced chunks have (multiples of 16, 100 and
1000), and half of the queries sit on those rows, so the ties reach the results. The one-chunk and the chunked results
are also held to the reference's exact search where it is built. In the process itself: strided and ragged host layouts,
the device entry in place and repacked on a non-default stream, the refusals of both entries with the device outputs
left untouched, and the top-level `search`."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import common  # noqa: E402
from oracle import bindings  # noqa: E402

N, NQ = 1200, 24
COUNTS = [1, 10, 256, 257, 700]
BOUNDARIES = sorted(set(range(16, N, 16)) | set(range(100, N, 100)) | {1000})
FAMILIES = [  # kind, dimensions (bits for b1), metrics
    ("f32", 96, ["cos", "l2sq", "ip"]),
    ("f16", 96, ["cos", "l2sq", "ip"]),
    ("bf16", 96, ["cos", "l2sq", "ip"]),
    ("f64", 48, ["cos", "l2sq", "ip"]),
    ("i8", 128, ["cos", "l2sq", "ip"]),
    ("b1", 256, ["hamming", "tanimoto", "sorensen"]),
]
KERNELS = ["default", "scan", "imma", "wgmma"]  # the forced ones run the i8 families only
CHUNK_ROWS = [16, 100, 1000]  # one tile or less for every scan, a few tiles, and a ragged last chunk of 200


def _one_ulp(row: np.ndarray, kind: str) -> np.ndarray:
    """`row` with its first element moved by one unit in the last place (one bit for b1)"""
    out = row.copy()
    if kind == "b1":
        out[0] ^= 1
    elif kind == "i8":
        out[0] = out[0] + 1 if out[0] < 127 else out[0] - 1
    else:
        as_int = {2: np.uint16, 4: np.uint32, 8: np.uint64}[out.itemsize]
        out.view(as_int)[0] += 1
    return out


def family_data(kind: str, d: int, n: int = N, seed: int = 7):
    """rows with a duplicate and a near tie across every forced boundary, and queries half of which sit on them"""
    base, queries = common.make_collection(n, d, "f32" if kind == "f64" else kind, NQ, seed=seed)
    if kind == "f64":
        base, queries = base.astype(np.float64), queries.astype(np.float64)
    for b in BOUNDARIES:
        if b + 1 < n:
            base[b] = base[b - 1]
            base[b + 1] = _one_ulp(base[b - 1], kind)
    on_boundaries = [b for b in BOUNDARIES if b + 1 < n]
    for i in range(NQ // 2):
        queries[i] = base[on_boundaries[(i * 7) % len(on_boundaries)] - 1]
    return np.ascontiguousarray(base), np.ascontiguousarray(queries)


def _search(results, key, *args, **kwargs):
    from usearch_b200.index import exact_search
    try:
        got = exact_search(*args, **kwargs)
        results[key] = (got.keys.copy(), got.distances.copy(), got.counts.copy())
    except RuntimeError as e:
        results[key] = str(e)


def _device_results(results):
    """the device entry on a non-default stream: in place (dense 384-byte rows) and repacked (a strided view, 388-byte rows)"""
    import torch
    from usearch_b200.index import exact_search_device
    base, queries = family_data("f32", 96)
    ragged, ragged_q = family_data("f32", 97)
    stream = torch.cuda.Stream()
    cases = {
        "in_place": (torch.from_numpy(base).cuda(), torch.from_numpy(queries).cuda()),
        "strided": (torch.from_numpy(np.repeat(base, 2, axis=0)).cuda()[::2], torch.from_numpy(queries).cuda()),
        "ragged": (torch.from_numpy(ragged).cuda(), torch.from_numpy(ragged_q).cuda()),
    }
    for name, (rows, q) in cases.items():
        for metric in ("cos", "l2sq"):
            for k in (10, 257):
                keys = torch.zeros((NQ, k), dtype=torch.int64, device="cuda")
                dists = torch.zeros((NQ, k), dtype=torch.float32, device="cuda")
                torch.cuda.synchronize()
                try:
                    exact_search_device(rows.data_ptr(), rows.shape[0], rows.stride(0) * 4, q.data_ptr(), q.shape[0], q.stride(0) * 4,
                                        rows.shape[1], k, keys.data_ptr(), dists.data_ptr(), metric=metric, dtype="f32",
                                        stream=stream.cuda_stream)
                    stream.synchronize()
                    results[("device", name, metric, k)] = (keys.cpu().numpy().view(np.uint64), dists.cpu().numpy(),
                                                            np.full(NQ, k, np.uint64))
                except RuntimeError as e:
                    results[("device", name, metric, k)] = str(e)


def run_worker(kernel: str, out_path: str) -> None:
    """every case of `kernel` under this process's chunk rows, pickled to `out_path`"""
    results = {}
    for kind, d, metrics in FAMILIES:
        if kernel != "default" and kind != "i8":
            continue
        base, queries = family_data(kind, d)
        small = np.ascontiguousarray(base[:300])
        for metric in metrics:
            for k in COUNTS:
                _search(results, (kind, metric, k), base, queries, k, metric=metric, dtype=kind)
            _search(results, (kind, metric, "k==n"), small, queries, 300, metric=metric, dtype=kind)
    if kernel == "default":
        base, queries = family_data("f32", 96)
        strided = np.repeat(base, 3, axis=0)[::3]
        assert not strided.flags.c_contiguous
        _search(results, ("strided", "cos", 10), strided, queries, 10, metric="cos", threads=3)
        ragged, ragged_q = family_data("f32", 97)
        for k in (10, 700):
            _search(results, ("ragged", "l2sq", k), ragged, ragged_q, k, metric="l2sq")
        _device_results(results)
    with open(out_path, "wb") as f:
        pickle.dump(results, f)


_DUMPS = {}


def _dump(kernel: str, rows, tmp_dir: str):
    if (kernel, rows) in _DUMPS:
        return _DUMPS[(kernel, rows)]
    out = os.path.join(tmp_dir, f"{kernel}_{rows}.pkl")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_exact_chunked as t\n"
            "t.run_worker(%r, %r)\n") % (ROOT, HERE, kernel, out)
    env = dict(os.environ)
    env.pop("USEARCH_B200_EXACT", None)
    env.pop("USEARCH_B200_EXACT_CHUNK_ROWS", None)
    if kernel != "default":
        env["USEARCH_B200_EXACT"] = kernel
    if rows:
        env["USEARCH_B200_EXACT_CHUNK_ROWS"] = str(rows)
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    with open(out, "rb") as f:
        _DUMPS[(kernel, rows)] = pickle.load(f)
    return _DUMPS[(kernel, rows)]


@pytest.fixture(scope="module")
def dump_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("exact_chunked"))


def _differences(what, want, got, limit=4):
    if isinstance(want, str) or isinstance(got, str):
        return [] if want == got else [f"{what}: want {want if isinstance(want, str) else 'results'}, got "
                                       f"{got if isinstance(got, str) else 'results'}"]
    wk, wd, wc = want
    gk, gd, gc = got
    lines = []
    if not np.array_equal(wc, gc):
        lines.append(f"{what}: counts differ")
    bad = np.argwhere((wk != gk) | (wd.view(np.uint32) != gd.view(np.uint32)))
    for q, pos in bad[:limit]:
        lines.append(f"{what}: query {q} position {pos}: key {int(wk[q, pos])} / {int(gk[q, pos])}, distance bits "
                     f"0x{int(wd.view(np.uint32)[q, pos]):08x} / 0x{int(gd.view(np.uint32)[q, pos]):08x}")
    return lines


@pytest.mark.gpu
@pytest.mark.parametrize("rows", CHUNK_ROWS)
@pytest.mark.parametrize("kernel", KERNELS)
def test_chunked_equals_one_chunk(kernel, rows, dump_dir):
    one = _dump(kernel, None, dump_dir)
    chunked = _dump(kernel, rows, dump_dir)
    assert set(one) == set(chunked)
    served = [key for key, value in one.items() if not isinstance(value, str)]
    assert len(served) >= len(one) // 2, {key: value for key, value in one.items() if isinstance(value, str)}
    report = []
    for key in sorted(one, key=str):
        report += _differences(f"{kernel} rows={rows} {key}", one[key], chunked[key])
    assert not report, "\n".join(report[:60])


def _hold_to_reference(what, got, base, queries, k, metric, kind, d):
    wk, wd = bindings.ref_exact_search(base, queries, min(k + 1, len(base)), metric=metric, scalar=kind, dims=d, pinned=True)
    keys, dists, _ = got
    assert np.array_equal(dists.view(np.uint32), wd[:, :k].view(np.uint32)), f"{what}: distance bits differ from the reference"
    unique = np.ones_like(wd[:, :k], dtype=bool)
    if k < wd.shape[1]:
        unique &= wd[:, :k] != wd[:, 1:k + 1]
    unique[:, 1:] &= wd[:, 1:k] != wd[:, :k - 1]
    assert np.array_equal(keys[unique], wk[:, :k][unique]), f"{what}: labels differ from the reference where distances are unique"


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [None, 16, 1000])
def test_chunked_matches_reference(rows, dump_dir):
    if not common.have_reference():
        pytest.skip("reference library not built")
    results = _dump("default", rows, dump_dir)
    checked = 0
    for kind, d, metrics in FAMILIES:
        if kind == "f64":  # the reference library takes no f64 rows
            continue
        base, queries = family_data(kind, d)
        for metric in metrics:
            for k in (1, 10, 257):
                got = results[(kind, metric, k)]
                assert not isinstance(got, str), got
                _hold_to_reference(f"{kind} {metric} k={k} rows={rows}", got, base, queries, k, metric, kind, d)
                checked += 1
    ragged, ragged_q = family_data("f32", 97)
    _hold_to_reference(f"ragged rows={rows}", results[("ragged", "l2sq", 700)], ragged, ragged_q, 700, "l2sq", "f32", 97)
    assert checked == 45


@pytest.mark.gpu
def test_host_layouts():
    """a strided, non-contiguous dataset and 388-byte rows give what their dense copies give"""
    from usearch_b200.index import exact_search
    base, queries = family_data("f32", 96)
    wide = np.zeros((N, 130), np.float32)
    wide[:, 7:103] = base
    view = wide[:, 7:103]
    assert not view.flags.c_contiguous and view.strides[0] == 130 * 4
    for threads in (0, 1, 5):
        got = exact_search(view, queries, 10, metric="cos", threads=threads)
        want = exact_search(base, queries, 10, metric="cos")
        assert not _differences("strided", (want.keys, want.distances, want.counts), (got.keys, got.distances, got.counts))
    ragged, ragged_q = family_data("f32", 97)
    assert ragged.strides[0] == 388
    got = exact_search(ragged, ragged_q, 10, metric="l2sq")
    exact = ((ragged_q[:, None, :].astype(np.float64) - ragged[None, :, :]) ** 2).sum(-1)
    assert np.allclose(got.distances, np.sort(exact, axis=1)[:, :10], rtol=1e-5, atol=1e-5)


@pytest.mark.gpu
def test_device_entry_equals_host_entry(dump_dir):
    """in place and repacked, on a non-default stream, unforced and with forced chunks"""
    from usearch_b200.index import exact_search
    base, queries = family_data("f32", 96)
    ragged, ragged_q = family_data("f32", 97)
    host = {"in_place": (base, queries), "strided": (base, queries), "ragged": (ragged, ragged_q)}
    report = []
    for rows in (None, 16):
        results = _dump("default", rows, dump_dir)
        for name, (rows_h, q_h) in host.items():
            for metric in ("cos", "l2sq"):
                for k in (10, 257):
                    want = exact_search(rows_h, q_h, k, metric=metric)
                    got = results[("device", name, metric, k)]
                    report += _differences(f"device {name} {metric} k={k} rows={rows}", (want.keys, want.distances, want.counts), got)
    assert not report, "\n".join(report[:40])


def _refusals():
    base, queries = family_data("f32", 96, n=300)
    long_rows = np.ones((300, 4096), np.float32)
    return [  # dataset, queries, count, metric, n override, message
        (base, queries, 301, "cos", None, "More neighbours requested than the dataset holds"),
        (base, queries, 10, "cos", 1 << 32, "Too many entries for 32-bit slots"),
        (long_rows, long_rows[:4], 257, "l2sq", None, "Exact search with count > 256 needs vectors that fit the tiled stage"),
        (base, queries, 10, "haversine", None, None),  # the host entry's message, whichever it is
    ]


@pytest.mark.gpu
def test_refusals_unchanged_on_both_entries():
    import ctypes as C

    import torch
    from usearch_b200.index import METRIC_KIND, SCALAR_KIND, exact_search, exact_search_device, load_library
    lib = load_library()
    for rows, q, k, metric, n_override, message in _refusals():
        n = n_override or rows.shape[0]
        keys = np.zeros((q.shape[0], k), np.uint64)
        dists = np.zeros((q.shape[0], k), np.float32)
        err = C.c_char_p()
        lib.usearch_exact_search(rows.ctypes.data_as(C.c_void_p), n, rows.strides[0], q.ctypes.data_as(C.c_void_p), q.shape[0],
                                 q.strides[0], SCALAR_KIND["f32"], rows.shape[1], METRIC_KIND[metric], k, 0,
                                 keys.ctypes.data_as(C.c_void_p), keys.strides[0], dists.ctypes.data_as(C.c_void_p),
                                 dists.strides[0], C.byref(err))
        assert err.value, f"host entry served {message}"
        host_message = err.value.decode()
        assert message is None or host_message == message
        if n_override is None and metric != "haversine":
            with pytest.raises(RuntimeError, match=host_message):
                exact_search(rows, q, k, metric=metric)
        d_rows, d_q = torch.from_numpy(rows).cuda(), torch.from_numpy(q).cuda()
        d_keys = torch.full((q.shape[0], k), 0x5A5A, dtype=torch.int64, device="cuda")
        d_dists = torch.full((q.shape[0], k), -7.25, dtype=torch.float32, device="cuda")
        before = (d_keys.clone(), d_dists.clone())
        with pytest.raises(RuntimeError) as refused:
            exact_search_device(d_rows.data_ptr(), n, rows.strides[0], d_q.data_ptr(), q.shape[0], q.strides[0], rows.shape[1], k,
                                d_keys.data_ptr(), d_dists.data_ptr(), metric=metric, stream=torch.cuda.Stream().cuda_stream)
        torch.cuda.synchronize()
        assert str(refused.value) == host_message
        assert torch.equal(d_keys, before[0]) and torch.equal(d_dists, before[1]), f"outputs written on {host_message}"


@pytest.mark.gpu
def test_top_level_search():
    from usearch_b200.index import Index, exact_search, search
    base, queries = family_data("f32", 96)
    want = exact_search(base, queries, 10, metric="l2sq")
    got = search(base, queries, 10, "l2sq", exact=True)
    assert not _differences("search(exact=True)", (want.keys, want.distances, want.counts), (got.keys, got.distances, got.counts))
    one = search(base, queries[3], 10, "l2sq", exact=True)
    assert np.array_equal(one.keys, want.keys[3]) and np.array_equal(one.distances.view(np.uint32), want.distances[3].view(np.uint32))
    index = Index(ndim=96, metric="cos", dtype="f32")
    index.add(None, base)
    want = index.search(queries, 10)
    got = search(base, queries, 10, "cos")
    assert not _differences("search(exact=False)", (want.keys, want.distances, want.counts), (got.keys, got.distances, got.counts))
