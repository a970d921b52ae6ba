"""f64 without a GPU: the lane split of the f64 metric structs, the fixture tests/golden/f64_cases.npz against the live
reference, the pinned f64 metric against the reference's own SimSIMD f64 kernels, and the reference's casts into and
out of f64 as the device and host casts restate them."""
import os
import subprocess

import numpy as np
import pytest

import common
import f64_reference as fr

NATIVE = os.path.join(common.ROOT, "tests", "native")
live = pytest.mark.skipif(not fr.available(), reason="reference sources unavailable")


def test_lane_split_matches_pinned_order(tmp_path):
    exe = tmp_path / "f64_lanes"
    subprocess.run(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror", "-I", NATIVE,
                    os.path.join(NATIVE, "test_f64_lanes_order.c"), "-o", str(exe), "-lm"], check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert "distances equal" in out


def test_fixture_native_labels_equal_pinned():
    fx = fr.load_fixture()
    for name in fr.case_names(fx):
        for tag in ("keys", "counts"):
            assert np.array_equal(fx[f"{name}/ef64_k10_native/{tag}"], fx[f"{name}/ef64_k10_pinned/{tag}"]), name


@live
@pytest.mark.parametrize("name", ["cos_d768", "l2sq_d97", "ip_d24", "l2sq_d3200"])
def test_fixture_reproduced_by_live_reference(name):
    fx = fr.load_fixture()
    blob, base = fr.case_blob(fx, name)
    q = fr.case_queries(fx, name)
    ref = fr.RefF64(fx[f"{name}/metric"].item(), int(fx[f"{name}/d"]), connectivity=int(fx[f"{name}/m"]))
    ref.view(blob)
    ref.pin(True)
    for key in fx:
        if not key.startswith(f"{name}/ef") or not key.endswith("_pinned/keys"):
            continue
        ef, k = (int(t[2:]) if t.startswith("ef") else int(t[1:]) for t in key.split("/")[1].split("_")[:2])
        ref.change_expansion_search(ef)
        got = ref.search(q, k)
        prefix = key[: -len("/keys")]
        common.assert_same_results(tuple(fx[f"{prefix}/{t}"] for t in ("keys", "distances", "counts", "computed", "visited")), got, prefix)
    ref.change_expansion_search(64)
    for k in (10, 300):
        if f"{name}/exact_k{k}/keys" in fx:
            got = ref.search(q, k, exact=True)
            assert np.array_equal(got[0], fx[f"{name}/exact_k{k}/keys"])
            keys, dist = fr.exact_search(base, q, k, fx[f"{name}/metric"].item())
            assert np.array_equal(dist.view(np.uint32), fx[f"{name}/free_k{k}/distances"].view(np.uint32))
    if f"{name}/max_level" in fx:
        for level in range(int(fx[f"{name}/max_level"]) + 2):
            got = ref.cluster(q, level)
            for tag, v in zip(("keys", "distances", "computed", "visited"), got):
                assert np.array_equal(np.asarray(v).view(np.uint32 if tag == "distances" else np.uint64),
                                      fx[f"{name}/cluster_l{level}/{tag}"].view(np.uint32 if tag == "distances" else np.uint64)), (level, tag)


@live
@pytest.mark.parametrize("metric", ["l2sq", "ip", "cos"])
def test_pinned_equals_native_simsimd(metric):
    """on an AVX-512 host the reference runs simsimd_*_f64_skylake: l2sq and ip give the pinned bits. cos is within 1 ULP, or
    within 2^-26 of a distance near 0, where rsqrt14_pd plus one Newton step leaves an absolute error of ~1e-10"""
    ref = fr.RefF64(metric, 8)
    if ref.isa_name not in ("skylake", "ice", "genoa", "sapphire", "turin"):
        pytest.skip(f"the reference dispatches f64 to {ref.isa_name}, not an AVX-512 kernel")
    rng = np.random.default_rng(5)
    worst = 0
    for n in (1, 3, 7, 8, 9, 24, 31, 97, 768, 3200):
        for scale in (1e-3, 1.0, 1e5):
            a, b = scale * rng.standard_normal(n), scale * rng.standard_normal(n)
            pinned = np.float32(fr.distance(metric, a, b, pinned=True))
            native = np.float32(fr.distance(metric, a, b, pinned=False))
            ulps = abs(int(pinned.view(np.int32)) - int(native.view(np.int32)))
            if metric == "cos":
                assert ulps <= 1 or abs(float(pinned) - float(native)) <= 2.0 ** -26, (n, scale, pinned, native)
                worst = max(worst, ulps if ulps <= 1 else 0)
            else:
                assert ulps == 0, (n, scale, pinned, native)
    assert worst <= 1


def test_fixture_casts_follow_cast_gt():
    """what the reference stored and returned, restated the way the device cast (into f64) and the host `get` cast
    (out of f64) compute it"""
    fx = fr.load_fixture()
    assert np.array_equal(fx["casts/in_f32_stored"], fx["casts/in_f32"].astype(np.float64))
    assert np.array_equal(fx["casts/in_f16_stored"], fx["casts/in_f16"].astype(np.float64))
    assert np.array_equal(fx["casts/in_i8_stored"], fx["casts/in_i8"].astype(np.float64) / 127.0)  # a double division
    assert not np.array_equal(fx["casts/in_i8_stored"], (fx["casts/in_i8"].astype(np.float32) / np.float32(127)).astype(np.float64))
    assert np.array_equal(fx["casts/in_b1_stored"], np.unpackbits(fx["casts/in_b1"], axis=1).astype(np.float64))
    x = fx["casts/out_rows"]
    assert np.array_equal(fx["casts/out_f32"].view(np.uint32), x.astype(np.float32).view(np.uint32))
    assert np.array_equal(fx["casts/out_f16"].view(np.uint16), x.astype(np.float32).astype(np.float16).view(np.uint16))
    assert np.array_equal(fx["casts/out_b1"], np.packbits(x > 0, axis=1))  # 1e-50 > 0 although (float)1e-50 == 0
    mag = np.sqrt(np.array([sum(float(v) * float(v) for v in row) for row in x]))
    want_i8 = np.clip(x * 127.0 / mag[:, None], -127, 127).astype(np.int8)
    assert np.array_equal(fx["casts/out_i8"], want_i8)


# ---- the port (oracle/hnsw_oracle.c with the f64 pinned metric, tests/native/port_f64.c) -------------------------------

@pytest.mark.parametrize("name", ["cos_d768", "l2sq_d97", "ip_d24", "l2sq_d3200"])
def test_port_matches_fixture(name):
    """labels, distance bits, counts and both counters of graph search, exact search and cluster, and pair distances"""
    fx = fr.load_fixture()
    blob, base = fr.case_blob(fx, name)
    q = fr.case_queries(fx, name)
    port = fr.PortF64(blob)
    want = lambda p: tuple(fx[f"{p}/{t}"] for t in ("keys", "distances", "counts", "computed", "visited"))
    for key in fx:
        if key.startswith(f"{name}/ef") and key.endswith("_pinned/keys"):
            ef, k = key.split("/")[1].split("_")[:2]
            port.change_expansion_search(int(ef[2:]))
            common.assert_same_results(want(key[: -len("/keys")]), port.search(q, int(k[1:])), key)
    for k in (10, 300):
        if f"{name}/exact_k{k}/keys" in fx:
            got = port.search(q, k, exact=True)
            common.assert_same_results(want(f"{name}/exact_k{k}")[:3], got[:3], f"{name} exact {k}")
    if f"{name}/max_level" in fx:
        for level in range(int(fx[f"{name}/max_level"]) + 2):
            got = port.cluster(q, level)
            for tag, v in zip(("keys", "distances", "computed", "visited"), got):
                w = fx[f"{name}/cluster_l{level}/{tag}"]
                assert np.array_equal(np.asarray(v).view(w.dtype), w), (level, tag)
        pairs = fx[f"{name}/pairs"]
        got = np.array([port.distance(base[i], base[j]) for i, j in pairs], dtype=np.float32)
        assert np.array_equal(got.view(np.uint32), fx[f"{name}/pairs_pinned"].view(np.uint32))
    if f"{name}/compact/graph" in fx:  # the reference's graph after more removals and isolate
        compact = np.concatenate([blob[: blob.size - fx[f"{name}/graph"].size], fx[f"{name}/compact/graph"]])
        port = fr.PortF64(compact)
        common.assert_same_results(want(f"{name}/compact/ef64_k10"), port.search(q, 10), "after isolate")


@live
@pytest.mark.parametrize("metric,d,n,m,removed", [("cos", 64, 800, 8, 0), ("l2sq", 33, 1200, 12, 90), ("ip", 7, 600, 4, 30),
                                                 ("cos", 257, 400, 16, 40), ("l2sq", 2, 300, 4, 0)])
def test_port_matches_live_reference(metric, d, n, m, removed):
    """seeded f64 graphs the reference builds: search at two ef, exact search and cluster on every level"""
    rng = np.random.default_rng(d * 1000 + n)
    base, q = rng.standard_normal((n, d)), rng.standard_normal((24, d))
    ref = fr.RefF64(metric, d, connectivity=m, expansion_add=64)
    ref.pin(True)
    ref.add(np.arange(n), base)
    for key in rng.choice(n, removed, replace=False):
        ref.remove(int(key))
    blob = ref.save()
    port = fr.PortF64(blob)
    for ef, k in ((16, 5), (128, 40)):
        ref.change_expansion_search(ef)
        port.change_expansion_search(ef)
        common.assert_same_results(ref.search(q, k), port.search(q, k), f"ef {ef} k {k}")
    assert np.array_equal(ref.search(q, 12, exact=True)[1].view(np.uint32), port.search(q, 12, exact=True)[1].view(np.uint32))
    top = int(np.frombuffer(blob[8 + n * d * 8 + 64 + 24:][:8].tobytes(), dtype=np.uint64)[0])
    for level in range(top + 2):
        for a, b in zip(ref.cluster(q, level), port.cluster(q, level)):
            assert np.array_equal(np.asarray(a), np.asarray(b)), level


# ---- the host casts of `get` out of an f64 index (usearch_b200/csrc/f64_casts.h) ---------------------------------------

@pytest.fixture(scope="module")
def casts(tmp_path_factory):
    import ctypes as C
    out = str(tmp_path_factory.mktemp("f64_casts") / "libf64_casts.so")
    subprocess.run(["g++", "-std=c++11", "-O2", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC", "-I",
                    os.path.join(common.ROOT, "usearch_b200", "csrc"), os.path.join(NATIVE, "f64_casts_shim.cpp"), "-o", out],
                   check=True, capture_output=True)
    lib = C.CDLL(out)
    for name in ("shim_f64_to_i8", "shim_f64_to_b1"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    return lib


def _host_cast(lib, rows, kind):
    rows = np.ascontiguousarray(rows, dtype=np.float64)
    d = rows.shape[1]
    out = np.zeros((len(rows), (d + 7) // 8 if kind == "b1" else d), dtype=np.uint8 if kind == "b1" else np.int8)
    fn = lib.shim_f64_to_b1 if kind == "b1" else lib.shim_f64_to_i8
    for r, o in zip(rows, out):
        fn(r.ctypes.data, d, o.ctypes.data)
    return out


def test_host_get_casts_match_fixture(casts):
    """the doubles include values below the f32 subnormal range (b1: > 0 all the same) and a row scaled by 1e-100, whose
    i8 magnitude only exists in f64"""
    fx = fr.load_fixture()
    for kind in ("i8", "b1"):
        assert np.array_equal(_host_cast(casts, fx["casts/out_rows"], kind), fx[f"casts/out_{kind}"]), kind


@live
def test_host_get_casts_match_live_reference(casts):
    rng = np.random.default_rng(17)
    for d in (1, 7, 8, 40, 97):
        rows = rng.standard_normal((12, d)) * np.logspace(-300, 300, 12)[:, None]
        rows[0, 0] = 1e-320
        ref = fr.RefF64("l2sq", d)
        ref.add(np.arange(len(rows)), rows)
        for kind in ("i8", "b1"):
            want = np.stack([ref.get(i, kind) for i in range(len(rows))])
            assert np.array_equal(_host_cast(casts, rows, kind).view(np.uint8), want.view(np.uint8)), (d, kind)
