"""The scalar casts (usearch_b200/csrc/scalar_casts.h) against the reference's own cast_gt, on the host.

The reference is the oracle's parity build (oracle/build.py), whose SimSIMD half-precision conversions round ties away from zero, turn
f16 overflow into NaN patterns, and decode the f16 exponent 31 as a finite number: an IEEE cast differs from it on about
one f32 element in 8192 of ordinary data and on every element of the edge tables in scalar_cast_edges.py."""
import os
import subprocess

import numpy as np
import pytest

import cast_reference as cr
import common
import scalar_cast_edges as edges

NATIVE = os.path.join(common.ROOT, "tests", "native")
CSRC = os.path.join(common.ROOT, "usearch_b200", "csrc")
live = pytest.mark.skipif(not cr.reference_available(), reason="reference sources unavailable")
KINDS = ("f64", "f32", "f16", "bf16", "i8", "b1")


def test_the_recipe_builds_the_reference_with_simsimd_casts():
    """The cast contract holds for this build only: without USEARCH_USE_FP16LIB=0 a reference built without AVX-512
    takes fp16lib, which rounds the IEEE way."""
    with open(os.path.join(common.ROOT, "oracle", "build.py")) as f:
        recipe = f.read()
    assert '"-DUSEARCH_USE_FP16LIB=0"' in recipe and '"-DUSEARCH_USE_SIMSIMD=1"' in recipe


@pytest.fixture(scope="module")
def shim():
    return cr.host()


def _bits(x: float) -> int:
    return int(np.float32(x).view(np.uint32))


def _value(bits: int) -> float:
    return float(np.uint32(bits).view(np.float32))


def test_the_reference_rows_of_the_cast_table(shim):
    """The conversions the reference makes and IEEE rounding does not, value by value."""
    assert shim.shim_f32_to_f16(_bits(1 + 2.0 ** -11)) == 0x3C01  # an exact tie, even below: away from zero
    assert shim.shim_f32_to_f16(_bits(-(1 + 2.0 ** -11))) == 0xBC01
    assert shim.shim_f32_to_f16(_bits(70000.0)) == 0x7C46  # f16 exponent 31 with mantissa bits: a NaN pattern
    assert shim.shim_f32_to_f16(_bits(65520.0)) == 0x7C00
    assert shim.shim_f32_to_f16(_bits(1e6)) == 0x7FFF and shim.shim_f32_to_f16(_bits(float("inf"))) == 0x7FFF
    assert shim.shim_f32_to_f16(_bits(float("-inf"))) == 0xFFFF
    assert shim.shim_f32_to_f16(0x7FFFF000) == 0x8000  # the rounding carry runs into the sign bit
    assert shim.shim_f32_to_f16(_bits(2.0 ** -26)) == 0x0000 and shim.shim_f32_to_f16(_bits(2.0 ** -25)) == 0x0001
    assert shim.shim_f32_to_bf16(0x3F808000) == 0x3F81  # a tie: away from zero
    assert shim.shim_f32_to_bf16(0x7F800001) == 0x7F80  # a signalling NaN becomes +inf
    assert shim.shim_f32_to_bf16(0x7F7F8000) == 0x7F80
    assert _value(shim.shim_f16_to_f32(0x7C00)) == 65536.0 and _value(shim.shim_f16_to_f32(0xFC00)) == -65536.0
    assert _value(shim.shim_f16_to_f32(0x7FFF)) == 131008.0
    assert _value(shim.shim_f16_to_f32(0x0001)) == 2.0 ** -24 and _value(shim.shim_f16_to_f32(0x03FF)) == 1023 * 2.0 ** -24


@live
def test_every_f32_and_half_pattern_casts_like_the_reference(tmp_path):
    """All 2^32 f32 patterns through f32 -> f16 and f32 -> bf16, all 2^16 f16 and bf16 patterns back to f32, natively.
    USEARCH_B200_CAST_STRIDE=k checks every k-th f32 pattern only."""
    exe = str(tmp_path / "test_scalar_casts")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-I", CSRC,
                    os.path.join(NATIVE, "test_scalar_casts.cpp"), "-o", exe, "-ldl"], check=True)
    lib = cr.ref_lib_path()
    stride = os.environ.get("USEARCH_B200_CAST_STRIDE", "1")
    out = subprocess.run([exe, lib, stride], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "failures: 0" in out.stdout


# ---- whole rows: cast_row_host (the casts of `get`) against the reference's cast_gt ---------------------------------

def _as_kind(rows: np.ndarray, kind: str) -> np.ndarray:
    """rows as f64 or f32 (an f32 table stays bit for bit, signalling NaNs included)"""
    with np.errstate(invalid="ignore", over="ignore"):
        return np.ascontiguousarray(rows, dtype=np.float64 if kind == "f64" else np.float32)


def _compare(shim, src: np.ndarray, from_kind: str, to_kind: str, dims: int, what: str):
    cr.assert_same_casts(cr.ref_cast(src, from_kind, to_kind, dims), cr.host_cast(src, from_kind, to_kind, dims), src,
                         from_kind, to_kind, dims, what)


def _i8_rows(dims: int, wide: bool) -> np.ndarray:
    """rows where the i8 cast (x * 127 / |x| in f64, clamped, truncated) is delicate"""
    rng = np.random.default_rng(dims)
    rows = []
    zero = np.zeros(dims)
    rows.append(zero)
    for special in (np.inf, -np.inf, np.nan):
        r = rng.standard_normal(dims)
        r[dims // 2] = special
        rows.append(r)
    for big in (1e30, -1e30, 3e38):  # one dominant element: 127 or -127 there, zeros elsewhere
        r = rng.standard_normal(dims)
        r[0] = big
        rows.append(r)
    for x in (1.0, -1.0, 3.0, 1e-30, 2.0 ** -149):  # a single non-zero: exactly +-127 (or more, before the clamp)
        r = zero.copy()
        r[-1] = x
        rows.append(r)
    r = np.full(dims, 0.1)
    rows.append(r)
    rows.append(rng.standard_normal(dims) * 1e-20)
    if wide:  # magnitudes only f64 holds, and squares that overflow or underflow it
        for scale in (1e200, -1e300, 1e-200, 1e-320):
            rows.append(rng.standard_normal(dims) * scale)
        r = rng.standard_normal(dims)
        r[1 % dims] = 1e300
        rows.append(r)
    return np.stack(rows)


def _b1_rows(dims: int, wide: bool) -> np.ndarray:
    vals = [0.0, -0.0, np.nan, -np.nan, 1e-45, -1e-45, 1e-40, 2.0 ** -149, np.inf, -np.inf, 1.0, -1.0]
    if wide:
        vals += [1e-320, -1e-320, 1e-200, 1e300]
    vals = np.asarray(vals)
    idx = (np.arange(dims)[None, :] + np.arange(len(vals))[:, None] * 5) % len(vals)
    return vals[idx]


@live
@pytest.mark.parametrize("from_kind", ["f32", "f64"])
@pytest.mark.parametrize("dims", [1, 7, 8, 9, 97, 768])
def test_float_rows_cast_into_every_kind(shim, from_kind, dims):
    """f32 / f64 rows of the edge tables, and the i8 and b1 edge rows, into every kind"""
    wide = from_kind == "f64"
    tables = {"edges": edges.edge_rows(24, dims), "i8 edges": _i8_rows(dims, wide),
              "b1 edges": _b1_rows(dims, wide)}
    if wide:  # doubles just off the edge values (narrowed to f32 before a half cast), and ones beyond the f32 range
        t = _as_kind(tables["edges"], "f64")
        t[:, ::3] *= 1 + 2.0 ** -40
        t[:, 1::5] = 1e39
        tables["f64 edges"] = t
    for what, rows in tables.items():
        src = _as_kind(rows, from_kind)
        for to_kind in KINDS:
            _compare(shim, src, from_kind, to_kind, dims, what)


@live
@pytest.mark.parametrize("from_kind", ["f16", "bf16", "i8", "b1"])
@pytest.mark.parametrize("dims", [1, 9, 97])
def test_stored_rows_cast_into_every_kind(shim, from_kind, dims):
    """What `get` casts out of a half, i8 or b1 index: raw rows that include every f16 / bf16 exponent-31 and NaN
    pattern class, i8 -128 and packed bits, into every kind"""
    rng = np.random.default_rng(dims)
    nbytes = cr.bindings.bytes_per_vector(dims, from_kind)
    raw = rng.integers(0, 256, size=(64, nbytes), dtype=np.uint8)
    if from_kind in ("f16", "bf16"):
        words = raw.view(np.uint16)
        exp_mask = 0x7C00 if from_kind == "f16" else 0x7F80
        words[::4] |= exp_mask  # a quarter of the rows: exponent all ones (inf / NaN / the finite 2^16 band)
        words[1::4] &= ~np.uint16(exp_mask)  # a quarter: zeros and subnormals
    for to_kind in KINDS:
        _compare(shim, raw, from_kind, to_kind, dims, "raw rows")
