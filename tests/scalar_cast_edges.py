"""Edge values of the scalar casts (usearch_b200/csrc/scalar_casts.h), shared by the CPU and GPU cast tests.

Every table is a set of f32 bit patterns (or f64 values) where an IEEE cast and the reference's differ, or where a cast is
easy to get wrong: half-precision ties, the top of the f16 range, inf and NaN payloads, the f16 subnormal range, bf16 ties
and signed zeros."""
from __future__ import annotations

import numpy as np


def _f32(bits) -> np.ndarray:
    return np.asarray(bits, dtype=np.uint32).view(np.float32)


def f16_ties() -> np.ndarray:
    """f32 values exactly halfway between two f16 values: below-even and below-odd, both signs, at every f16 exponent,
    in the subnormal range, and at the top of the range (65520 rounds up to the f16 exponent 31)."""
    out = []
    for e in range(-14, 16):
        for m in (0, 1, 2, 3, 511, 1022, 1023):  # ten-bit f16 mantissa below the tie
            out.append((1 + (m + 0.5) / 1024) * 2.0 ** e)
    for m in (0, 1, 2, 3, 100, 101, 1022, 1023):  # subnormal ties: (m + 1/2) 2^-24
        out.append((m + 0.5) * 2.0 ** -24)
    out = np.asarray(out, dtype=np.float64)
    return np.concatenate([out, -out]).astype(np.float32)


def f16_overflow() -> np.ndarray:
    v = np.array([65504, 65505, 65519, 65519.99, 65520, 65535, 65536, 70000, 131056, 131071, 131072, 2.0 ** 17 + 1, 1e5,
                  5e5, 1e6, 3.0e38], dtype=np.float32)
    return np.concatenate([v, -v])


def specials() -> np.ndarray:
    """inf, quiet and signalling NaNs with small and large payloads (the large ones carry into the sign bit or out of
    the word when half an ulp is added), and signed zeros"""
    return _f32([0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FA00000, 0x7F801000,
                 0x7FBFFFFF, 0x7FFFEFFF, 0x7FFFF000, 0x7FFFFFFF, 0xFFFFF000, 0xFFFFFFFF, 0x7FFF8000, 0xFFFF8000,
                 0x00000000, 0x80000000])


def f16_subnormals() -> np.ndarray:
    """2^-26 .. 2^-14: the flush threshold, the first subnormals and the boundary with the normal range"""
    v = [2.0 ** -27, 2.0 ** -26, 2.0 ** -26 * 1.5, 2.0 ** -25, np.nextafter(2.0 ** -25, 0), np.nextafter(2.0 ** -25, 1),
         2.0 ** -24, 1.5 * 2.0 ** -24, 2.0 ** -23, 3 * 2.0 ** -24, 2.0 ** -15, 2.0 ** -14 - 2.0 ** -25,
         np.nextafter(np.float32(2.0 ** -14), np.float32(0)), 2.0 ** -14, 1e-45, 1e-40]
    v = np.asarray(v, dtype=np.float64)
    grid = 2.0 ** np.linspace(-26, -14, 61)
    v = np.concatenate([v, grid]).astype(np.float32)
    return np.concatenate([v, -v])


def bf16_ties() -> np.ndarray:
    """f32 patterns with exactly 0x8000 in the low half: below-even and below-odd, the largest finite bf16's tie (rounds to
    inf) and a subnormal tie"""
    b = np.array([0x3F808000, 0x3F818000, 0x40490000 | 0x8000, 0x42F68000, 0x7F7F8000, 0x7F7E8000, 0x00008000, 0x00018000,
                  0x33808000], dtype=np.uint32)
    return np.concatenate([_f32(b), _f32(b | 0x80000000)])


def edge_table(finite_only: bool = False) -> np.ndarray:
    t = np.concatenate([f16_ties(), f16_overflow(), specials(), f16_subnormals(), bf16_ties()])
    return t[np.isfinite(t)] if finite_only else t


def edge_rows(n: int, dims: int, seed: int = 0, finite_only: bool = False) -> np.ndarray:
    """n x dims f32 rows: every element an edge value, the table cycled with a different offset and order per row so that
    every value meets every column position across the rows"""
    t = edge_table(finite_only)
    rng = np.random.default_rng(seed)
    idx = (np.arange(dims)[None, :] * 7 + np.arange(n)[:, None] * 13) % t.size
    rows = t[idx]
    rng.shuffle(rows, axis=1)
    return np.ascontiguousarray(rows)


def tie_rows(n: int, dims: int, kind: str, seed: int = 0) -> np.ndarray:
    """finite f32 rows whose every element is an exact tie of `kind` (f16 or bf16), the scale of a row random: the casts
    of such queries differ from IEEE rounding in every element whose lower neighbour is even"""
    rng = np.random.default_rng(seed)
    sign = rng.choice([-1.0, 1.0], size=(n, dims))
    if kind == "f16":
        m = rng.integers(0, 1024, size=(n, dims))
        e = rng.integers(-6, 4, size=(n, dims))
        return ((1 + (m + 0.5) / 1024) * 2.0 ** e * sign).astype(np.float32)
    hi = rng.integers(0x3C00, 0x4200, size=(n, dims)).astype(np.uint32)  # bf16 magnitudes ~2^-7 .. 2^5
    return (_f32((hi << 16) | 0x8000).astype(np.float64) * sign).astype(np.float32)
