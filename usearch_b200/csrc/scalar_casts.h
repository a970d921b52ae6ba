/*
 *  scalar_casts.h — the reference's scalar conversions (cast_gt, index_plugins.hpp:1105-1224), host and device.
 *
 *  The reference is the test oracle's build: USEARCH_USE_SIMSIMD=1 with USEARCH_USE_FP16LIB=0, so f16 and bf16 go
 *  through SimSIMD's portable bit-twiddling conversions, and those do not round the IEEE way. What they do, pinned over
 *  every input by tests/native/test_scalar_casts.cpp:
 *
 *  f32 -> f16   Half an f16 ulp (0x1000) is added to the raw f32 bits, unsigned and modulo 2^32, and the sum r is read:
 *               ties round away from zero, and the carry may ripple into the exponent, or for a NaN whose top eleven
 *               mantissa bits are set into the sign (0x7FFFFxxx -> 0x8000) or out of the word (0xFFFFFxxx -> 0x0000).
 *               With E the biased f32 exponent of r and m its mantissa bits:
 *                 E >= 144   sign | 0x7FFF: every |x| >= 2^17 - 2^4, inf and (most) NaN become a NaN pattern
 *                 E == 143   sign | 0x7C00 | m >> 13: 65520 <= |x| < 2^17 - 2^4 gives inf or a NaN (70000 -> 0x7C46)
 *                 113..142   sign | (E - 112) << 10 | m >> 13: the normal range
 *                 102..112   sign | the f16 subnormal: the significand (0x800000 | m) less the 0x1000 added above,
 *                            shifted right by 126 - E with ties away from zero (values from 2^-26 up)
 *                 <= 101     sign | 0: a signed zero
 *  f32 -> bf16  Half a bf16 ulp (0x8000) added to the raw bits, modulo 2^32, then the top 16 bits: ties away from zero,
 *               finite values that round past the largest bf16 become inf, and a NaN is not quieted, so a signalling
 *               NaN with a small payload becomes inf (0x7F800001 -> 0x7F80); the same carries as f16.
 *  f16 -> f32   Exact for biased exponents 0..30, subnormals included. Exponent 31 is not special: 0x7C00 is 65536 and
 *               every "NaN" the finite 2^16 (1 + m / 1024).
 *  bf16 -> f32  The 16 bits shifted into the top of the word (exact).
 *
 *  A reference built without AVX-512 and without these two defines takes fp16lib, which rounds the IEEE way; DESIGN.md
 *  records which one the project matches. The distance kernels decode stored halves with the hardware conversion
 *  (metrics.cuh), like the reference's SIMD kernels do; only the casts between kinds use these functions.
 *
 *  The second half is the whole cast_gt matrix for one row on the host (`get`, and tests): the device runs the same element
 *  functions in builder.cu's cast kernels. Plain C++ (no CUDA) when compiled by a host compiler.
 */
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "device_index.h"
#include "f64_casts.h"

#if defined(__CUDACC__)
#define SC_HD __host__ __device__ __forceinline__
#else
#define SC_HD inline
#endif

namespace usearch_b200 {

SC_HD uint32_t sc_f32_bits(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t x;
    std::memcpy(&x, &f, 4);
    return x;
#endif
}

SC_HD float sc_bits_f32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(x);
#else
    float f;
    std::memcpy(&f, &x, 4);
    return f;
#endif
}

SC_HD uint16_t f32_to_f16_bits(float f) {
    uint32_t const r = sc_f32_bits(f) + 0x1000u;
    uint32_t const sign = (r >> 16) & 0x8000u, e = (r >> 23) & 0xFFu, m = r & 0x7FFFFFu;
    if (e >= 144) return (uint16_t)(sign | 0x7FFFu);
    if (e >= 113) return (uint16_t)(sign | ((e - 112) << 10) | (m >> 13));
    if (e >= 102) {
        uint32_t const significand = (0x800000u | m) - 0x1000u, shift = 126 - e;
        return (uint16_t)(sign | ((significand + (1u << (shift - 1))) >> shift));
    }
    return (uint16_t)sign;
}

SC_HD uint16_t f32_to_bf16_bits(float f) { return (uint16_t)((sc_f32_bits(f) + 0x8000u) >> 16); }

SC_HD float f16_bits_to_f32(uint16_t h) {
    uint32_t const sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    if (e) return sc_bits_f32(sign | ((e + 112) << 23) | (m << 13));
    float const magnitude = (float)m * 0x1p-24f; /* subnormal or zero: m 2^-24, exact in f32 */
    return sign ? -magnitude : magnitude;
}

SC_HD float bf16_bits_to_f32(uint16_t h) { return sc_bits_f32((uint32_t)h << 16); }

/* f64 -> f32 as the reference's host build narrows (x86 cvtsd2ss): round to nearest, and a NaN keeps its sign and the top
 * 22 bits of its payload and becomes quiet. The device conversion would return the canonical NaN instead. */
SC_HD float f64_to_f32(double x) {
#if defined(__CUDA_ARCH__)
    if (x != x) {
        uint64_t const b = (uint64_t)__double_as_longlong(x);
        return __uint_as_float(((uint32_t)(b >> 32) & 0x80000000u) | 0x7FC00000u | ((uint32_t)(b >> 29) & 0x3FFFFFu));
    }
    return __double2float_rn(x);
#else
    return (float)x;
#endif
}

/* ---- one row, any kind to any kind, on the host ---------------------------------------------------------------------- */

inline size_t sc_row_bytes(uint32_t kind, size_t dims) {
    switch (kind) {
    case SCALAR_B1: return (dims + 7) / 8;
    case SCALAR_I8: return dims;
    case SCALAR_F16: case SCALAR_BF16: return dims * 2;
    case SCALAR_F32: return dims * 4;
    case SCALAR_F64: return dims * 8;
    default: return 0;
    }
}

/* cast_gt<from, to>::try_ for one row of `dims` elements; returns an error or nullptr. A b1 target is written whole, its
 * padding bits zero. */
inline char const* cast_row_host(uint32_t from, uint32_t to, size_t dims, uint8_t const* src, uint8_t* dst) {
    size_t const to_bytes = sc_row_bytes(to, dims);
    if (!to_bytes || !sc_row_bytes(from, dims)) return dims ? "Unsupported scalar kind" : nullptr;
    if (from == to) { std::memcpy(dst, src, to_bytes); return nullptr; }
    auto store_f32 = [&](size_t j, float v) { /* a float value into a float target: to_scalar_at(float) */
        uint16_t h;
        switch (to) {
        case SCALAR_F32: std::memcpy(dst + 4 * j, &v, 4); break;
        case SCALAR_F64: { double w = v; std::memcpy(dst + 8 * j, &w, 8); break; }
        case SCALAR_F16: h = f32_to_f16_bits(v); std::memcpy(dst + 2 * j, &h, 2); break;
        case SCALAR_BF16: h = f32_to_bf16_bits(v); std::memcpy(dst + 2 * j, &h, 2); break;
        default: break;
        }
    };
    if (from == SCALAR_B1) { /* cast_from_b1x8_gt: a set bit is to_scalar_at(true) -- 1, also for i8 */
        for (size_t j = 0; j < dims; ++j) {
            bool const bit = (src[j >> 3] & (128u >> (j & 7u))) != 0;
            if (to == SCALAR_I8) reinterpret_cast<int8_t*>(dst)[j] = bit ? 1 : 0;
            else store_f32(j, bit ? 1.f : 0.f);
        }
        return nullptr;
    }
    if (from == SCALAR_I8 && to != SCALAR_B1) { /* cast_from_i8_gt: x / 127.f, a double division for f64 */
        int8_t const* x = reinterpret_cast<int8_t const*>(src);
        for (size_t j = 0; j < dims; ++j) {
            if (to == SCALAR_F64) { double w = (double)x[j] / 127.0; std::memcpy(dst + 8 * j, &w, 8); }
            else store_f32(j, (float)x[j] / 127.f);
        }
        return nullptr;
    }
    /* every other source as the value cast_gt reads: an f32 (the halves decoded), the f64 as stored, i8 (into b1 only)
     * as the integer -- its sign is all b1 needs */
    auto load = [&](size_t j) -> double {
        uint16_t h;
        switch (from) {
        case SCALAR_F64: { double v; std::memcpy(&v, src + 8 * j, 8); return v; }
        case SCALAR_F32: { float v; std::memcpy(&v, src + 4 * j, 4); return v; }
        case SCALAR_F16: std::memcpy(&h, src + 2 * j, 2); return f16_bits_to_f32(h);
        case SCALAR_BF16: std::memcpy(&h, src + 2 * j, 2); return bf16_bits_to_f32(h);
        default: return reinterpret_cast<int8_t const*>(src)[j];
        }
    };
    if (from != SCALAR_F64 && from != SCALAR_F32 && from != SCALAR_F16 && from != SCALAR_BF16 && from != SCALAR_I8)
        return "Unsupported scalar kind";
    if (to == SCALAR_I8 || to == SCALAR_B1 || to == SCALAR_F64) {
        std::vector<double> x(dims);
        for (size_t j = 0; j < dims; ++j) x[j] = load(j);
        if (to == SCALAR_I8) cast_f64_to_i8(x.data(), dims, reinterpret_cast<int8_t*>(dst));
        else if (to == SCALAR_B1) cast_f64_to_b1(x.data(), dims, dst);
        else std::memcpy(dst, x.data(), dims * 8);
        return nullptr;
    }
    /* into f32 / f16 / bf16 the value stays an f32 (a round trip through f64 would quiet a signalling NaN); an f64
     * narrows to f32 first, as f16_bits_t(double) does */
    for (size_t j = 0; j < dims; ++j) {
        uint16_t h;
        float v;
        switch (from) {
        case SCALAR_F64: v = f64_to_f32(load(j)); break;
        case SCALAR_F32: std::memcpy(&v, src + 4 * j, 4); break;
        case SCALAR_F16: std::memcpy(&h, src + 2 * j, 2); v = f16_bits_to_f32(h); break;
        default: std::memcpy(&h, src + 2 * j, 2); v = bf16_bits_to_f32(h); break;
        }
        store_f32(j, v);
    }
    return nullptr;
}

} // namespace usearch_b200
