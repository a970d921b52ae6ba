/*
 *  f64_casts.h — cast_gt<f64, i8> and cast_gt<f64, b1x8> (index_plugins.hpp:1139-1191) on the host, for `get` out of an
 *  f64 index. Both read the doubles themselves: the i8 magnitude is the sequential f64 sum of squares of the f64 values,
 *  and a double below the f32 range is still > 0 for b1. Plain C++ (no CUDA), so the tests compile it on its own.
 */
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>

namespace usearch_b200 {

inline void cast_f64_to_i8(double const* x, size_t dims, int8_t* out) {
    double magnitude = 0;
    for (size_t j = 0; j < dims; ++j) magnitude += x[j] * x[j];
    magnitude = std::sqrt(magnitude);
    for (size_t j = 0; j < dims; ++j) {
        double v = x[j] * 127.0 / magnitude;
        v = v > 127.0 ? 127.0 : (v < -127.0 ? -127.0 : v); /* NaN (zero vector) passes through, like usearch::clamp */
        out[j] = (int8_t)v;
    }
}

inline void cast_f64_to_b1(double const* x, size_t dims, uint8_t* out) {
    std::memset(out, 0, (dims + 7) / 8);
    for (size_t j = 0; j < dims; ++j)
        if (x[j] > 0) out[j / 8] |= (uint8_t)(128 >> (j & 7));
}

} // namespace usearch_b200
