/*
 *  tests/native/f64_pinned.h — the f64 distances an AVX-512 host computes, restated in portable C for the tests.
 *
 *  simsimd_l2sq_f64_skylake, simsimd_dot_f64_skylake and simsimd_cos_f64_skylake (spatial.h:1622-1674, dot.h:1320-1341)
 *  keep 8 f64 accumulators: element i goes to accumulator i mod 8 through one fma. _mm512_reduce_add_pd is, in GCC's
 *  avx512fintrin.h, ((v0+v4)+(v2+v6)) + ((v1+v5)+(v3+v7)). The masked tail adds fma(0, 0, acc) = acc to the padded
 *  accumulators, so it changes nothing. Each result is then cast to f32 (index_plugins.hpp:1914-1916); ip subtracts
 *  from 1 in f32 after that cast. The cosine normalisation is the IEEE form of _simsimd_cos_normalize_f64_skylake
 *  (spatial.h:1544-1585), whose rsqrt14_pd + Newton step differs from it by at most 1 ULP(f32) after the cast.
 *
 *  Compile with -ffp-contract=off and without -ffast-math, so that only the explicit fma calls fuse.
 */
#ifndef USEARCH_B200_TESTS_F64_PINNED_H
#define USEARCH_B200_TESTS_F64_PINNED_H

#include <math.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

static inline double pinned_reduce8_f64_(double const v[8]) {
    return ((v[0] + v[4]) + (v[2] + v[6])) + ((v[1] + v[5]) + (v[3] + v[7]));
}

static inline float pinned_l2sq_f64(double const* a, double const* b, size_t n) {
    double acc[8] = {0};
    for (size_t i = 0; i < n; ++i) {
        double x = a[i] - b[i];
        acc[i & 7] = fma(x, x, acc[i & 7]);
    }
    return (float)pinned_reduce8_f64_(acc);
}

static inline float pinned_ip_f64(double const* a, double const* b, size_t n) {
    double acc[8] = {0};
    for (size_t i = 0; i < n; ++i) acc[i & 7] = fma(a[i], b[i], acc[i & 7]);
    return 1.0f - (float)pinned_reduce8_f64_(acc);
}

static inline float pinned_cos_f64(double const* a, double const* b, size_t n) {
    double ab[8] = {0}, a2[8] = {0}, b2[8] = {0};
    for (size_t i = 0; i < n; ++i) {
        ab[i & 7] = fma(a[i], b[i], ab[i & 7]);
        a2[i & 7] = fma(a[i], a[i], a2[i & 7]);
        b2[i & 7] = fma(b[i], b[i], b2[i & 7]);
    }
    double sab = pinned_reduce8_f64_(ab), sa2 = pinned_reduce8_f64_(a2), sb2 = pinned_reduce8_f64_(b2);
    if (sa2 == 0 && sb2 == 0) return 0.f;
    if (sab == 0) return 1.f;
    double r = 1.0 - (sab * (1.0 / sqrt(sa2))) * (1.0 / sqrt(sb2));
    return r > 0 ? (float)r : 0.f;
}

#ifdef __cplusplus
}
#endif
#endif
