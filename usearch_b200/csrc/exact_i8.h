/*
 *  exact_i8.h — the three i8 metrics as functions of the integer triple (ab, a2, b2), shared by the tensor-core scans
 *  (exact_imma.cu: mma.sync; exact_wgmma.cu: wgmma), and the wgmma scan's conservative filter on ab:
 *      ip    1 - float(ab)                               index_plugins.hpp:1914-1916 over simsimd_dot_i8
 *      l2sq  float(a2 + b2 - 2 ab)  == sum (a-b)^2       spatial.h l2sq_i8 (i32 accumulation)
 *      cos   normalise(float(ab), float(a2), float(b2))  spatial.h:1904-1972 -> the f32 normaliser
 *  Plain C++ on the host (g++ -ffp-contract=off), the same IEEE operations through intrinsics on the device:
 *  tests/native/test_exact_i8_filter.cpp holds the filter sound against these distances and the distances equal to the
 *  pinned reference metrics (the metrics_pinned.h of the test oracle).
 *
 *  The filter (i8_filter_t). Once a row's k-best list is full with worst entry w, a column can only enter with d <= w
 *  (a tie enters when its slot is larger). The filter must pass every such column; it may pass more.
 *
 *  ip: d = fl(1 - F), F = fl(ab). |ab| <= 128^2 d fits 2^27 for d <= 8192, where |F - ab| <= 4 (ulp 8 below 2^27).
 *      d <= w  =>  1 - F <= w + 2^-24 |w| (the subtraction's rounding, at most half an ulp of its result)
 *              =>  ab >= (1 - w) - 2^-24 |w| - 4. t = rd(1 - w) <= 1 - w, lowered by 4.8e-7 |t| (> 2^-24 |w| + the
 *      rounding of that fma, since |w| <= |t| + 1 and integers below 2^24 are exact), floored, minus 4 units.
 *  l2sq: d = fl(S), S = a2 + b2 - 2 ab exact in i32. d <= w  =>  S <= w + 2^-24 w  =>  S <= ru(w + 4.8e-7 w) + 4, i.e.
 *      2 ab - b2 >= a2 - ru(w + 4.8e-7 w) - 4.
 *  cos: d = max(fl(1 - p), 0) with p = fl(fl(A qr) vr) (fl(fl(A vr) qr) for SWAP), A = fl(ab), qr / vr the reciprocal
 *      norms (i8_rnorm; in [2^-16, 1] for non-zero rows, so no product underflows). The filter tests x = fl(A vr) >= thr.
 *      (1) d <= w  =>  fl(1 - p) <= w  =>  1 - p <= w + 2^-23, u = 2^-24: the subtraction errs by at most half an ulp of
 *          its result, which is below 4 (w <= 2 + a few ulps); for d in (0.5, 1) the error alone is up to 2^-25. So
 *          p >= L = (1 - w) - 2^-23. This ABSOLUTE term is what a relative slack on (1 - w) misses as w -> 1.
 *      (2) x = (p / qr)(1 + theta), |theta| <= 4u: three roundings (two of p, one of x) between them, in either order.
 *          So x >= L / qr - 4u |L| / qr.
 *      (3) thr = fl(fl(fl(1 - w) - 2^-22) / qr) lowered by 1e-5 of itself (and 1e-30, so that thr < 0 whenever w >= 1).
 *          fl(1 - w) - 2^-22 = T + E with T = (1 - w) - 2^-22 = L - 2^-23 and |E| <= 2u (|1 - w| + 2^-22); the division
 *          adds u. So qr thr <= T + 3u |T| + 2^-21 u - 0.9e-5 |T|, and qr x - qr thr >= 2^-23 - 4u |L| - 3u |T| + 0.9e-5 |T|
 *          - 2^-21 u > 0, because 4u |L| + 3u |T| <= 7u |T| + 2^-21 u and 7u < 0.9e-5.
 *      The special rules: ab == 0 gives d = 1, which needs w >= 1, where fl(1 - w) <= 0 and thr < 0 <= x; a zero row or
 *      query has a reciprocal norm of +inf, so x = 0 * inf is NaN (passes) or thr = (<= 0) / inf - 1e-30 < 0 = x.
 */
#pragma once
#include <cmath>
#include <cstdint>

#include "device_index.h"

#if defined(__CUDACC__)
#define I8_HD __host__ __device__ __forceinline__
#else
#define I8_HD inline
#endif

namespace usearch_b200 {

/* ---- round-to-nearest / directed f32 operations: device intrinsics, and their host equivalents ---- */
I8_HD float i8_int2float_rn(int x) {
#if defined(__CUDA_ARCH__)
    return __int2float_rn(x);
#else
    return (float)x;
#endif
}
I8_HD float i8_fsub_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
I8_HD float i8_fmul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
I8_HD float i8_fdiv_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
/* c + a * b and c - a * b in one rounding: nvcc contracts the device expressions into an fma (--fmad=true, the default),
 * and folds them where the operands are constants; the host states the fma */
I8_HD float i8_add_mul(float c, float a, float b) {
#if defined(__CUDA_ARCH__)
    return c + a * b;
#else
    return std::fmaf(a, b, c);
#endif
}
I8_HD float i8_sub_mul(float c, float a, float b) {
#if defined(__CUDA_ARCH__)
    return c - a * b;
#else
    return std::fmaf(-a, b, c);
#endif
}
/* a - b rounded toward -inf: on the host the nearest difference, one step down when the exact error (two-sum) is negative */
I8_HD float i8_fsub_rd(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rd(a, b);
#else
    float const s = a - b, bb = s - a, err = (a - (s - bb)) + (-b - bb);
    return err < 0.0f ? std::nextafterf(s, -INFINITY) : s;
#endif
}
I8_HD int i8_float2int_rd(float x) {
#if defined(__CUDA_ARCH__)
    return __float2int_rd(x);
#else
    return (int)std::floor(x);
#endif
}
I8_HD int i8_float2int_ru(float x) {
#if defined(__CUDA_ARCH__)
    return __float2int_ru(x);
#else
    return (int)std::ceil(x);
#endif
}
/* 1 / sqrt(x), both correctly rounded: the reciprocal root of cos_normalize_f32 */
I8_HD float i8_rnorm(int x2) {
#if defined(__CUDA_ARCH__)
    return __frcp_rn(__fsqrt_rn(__int2float_rn(x2)));
#else
    return 1.0f / std::sqrt((float)x2);
#endif
}

/* cos: the two reciprocal roots of cos_normalize_f32 are per-operand (qr, vr), computed once per row / column of
 * the tile; the per-pair remainder is the same two multiplies and the subtraction, in the operand order of the
 * call (`metric(query, stored)` for an index, `metric(stored, query)` for exact_search_t) */
template <uint32_t METRIC, bool SWAP>
I8_HD float i8_distance(int ab, int qa2, int vb2, float qr, float vr) {
    if constexpr (METRIC == METRIC_IP) return i8_fsub_rn(1.0f, i8_int2float_rn(ab));
    else if constexpr (METRIC == METRIC_L2SQ) return i8_int2float_rn(qa2 + vb2 - 2 * ab);
    else {
        if (qa2 == 0 && vb2 == 0) return 0.0f;
        if (ab == 0) return 1.0f;
        float const abf = i8_int2float_rn(ab);
        float const r = SWAP ? i8_fsub_rn(1.0f, i8_fmul_rn(i8_fmul_rn(abf, vr), qr)) : i8_fsub_rn(1.0f, i8_fmul_rn(i8_fmul_rn(abf, qr), vr));
        return r > 0 ? r : 0.f;
    }
}

/* the filter of one query row (derivation above): thresholds from the list's worst, then one test per column */
template <uint32_t METRIC> struct i8_filter_t {
    int thr_i; /* ip / l2sq; while the list is not full everything passes */
    float thr_f; /* cos */

    /* qa2 / qr: the row's squared norm and reciprocal norm */
    I8_HD void set_thresholds(uint32_t size, uint32_t k, float worst, int qa2, float qr) {
        thr_i = INT32_MIN;
        thr_f = -INFINITY;
        if (size < k) return;
        if constexpr (METRIC == METRIC_IP) { /* d = 1 - float(ab), non-increasing in ab */
            float const t = i8_fsub_rd(1.0f, worst);
            thr_i = i8_float2int_rd(i8_sub_mul(t, fabsf(t), 4.8e-7f)) - 4;
        } else if constexpr (METRIC == METRIC_L2SQ) /* d = float(a2 + b2 - 2ab) <= worst  <=>  2ab - b2 >= a2 - floor(worst) (- slack) */
            thr_i = qa2 - (i8_float2int_ru(i8_add_mul(worst, fabsf(worst), 4.8e-7f)) + 4);
        else { /* d = 1 - ab*qr*vr <= worst  =>  ab*vr >= (1 - worst - 2^-22) / qr, lowered by a relative 1e-5 */
            float const base = i8_fdiv_rn(i8_fsub_rn(i8_fsub_rn(1.0f, worst), 0x1p-22f), qr);
            thr_f = i8_fsub_rn(i8_sub_mul(base, fabsf(base), 1e-5f), 1e-30f);
        }
    }

    /* may the column with dot product ab (squared norm vb2, reciprocal norm vr) enter the list? */
    I8_HD bool maybe(int ab, int vb2, float vr) const {
        if constexpr (METRIC == METRIC_IP) return ab >= thr_i;
        else if constexpr (METRIC == METRIC_L2SQ) return 2 * ab - vb2 >= thr_i;
        else return !(i8_fmul_rn(i8_int2float_rn(ab), vr) < thr_f); /* a NaN (zero vector) passes */
    }
};

} // namespace usearch_b200
