/*
 *  metrics.cuh — SimSIMD's distance kernels re-expressed for a sub-warp of LPV lanes walking one
 *  stored vector with 128-bit loads (metric_punned_t, index_plugins.hpp:1678-2015, resolves the
 *  builtin metrics to these SimSIMD kernels at index_plugins.hpp:1863-1916).
 *
 *  Parity contract: every floating-point kernel reproduces the SUMMATION ORDER of the SimSIMD
 *  kernel it replaces, using explicit round-to-nearest intrinsics so that nvcc neither contracts
 *  nor re-associates anything. Integer kernels are exact in any order.
 *
 *    f32  : 16 virtual accumulators, element i -> accumulator i mod 16, one fma per element
 *           (spatial.h:1520-1542 l2sq_f32_skylake, :1587-1615 cos_f32_skylake,
 *           dot.h:1297-1318 dot_f32_skylake). A 16-byte chunk j holds elements 4j..4j+3, i.e.
 *           accumulators 4(j mod 4)..+3, so exactly FOUR lanes share a vector: lane `sub` owns
 *           chunks sub, sub+4, ... and accumulators 4*sub..4*sub+3. The horizontal reduce
 *           (dot.h:1279-1284) r_i = (v[i]+v[i+8]) + (v[i+4]+v[i+12]); (r0+r1)+(r2+r3) becomes two
 *           xor-shuffles (2 then 1) and three adds.
 *    cos  : normalisation is the IEEE restatement 1 - ab*(1/sqrt(a2))*(1/sqrt(b2)) in f64 with
 *           SimSIMD's zero rules and clamp (spatial.h:1544-1585 uses rsqrt14+Newton, which differs
 *           by <= 1 ULP(f32) and cannot be reproduced off-x86; see oracle/metrics_pinned.h).
 *    ip   : 1.0f - dot in f32 (index_plugins.hpp:1914-1916: the f64 result is cast to f32 first).
 *    f64  : 8 accumulators, element i -> accumulator i mod 8; lane `sub` owns accumulators 2 sub, 2 sub + 1
 *           (spatial.h:1622-1674, dot.h:1320-1341), see the f64 section below.
 *    i8   : exact i32 sums via dp4a (dot.h:1749-1775, spatial.h:1880-1972).
 *    b1   : exact popcounts (binary.h:92-105, :271-347).
 */
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "device_index.h"
#include "prefilter_bound.h"

namespace usearch_b200 {

__device__ __forceinline__ uint4 ldg_stream(uint4 const* p) {
    /* vectors are touched once per query: keep them out of L1 */
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

template <int LPV> __device__ __forceinline__ int reduce_add_i32(int v) {
#pragma unroll
    for (int o = LPV / 2; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

/* ---- f32 -------------------------------------------------------------------------------- */

__device__ __forceinline__ float reduce16_f32(float const v[4]) {
    /* lanes sub=0..3 of a 4-lane group hold accumulators 4*sub..4*sub+3 */
    float u[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float t = __fadd_rn(v[c], __shfl_xor_sync(0xffffffffu, v[c], 2)); /* v[i]+v[i+8] | v[i+4]+v[i+12] */
        u[c] = __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, 1));
    }
    return __fadd_rn(__fadd_rn(u[0], u[1]), __fadd_rn(u[2], u[3]));
}

__device__ __forceinline__ float cos_normalize_f64(float ab_f, float a2_f, float b2_f) {
    double ab = (double)ab_f, a2 = (double)a2_f, b2 = (double)b2_f;
    if (a2 == 0 && b2 == 0) return 0.f;
    if (ab == 0) return 1.f;
    double ra = __drcp_rn(__dsqrt_rn(a2));
    double rb = __drcp_rn(__dsqrt_rn(b2));
    double r = __dsub_rn(1.0, __dmul_rn(__dmul_rn(ab, ra), rb));
    return r > 0 ? __double2float_rn(r) : 0.f;
}

__device__ __forceinline__ float cos_normalize_f32(float ab, float a2, float b2) {
    if (a2 == 0.0f && b2 == 0.0f) return 0.0f;
    if (ab == 0.0f) return 1.0f;
    float ra = __frcp_rn(__fsqrt_rn(a2));
    float rb = __frcp_rn(__fsqrt_rn(b2));
    float r = __fsub_rn(1.0f, __fmul_rn(__fmul_rn(ab, ra), rb));
    return r > 0 ? r : 0.f;
}

struct l2sq_f32_t {
    static constexpr int LPV = 4;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { float v[4]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.v[0] = a.v[1] = a.v[2] = a.v[3] = 0.f; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        float x;
        x = __fsub_rn(__uint_as_float(q.x), __uint_as_float(b.x)); a.v[0] = __fmaf_rn(x, x, a.v[0]);
        x = __fsub_rn(__uint_as_float(q.y), __uint_as_float(b.y)); a.v[1] = __fmaf_rn(x, x, a.v[1]);
        x = __fsub_rn(__uint_as_float(q.z), __uint_as_float(b.z)); a.v[2] = __fmaf_rn(x, x, a.v[2]);
        x = __fsub_rn(__uint_as_float(q.w), __uint_as_float(b.w)); a.v[3] = __fmaf_rn(x, x, a.v[3]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) { return reduce16_f32(a.v); }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

struct ip_f32_t {
    static constexpr int LPV = 4;
    static constexpr bool NORMS = false;
    /* layer-0 prefilter through the int8 shadow (search_kernel.cu, measure_prefiltered; bound: prefilter_bound.h) */
    static constexpr bool PREFILTER = true;
    static __device__ __forceinline__ double pf_lower(float dot, pf_record_t r, pf_query_bound_t const& q) {
        return pf_ip_lower_q(dot, r.s, r.rho, r.bnorm, q);
    }
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { float v[4]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.v[0] = a.v[1] = a.v[2] = a.v[3] = 0.f; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.v[0] = __fmaf_rn(__uint_as_float(q.x), __uint_as_float(b.x), a.v[0]);
        a.v[1] = __fmaf_rn(__uint_as_float(q.y), __uint_as_float(b.y), a.v[1]);
        a.v[2] = __fmaf_rn(__uint_as_float(q.z), __uint_as_float(b.z), a.v[2]);
        a.v[3] = __fmaf_rn(__uint_as_float(q.w), __uint_as_float(b.w), a.v[3]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        return __fsub_rn(1.0f, reduce16_f32(a.v));
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

/*  cos f32 reads ||b||^2 from `device_index_t::norms`, computed once at freeze time by the very same
 *  16-accumulator fma chain (norms_f32_kernel), so the value is bit-identical to what
 *  simsimd_cos_f32_skylake accumulates in its b2 register (spatial.h:1587-1615) while halving the
 *  FMAs of the hot loop. The f64 normalisation is deferred: `finish` returns the raw dot product and
 *  `finalize` is run once per hop, one candidate per lane. */
struct cos_f32_t {
    static constexpr int LPV = 4;
    static constexpr bool NORMS = true;
    static constexpr bool PREFILTER = true; /* see ip_f32_t */
    static __device__ __forceinline__ double pf_lower(float dot, pf_record_t r, pf_query_bound_t const& q) {
        return pf_cos_lower_q(dot, r.s, r.rho, r.b2, q);
    }
    struct acc_t { float ab[4]; };
    struct qconst_t { float a2; };
    static __device__ __forceinline__ void init(acc_t& a) { a.ab[0] = a.ab[1] = a.ab[2] = a.ab[3] = 0.f; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.ab[0] = __fmaf_rn(__uint_as_float(q.x), __uint_as_float(b.x), a.ab[0]);
        a.ab[1] = __fmaf_rn(__uint_as_float(q.y), __uint_as_float(b.y), a.ab[1]);
        a.ab[2] = __fmaf_rn(__uint_as_float(q.z), __uint_as_float(b.z), a.ab[2]);
        a.ab[3] = __fmaf_rn(__uint_as_float(q.w), __uint_as_float(b.w), a.ab[3]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) { return reduce16_f32(a.ab); }
    static __device__ __forceinline__ float finalize(float ab, qconst_t qc, float b2) { return cos_normalize_f64(ab, qc.a2, b2); }
    /* metric(stored, query) instead of metric(query, stored): exact_search_t calls it that way (index_plugins.hpp:2112) */
    static __device__ __forceinline__ float finalize_sw(float ab, qconst_t qc, float b2) { return cos_normalize_f64(ab, b2, qc.a2); }
    /* the two reciprocal roots of cos_normalize_f64 depend on one operand each: a dense scan computes them once per
     * query / per stored vector and finishes every pair with two multiplies — same operations, same bits */
    using rn_t = double;
    static __device__ __forceinline__ rn_t rnorm(float x2) { return __drcp_rn(__dsqrt_rn((double)x2)); }
    static __device__ __forceinline__ float finalize_rn(float ab, float first2, float second2, rn_t rfirst, rn_t rsecond) {
        if (first2 == 0.f && second2 == 0.f) return 0.f;
        if (ab == 0.f) return 1.f;
        double r = __dsub_rn(1.0, __dmul_rn(__dmul_rn((double)ab, rfirst), rsecond));
        return r > 0 ? __double2float_rn(r) : 0.f;
    }
    /* dot(v, v) in the 16-accumulator order; every 4-lane group computes the same value */
    static __device__ __forceinline__ float self_dot(uint4 const* v4, uint32_t chunks16, int lane) {
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        for (uint32_t j = lane & 3; j < chunks16; j += 4) {
            uint4 q = v4[j];
            v[0] = __fmaf_rn(__uint_as_float(q.x), __uint_as_float(q.x), v[0]);
            v[1] = __fmaf_rn(__uint_as_float(q.y), __uint_as_float(q.y), v[1]);
            v[2] = __fmaf_rn(__uint_as_float(q.z), __uint_as_float(q.z), v[2]);
            v[3] = __fmaf_rn(__uint_as_float(q.w), __uint_as_float(q.w), v[3]);
        }
        return reduce16_f32(v);
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const* q4, uint32_t chunks16, int lane) {
        return {self_dot(q4, chunks16, lane)};
    }
};

/* ---- f64 -------------------------------------------------------------------------------- */
/*
 *  simsimd_{l2sq,dot,cos}_f64_skylake (spatial.h:1622-1674, dot.h:1320-1341): 8 f64 accumulators, element i ->
 *  accumulator i mod 8, one fma per element, then _mm512_reduce_add_pd, which GCC's avx512fintrin.h evaluates as
 *  ((v0+v4)+(v2+v6)) + ((v1+v5)+(v3+v7)). A 16-byte chunk j holds elements 2j and 2j+1, i.e. accumulators
 *  2(j mod 4) and 2(j mod 4)+1, so FOUR lanes share a vector as for f32: lane `sub` owns chunks sub, sub+4, ... and
 *  accumulators 2 sub and 2 sub + 1. The tree is the one of reduce_words_f64 without the widening from f32.
 *  The f64 rows have no stored norm (`norms` is f32): cos accumulates b2 in the loop, like cos_i8_t.
 */
__device__ __forceinline__ double reduce8_lanes_f64(double a, double b) {
    a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 2)); /* lanes 0,2: v0+v4 | lanes 1,3: v2+v6 */
    b = __dadd_rn(b, __shfl_xor_sync(0xffffffffu, b, 2)); /* lanes 0,2: v1+v5 | lanes 1,3: v3+v7 */
    a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 1)); /* (v0+v4)+(v2+v6) */
    b = __dadd_rn(b, __shfl_xor_sync(0xffffffffu, b, 1)); /* (v1+v5)+(v3+v7) */
    return __dadd_rn(a, b);
}

__device__ __forceinline__ double lo_f64(uint4 x) { return __hiloint2double((int)x.y, (int)x.x); }
__device__ __forceinline__ double hi_f64(uint4 x) { return __hiloint2double((int)x.w, (int)x.z); }

/* _simsimd_cos_normalize_f64_skylake (spatial.h:1544-1585) on the f64 sums themselves, restated in IEEE like the f32
 * cosine (rsqrt14_pd + one Newton step differs by <= 1 ULP(f32) after the cast) */
__device__ __forceinline__ float cos_normalize_wide_f64(double ab, double a2, double b2) {
    if (a2 == 0 && b2 == 0) return 0.f;
    if (ab == 0) return 1.f;
    double ra = __drcp_rn(__dsqrt_rn(a2));
    double rb = __drcp_rn(__dsqrt_rn(b2));
    double r = __dsub_rn(1.0, __dmul_rn(__dmul_rn(ab, ra), rb));
    return r > 0 ? __double2float_rn(r) : 0.f;
}

struct l2sq_f64_t {
    static constexpr int LPV = 4;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { double v[2]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.v[0] = a.v[1] = 0.0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        double const x0 = __dsub_rn(lo_f64(q), lo_f64(b)), x1 = __dsub_rn(hi_f64(q), hi_f64(b));
        a.v[0] = __fma_rn(x0, x0, a.v[0]);
        a.v[1] = __fma_rn(x1, x1, a.v[1]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) { return __double2float_rn(reduce8_lanes_f64(a.v[0], a.v[1])); }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

struct ip_f64_t {
    static constexpr int LPV = 4;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { double v[2]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.v[0] = a.v[1] = 0.0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.v[0] = __fma_rn(lo_f64(q), lo_f64(b), a.v[0]);
        a.v[1] = __fma_rn(hi_f64(q), hi_f64(b), a.v[1]);
    }
    /* index_plugins.hpp:1914-1916: the f64 dot is cast to f32 before `1 - x` */
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        return __fsub_rn(1.0f, __double2float_rn(reduce8_lanes_f64(a.v[0], a.v[1])));
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

struct cos_f64_t {
    static constexpr int LPV = 4;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { double ab[2], b2[2]; };
    struct qconst_t { double a2; };
    static __device__ __forceinline__ void init(acc_t& a) { a.ab[0] = a.ab[1] = a.b2[0] = a.b2[1] = 0.0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        double const b0 = lo_f64(b), b1 = hi_f64(b);
        a.ab[0] = __fma_rn(lo_f64(q), b0, a.ab[0]);
        a.ab[1] = __fma_rn(hi_f64(q), b1, a.ab[1]);
        a.b2[0] = __fma_rn(b0, b0, a.b2[0]);
        a.b2[1] = __fma_rn(b1, b1, a.b2[1]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t qc) {
        double const ab = reduce8_lanes_f64(a.ab[0], a.ab[1]), b2 = reduce8_lanes_f64(a.b2[0], a.b2[1]);
        return cos_normalize_wide_f64(ab, qc.a2, b2);
    }
    /* metric(stored, query): exact_search_t's argument order (index_plugins.hpp:2112) */
    static __device__ __forceinline__ float finish_sw(acc_t const& a, qconst_t qc) {
        double const ab = reduce8_lanes_f64(a.ab[0], a.ab[1]), b2 = reduce8_lanes_f64(a.b2[0], a.b2[1]);
        return cos_normalize_wide_f64(ab, b2, qc.a2);
    }
    /* dot(q, q) in the 8-accumulator order; every 4-lane group computes the same value */
    static __device__ __forceinline__ qconst_t prepare(uint4 const* q4, uint32_t chunks16, int lane) {
        double v0 = 0.0, v1 = 0.0;
        for (uint32_t j = lane & 3; j < chunks16; j += 4) {
            uint4 const q = q4[j];
            double const q0 = lo_f64(q), q1 = hi_f64(q);
            v0 = __fma_rn(q0, q0, v0);
            v1 = __fma_rn(q1, q1, v1);
        }
        return {reduce8_lanes_f64(v0, v1)};
    }
};

/* ---- f16 / bf16 --------------------------------------------------------------------------- */
/*
 *  simsimd_{l2sq,dot,cos}_{f16,bf16}_haswell (spatial.h:1098-1200): 8 f32 accumulators, element i ->
 *  accumulator i mod 8, operands widened to f32, one fma per element; horizontal reduce through f64
 *  (dot.h:857-869, :844-855): s_k = (double)v[k] + (double)v[k+4]; (s0 + s2) + (s1 + s3).
 *  A 16-byte chunk holds one element of EVERY accumulator, so the chains cannot be split across lanes:
 *  ONE lane walks a whole vector (LPV = 1, 32 candidate vectors per pass, no cross-lane reduction) and
 *  the query chunk it needs is the same address for all 32 lanes — a shared-memory broadcast.
 *  The native AVX512-FP16 kernel of a Sapphire Rapids host accumulates in fp16 and is not reproducible
 *  (SURVEY.md finding 5); the oracle pins this f32-accumulating order instead.
 */
struct f16_conv_t {
    static __device__ __forceinline__ void widen(uint32_t w, float& lo, float& hi) {
        float2 f = __half22float2(*reinterpret_cast<__half2 const*>(&w));
        lo = f.x;
        hi = f.y;
    }
};
struct bf16_conv_t {
    static __device__ __forceinline__ void widen(uint32_t w, float& lo, float& hi) {
        lo = __uint_as_float(w << 16);
        hi = __uint_as_float(w & 0xFFFF0000u);
    }
};

__device__ __forceinline__ double reduce8_f64(float const v[8]) {
    double s0 = __dadd_rn((double)v[0], (double)v[4]), s1 = __dadd_rn((double)v[1], (double)v[5]);
    double s2 = __dadd_rn((double)v[2], (double)v[6]), s3 = __dadd_rn((double)v[3], (double)v[7]);
    return __dadd_rn(__dadd_rn(s0, s2), __dadd_rn(s1, s3));
}

template <class C> __device__ __forceinline__ void widen8(uint4 x, float (&f)[8]) {
    C::widen(x.x, f[0], f[1]);
    C::widen(x.y, f[2], f[3]);
    C::widen(x.z, f[4], f[5]);
    C::widen(x.w, f[6], f[7]);
}

template <class C> struct l2sq_half_t {
    static constexpr int LPV = 1;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { float v[8]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a.v[k] = 0.f;
    }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        float fb[8], fq[8];
        widen8<C>(b, fb);
        widen8<C>(q, fq);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float x = __fsub_rn(fq[k], fb[k]);
            a.v[k] = __fmaf_rn(x, x, a.v[k]);
        }
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) { return __double2float_rn(reduce8_f64(a.v)); }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

template <class C> struct ip_half_t {
    static constexpr int LPV = 1;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { float v[8]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a.v[k] = 0.f;
    }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        float fb[8], fq[8];
        widen8<C>(b, fb);
        widen8<C>(q, fq);
#pragma unroll
        for (int k = 0; k < 8; ++k) a.v[k] = __fmaf_rn(fq[k], fb[k], a.v[k]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        return __fsub_rn(1.0f, __double2float_rn(reduce8_f64(a.v)));
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

/* cos: ||b||^2 comes from `norms` (same chain, computed at freeze); normalisation in f32 like
 * _simsimd_cos_normalize_f32_haswell (spatial.h:1050-1080), IEEE instead of rsqrt_ps + Newton. */
template <class C> struct cos_half_t {
    static constexpr int LPV = 1;
    static constexpr bool NORMS = true;
    struct acc_t { float v[8]; };
    struct qconst_t { float a2; };
    static __device__ __forceinline__ void init(acc_t& a) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a.v[k] = 0.f;
    }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        float fb[8], fq[8];
        widen8<C>(b, fb);
        widen8<C>(q, fq);
#pragma unroll
        for (int k = 0; k < 8; ++k) a.v[k] = __fmaf_rn(fq[k], fb[k], a.v[k]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) { return __double2float_rn(reduce8_f64(a.v)); }
    static __device__ __forceinline__ float finalize(float ab, qconst_t qc, float b2) { return cos_normalize_f32(ab, qc.a2, b2); }
    static __device__ __forceinline__ float finalize_sw(float ab, qconst_t qc, float b2) { return cos_normalize_f32(ab, b2, qc.a2); }
    using rn_t = float;
    static __device__ __forceinline__ rn_t rnorm(float x2) { return __frcp_rn(__fsqrt_rn(x2)); }
    static __device__ __forceinline__ float finalize_rn(float ab, float first2, float second2, rn_t rfirst, rn_t rsecond) {
        if (first2 == 0.0f && second2 == 0.0f) return 0.0f;
        if (ab == 0.0f) return 1.0f;
        float r = __fsub_rn(1.0f, __fmul_rn(__fmul_rn(ab, rfirst), rsecond));
        return r > 0 ? r : 0.f;
    }
    static __device__ __forceinline__ float self_dot(uint4 const* v4, uint32_t chunks16, int) {
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (uint32_t j = 0; j < chunks16; ++j) {
            float f[8];
            widen8<C>(v4[j], f);
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = __fmaf_rn(f[k], f[k], v[k]);
        }
        return __double2float_rn(reduce8_f64(v));
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const* q4, uint32_t chunks16, int lane) {
        return {self_dot(q4, chunks16, lane)};
    }
};

/*
 *  WORD variants of the half-precision metrics (lane group of 4, STAGED kernel only).
 *
 *  The reference keeps 8 f32 accumulators; a 16-byte chunk holds exactly one element of each, so accumulator i sees
 *  elements i, i+8, i+16, ... in order. Splitting the work over lanes BY ACCUMULATOR keeps every fma chain intact:
 *  lane s of the group owns accumulators 2s and 2s+1 and reads the 32-bit word s of every chunk (unit = one word,
 *  4 units per chunk). The f64 tree of reduce8_f64, ((v0+v4)+(v2+v6)) + ((v1+v5)+(v3+v7)), becomes an xor-2 shuffle
 *  (v_i + v_{i+4}) followed by an xor-1 shuffle ((..)+(..)); f64 addition is commutative, so the lanes that see the
 *  operands swapped produce the same bits. Compared with one lane per vector this gives 8 vectors per pass in two
 *  double-buffered sets (like f32) instead of 32 in one, and a quarter of the shared memory per warp.
 */
__device__ __forceinline__ float reduce_words_f64(float const v[2]) {
    double a = (double)v[0], b = (double)v[1];
    a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 2)); /* lanes 0,2: v0+v4 | lanes 1,3: v2+v6 */
    b = __dadd_rn(b, __shfl_xor_sync(0xffffffffu, b, 2)); /* lanes 0,2: v1+v5 | lanes 1,3: v3+v7 */
    a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, 1)); /* (v0+v4)+(v2+v6) */
    b = __dadd_rn(b, __shfl_xor_sync(0xffffffffu, b, 1)); /* (v1+v5)+(v3+v7) */
    return __double2float_rn(__dadd_rn(a, b));
}

template <class C> struct l2sq_halfw_t {
    static constexpr int LPV = 4, UPC = 4;
    static constexpr bool NORMS = false;
    using unit_t = uint32_t;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    struct acc_t { float v[2]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.v[0] = a.v[1] = 0.f; }
    static __device__ __forceinline__ void step(acc_t& a, uint32_t b, uint32_t q) {
        float b0, b1, q0, q1;
        C::widen(b, b0, b1);
        C::widen(q, q0, q1);
        float const x0 = __fsub_rn(q0, b0), x1 = __fsub_rn(q1, b1);
        a.v[0] = __fmaf_rn(x0, x0, a.v[0]);
        a.v[1] = __fmaf_rn(x1, x1, a.v[1]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) { return reduce_words_f64(a.v); }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

template <class C> struct ip_halfw_t {
    static constexpr int LPV = 4, UPC = 4;
    static constexpr bool NORMS = false;
    using unit_t = uint32_t;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    struct acc_t { float v[2]; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.v[0] = a.v[1] = 0.f; }
    static __device__ __forceinline__ void step(acc_t& a, uint32_t b, uint32_t q) {
        float b0, b1, q0, q1;
        C::widen(b, b0, b1);
        C::widen(q, q0, q1);
        a.v[0] = __fmaf_rn(q0, b0, a.v[0]);
        a.v[1] = __fmaf_rn(q1, b1, a.v[1]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        float const* v = a.v;
        return __fsub_rn(1.0f, reduce_words_f64(v));
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

template <class C> struct cos_halfw_t {
    static constexpr int LPV = 4, UPC = 4;
    static constexpr bool NORMS = true;
    using unit_t = uint32_t;
    struct acc_t { float v[2]; };
    using qconst_t = typename cos_half_t<C>::qconst_t;
    static __device__ __forceinline__ void init(acc_t& a) { a.v[0] = a.v[1] = 0.f; }
    static __device__ __forceinline__ void step(acc_t& a, uint32_t b, uint32_t q) {
        float b0, b1, q0, q1;
        C::widen(b, b0, b1);
        C::widen(q, q0, q1);
        a.v[0] = __fmaf_rn(q0, b0, a.v[0]);
        a.v[1] = __fmaf_rn(q1, b1, a.v[1]);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        float const* v = a.v;
        return reduce_words_f64(v);
    }
    static __device__ __forceinline__ float finalize(float ab, qconst_t qc, float b2) { return cos_normalize_f32(ab, qc.a2, b2); }
    static __device__ __forceinline__ qconst_t prepare(uint4 const* q4, uint32_t chunks16, int lane) {
        return cos_half_t<C>::prepare(q4, chunks16, lane); /* the query's own norm: same chain as the stored norms */
    }
};

/* the unit a lane reads per step: a 16-byte chunk, or one 32-bit word of it (the WORD variants above) */
template <class M, class = void> struct unit_of {
    using type = uint4;
    static constexpr uint32_t UPC = 1;
};
template <class M> struct unit_of<M, decltype((void)sizeof(typename M::unit_t), void())> {
    using type = typename M::unit_t;
    static constexpr uint32_t UPC = (uint32_t)M::UPC;
};

/* M::PREFILTER where the metric declares it, else false: every other metric keeps the plain search */
template <class M, class = void> struct prefilter_of {
    static constexpr bool value = false;
};
template <class M> struct prefilter_of<M, decltype((void)M::PREFILTER, void())> {
    static constexpr bool value = M::PREFILTER;
};

/* ---- i8 --------------------------------------------------------------------------------- */

template <int LPV_> struct ip_i8_t {
    static constexpr int LPV = LPV_;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { int ab; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.ab = 0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.ab = __dp4a((int)q.x, (int)b.x, a.ab);
        a.ab = __dp4a((int)q.y, (int)b.y, a.ab);
        a.ab = __dp4a((int)q.z, (int)b.z, a.ab);
        a.ab = __dp4a((int)q.w, (int)b.w, a.ab);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        int ab = reduce_add_i32<LPV>(a.ab);
        return __fsub_rn(1.0f, __int2float_rn(ab));
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

template <int LPV_> struct l2sq_i8_t {
    static constexpr int LPV = LPV_;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { int d2; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.d2 = 0; }
    static __device__ __forceinline__ void word(acc_t& a, uint32_t b, uint32_t q) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int x = (int)(int8_t)(q >> (8 * i)) - (int)(int8_t)(b >> (8 * i));
            a.d2 += x * x;
        }
    }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        word(a, b.x, q.x); word(a, b.y, q.y); word(a, b.z, q.z); word(a, b.w, q.w);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        return (float)reduce_add_i32<LPV>(a.d2);
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

template <int LPV_> struct cos_i8_t {
    static constexpr int LPV = LPV_;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { int ab, b2; };
    struct qconst_t { int a2; };
    static __device__ __forceinline__ void init(acc_t& a) { a.ab = a.b2 = 0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.ab = __dp4a((int)q.x, (int)b.x, a.ab); a.b2 = __dp4a((int)b.x, (int)b.x, a.b2);
        a.ab = __dp4a((int)q.y, (int)b.y, a.ab); a.b2 = __dp4a((int)b.y, (int)b.y, a.b2);
        a.ab = __dp4a((int)q.z, (int)b.z, a.ab); a.b2 = __dp4a((int)b.z, (int)b.z, a.b2);
        a.ab = __dp4a((int)q.w, (int)b.w, a.ab); a.b2 = __dp4a((int)b.w, (int)b.w, a.b2);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t qc) {
        int ab = reduce_add_i32<LPV>(a.ab), b2 = reduce_add_i32<LPV>(a.b2);
        return cos_normalize_f32((float)ab, (float)qc.a2, (float)b2);
    }
    static __device__ __forceinline__ float finish_sw(acc_t const& a, qconst_t qc) {
        int ab = reduce_add_i32<LPV>(a.ab), b2 = reduce_add_i32<LPV>(a.b2);
        return cos_normalize_f32((float)ab, (float)b2, (float)qc.a2);
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const* q4, uint32_t chunks16, int lane) {
        int a2 = 0;
        for (uint32_t j = lane; j < chunks16; j += 32) {
            uint4 q = q4[j];
            a2 = __dp4a((int)q.x, (int)q.x, a2); a2 = __dp4a((int)q.y, (int)q.y, a2);
            a2 = __dp4a((int)q.z, (int)q.z, a2); a2 = __dp4a((int)q.w, (int)q.w, a2);
        }
        return {reduce_add_i32<32>(a2)};
    }
};

/* ---- b1x8 ------------------------------------------------------------------------------- */

template <int LPV_> struct hamming_b1_t {
    static constexpr int LPV = LPV_;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { int d; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.d = 0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.d += __popc(b.x ^ q.x) + __popc(b.y ^ q.y) + __popc(b.z ^ q.z) + __popc(b.w ^ q.w);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) { return (float)reduce_add_i32<LPV>(a.d); }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

template <int LPV_> struct tanimoto_b1_t {
    static constexpr int LPV = LPV_;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { int and_, or_; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.and_ = a.or_ = 0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.and_ += __popc(b.x & q.x) + __popc(b.y & q.y) + __popc(b.z & q.z) + __popc(b.w & q.w);
        a.or_ += __popc(b.x | q.x) + __popc(b.y | q.y) + __popc(b.z | q.z) + __popc(b.w | q.w);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        int and_ = reduce_add_i32<LPV>(a.and_), or_ = reduce_add_i32<LPV>(a.or_);
        return or_ ? __double2float_rn(__dsub_rn(1.0, __ddiv_rn((double)and_, (double)or_))) : 1.f;
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

template <int LPV_> struct sorensen_b1_t {
    static constexpr int LPV = LPV_;
    static constexpr bool NORMS = false;
    template <class Q> static __device__ __forceinline__ float finalize(float raw, Q, float) { return raw; }
    template <class Q> static __device__ __forceinline__ float finalize_sw(float raw, Q, float) { return raw; }
    struct acc_t { int and_, any_; };
    struct qconst_t {};
    static __device__ __forceinline__ void init(acc_t& a) { a.and_ = a.any_ = 0; }
    static __device__ __forceinline__ void step(acc_t& a, uint4 b, uint4 q) {
        a.and_ += __popc(b.x & q.x) + __popc(b.y & q.y) + __popc(b.z & q.z) + __popc(b.w & q.w);
        a.any_ += __popc(b.x) + __popc(b.y) + __popc(b.z) + __popc(b.w) + __popc(q.x) + __popc(q.y) + __popc(q.z) + __popc(q.w);
    }
    static __device__ __forceinline__ float finish(acc_t const& a, qconst_t) {
        int and_ = reduce_add_i32<LPV>(a.and_), any_ = reduce_add_i32<LPV>(a.any_);
        return __fsub_rn(1.f, __fdiv_rn(__fmul_rn(2.f, (float)and_), (float)any_));
    }
    static __device__ __forceinline__ qconst_t prepare(uint4 const*, uint32_t, int) { return {}; }
};

} // namespace usearch_b200
