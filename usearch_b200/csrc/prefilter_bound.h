/*
 *  prefilter_bound.h — a proved lower bound on the f32 distance the reference computes for cos / ip f32, from the int8
 *  shadow code of the stored vector. Plain C++ (host and device): tests/native/test_prefilter_bound.cpp checks the same
 *  functions against the pinned reference metrics (the metrics_pinned.h of the test oracle).
 *
 *  Stored vector b (n = dims f32 elements), its shadow: codes c (int8, c_i = clamp(rint(b_i / s), -127, 127)), the scale
 *  s = max|b_i| / 127 (f32), rho >= ||b - s c|| (computed in f64, rounded up) and bnorm >= ||b|| (same). Query a (f32).
 *  `dot` stands for a.c, rounded to f32 (step 1 below bounds how); s dot is formed in f64 (an exact product), and every
 *  f64 operation of the bound itself errs by 2^-53 relative, far inside the margin below. Then, with ||.|| the exact
 *  Euclidean norm:
 *
 *    a.b = s (a.c) + a.(b - s c) <= s (a.c) + ||a|| rho                                      (Cauchy-Schwarz)
 *
 *  and what remains is the rounding of four computations, g = gamma_n = n u / (1 - n u), u = 2^-24 (Higham, Accuracy
 *  and Stability of Numerical Algorithms, 2nd ed., Lemma 3.1 / (3.5): any summation order of n products with an fma
 *  chain or a tree has |computed - exact| <= gamma_n sum |x_i y_i|):
 *    1. `dot`:                 |dot - a.c| <= g ||a|| ||c||, and s ||c|| <= ||b - s c|| + ||b|| <= rho + ||b||;
 *    2. the reference's ab:    |ab_ref - a.b| <= g ||a|| ||b||  (16 accumulators then a tree: still one sum of n terms);
 *    3. its norms:             a2_ref = ||a||^2 (1 + t), |t| <= g, so ||a|| <= A (1 + g) with A = sqrt(a2_ref) (same
 *                              for b); cos divides by A B in f64, ip needs no norm of its own;
 *    4. its last roundings:    cos: four f64 operations (relative 2^-53 each) and the cast to f32 (2^-24 relative,
 *                              |r| <= 2 + rho / B + ... <= 4 on the values that reach it); ip: 1 - ab in f32, at most
 *                              2^-24 (1 + |ab_ref|) with |ab_ref| <= (1 + g)^3 A B <= 2 A B.
 *  Products that underflow add at most 2^-150 each (n of them) to (1) and (2): the term n 2^-148 (1 + s).
 *  Summing (the g ||a|| rho of step 3 is the second `2 rho`):
 *
 *    ab_ref <= s dot + A rho + (1 + g)^2 delta0,  delta0 = g A (2 B + 2 rho) + n 2^-148 (1 + s)
 *    cos: d_ref >= 1 - ab_ref / (A B) - 2^-22           ip: d_ref >= 1 - ab_ref - 2^-24 (1 + 2 A B)
 *
 *  (1 + g)^2 <= 1.04 for n <= 2^18, so the margin PF_MARGIN = 16 is more than ten times that worst case:
 *    cos: d_lo = 1 - (s dot + A rho + delta) / (A B),  delta = 16 (delta0 + 2^-22 A B)
 *    ip:  d_lo = 1 - (s dot + A rho + delta),          delta = 16 (delta0 + 2^-24 (1 + 2 A B))   (B = bnorm for ip)
 *
 *  The query split (what the kernel computes, pf_split_query). Step 1 above is how `dot` errs when it is a.c summed in
 *  f32. The kernel instead splits the query once into two int8 levels, q1 = code(a, sa1) and q2 = code(r1, sa2) of the
 *  residual r1 = a - sa1 q1, with sa1 = max|a_i| / 127 and sa2 = max|r1_i| / 127 (f32 scales), leaving
 *  r2 = r1 - sa2 q2 and rho_a >= ||r2|| (f64, rounded up). Every r1_i and r2_i is exact in f64: an f32 minus an f32 scale
 *  times |q| <= 127 spans fewer than 53 bits. So a.c = sa1 D1 + sa2 D2 + r2.c with the exact integers D1 = q1.c and
 *  D2 = q2.c (tensor-core products in s32, exact while n 127^2 < 2^31), and `dot` = fl32(sa1 D1 + sa2 D2), formed in f64.
 *  Then |dot - a.c| <= 2^-24 |a.c| + rho_a ||c|| (+ f64 and 2^-24 rho_a ||c|| roundings, inside the margin), and
 *  2^-24 |a.c| <= g ||a|| ||c|| for n >= 1, so step 1 still holds with the extra term rho_a ||c||. Multiplied by s, with
 *  s ||c|| <= rho + ||b||, that adds
 *
 *    T = rho_a (rho + ||b||),   ||b|| <= B (1 + g) for cos (step 3), ||b|| <= bnorm = B for ip,
 *
 *  to ab_ref, outside the margin like A rho: d_lo is then 1 - (s dot + A rho + T + delta) / (A B) for cos and
 *  1 - (s dot + A rho + T + delta) for ip. rho_a = 0 (the default) is the bound for an f32 `dot`. A query whose split is
 *  unusable (a non-finite element, or a zero scale) gets rho_a = +inf: it never rejects.
 *
 *  The reference's special cases stay exact: a2 == b2 == 0 is a "never reject" (zero norm), ab == 0 gives d = 1 and the
 *  bound is below it (ab_ref <= s dot + A rho + delta0 forces that sum >= 0), and the clamp at 0 only raises d. Norms
 *  that are zero, below 2^-100 (where underflow inside the chains could matter), non-finite, or so large that a
 *  product could overflow (A B > 2^120), and a shadow that is non-finite (rho = +inf marks an all-zero or non-finite
 *  row), all return -inf: such a candidate is never rejected. A caller rejects iff `d_lo >= radius`: NaN never rejects.
 */
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define PF_HD __host__ __device__ __forceinline__
#else
#define PF_HD inline
#endif

namespace usearch_b200 {

constexpr double PF_MARGIN = 16.0;

/* 16-byte shadow record of one slot (one sector per candidate) */
struct alignas(16) pf_record_t {
    float s;     /* scale of the int8 code: max|b_i| / 127 */
    float rho;   /* >= ||b - s c||, +inf = never reject */
    float bnorm; /* >= ||b|| */
    float b2;    /* cos: the stored squared norm (bit copy of `norms`), so that one record serves the whole bound */
};

PF_HD double pf_gamma(uint32_t n) {
    double const nu = (double)n * 0x1p-24;
    return nu / (1.0 - nu);
}

/* never reject: -inf. Every comparison is written so that a NaN lands on "usable == false". */
PF_HD bool pf_usable(double A, double B, float s, float rho) {
    return A >= 0x1p-50 && B >= 0x1p-50 && A * B <= 0x1p120 && rho >= 0.0f && rho < INFINITY && s > 0.0f && s < INFINITY;
}

PF_HD double pf_delta0(double A, double B, double s, double rho, uint32_t n) {
    return pf_gamma(n) * A * (2.0 * B + 2.0 * rho) + (double)n * 0x1p-148 * (1.0 + s);
}

/* the query split's term T = rho_a (rho + ||b||), with nb >= ||b|| */
PF_HD double pf_split_term(float rho_a, float rho, double nb) { return (double)rho_a * ((double)rho + nb); }

/* cos f32: a2 = the query's squared norm and b2 = the stored one, both as the reference accumulates them; rho_a: the
 * query split's residual bound when `dot` comes from it (pf_split_query), 0 for an f32 `dot` */
PF_HD double pf_cos_lower(float dot, float s, float rho, float a2, float b2, uint32_t n, float rho_a = 0.0f) {
    double const A = sqrt((double)a2), B = sqrt((double)b2);
    if (!pf_usable(A, B, s, rho) || !(rho_a >= 0.0f && rho_a < INFINITY)) return -INFINITY;
    double const delta = PF_MARGIN * (pf_delta0(A, B, s, rho, n) + 0x1p-22 * A * B);
    double const T = pf_split_term(rho_a, rho, B * (1.0 + pf_gamma(n)));
    return 1.0 - ((double)s * (double)dot + A * (double)rho + T + delta) / (A * B);
}

/* ip f32: a2 = the query's squared norm accumulated in f32, bnorm >= ||b|| from the record */
PF_HD double pf_ip_lower(float dot, float s, float rho, float a2, float bnorm, uint32_t n, float rho_a = 0.0f) {
    double const A = sqrt((double)a2), B = (double)bnorm;
    if (!pf_usable(A, B, s, rho) || !(rho_a >= 0.0f && rho_a < INFINITY)) return -INFINITY;
    double const delta = PF_MARGIN * (pf_delta0(A, B, s, rho, n) + 0x1p-24 * (1.0 + 2.0 * A * B));
    double const T = pf_split_term(rho_a, rho, B);
    return 1.0 - ((double)s * (double)dot + A * (double)rho + T + delta);
}

/* The same two bounds with what depends only on the query (A = sqrt(a2), gamma_n and its products, the rho_a test)
 * computed once per query: every candidate then runs the f64 operations above that involve its own record, on the same
 * operands in the same order, so d_lo is the same bits. */
struct pf_query_bound_t {
    double A;      /* sqrt(a2) */
    double gA;     /* pf_gamma(n) * A, the first product of pf_delta0 */
    double n148;   /* n 2^-148, the first product of pf_delta0's underflow term */
    double one_g;  /* 1 + pf_gamma(n) */
    bool split_ok; /* rho_a is finite and not negative */
    float rho_a;
};

PF_HD pf_query_bound_t pf_query_bound(float a2, uint32_t n, float rho_a) {
    double const A = sqrt((double)a2), g = pf_gamma(n);
    return pf_query_bound_t{A, g * A, (double)n * 0x1p-148, 1.0 + g, rho_a >= 0.0f && rho_a < INFINITY, rho_a};
}

PF_HD double pf_delta0_q(pf_query_bound_t const& q, double B, double s, double rho) {
    return q.gA * (2.0 * B + 2.0 * rho) + q.n148 * (1.0 + s);
}

PF_HD double pf_cos_lower_q(float dot, float s, float rho, float b2, pf_query_bound_t const& q) {
    double const A = q.A, B = sqrt((double)b2);
    if (!pf_usable(A, B, s, rho) || !q.split_ok) return -INFINITY;
    double const delta = PF_MARGIN * (pf_delta0_q(q, B, s, rho) + 0x1p-22 * A * B);
    double const T = pf_split_term(q.rho_a, rho, B * q.one_g);
    return 1.0 - ((double)s * (double)dot + A * (double)rho + T + delta) / (A * B);
}

PF_HD double pf_ip_lower_q(float dot, float s, float rho, float bnorm, pf_query_bound_t const& q) {
    double const A = q.A, B = (double)bnorm;
    if (!pf_usable(A, B, s, rho) || !q.split_ok) return -INFINITY;
    double const delta = PF_MARGIN * (pf_delta0_q(q, B, s, rho) + 0x1p-24 * (1.0 + 2.0 * A * B));
    double const T = pf_split_term(q.rho_a, rho, B);
    return 1.0 - ((double)s * (double)dot + A * (double)rho + T + delta);
}

/* what the tightness checks compare against: d_ref - d_lo stays below this */
PF_HD double pf_cos_gap_limit(float s, float rho, float a2, float b2, uint32_t n, float rho_a = 0.0f) {
    double const A = sqrt((double)a2), B = sqrt((double)b2);
    double const delta = PF_MARGIN * (pf_delta0(A, B, s, rho, n) + 0x1p-22 * A * B);
    double const T = pf_split_term(rho_a, rho, B * (1.0 + pf_gamma(n)));
    return 2.0 * (double)rho / B + 2.0 * (delta + T) / (A * B);
}
PF_HD double pf_ip_gap_limit(float s, float rho, float a2, float bnorm, uint32_t n, float rho_a = 0.0f) {
    double const A = sqrt((double)a2), B = (double)bnorm;
    double const delta = PF_MARGIN * (pf_delta0(A, B, s, rho, n) + 0x1p-24 * (1.0 + 2.0 * A * B));
    double const T = pf_split_term(rho_a, rho, B);
    return 2.0 * A * (double)rho + 2.0 * (delta + T);
}

/* The pieces of one row's shadow, shared by the device kernel (a warp per row, search_kernel.cu) and the host test. */
PF_HD float pf_scale(double max_abs) { return (float)(max_abs / 127.0); }
PF_HD int8_t pf_code_f64(double x, float s) {
    double q = rint(x / (double)s);
    q = q > 127.0 ? 127.0 : (q < -127.0 ? -127.0 : q);
    return (int8_t)q;
}
PF_HD int8_t pf_code(float x, float s) { return pf_code_f64((double)x, s); }
/* sqrt of an f64 sum of n squares (relative error <= (n + 2) 2^-53 in any order), lifted by 2^-30 (covers n < 2^22)
 * and rounded up to f32: never below the exact norm. Overflow gives +inf. */
PF_HD float pf_round_up_norm(double sum_sq) { return nextafterf((float)(sqrt(sum_sq) * (1.0 + 0x1p-30)), INFINITY); }

/* The whole shadow of one row: the record, and `code_stride` int8 codes (zero padding). A row that is all zero or holds
 * a non-finite element gets rho = +inf (never rejected) and zero codes. */
PF_HD pf_record_t pf_encode_row(float const* b, uint32_t n, int8_t* codes, uint32_t code_stride, float b2) {
    double mx = 0.0;
    bool finite = true;
    for (uint32_t i = 0; i < n; ++i) {
        double const x = fabs((double)b[i]);
        finite = finite && x < INFINITY; /* NaN fails too */
        mx = x > mx ? x : mx;
    }
    float const s = pf_scale(mx);
    pf_record_t r{0.f, INFINITY, INFINITY, b2};
    for (uint32_t i = 0; i < code_stride; ++i) codes[i] = 0;
    if (!finite || !(s > 0.0f)) return r;
    double e2 = 0.0, n2 = 0.0;
    for (uint32_t i = 0; i < n; ++i) {
        codes[i] = pf_code(b[i], s);
        double const e = (double)b[i] - (double)s * (double)codes[i];
        e2 += e * e;
        n2 += (double)b[i] * (double)b[i];
    }
    r.s = s;
    r.rho = pf_round_up_norm(e2);
    r.bnorm = pf_round_up_norm(n2);
    return r;
}

/* ---- the query split (derivation above): two int8 levels of the f32 query ---- */
struct pf_query_split_t {
    float sa1, sa2; /* scales of q1 and q2 */
    float rho_a;    /* >= ||a - sa1 q1 - sa2 q2||, +inf = never reject */
};

/* One element's two steps, shared by the kernel (a warp per query, search_kernel.cu) and the host: q1 and the exact
 * residual r1 = x - sa1 q1, then q2 and r2 = r1 - sa2 q2. A zero scale codes everything as 0. */
PF_HD double pf_split_step(double x, float scale, int8_t& q) {
    q = scale > 0.0f ? pf_code_f64(x, scale) : (int8_t)0;
    return x - (double)scale * (double)q;
}

/* The whole split of one query: `q1` and `q2` get `code_len` int8 codes each, zero beyond n. A query with a non-finite
 * element or a zero norm gets zero codes and rho_a = +inf. */
PF_HD pf_query_split_t pf_split_query(float const* a, uint32_t n, int8_t* q1, int8_t* q2, uint32_t code_len) {
    double mx1 = 0.0;
    bool finite = true;
    for (uint32_t i = 0; i < n; ++i) {
        double const x = fabs((double)a[i]);
        finite = finite && x < INFINITY; /* NaN fails too */
        mx1 = x > mx1 ? x : mx1;
    }
    pf_query_split_t sp{pf_scale(mx1), 0.0f, INFINITY};
    for (uint32_t i = 0; i < code_len; ++i) q1[i] = q2[i] = 0;
    if (!finite || !(sp.sa1 > 0.0f)) return pf_query_split_t{0.0f, 0.0f, INFINITY};
    double mx2 = 0.0;
    for (uint32_t i = 0; i < n; ++i) {
        double const r1 = fabs(pf_split_step((double)a[i], sp.sa1, q1[i]));
        mx2 = r1 > mx2 ? r1 : mx2;
    }
    sp.sa2 = pf_scale(mx2);
    double e2 = 0.0;
    for (uint32_t i = 0; i < n; ++i) {
        double const r2 = pf_split_step(pf_split_step((double)a[i], sp.sa1, q1[i]), sp.sa2, q2[i]);
        e2 += r2 * r2;
    }
    sp.rho_a = pf_round_up_norm(e2);
    return sp;
}

} // namespace usearch_b200
