/*
 *  The prefilter's query split (pf_split_query in usearch_b200/csrc/prefilter_bound.h) and the bound it feeds, against
 *  the pinned reference metrics (oracle/metrics_pinned.h). The kernel multiplies the int8 codes of a row with the two
 *  int8 levels of the query on the tensor cores; here the same integers are formed on the host:
 *    - rho_a >= the long-double norm of a - sa1 q1 - sa2 q2, and the codes are zero past the query;
 *    - d_lo <= d_pinned for cos and ip, with dot = fl32(sa1 D1 + sa2 D2) and the rho_a term;
 *    - d_pinned - d_lo stays under the gap limit that includes that term.
 *  Random pairs (10^7, dims 1..32, plus 768-d and 97-d ones), the adversarial pairs of test_prefilter_bound.cpp, and
 *  queries made for the split: one huge element among tiny ones, queries on the sa1 grid (sa2 = 0), subnormal
 *  elements, zero and non-finite queries.
 *  Build: g++ -O2 -ffp-contract=off -std=c++17 -I oracle -I usearch_b200/csrc; run: ./a.out [pairs]
 */
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "metrics_pinned.h"
#include "prefilter_bound.h"

using namespace usearch_b200;

static uint64_t checked = 0, applied = 0, failures = 0, split_checked = 0;
static double worst_gap_share = 0; /* max over pairs of (d - d_lo) / limit */

static void fail(char const* what, uint32_t n, double d, double lo, double limit) {
    if (failures < 20) std::printf("FAIL %s n=%u d=%.9g d_lo=%.9g limit=%.3g\n", what, n, d, lo, limit);
    ++failures;
}

/* the split of `a` and its own checks; returns it with q1, q2 filled (code_len bytes each) */
static pf_query_split_t split_checked_query(std::vector<float> const& a, std::vector<int8_t>& q1, std::vector<int8_t>& q2,
                                            uint32_t code_len) {
    uint32_t const n = (uint32_t)a.size();
    q1.assign(code_len, 7);
    q2.assign(code_len, 7);
    pf_query_split_t const sp = pf_split_query(a.data(), n, q1.data(), q2.data(), code_len);
    ++split_checked;
    for (uint32_t i = n; i < code_len; ++i)
        if (q1[i] != 0 || q2[i] != 0) fail("split padding", n, 0, 0, 0);
    for (uint32_t i = 0; i < n; ++i)
        if (q1[i] < -127 || q2[i] < -127) fail("split code -128", n, 0, 0, 0);
    if (sp.rho_a < INFINITY) {
        long double e2 = 0;
        for (uint32_t i = 0; i < n; ++i) {
            long double const e = (long double)a[i] - (long double)sp.sa1 * q1[i] - (long double)sp.sa2 * q2[i];
            e2 += e * e;
        }
        if (!((long double)sp.rho_a >= sqrtl(e2))) fail("rho_a below the residual", n, (double)sqrtl(e2), sp.rho_a, 0);
        if (!(sp.sa1 > 0.0f)) fail("usable split with a zero scale", n, 0, sp.sa1, 0);
        if (sp.sa2 == 0.0f)
            for (uint32_t i = 0; i < n; ++i)
                if (q2[i] != 0) fail("q2 without a scale", n, 0, 0, 0);
    } else {
        for (uint32_t i = 0; i < n; ++i)
            if (q1[i] != 0 || q2[i] != 0) fail("unusable split with codes", n, 0, 0, 0);
    }
    return sp;
}

static void check_pair(std::vector<float> const& a, std::vector<float> const& b) {
    uint32_t const n = (uint32_t)a.size(), cs = (n + 15) & ~15u, len = (cs + 31) & ~31u;
    std::vector<int8_t> codes(cs), q1, q2;
    float const b2 = pinned_dot_f32_(b.data(), b.data(), n);
    pf_record_t const r = pf_encode_row(b.data(), n, codes.data(), cs, b2);
    pf_query_split_t const sp = split_checked_query(a, q1, q2, len);
    int64_t D1 = 0, D2 = 0; /* the tensor cores' s32 sums; a 32-byte k-step reads past `cs`, where the split is zero */
    for (uint32_t i = 0; i < cs; ++i) { D1 += (int64_t)q1[i] * codes[i]; D2 += (int64_t)q2[i] * codes[i]; }
    if (D1 != (int32_t)D1 || D2 != (int32_t)D2) fail("s32 overflow", n, 0, 0, 0);
    float const dot = (float)((double)sp.sa1 * (double)D1 + (double)sp.sa2 * (double)D2);
    float const a2 = pinned_dot_f32_(a.data(), a.data(), n);
    struct { char const* name; double d, lo, limit; } const m[2] = {
        {"cos", pinned_cos_f32(a.data(), b.data(), n), pf_cos_lower(dot, r.s, r.rho, a2, r.b2, n, sp.rho_a),
         pf_cos_gap_limit(r.s, r.rho, a2, r.b2, n, sp.rho_a)},
        {"ip", pinned_ip_f32(a.data(), b.data(), n), pf_ip_lower(dot, r.s, r.rho, a2, r.bnorm, n, sp.rho_a),
         pf_ip_gap_limit(r.s, r.rho, a2, r.bnorm, n, sp.rho_a)},
    };
    for (auto const& x : m) {
        ++checked;
        if (std::isnan(x.d)) { /* a NaN distance must never be rejected: only -inf or NaN bounds */
            if (!(x.lo == -INFINITY || std::isnan(x.lo))) fail(x.name, n, x.d, x.lo, x.limit);
            continue;
        }
        if (!(x.lo <= x.d) && !std::isnan(x.lo)) { fail(x.name, n, x.d, x.lo, x.limit); continue; }
        if (x.lo == -INFINITY || std::isnan(x.lo)) continue; /* never rejects */
        ++applied;
        double const gap = x.d - x.lo;
        if (!(gap < x.limit)) { fail(x.name, n, x.d, x.lo, x.limit); continue; }
        if (gap / x.limit > worst_gap_share) worst_gap_share = gap / x.limit;
    }
}

int main(int argc, char** argv) {
    uint64_t const pairs = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 10000000ull;
    uint64_t state = 4242;
    auto rng = [&]() { /* splitmix64 */
        uint64_t z = (state += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    };
    auto unif = [&](decltype(rng)&) { return (float)((double)(rng() >> 11) * 0x1p-52 - 1.0); }; /* [-1, 1) */
    auto gauss = [&](decltype(rng)& r) { return unif(r) + unif(r) + unif(r); };             /* bell-shaped */
    auto expo = [&](decltype(rng)&) { return (int)(rng() % 81) - 40; };                      /* -40 .. 40 */
    float const corr[] = {0.f, 1e-7f, 1e-5f, 1e-3f, 1e-2f, 0.1f, 0.5f, 1.f};
    std::vector<float> a, b;
    auto random_pair = [&](uint32_t n) {
        a.resize(n);
        b.resize(n);
        float const sa = std::ldexp(1.f, expo(rng)), sb = std::ldexp(1.f, expo(rng) / 4);
        float const eps = corr[rng() % 8];
        bool const uniform = rng() & 1;
        for (uint32_t i = 0; i < n; ++i) a[i] = uniform ? unif(rng) : gauss(rng);
        for (uint32_t i = 0; i < n; ++i) {
            float const noise = uniform ? unif(rng) : gauss(rng);
            b[i] = eps == 1.f ? noise * sb : (a[i] + eps * noise) * sb; /* b near a (up to scale) or independent */
        }
        for (uint32_t i = 0; i < n; ++i) a[i] *= sa;
        if (rng() % 4 == 0) std::swap(a, b);
    };
    for (uint64_t p = 0; p < pairs; ++p) { random_pair(1 + (uint32_t)(rng() % 32)); check_pair(a, b); }
    for (int p = 0; p < 20000; ++p) { random_pair(768); check_pair(a, b); }
    for (int p = 0; p < 20000; ++p) { random_pair(97); check_pair(a, b); }
    uint64_t const random_checked = checked;

    /* adversarial pairs, as in test_prefilter_bound.cpp */
    for (uint32_t n : {1u, 3u, 16u, 64u, 97u, 768u}) {
        for (int rep = 0; rep < 200; ++rep) {
            random_pair(n);
            check_pair(a, a);
            std::vector<float> c = a;
            uint32_t const j = (uint32_t)(rng() % n);
            c[j] = std::nextafter(c[j], INFINITY);
            check_pair(a, c);
            check_pair(c, a);
            for (uint32_t i = 0; i < n; ++i) c[i] = std::nextafter(a[i], -INFINITY);
            check_pair(a, c);
            for (uint32_t i = 0; i < n; ++i) c[i] = -a[i];
            check_pair(a, c);
        }
        std::vector<float> z(n, 0.f), h(n, 0.f), h2(n, 0.f), w(n), sub(n), big(n);
        h[0] = 1.f;
        h2[n - 1] = -3.f;
        for (uint32_t i = 0; i < n; ++i) {
            w[i] = std::ldexp(unif(rng), (int)(i % 60) - 30);
            sub[i] = std::ldexp(unif(rng), -140 + (int)(i % 10));
            big[i] = std::ldexp(unif(rng), 60);
        }
        std::vector<float> wn = w, bad = h;
        wn[n / 2] = std::nextafter(wn[n / 2], 0.f);
        for (auto const& p : {std::make_pair(&z, &z), std::make_pair(&z, &h), std::make_pair(&h, &z), std::make_pair(&h, &h),
                              std::make_pair(&h, &h2), std::make_pair(&w, &w), std::make_pair(&w, &h), std::make_pair(&h, &w),
                              std::make_pair(&w, &wn), std::make_pair(&sub, &sub), std::make_pair(&sub, &h),
                              std::make_pair(&h, &sub), std::make_pair(&big, &big), std::make_pair(&big, &h)})
            check_pair(*p.first, *p.second);
        bad[n - 1] = INFINITY;
        check_pair(h, bad);
        check_pair(bad, h);
        bad[n - 1] = NAN;
        check_pair(h, bad);
        check_pair(bad, h);

        /* queries made for the split, each against a random row and against itself */
        std::vector<std::vector<float>> qs;
        std::vector<float> x(n);
        for (uint32_t i = 0; i < n; ++i) x[i] = std::ldexp(unif(rng), -30); /* one huge element among tiny ones: */
        x[n / 3] = 1e6f;                                                   /* q1 saturates, q2 carries the rest */
        qs.push_back(x);
        float const grid = std::ldexp(1.f, -7); /* on the sa1 grid: max = 127 grid, every element a multiple of it */
        for (uint32_t i = 0; i < n; ++i) x[i] = grid * (float)((int)(rng() % 255) - 127);
        x[0] = 127.f * grid;
        qs.push_back(x);
        for (uint32_t i = 0; i < n; ++i) x[i] = std::ldexp(unif(rng), -149 + (int)(i % 24)); /* subnormal */
        qs.push_back(x);
        for (uint32_t i = 0; i < n; ++i) x[i] = i % 2 ? std::ldexp(unif(rng), -130) : unif(rng); /* mixed */
        qs.push_back(x);
        qs.push_back(z);
        x = h;
        x[n - 1] = -INFINITY;
        qs.push_back(x);
        x[n - 1] = NAN;
        qs.push_back(x);
        std::vector<int8_t> q1, q2;
        uint32_t const len = (((n + 15) & ~15u) + 31) & ~31u;
        for (auto const& q : qs) {
            for (int rep = 0; rep < 20; ++rep) {
                random_pair(n);
                check_pair(q, b);
                check_pair(q, a);
            }
            check_pair(q, q);
        }
        pf_query_split_t const on_grid = split_checked_query(qs[1], q1, q2, len);
        if (on_grid.sa2 != 0.0f || !(on_grid.rho_a <= std::nextafter(0.0f, 1.0f))) fail("grid query: sa2 or rho_a not zero", n, on_grid.sa2, on_grid.rho_a, 0);
        for (size_t k : {(size_t)4, (size_t)5, (size_t)6})
            if (split_checked_query(qs[k], q1, q2, len).rho_a != INFINITY) fail("zero or non-finite query usable", n, 0, 0, 0);
    }
    std::printf("pairs checked: %llu random + %llu adversarial (cos and ip each counted); splits checked: %llu; bound "
                "applied on %llu; worst gap / limit = %.4f; failures: %llu\n",
                (unsigned long long)random_checked, (unsigned long long)(checked - random_checked),
                (unsigned long long)split_checked, (unsigned long long)applied, worst_gap_share, (unsigned long long)failures);
    return failures ? 1 : 0;
}
