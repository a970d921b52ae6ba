/*
 *  The int8-shadow lower bound (usearch_b200/csrc/prefilter_bound.h) against the pinned reference metrics
 *  (oracle/metrics_pinned.h): for cos and ip f32, d_lo <= d_pinned on every pair, and d_pinned - d_lo stays under the
 *  gap limit (2 rho / ||b|| + 2 delta, normalised, for cos; 2 ||a|| rho + 2 delta for ip) wherever the bound applies.
 *  Random pairs (10^7, dims 1..32, plus 768-d and 97-d ones, at magnitudes from 2^-40 to 2^40 and correlations from
 *  duplicates to independent), then adversarial ones: last-ULP differences, duplicates, opposite vectors, huge dynamic
 *  range inside one vector, one-hot, zero, subnormal and non-finite vectors.
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

static uint64_t checked = 0, applied = 0, failures = 0;
static double worst_gap_share = 0; /* max over pairs of (d - d_lo) / limit */

/* a.c in f32 the way the kernel groups it: word u = i / 4 goes to lane u % 4, element i % 4 of the word to that lane's
 * accumulator i % 4; then the 4 accumulators of a lane, then the 4 lanes (xor 1, xor 2) */
static float shadow_dot(float const* a, int8_t const* c, uint32_t n) {
    float acc[4][4] = {};
    for (uint32_t i = 0; i < n; ++i) acc[(i / 4) % 4][i % 4] = fmaf(a[i], (float)c[i], acc[(i / 4) % 4][i % 4]);
    float l[4];
    for (int s = 0; s < 4; ++s) l[s] = (acc[s][0] + acc[s][1]) + (acc[s][2] + acc[s][3]);
    float const x0 = l[0] + l[1], x2 = l[2] + l[3];
    return x0 + x2;
}

static void fail(char const* what, uint32_t n, double d, double lo, double limit) {
    if (failures < 20) std::printf("FAIL %s n=%u d=%.9g d_lo=%.9g limit=%.3g\n", what, n, d, lo, limit);
    ++failures;
}

static void check_pair(std::vector<float> const& a, std::vector<float> const& b) {
    uint32_t const n = (uint32_t)a.size(), cs = (n + 15) & ~15u;
    std::vector<int8_t> codes(cs);
    float const b2 = pinned_dot_f32_(b.data(), b.data(), n);
    pf_record_t const r = pf_encode_row(b.data(), n, codes.data(), cs, b2);
    for (uint32_t i = n; i < cs; ++i)
        if (codes[i] != 0) fail("code padding", n, 0, 0, 0);
    if (r.rho < INFINITY) { /* the record's bounds hold in long double */
        long double e2 = 0, n2 = 0;
        for (uint32_t i = 0; i < n; ++i) {
            long double const e = (long double)b[i] - (long double)r.s * codes[i];
            e2 += e * e;
            n2 += (long double)b[i] * b[i];
        }
        if (!((long double)r.rho >= sqrtl(e2))) fail("rho below the residual", n, (double)sqrtl(e2), r.rho, 0);
        if (!((long double)r.bnorm >= sqrtl(n2))) fail("bnorm below the norm", n, (double)sqrtl(n2), r.bnorm, 0);
    }
    float const dot = shadow_dot(a.data(), codes.data(), n);
    float const a2 = pinned_dot_f32_(a.data(), a.data(), n);
    struct { char const* name; double d, lo, limit; } const m[2] = {
        {"cos", pinned_cos_f32(a.data(), b.data(), n), pf_cos_lower(dot, r.s, r.rho, a2, r.b2, n),
         pf_cos_gap_limit(r.s, r.rho, a2, r.b2, n)},
        {"ip", pinned_ip_f32(a.data(), b.data(), n), pf_ip_lower(dot, r.s, r.rho, a2, r.bnorm, n),
         pf_ip_gap_limit(r.s, r.rho, a2, r.bnorm, n)},
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
    uint64_t state = 42;
    auto rng = [&]() { /* splitmix64: cheap enough for 10^7 pairs */
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

    /* adversarial pairs */
    for (uint32_t n : {1u, 3u, 16u, 64u, 97u, 768u}) {
        for (int rep = 0; rep < 200; ++rep) {
            random_pair(n);
            check_pair(a, a); /* exact duplicates */
            std::vector<float> c = a;
            uint32_t const j = (uint32_t)(rng() % n);
            c[j] = std::nextafter(c[j], INFINITY); /* one element one ULP apart */
            check_pair(a, c);
            check_pair(c, a);
            for (uint32_t i = 0; i < n; ++i) c[i] = std::nextafter(a[i], -INFINITY); /* every element */
            check_pair(a, c);
            for (uint32_t i = 0; i < n; ++i) c[i] = -a[i]; /* opposite */
            check_pair(a, c);
        }
        std::vector<float> z(n, 0.f), h(n, 0.f), h2(n, 0.f), w(n), sub(n), big(n);
        h[0] = 1.f;
        h2[n - 1] = -3.f;
        check_pair(z, z);
        check_pair(z, h);
        check_pair(h, z);
        check_pair(h, h);  /* one-hot, same */
        check_pair(h, h2); /* one-hot, apart (or opposite when n == 1) */
        for (uint32_t i = 0; i < n; ++i) {
            w[i] = std::ldexp(unif(rng), (int)(i % 60) - 30);        /* 2^-30 .. 2^29 inside one vector */
            sub[i] = std::ldexp(unif(rng), -140 + (int)(i % 10));    /* subnormal and barely normal */
            big[i] = std::ldexp(unif(rng), 60);                      /* squares near the top of the range */
        }
        check_pair(w, w);
        check_pair(w, h);
        check_pair(h, w);
        std::vector<float> wn = w;
        wn[n / 2] = std::nextafter(wn[n / 2], 0.f);
        check_pair(w, wn);
        check_pair(sub, sub);
        check_pair(sub, h);
        check_pair(h, sub);
        check_pair(big, big);
        check_pair(big, h);
        std::vector<float> bad = h;
        bad[n - 1] = INFINITY;
        check_pair(h, bad);
        bad[n - 1] = NAN;
        check_pair(h, bad);
        check_pair(bad, h);
    }
    std::printf("pairs checked: %llu random + %llu adversarial (cos and ip each counted); bound applied on %llu; "
                "worst gap / limit = %.4f; failures: %llu\n",
                (unsigned long long)random_checked, (unsigned long long)(checked - random_checked),
                (unsigned long long)applied, worst_gap_share, (unsigned long long)failures);
    return failures ? 1 : 0;
}
