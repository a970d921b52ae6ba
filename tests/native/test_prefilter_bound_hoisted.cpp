/*
 *  The per-query form of the int8-shadow bound (pf_query_bound + pf_cos_lower_q / pf_ip_lower_q, what the search kernel
 *  evaluates) against the per-candidate form (pf_cos_lower / pf_ip_lower): the same bits on every pair, for the split's
 *  own rho_a and for rho_a = 0, +inf, NaN and a negative value. The pairs are those of test_prefilter_bound.cpp: 10^7
 *  random ones (dims 1..32, plus 768-d and 97-d ones) and the adversarial set.
 *  Build: g++ -O2 -ffp-contract=off -std=c++17 -I oracle -I usearch_b200/csrc; run: ./a.out [pairs]
 */
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "metrics_pinned.h"
#include "prefilter_bound.h"

using namespace usearch_b200;

static uint64_t checked = 0, failures = 0;

static bool same_bits(double x, double y) { return std::memcmp(&x, &y, sizeof x) == 0; }

static void compare(char const* what, uint32_t n, double want, double got) {
    ++checked;
    if (same_bits(want, got)) return;
    if (failures < 20) std::printf("FAIL %s n=%u per-candidate=%a per-query=%a\n", what, n, want, got);
    ++failures;
}

static void check_pair(std::vector<float> const& a, std::vector<float> const& b) {
    uint32_t const n = (uint32_t)a.size(), cs = (n + 15) & ~15u, len = (cs + 31) & ~31u;
    std::vector<int8_t> codes(cs), q1(len), q2(len);
    float const b2 = pinned_dot_f32_(b.data(), b.data(), n);
    pf_record_t const r = pf_encode_row(b.data(), n, codes.data(), cs, b2);
    pf_query_split_t const sp = pf_split_query(a.data(), n, q1.data(), q2.data(), len);
    int64_t d1 = 0, d2 = 0;
    for (uint32_t i = 0; i < n; ++i) { d1 += (int64_t)q1[i] * codes[i]; d2 += (int64_t)q2[i] * codes[i]; }
    float const dot = (float)((double)sp.sa1 * (double)d1 + (double)sp.sa2 * (double)d2);
    float const a2 = pinned_dot_f32_(a.data(), a.data(), n);
    for (float const rho_a : {sp.rho_a, 0.0f, INFINITY, NAN, -1.0f}) {
        pf_query_bound_t const q = pf_query_bound(a2, n, rho_a);
        compare("cos", n, pf_cos_lower(dot, r.s, r.rho, a2, r.b2, n, rho_a), pf_cos_lower_q(dot, r.s, r.rho, r.b2, q));
        compare("ip", n, pf_ip_lower(dot, r.s, r.rho, a2, r.bnorm, n, rho_a), pf_ip_lower_q(dot, r.s, r.rho, r.bnorm, q));
    }
}

int main(int argc, char** argv) {
    uint64_t const pairs = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 10000000ull;
    uint64_t state = 42;
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
            b[i] = eps == 1.f ? noise * sb : (a[i] + eps * noise) * sb;
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
        check_pair(z, z);
        check_pair(z, h);
        check_pair(h, z);
        check_pair(h, h);
        check_pair(h, h2);
        for (uint32_t i = 0; i < n; ++i) {
            w[i] = std::ldexp(unif(rng), (int)(i % 60) - 30);
            sub[i] = std::ldexp(unif(rng), -140 + (int)(i % 10));
            big[i] = std::ldexp(unif(rng), 60);
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
    std::printf("bounds compared: %llu random + %llu adversarial; failures: %llu\n", (unsigned long long)random_checked,
                (unsigned long long)(checked - random_checked), (unsigned long long)failures);
    return failures ? 1 : 0;
}
