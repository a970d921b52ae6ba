/*
 *  The wgmma exact scan's integer filter (usearch_b200/csrc/exact_i8.h, i8_filter_t) against the i8 distances it guards:
 *  for ip, l2sq and cos, in both operand orders, every column whose distance is <= the list's worst must pass the filter
 *  (a tie at the worst enters the list when its slot is larger). The distances themselves (i8_distance) are held equal,
 *  bit for bit, to the pinned reference metrics (oracle/metrics_pinned.h) on every triple.
 *  Triples (ab, a2, b2) of vectors of d <= 8192 elements in [-128, 127]: 10^7 random ones at every magnitude, then
 *  adversarial families: a constructed tie at cos distance 0.99996, worst in (0.99, 1), worst = 0 (duplicates and scaled
 *  copies, p >= 1 clamped), zero norms, and saturated rows whose sums pass 2^24.
 *  Build: g++ -O2 -ffp-contract=off -std=c++17 -I oracle -I usearch_b200/csrc; run: ./a.out [triples]
 */
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>

#include "exact_i8.h"
#include "metrics_pinned.h"

using namespace usearch_b200;

static uint64_t checked = 0, entered = 0, failures = 0;

static uint32_t bits(float x) {
    uint32_t u;
    std::memcpy(&u, &x, 4);
    return u;
}

/* the reference's distance of the pair: metric(query, stored), or metric(stored, query) under SWAP */
template <uint32_t METRIC, bool SWAP> static float reference(int ab, int qa2, int vb2) {
    if (METRIC == METRIC_IP) return 1.0f - (float)ab;
    if (METRIC == METRIC_L2SQ) return (float)(qa2 + vb2 - 2 * ab);
    return SWAP ? pinned_cos_normalize_f32((float)ab, (float)vb2, (float)qa2) : pinned_cos_normalize_f32((float)ab, (float)qa2, (float)vb2);
}

static char const* name(uint32_t metric) { return metric == METRIC_IP ? "ip" : (metric == METRIC_L2SQ ? "l2sq" : "cos"); }

/* one column (ab, vb2) of the query row qa2 against a full list whose worst entry is `worst` */
template <uint32_t METRIC, bool SWAP> static void check_one(int ab, int qa2, int vb2, float worst) {
    float const qr = i8_rnorm(qa2), vr = i8_rnorm(vb2);
    float const d = i8_distance<METRIC, SWAP>(ab, qa2, vb2, qr, vr);
    ++checked;
    float const want = reference<METRIC, SWAP>(ab, qa2, vb2);
    if (bits(d) != bits(want)) {
        if (failures < 20)
            std::printf("FAIL distance %s swap=%d ab=%d a2=%d b2=%d: %a (0x%08x), reference %a (0x%08x)\n", name(METRIC), (int)SWAP, ab, qa2,
                        vb2, d, bits(d), want, bits(want));
        ++failures;
    }
    if (!(d <= worst)) return;
    ++entered;
    i8_filter_t<METRIC> f;
    f.set_thresholds(1, 1, worst, qa2, qr);
    if (!f.maybe(ab, vb2, vr)) {
        if (failures < 20)
            std::printf("FAIL filter %s swap=%d ab=%d a2=%d b2=%d: d=%.9g (0x%08x) <= worst=%.9g (0x%08x) but rejected (thr_i=%d thr_f=%a)\n",
                        name(METRIC), (int)SWAP, ab, qa2, vb2, d, bits(d), worst, bits(worst), f.thr_i, f.thr_f);
        ++failures;
    }
}

template <uint32_t METRIC, bool SWAP> static float dist(int ab, int qa2, int vb2) {
    return i8_distance<METRIC, SWAP>(ab, qa2, vb2, i8_rnorm(qa2), i8_rnorm(vb2));
}

/* the column against a list whose worst is its own distance (the tie), one ulp above it, and `other` (another column's
 * distance for the same query row) */
template <uint32_t METRIC, bool SWAP> static void check_worsts(int ab, int qa2, int vb2, float other) {
    float const d = dist<METRIC, SWAP>(ab, qa2, vb2);
    check_one<METRIC, SWAP>(ab, qa2, vb2, d);
    check_one<METRIC, SWAP>(ab, qa2, vb2, std::nextafterf(d, INFINITY));
    check_one<METRIC, SWAP>(ab, qa2, vb2, other);
}

static void check_all(int ab, int qa2, int vb2, int ab2, int vb2b) {
    /* `other` comes from a second column (ab2, vb2b) of the same query row */
    check_worsts<METRIC_IP, false>(ab, qa2, vb2, dist<METRIC_IP, false>(ab2, qa2, vb2b));
    check_worsts<METRIC_IP, true>(ab, qa2, vb2, dist<METRIC_IP, true>(ab2, qa2, vb2b));
    check_worsts<METRIC_L2SQ, false>(ab, qa2, vb2, dist<METRIC_L2SQ, false>(ab2, qa2, vb2b));
    check_worsts<METRIC_L2SQ, true>(ab, qa2, vb2, dist<METRIC_L2SQ, true>(ab2, qa2, vb2b));
    check_worsts<METRIC_COS, false>(ab, qa2, vb2, dist<METRIC_COS, false>(ab2, qa2, vb2b));
    check_worsts<METRIC_COS, true>(ab, qa2, vb2, dist<METRIC_COS, true>(ab2, qa2, vb2b));
}

int main(int argc, char** argv) {
    uint64_t const triples = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 10000000ull;
    uint64_t state = 7;
    auto rng = [&]() { /* splitmix64 */
        uint64_t z = (state += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    };
    auto unit = [&]() { return (double)(rng() >> 11) * 0x1p-53; }; /* [0, 1) */
    /* a squared norm of a d-element row: log-uniform up to 128^2 d, sometimes exactly 0 or the saturated maximum */
    auto norm2 = [&](int d) -> int {
        uint64_t const r = rng() % 64;
        if (r == 0) return 0;
        if (r == 1) return 16384 * d;
        if (r == 2) return 16129 * d;
        return (int)std::floor(std::exp2(unit() * std::log2(16384.0 * d)));
    };
    /* a dot product the two norms allow: |ab| <= sqrt(a2 b2), near the bound, near 0, or anywhere between */
    auto dot = [&](int a2, int b2) -> int {
        double const lim = std::floor(std::sqrt((double)a2 * (double)b2));
        uint64_t const r = rng() % 4;
        double x;
        if (r == 0) x = lim - (double)(rng() % 64);                  /* near-duplicates */
        else if (r == 1) x = (double)(rng() % 200) - 100.0;          /* near-orthogonal: cos distance near 1 */
        else if (r == 2) x = lim * unit() * unit();                  /* small correlations */
        else x = lim * unit();
        x = x > lim ? lim : (x < 0 && a2 * (double)b2 == 0 ? 0 : x);
        if (x < -lim) x = -lim;
        return (rng() & 1) ? (int)x : -(int)x;
    };
    for (uint64_t t = 0; t < triples; ++t) {
        int const d = 1 + (int)(rng() % 8192);
        int const qa2 = norm2(d), vb2 = norm2(d), vb2b = norm2(d);
        check_all(dot(qa2, vb2), qa2, vb2, dot(qa2, vb2b), vb2b);
    }
    uint64_t const random_checked = checked;

    /* the constructed tie (d = 128): q = 127 x 63, 1; W and C share the cos distance 0.9999571 with the query */
    {
        int const qa2 = 63 * 127 * 127 + 1, ab_w = 33, b2_w = 33 * 33 + 36 * 127 * 127 + 2 * 18 * 18;
        int const ab_c = 43, b2_c = 43 * 43 + 61 * 127 * 127 + 23 * 23 + 51 * 51;
        check_all(ab_c, qa2, b2_c, ab_w, b2_w);
        check_all(ab_w, qa2, b2_w, ab_c, b2_c);
        if (bits(dist<METRIC_COS, false>(ab_w, qa2, b2_w)) != bits(dist<METRIC_COS, false>(ab_c, qa2, b2_c))) {
            std::printf("FAIL: the constructed pair does not tie\n");
            ++failures;
        }
    }
    /* worst in (0.99, 1): small positive correlations of long rows, every column tied or nearly tied with its neighbour */
    for (int rep = 0; rep < 2000000; ++rep) {
        int const d = 16 + (int)(rng() % 8177);
        int const qa2 = 1 + (int)(unit() * 16129.0 * d), vb2 = 1 + (int)(unit() * 16129.0 * d);
        double const lim = std::sqrt((double)qa2 * vb2);
        int const ab = 1 + (int)(lim * 0.01 * unit());
        check_all(ab, qa2, vb2, ab + (int)(rng() % 3) - 1, vb2 + (int)(rng() % 2001) - 1000);
    }
    /* worst = 0: duplicates and positive multiples (the clamp at p >= 1), and their opposites (cos 2) */
    for (int d : {1, 15, 16, 17, 128, 129, 1040, 4096, 8192}) {
        for (int rep = 0; rep < 2000; ++rep) {
            int const a2 = 1 + (int)(rng() % (16384ull * d));
            int const m = 1 + (int)(rng() % 4);
            long long const b2 = (long long)a2 * m * m;
            if (b2 > 16384ll * d) continue;
            check_all(a2 * m, a2, (int)b2, a2, a2);
            check_all(-a2 * m, a2, (int)b2, a2, a2);
            check_all(a2, a2, a2, a2 * m, (int)b2);
        }
    }
    /* zero norms: zero query, zero row, both (cos 0/0 -> 0, ab = 0 -> 1, ip -> 1) */
    for (int d : {1, 16, 128, 4096, 8192}) {
        for (int x2 : {1, 127 * 127, 16129 * d, 16384 * d}) {
            check_all(0, 0, x2, 0, 0);
            check_all(0, x2, 0, 0, x2);
            check_all(0, 0, 0, 0, x2);
            check_all(0, x2, x2, x2, x2);
            check_all(0, 0, 0, 0, 0);
        }
    }
    /* saturated rows whose sums pass 2^24: all -128, all 127, alternating, against each other, and one unit apart */
    for (int d = 1024; d <= 8192; d += 16) {
        int const n128 = 16384 * d, n127 = 16129 * d, nmix = (16384 + 16129) / 2 * d - (d & 1 ? 16129 / 2 : 0);
        int const rows[3] = {n128, n127, nmix};
        int const dots[][3] = {
            {n128, n128, n128},         /* -128 . -128 */
            {-128 * 127 * d, n128, n127}, /* -128 . 127 */
            {n127, n127, n127},         /* 127 . 127 */
            {-n127, n127, n127},        /* 127 . -127 */
        };
        for (auto const& t : dots)
            for (int j = -8; j <= 8; ++j) {
                int const ab = t[0] + j;
                if ((double)ab * ab > (double)t[1] * t[2]) continue;
                check_all(ab, t[1], t[2], t[0], t[2]);
                check_all(ab, t[1], t[2], t[0] - j, t[2]);
            }
        for (int a : rows)
            for (int b : rows)
                for (int j = 0; j < 64; ++j) {
                    int const ab = (int)std::floor(std::sqrt((double)a * b)) - j * 97;
                    check_all(ab, a, b, ab + 1, b);
                    check_all(-ab, a, b, -ab - 1, b);
                }
    }
    std::printf("columns checked: %llu random + %llu adversarial (3 metrics x 2 orders x 3 worsts each); inside the worst: %llu; "
                "failures: %llu\n",
                (unsigned long long)random_checked, (unsigned long long)(checked - random_checked), (unsigned long long)entered,
                (unsigned long long)failures);
    return failures ? 1 : 0;
}
