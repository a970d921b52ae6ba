/*
 *  Host emulation of the f64 metric structs (usearch_b200/csrc/metrics.cuh): four lanes share a vector, lane `s` reads
 *  the 16-byte chunks s, s+4, ... (two doubles each) into accumulators 2s and 2s+1, and the group reduces with an xor-2
 *  then an xor-1 exchange before adding its two halves. The result must equal tests/native/f64_pinned.h, which follows
 *  the reference's 8-accumulator order, bit for bit, for every length including ragged ones (a zero-padded last chunk).
 *  Build: cc -O2 -ffp-contract=off test_f64_lanes_order.c -lm. Exit status 0 on success.
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "f64_pinned.h"

enum { L2SQ, IP, COS };

/* one lane group: acc[s][0..1] are lane s's two accumulators */
static double reduce_group(double acc[4][2]) {
    double a[4], b[4], a2[4], b2[4];
    for (int s = 0; s < 4; ++s) { a[s] = acc[s][0] + acc[s ^ 2][0]; b[s] = acc[s][1] + acc[s ^ 2][1]; } /* xor 2 */
    for (int s = 0; s < 4; ++s) { a2[s] = a[s] + a[s ^ 1]; b2[s] = b[s] + b[s ^ 1]; }                 /* xor 1 */
    double r = a2[0] + b2[0];
    for (int s = 1; s < 4; ++s) /* every lane of the group holds the same bits */
        if (memcmp(&r, &(double){a2[s] + b2[s]}, 8) != 0) { fprintf(stderr, "lanes disagree\n"); exit(2); }
    return r;
}

static float lanes(int metric, double const* q, double const* v, size_t n) {
    size_t const chunks = (n + 1) / 2;
    double ab[4][2] = {{0}}, bb[4][2] = {{0}}, qq[4][2] = {{0}};
    for (int s = 0; s < 4; ++s)
        for (size_t j = (size_t)s; j < chunks; j += 4)
            for (int h = 0; h < 2; ++h) {
                size_t const i = 2 * j + (size_t)h;
                double const x = i < n ? q[i] : 0.0, y = i < n ? v[i] : 0.0; /* zero padding of the last chunk */
                if (metric == L2SQ) { double const d = x - y; ab[s][h] = fma(d, d, ab[s][h]); }
                else {
                    ab[s][h] = fma(x, y, ab[s][h]);
                    bb[s][h] = fma(y, y, bb[s][h]);
                    qq[s][h] = fma(x, x, qq[s][h]);
                }
            }
    double const sab = reduce_group(ab);
    if (metric == L2SQ) return (float)sab;
    if (metric == IP) return 1.0f - (float)sab;
    double const sb2 = reduce_group(bb), sa2 = reduce_group(qq);
    if (sa2 == 0 && sb2 == 0) return 0.f;
    if (sab == 0) return 1.f;
    double const r = 1.0 - (sab * (1.0 / sqrt(sa2))) * (1.0 / sqrt(sb2));
    return r > 0 ? (float)r : 0.f;
}

static double gauss(void) {
    double u = (rand() + 1.0) / ((double)RAND_MAX + 2.0), w = (rand() + 1.0) / ((double)RAND_MAX + 2.0);
    return sqrt(-2.0 * log(u)) * cos(6.283185307179586 * w);
}

int main(void) {
    srand(7);
    size_t const lengths[] = {1, 2, 3, 7, 8, 9, 15, 16, 17, 24, 31, 33, 97, 128, 255, 768, 769, 3200};
    static double q[4096], v[4096];
    size_t checked = 0;
    for (size_t li = 0; li < sizeof lengths / sizeof *lengths; ++li)
        for (int trial = 0; trial < 20; ++trial) {
            size_t const n = lengths[li];
            double const scale = trial % 3 == 0 ? 1e-3 : (trial % 3 == 1 ? 1.0 : 1e4);
            for (size_t i = 0; i < n; ++i) { q[i] = scale * gauss(); v[i] = trial == 19 ? q[i] : scale * gauss(); }
            float const want[3] = {pinned_l2sq_f64(q, v, n), pinned_ip_f64(q, v, n), pinned_cos_f64(q, v, n)};
            for (int m = 0; m < 3; ++m) {
                float const got = lanes(m, q, v, n);
                if (memcmp(&got, &want[m], 4) != 0) {
                    fprintf(stderr, "metric %d, n %zu, trial %d: %.9g != %.9g\n", m, n, trial, got, want[m]);
                    return 1;
                }
                ++checked;
            }
        }
    printf("%zu distances equal\n", checked);
    return 0;
}
