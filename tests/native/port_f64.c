/*
 *  tests/native/port_f64.c — the plain-C port of the reference's search (oracle/hnsw_oracle.c, included unchanged) over
 *  f64 graphs, with the metric of tests/native/f64_pinned.h. Needs no reference sources, so it also runs where only the
 *  repository is. Build: cc -O2 -ffp-contract=off -I oracle -I tests/native -shared -fPIC port_f64.c -lm -lpthread.
 *
 *  The port's blob parser knows the f64 row width (bits_per_scalar) but has no f64 metric. `oracle_open_f64` lets it parse
 *  a private copy of the blob whose head names f32 rows of twice the dimensions (the same bytes per row, so every offset
 *  is the same), then puts the f64 kind, the real dimensions and the f64 metric back. The search path itself is the
 *  port's, untouched.
 */
#include "../../oracle/hnsw_oracle.c"

#include "f64_pinned.h"

static float wrap_l2sq_f64(void const* a, void const* b, size_t n) { return pinned_l2sq_f64((double const*)a, (double const*)b, n); }
static float wrap_ip_f64(void const* a, void const* b, size_t n) { return pinned_ip_f64((double const*)a, (double const*)b, n); }
static float wrap_cos_f64(void const* a, void const* b, size_t n) { return pinned_cos_f64((double const*)a, (double const*)b, n); }

oracle_index_t* oracle_open_f64(void const* buffer, size_t length, char const** error) {
    *error = NULL;
    if (length < 8 + 64 + 40) { *error = "File is corrupted and lacks matrix dimensions"; return NULL; }
    uint8_t* copy = (uint8_t*)malloc(length);
    if (!copy) { *error = "Out of memory!"; return NULL; }
    memcpy(copy, buffer, length);
    uint64_t const head = 8 + (uint64_t)rd_u32(copy) * rd_u32(copy + 4);
    if (head + 64 + 40 > length || copy[head + 14] != SK_F64) { free(copy); *error = "Not an f64 index"; return NULL; }
    uint8_t const metric = copy[head + 13];
    oracle_metric_t const fn = metric == 'e' ? wrap_l2sq_f64 : metric == 'i' ? wrap_ip_f64 : metric == 'c' ? wrap_cos_f64 : NULL;
    if (!fn) { free(copy); *error = "Unknown metric kind!"; return NULL; }
    uint64_t const dims = rd_u64(copy + head + 33), twice = 2 * dims;
    copy[head + 14] = SK_F32;
    memcpy(copy + head + 33, &twice, 8);
    oracle_index_t* ix = oracle_open(copy, length, error);
    if (!ix) { free(copy); return NULL; }
    ix->scalar_kind = SK_F64;
    ix->dimensions = dims;
    ix->metric = fn;
    ix->metric_third = dims;
    return ix;
}

void oracle_close_f64(oracle_index_t* ix) {
    if (!ix) return;
    free((void*)ix->blob);
    oracle_close(ix);
}
