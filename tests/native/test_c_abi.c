/*
 *  C99 client of the drop-in C ABI, in the spirit of the reference's c/test.c (init / load / search /
 *  save-load sections, c/test.c:52-391), restricted to the search path.
 *
 *  usage: test_c_abi <index.usearch> <cases.bin>
 *  cases.bin: u64 nq, u64 dims, u64 k, f32 queries[nq*dims], u64 keys[nq*k], f32 distances[nq*k], u64 counts[nq]
 *             (the expected rows come from the oracle at the index's default expansion of 64)
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "usearch_b200.h"

#define EXPECT(cond)                                                          \
    do {                                                                      \
        if (!(cond)) {                                                        \
            fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            return 1;                                                         \
        }                                                                     \
    } while (0)

static int even_keys_only(usearch_key_t key, void* state) { (void)state; return key % 2 == 0; }

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    usearch_error_t error = NULL;

    /* metadata sniffing (usearch.h:186) */
    usearch_init_options_t meta;
    usearch_metadata(argv[1], &meta, &error);
    EXPECT(!error);
    EXPECT(meta.metric_kind == usearch_metric_cos_k && meta.quantization == usearch_scalar_f32_k);

    FILE* f = fopen(argv[2], "rb");
    EXPECT(f);
    unsigned long long nq, dims, k;
    EXPECT(fread(&nq, 8, 1, f) == 1 && fread(&dims, 8, 1, f) == 1 && fread(&k, 8, 1, f) == 1);
    EXPECT(meta.dimensions == dims);
    float* queries = (float*)malloc(nq * dims * 4);
    usearch_key_t* want_keys = (usearch_key_t*)malloc(nq * k * 8);
    float* want_dist = (float*)malloc(nq * k * 4);
    unsigned long long* want_counts = (unsigned long long*)malloc(nq * 8);
    EXPECT(fread(queries, 4, nq * dims, f) == nq * dims);
    EXPECT(fread(want_keys, 8, nq * k, f) == nq * k);
    EXPECT(fread(want_dist, 4, nq * k, f) == nq * k);
    EXPECT(fread(want_counts, 8, nq, f) == nq);
    fclose(f);

    /* init with NULL options = empty index awaiting load (c/lib.cpp:142-147) */
    usearch_index_t index = usearch_init(NULL, &error);
    EXPECT(index && !error);
    EXPECT(usearch_size(index, &error) == 0);
    usearch_load(index, argv[1], &error);
    EXPECT(!error);
    EXPECT(usearch_size(index, &error) > 0 && usearch_dimensions(index, &error) == dims);
    EXPECT(usearch_connectivity(index, &error) >= 2);
    EXPECT(strcmp(usearch_hardware_acceleration(index, &error), "sm_90a") == 0);
    EXPECT(usearch_memory_usage(index, &error) > 0);

    /* single-query searches, one call per query like Go / C# callers (golang/lib.go:628) */
    usearch_key_t* keys = (usearch_key_t*)malloc(k * 8);
    float* dist = (float*)malloc(k * 4);
    for (unsigned long long q = 0; q < nq && q < 16; ++q) {
        size_t found = usearch_search(index, queries + q * dims, usearch_scalar_f32_k, k, keys, dist, &error);
        EXPECT(!error && found == want_counts[q]);
        EXPECT(memcmp(keys, want_keys + q * k, k * 8) == 0);
        EXPECT(memcmp(dist, want_dist + q * k, k * 4) == 0);
        for (size_t i = 1; i < found; ++i) EXPECT(dist[i - 1] <= dist[i]); /* cpp/test.cpp:499-503 */
    }

    /* the additive batch entry: strided outputs */
    size_t const key_stride = (k + 3) * 8, dist_stride = (k + 1) * 4;
    char* keys_many = (char*)calloc(nq, key_stride);
    char* dist_many = (char*)calloc(nq, dist_stride);
    size_t* counts = (size_t*)malloc(nq * sizeof(size_t));
    size_t total = usearch_search_many(index, queries, nq, dims * 4, usearch_scalar_f32_k, k, (usearch_key_t*)keys_many,
                                       key_stride, (usearch_distance_t*)dist_many, dist_stride, counts, &error);
    EXPECT(!error);
    size_t expect_total = 0;
    for (unsigned long long q = 0; q < nq; ++q) {
        expect_total += want_counts[q];
        EXPECT(counts[q] == want_counts[q]);
        EXPECT(memcmp(keys_many + q * key_stride, want_keys + q * k, k * 8) == 0);
        EXPECT(memcmp(dist_many + q * dist_stride, want_dist + q * k, k * 4) == 0);
    }
    EXPECT(total == expect_total);

    /* count == 0 is an empty result, not an error (index.hpp:3025-3026) */
    EXPECT(usearch_search(index, queries, usearch_scalar_f32_k, 0, keys, dist, &error) == 0 && !error);

    /* save -> load into a second handle -> identical answers (c/test.c save/load section) */
    size_t length = usearch_serialized_length(index, &error);
    void* buffer = malloc(length);
    usearch_save_buffer(index, buffer, length, &error);
    EXPECT(!error);
    usearch_index_t copy = usearch_init(NULL, &error);
    usearch_load_buffer(copy, buffer, length, &error);
    EXPECT(!error && usearch_size(copy, &error) == usearch_size(index, &error));
    size_t found = usearch_search(copy, queries, usearch_scalar_f32_k, k, keys, dist, &error);
    EXPECT(!error && found == want_counts[0] && memcmp(keys, want_keys, k * 8) == 0 && memcmp(dist, want_dist, k * 4) == 0);
    usearch_free(copy, &error);

    /* a corrupted buffer is refused with the reference's message */
    memset(buffer, 0, 256);
    usearch_index_t broken = usearch_init(NULL, &error);
    usearch_load_buffer(broken, buffer, length, &error);
    EXPECT(error);
    error = NULL;
    usearch_free(broken, &error);

    /* lookups by key (c/test.c "contains/count/get" sections) */
    EXPECT(usearch_contains(index, want_keys[0], &error) && !error);
    EXPECT(usearch_count(index, want_keys[0], &error) == 1 && !error);
    EXPECT(!usearch_contains(index, 0xDEADBEEFull, &error) && !error);
    float* stored = (float*)malloc(dims * 4);
    EXPECT(usearch_get(index, want_keys[0], 1, stored, usearch_scalar_f32_k, &error) == 1 && !error);
    EXPECT(usearch_get(index, 0xDEADBEEFull, 1, stored, usearch_scalar_f32_k, &error) == 0 && !error);
    /* the closest match of query 0 is at the distance the index reports for that pair (usearch_distance) */
    {
        float d = usearch_distance(queries, stored, usearch_scalar_f32_k, dims, usearch_metric_cos_k, &error);
        EXPECT(!error && memcmp(&d, want_dist, 4) == 0);
    }

    /* a host predicate (c/test.c test_filtered_search): only even keys may be returned */
    {
        size_t found = usearch_filtered_search(index, queries, usearch_scalar_f32_k, k, even_keys_only, NULL, keys, dist, &error);
        EXPECT(!error && found > 0);
        for (size_t i = 0; i < found; ++i) EXPECT(keys[i] % 2 == 0);
    }

    /* add -> found -> remove -> gone (c/test.c test_add_vector / test_remove_vector) */
    {
        size_t const before = usearch_size(index, &error);
        usearch_key_t const fresh = 0x7000000000ull;
        usearch_add(index, fresh, queries, usearch_scalar_f32_k, &error);
        EXPECT(!error);
        EXPECT(usearch_size(index, &error) == before + 1 && usearch_contains(index, fresh, &error));
        size_t found = usearch_search(index, queries, usearch_scalar_f32_k, k, keys, dist, &error);
        EXPECT(!error && found >= 1 && keys[0] == fresh);
        usearch_add(index, fresh, queries, usearch_scalar_f32_k, &error); /* duplicates are refused (not a multi-index) */
        EXPECT(error);
        error = NULL;
        EXPECT(usearch_rename(index, fresh, fresh + 1, &error) == 1 && !error && usearch_contains(index, fresh + 1, &error));
        EXPECT(usearch_remove(index, fresh + 1, &error) == 1 && !error);
        EXPECT(usearch_remove(index, fresh + 1, &error) == 0 && !error);
        EXPECT(usearch_size(index, &error) == before && !usearch_contains(index, fresh + 1, &error));
        found = usearch_search(index, queries, usearch_scalar_f32_k, k, keys, dist, &error);
        EXPECT(!error);
        for (size_t i = 0; i < found; ++i) EXPECT(keys[i] != fresh + 1 && keys[i] != fresh);
    }
    free(stored);

    usearch_clear(index, &error);
    EXPECT(usearch_size(index, &error) == 0);
    usearch_free(index, &error);
    printf("C_ABI_OK %llu queries\n", nq);
    return 0;
}
