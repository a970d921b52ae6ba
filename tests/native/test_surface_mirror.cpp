// C++11 client of the reading-back surface of include/usearch_b200.hpp: `get` for many keys, `export_keys`, `copy()` and
// the three `stats` functions, shaped like index_dense_gt's. Usage: test_surface_mirror <index.usearch>. Prints
// SURFACE_MIRROR_OK when every check holds.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "usearch_b200.hpp"

#define CHECK(cond)                                                                    \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);     \
            return 1;                                                                  \
        }                                                                              \
    } while (0)

using namespace usearch_b200;

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    index_dense_t::state_result_t state = index_dense_t::make(argv[1]);
    CHECK(state);
    index_dense_t& index = state.index;
    std::size_t const n = index.size(), dims = index.dimensions();
    CHECK(n > 0);

    std::vector<vector_key_t> keys(n + 1);
    index.export_keys(keys.data(), 0, n);
    keys[n] = 0xFFFFFFFFFFFFFFF0ull; /* absent */

    /* many keys at once == one key at a time */
    std::vector<float> many((n + 1) * dims), one(dims);
    std::vector<std::size_t> counts(n + 1);
    std::size_t const rows = index.get(keys.data(), n + 1, many.data(), counts.data());
    CHECK(rows == n && counts[n] == 0);
    for (std::size_t i = 0; i < n; i += 97) {
        CHECK(counts[i] == 1);
        CHECK(index.get(keys[i], one.data()) == 1);
        CHECK(std::memcmp(one.data(), many.data() + i * dims, dims * sizeof(float)) == 0);
    }

    /* stats: the total equals the per-level sum; stats(level) adds the 10-byte head above level 0 */
    index_dense_t::stats_t const total = index.stats();
    std::size_t const top = index.max_level();
    std::vector<index_dense_t::stats_t> per(top + 1);
    index_dense_t::stats_t const sum = index.stats(per.data(), top);
    CHECK(total.nodes == n && sum.nodes >= n && total.edges == sum.edges && total.max_edges == sum.max_edges);
    CHECK(total.allocated_bytes == sum.allocated_bytes);
    for (std::size_t l = 0; l <= top; ++l) {
        index_dense_t::stats_t const s = index.stats(l);
        CHECK(s.nodes == per[l].nodes && s.edges == per[l].edges);
        CHECK(s.allocated_bytes == per[l].allocated_bytes + (l ? 10 * s.nodes : 0));
    }
    CHECK(index.stats(top + 1).nodes == 0);

    /* copy: same file, and it outlives the original */
    index_dense_t::state_result_t copied = index.copy();
    CHECK(copied);
    std::size_t const length = index.serialized_length();
    CHECK(copied.index.serialized_length() == length);
    std::vector<unsigned char> a(length), b(length);
    usearch_error_t error = nullptr;
    usearch_save_buffer(index.native_handle(), a.data(), length, &error);
    CHECK(!error);
    usearch_save_buffer(copied.index.native_handle(), b.data(), length, &error);
    CHECK(!error);
    CHECK(a == b);
    { index_dense_t gone(std::move(index)); }
    CHECK(copied.index.get(keys[0], one.data()) == 1);
    CHECK(std::memcmp(one.data(), many.data(), dims * sizeof(float)) == 0);
    CHECK(copied.index.stats().edges == total.edges && !copied.index.multi());

    std::printf("SURFACE_MIRROR_OK\n");
    return 0;
}
