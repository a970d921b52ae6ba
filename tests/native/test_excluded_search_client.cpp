// C++11 client of excluded search through include/usearch_b200.hpp: the graph and exact forms, host and device. Compiled,
// not run: the calls need a GPU.
#include <cstdint>

#include "usearch_b200.hpp"

using namespace usearch_b200;

int not_these(index_dense_t const& index, float const* queries, std::size_t n, std::uint32_t const* groups, std::uint64_t const* offsets,
              std::size_t sets, vector_key_t const* set_keys, vector_key_t* found, distance_t* distances, std::size_t* counts,
              std::uint32_t* d_counts, void* stream) {
    std::size_t const stride = index.dimensions() * sizeof(float);
    std::uint64_t computed[4] = {0, 0, 0, 0}, visited[4] = {0, 0, 0, 0};
    if (error_t e = index.grouped_excluded_search(queries, n, stride, 10, groups, offsets, sets, set_keys, found, distances, counts, computed,
                                                  visited))
        return 1;
    // one set, no groups
    if (error_t e = index.grouped_excluded_search(queries, n, stride, 10, nullptr, offsets, 1, set_keys, found, distances, counts))
        return 2;
    if (error_t e = index.grouped_excluded_search_device(queries, n, stride, 10, groups, offsets, sets, set_keys, found, distances, d_counts,
                                                         nullptr, nullptr, stream))
        return 3;
    if (error_t e = index.grouped_excluded_exact_search(queries, n, stride, 10, groups, offsets, sets, set_keys, found, distances, counts,
                                                        computed))
        return 4;
    if (error_t e = index.grouped_excluded_exact_search_device(queries, n, stride, 10, nullptr, offsets, 1, set_keys, found, distances,
                                                               d_counts, nullptr, stream))
        return 5;
    return 0;
}
