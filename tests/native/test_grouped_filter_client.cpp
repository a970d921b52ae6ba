// C++11 client of grouped filtered search through include/usearch_b200.hpp: a tenant's queries, each with the key set of
// its tenant, as CSR. Compiled, not run: the calls need a GPU.
#include <cstdint>

#include "usearch_b200.hpp"

using namespace usearch_b200;

int tenants(index_dense_t const& index, float const* queries, std::size_t n, std::uint32_t const* groups, std::uint64_t const* offsets,
            std::size_t sets, vector_key_t const* set_keys, vector_key_t* found, distance_t* distances, std::size_t* counts,
            std::uint32_t* d_counts, void* stream) {
    std::size_t const stride = index.dimensions() * sizeof(float);
    if (error_t e = index.grouped_filtered_search(queries, n, stride, 10, groups, offsets, sets, set_keys, found, distances, counts))
        return 1;
    std::uint64_t computed = 0, visited = 0;
    if (error_t e = index.grouped_filtered_search(queries, 1, 0, 10, groups, offsets, sets, set_keys, found, distances, counts, &computed,
                                                  &visited))
        return 2;
    // the same arrays as device pointers
    if (error_t e = index.grouped_filtered_search_device(queries, n, stride, 10, groups, offsets, sets, set_keys, found, distances,
                                                         d_counts, nullptr, nullptr, stream))
        return 3;
    return 0;
}
