// C++11 client of the device lookups of include/usearch_b200.hpp: every pointer below stands for device memory that a
// caller's pipeline filled (search results, a model's filter set). Compiled, not run: the calls need a GPU.
#include <cstdint>

#include "usearch_b200.hpp"

using namespace usearch_b200;

int lookups(index_dense_t const& index, vector_key_t const* d_keys, std::size_t n, float* d_rows,
            std::uint32_t* d_counts, float const* d_queries, vector_key_t const* d_allowed, std::size_t allowed,
            vector_key_t* d_found, distance_t* d_distances, void* stream) {
    if (error_t e = index.count_device(d_keys, n, d_counts, stream)) return 1;
    if (error_t e = index.get_device(d_keys, n, d_rows, d_counts)) return 2;
    if (error_t e = index.get_device(d_keys, n, d_rows, d_counts, 4, index.dimensions() * sizeof(float) * 2, stream)) return 3;
    if (error_t e = index.filtered_search_device(d_queries, n, index.dimensions() * sizeof(float), 10, d_allowed, allowed, d_found,
                                                 d_distances, d_counts, nullptr, nullptr, stream))
        return 4;
    return 0;
}
