// C++11 client of exact filtered search through include/usearch_b200.hpp: the set-based batch forms and the reference's
// own `filtered_search(vector, wanted, predicate, thread, exact)`. Compiled, not run: the calls need a GPU.
#include <cstdint>

#include "usearch_b200.hpp"

using namespace usearch_b200;

struct even_keys_t {
    bool operator()(vector_key_t key) const { return key % 2 == 0; }
};

int ground_truth(index_dense_t const& index, float const* queries, std::size_t n, std::uint32_t const* groups, std::uint64_t const* offsets,
                 std::size_t sets, vector_key_t const* set_keys, vector_key_t* found, distance_t* distances, std::size_t* counts,
                 std::uint32_t* d_counts, void* stream) {
    std::size_t const stride = index.dimensions() * sizeof(float);
    std::uint64_t computed[4] = {0, 0, 0, 0};
    if (error_t e = index.grouped_filtered_exact_search(queries, n, stride, 10, groups, offsets, sets, set_keys, found, distances, counts,
                                                         computed))
        return 1;
    // one set, no groups
    if (error_t e = index.grouped_filtered_exact_search(queries, n, stride, 10, nullptr, offsets, 1, set_keys, found, distances, counts))
        return 2;
    if (error_t e = index.grouped_filtered_exact_search_device(queries, n, stride, 10, groups, offsets, sets, set_keys, found, distances,
                                                               d_counts, nullptr, stream))
        return 3;
    // the reference's signature: a predicate object, and a lambda
    index_dense_t::search_result_t exact = index.filtered_search(queries, 10, even_keys_t(), 0, true);
    if (!exact) return 4;
    index_dense_t::search_result_t graph = index.filtered_search(queries, 10, [](vector_key_t key) { return key > 100; });
    if (!graph) return 5;
    // const lvalue predicates, as the reference accepts them, in both modes
    even_keys_t const even = even_keys_t();
    index_dense_t::search_result_t const_exact = index.filtered_search(queries, 10, even, 0, true);
    index_dense_t::search_result_t const_graph = index.filtered_search(queries, 10, even);
    return const_exact && const_graph ? 0 : 6;
}
