// C++11 client of the free exact search through include/usearch_b200.hpp: host matrices of any size, and device
// matrices on a caller's stream. Compiled, not run: the calls need a GPU.
#include <cstdint>

#include "usearch_b200.hpp"

using namespace usearch_b200;

int ground_truth(float const* dataset, std::size_t n, float const* queries, std::size_t nq, std::size_t dims, vector_key_t* keys,
                 distance_t* distances, void const* d_dataset, void const* d_queries, vector_key_t* d_keys, distance_t* d_distances,
                 void* stream) {
    std::size_t const stride = dims * sizeof(float);
    if (error_t e = exact_search(dataset, n, stride, queries, nq, stride, dims, usearch_metric_cos_k, 10, keys, 10 * sizeof(vector_key_t),
                                 distances, 10 * sizeof(distance_t)))
        return 1;
    // with four host threads staging the rows
    if (error_t e = exact_search(dataset, n, stride, queries, nq, stride, dims, usearch_metric_l2sq_k, 10, keys, 10 * sizeof(vector_key_t),
                                 distances, 10 * sizeof(distance_t), 4))
        return 2;
    if (error_t e = exact_search_device(d_dataset, n, stride, d_queries, nq, stride, usearch_scalar_f32_k, dims, usearch_metric_ip_k, 10,
                                        d_keys, 0, d_distances, 0, stream))
        return 3;
    // the default stream
    error_t e = exact_search_device(d_dataset, n, stride, d_queries, nq, stride, usearch_scalar_f32_k, dims, usearch_metric_ip_k, 10,
                                    d_keys, 0, d_distances, 0);
    return e ? 4 : 0;
}
