/*
 *  cuda_check.h — the one place that turns a cudaError_t into the library's error text, and CU(), which returns that
 *  text from the calling function.
 */
#pragma once
#include <cuda_runtime_api.h>

#include <cstdio>

namespace usearch_b200 {

inline char const* cuda_error(cudaError_t e) {
    if (e == cudaSuccess) return nullptr;
    cudaGetLastError();
    if (e == cudaErrorMemoryAllocation) return "Out of GPU memory!";
    static thread_local char message[160];
    std::snprintf(message, sizeof(message), "CUDA failure: %s", cudaGetErrorString(e));
    return message;
}

} // namespace usearch_b200

#define CU(call)                                                              \
    do {                                                                      \
        if (char const* err_ = ::usearch_b200::cuda_error((call))) return err_; \
    } while (0)
