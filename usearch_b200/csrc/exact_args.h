/*
 *  exact_args.h — launch arguments shared by the exact-search kernels (exact_kernel.cu, exact_imma.cu, exact_wgmma.cu).
 */
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "device_index.h"

namespace usearch_b200 {

struct exact_args_t {
    uint8_t const* queries = nullptr; /* rows padded to vec_stride, index scalar kind */
    uint64_t query_stride = 0;
    uint32_t nq = 0, k = 0;
    uint32_t segments = 1, segment_len = 0; /* dataset cut into `segments` runs of `segment_len` slots (multiple of VPP) */
    float* part_d = nullptr;                /* [nq x segments x k] */
    uint32_t* part_s = nullptr;
    uint32_t* part_n = nullptr;             /* [nq x segments] */
    uint64_t* out_keys = nullptr;           /* [nq x k] */
    float* out_dists = nullptr;
    uint32_t* out_counts = nullptr;
    uint32_t stage_stride = 0, off_bars = 0, off_stage = 0;
    uint32_t slots_as_keys = 0;             /* 1: report the slot number as the key (free-function mode) */
    uint32_t off_queries = 0;               /* tiled kernel: queries region precedes the barriers */
    int const* query_norms = nullptr;       /* IMMA kernel (i8): sum of squares per query / per stored vector */
    int const* vector_norms = nullptr;
};

/* exact_imma.cu: i8 on the tensor cores */
size_t exact_imma_smem_bytes();
int exact_imma_tile_queries();
int exact_imma_tile_vectors();
cudaError_t exact_imma_self_dots(uint8_t const* rows, uint64_t stride, uint32_t chunks16, uint32_t count, int* out, cudaStream_t stream);
cudaError_t exact_imma_launch(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, cudaStream_t stream);

/* exact_wgmma.cu: the same scan on warpgroup MMAs (wgmma, TMA operand loads) */
size_t exact_wgmma_smem_bytes();
int exact_wgmma_tile_queries();
int exact_wgmma_tile_vectors();
bool exact_wgmma_usable(device_index_t const& ix, exact_args_t const& a);
cudaError_t exact_wgmma_launch(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, cudaStream_t stream);

} // namespace usearch_b200
