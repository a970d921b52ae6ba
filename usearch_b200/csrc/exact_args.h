/*
 *  exact_args.h — launch arguments shared by the exact-search kernels (exact_kernel.cu, exact_imma.cu, exact_wgmma.cu).
 */
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

#include "device_index.h"

namespace usearch_b200 {

/* one CTA row of a listed launch: `count` queries from `first` (sorted by set) against one set's ascending slot list */
struct exact_item_t {
    uint32_t first, count, list_begin, list_len;
};

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

/* the LISTED kernels' arguments (exact filtered search): the fields above, then the lists. CTA x serves items[x], whose
 * queries are `first ..` of the gathered batch and whose rows are slots rows[list_begin ..]; each list is cut into
 * `segments` runs of ceil(len / segments) rounded up to the tile, and vector_norms is indexed by list position. The
 * kernels that serve every slot, and the merge, keep exact_args_t itself. */
struct exact_listed_args_t : exact_args_t {
    exact_item_t const* items = nullptr;
    uint32_t const* rows = nullptr;
};
template <bool LISTED> using exact_args_of = typename std::conditional<LISTED, exact_listed_args_t, exact_args_t>::type;

/* positions [lo, hi) of segment `seg` of a listed item, segments a multiple of `tile` long */
__device__ __forceinline__ void listed_segment(exact_item_t const& it, uint32_t segments, uint32_t seg, uint32_t tile, uint32_t& lo,
                                               uint32_t& hi) {
    uint32_t len = (it.list_len + segments - 1) / segments;
    len = (len + tile - 1) / tile * tile;
    lo = min(it.list_len, seg * len);
    hi = min(it.list_len, lo + len);
}

/* exact_imma.cu: i8 on the tensor cores */
size_t exact_imma_smem_bytes();
int exact_imma_tile_queries();
int exact_imma_tile_vectors();
cudaError_t exact_imma_self_dots(uint8_t const* rows, uint64_t stride, uint32_t chunks16, uint32_t count, int* out, cudaStream_t stream);
cudaError_t exact_imma_launch(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, cudaStream_t stream);
/* listed (exact filtered) twins: b2 of slots rows[0 .. count) by list position, and the LISTED kernel (metric(query, stored)) */
cudaError_t exact_imma_listed_self_dots(uint8_t const* vectors, uint64_t stride, uint32_t chunks16, uint32_t const* rows, uint32_t count,
                                        int* out, cudaStream_t stream);
cudaError_t exact_imma_listed_launch(device_index_t const& ix, exact_listed_args_t const& a, dim3 grid, cudaStream_t stream);

/* exact_wgmma.cu: the same scan on warpgroup MMAs (wgmma, TMA operand loads) */
size_t exact_wgmma_smem_bytes();
int exact_wgmma_tile_queries();
int exact_wgmma_tile_vectors();
bool exact_wgmma_usable(device_index_t const& ix, exact_args_t const& a);
cudaError_t exact_wgmma_launch(device_index_t const& ix, exact_args_t const& a, bool swap, dim3 grid, cudaStream_t stream);

} // namespace usearch_b200
