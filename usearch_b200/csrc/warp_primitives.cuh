/*
 *  warp_primitives.cuh — device helpers shared by the search and the exact-scan kernels: TMA bulk copies
 *  with mbarrier completion, and the register-resident sorted list that plays `sorted_buffer_gt`.
 */
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "search_order.h"

namespace usearch_b200 {

/* ---- TMA bulk copy + mbarrier (PTX ISA: cp.async.bulk, mbarrier.*) ---------------------------- */

__device__ __forceinline__ uint32_t smem_u32(void const* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, void const* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}

/*
 *  Register-resident `top` for ef <= 256, BLOCKED layout: lane l holds elements 8l .. 8l+7. The same
 *  sorted_buffer_gt::insert semantics (index.hpp:928-939); the right-shift costs one shuffle per array:
 *  element g receives element g-1, which is the previous register of the same lane or register 7 of
 *  the lane below.
 */
constexpr int TOP_E = 8;

/* element g of a register `top`: register g % TOP_E of lane g / TOP_E; every lane calls it with the same g */
__device__ __forceinline__ float top_at_reg(float const (&td)[TOP_E], uint32_t g) {
    uint32_t const r = g & (TOP_E - 1);
    float sel = td[0];
#pragma unroll
    for (int j = 1; j < TOP_E; ++j)
        if ((uint32_t)j == r) sel = td[j];
    return __shfl_sync(0xffffffffu, sel, (int)(g / TOP_E));
}

/* `has_nan` (uniform): `top` may hold a NaN, and only the probe of libstdc++'s lower_bound places d as the
 * reference does (search_order.h); without one, the count of smaller elements is that position */
__device__ __forceinline__ void top_insert_reg(float (&td)[TOP_E], uint32_t (&ts)[TOP_E], uint32_t& size, uint32_t limit,
                                               float d, uint32_t s, bool& has_nan, int lane) {
    uint32_t const g0 = (uint32_t)lane * TOP_E;
    uint32_t pos;
    if (!has_nan) {
        uint32_t mine = 0; /* lower_bound: number of stored distances strictly below d */
#pragma unroll
        for (int j = 0; j < TOP_E; ++j) mine += (g0 + j < size && td[j] < d) ? 1u : 0u;
        pos = __reduce_add_sync(0xffffffffu, mine);
    } else
        pos = probe_lower_bound([&td](uint32_t g) { return top_at_reg(td, g); }, size, d);
    if (pos == limit) return;
    has_nan = top_may_hold_nan(has_nan, d);
    bool const full = size == limit;
    uint32_t const hi = size - (full ? 1u : 0u); /* old [pos, hi) becomes new (pos, hi] */
    float const up_d = __shfl_up_sync(0xffffffffu, td[TOP_E - 1], 1);
    uint32_t const up_s = __shfl_up_sync(0xffffffffu, ts[TOP_E - 1], 1);
#pragma unroll
    for (int j = TOP_E - 1; j >= 0; --j) {
        uint32_t const g = g0 + (uint32_t)j;
        if (g > pos && g <= hi) {
            td[j] = j ? td[j > 0 ? j - 1 : 0] : up_d;
            ts[j] = j ? ts[j > 0 ? j - 1 : 0] : up_s;
        } else if (g == pos) {
            td[j] = d;
            ts[j] = s;
        }
    }
    size += full ? 0u : 1u;
}

/* distance of the last (worst) element: sorted_buffer_gt::top() (index.hpp:891) */
__device__ __forceinline__ float top_back_reg(float const (&td)[TOP_E], uint32_t size) { return top_at_reg(td, size - 1); }

/* The same insert under the TOTAL order (distance ascending, slot descending): what a sequence of
 * sorted_buffer_gt::insert calls in ascending slot order converges to (each equal distance is placed BEFORE
 * the earlier ones, the last element is the one evicted) — see search_exact_, index.hpp:4251-4268. With an
 * explicit tie-break the insertion order no longer matters, so partial results can be merged in any order. */
__device__ __forceinline__ void top_insert_reg_keyed(float (&td)[TOP_E], uint32_t (&ts)[TOP_E], uint32_t& size, uint32_t limit,
                                                     float d, uint32_t s, int lane) {
    uint32_t const g0 = (uint32_t)lane * TOP_E;
    uint32_t mine = 0;
#pragma unroll
    for (int j = 0; j < TOP_E; ++j) mine += (g0 + j < size && (td[j] < d || (td[j] == d && ts[j] > s))) ? 1u : 0u;
    uint32_t const pos = __reduce_add_sync(0xffffffffu, mine);
    if (pos == limit) return;
    bool const full = size == limit;
    uint32_t const hi = size - (full ? 1u : 0u);
    float const up_d = __shfl_up_sync(0xffffffffu, td[TOP_E - 1], 1);
    uint32_t const up_s = __shfl_up_sync(0xffffffffu, ts[TOP_E - 1], 1);
#pragma unroll
    for (int j = TOP_E - 1; j >= 0; --j) {
        uint32_t const g = g0 + (uint32_t)j;
        if (g > pos && g <= hi) {
            td[j] = j ? td[j > 0 ? j - 1 : 0] : up_d;
            ts[j] = j ? ts[j > 0 ? j - 1 : 0] : up_s;
        } else if (g == pos) {
            td[j] = d;
            ts[j] = s;
        }
    }
    size += full ? 0u : 1u;
}

/* sorted insert into a k-best list in global memory under (distance asc, slot desc); whole warp, uniform arguments */
__device__ __forceinline__ void top_insert_global_keyed(float volatile* ld, uint32_t volatile* ls, uint32_t& size, uint32_t k, float cd,
                                                        uint32_t cs, int lane) {
    uint32_t pos = 0;
    for (uint32_t base = 0; base < size; base += 32) {
        uint32_t const i = base + (uint32_t)lane;
        bool before = false;
        if (i < size) {
            float const d = ld[i];
            before = d < cd || (d == cd && ls[i] > cs);
        }
        pos += __popc(__ballot_sync(0xffffffffu, before));
    }
    if (pos >= k) return;
    uint32_t const new_size = size < k ? size + 1 : k;
    for (int hi = (int)new_size - 1; hi > (int)pos; hi -= 32) { /* old [pos, new_size-1) moves one to the right, tail first */
        int const i = hi - lane;
        bool const mv = i > (int)pos;
        float d = 0.f;
        uint32_t sl = 0;
        if (mv) { d = ld[i - 1]; sl = ls[i - 1]; }
        __syncwarp();
        if (mv) { ld[i] = d; ls[i] = sl; }
        __syncwarp();
    }
    if (lane == 0) { ld[pos] = cd; ls[pos] = cs; }
    __syncwarp();
    size = new_size;
}

} // namespace usearch_b200
