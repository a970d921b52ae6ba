/*
 *  exact_i8.cuh — the three i8 metrics as functions of the integer triple (ab, a2, b2), shared by the tensor-core scans
 *  (exact_imma.cu: mma.sync; exact_wgmma.cu: wgmma):
 *      ip    1 - float(ab)                               index_plugins.hpp:1914-1916 over simsimd_dot_i8
 *      l2sq  float(a2 + b2 - 2 ab)  == sum (a-b)^2       spatial.h l2sq_i8 (i32 accumulation)
 *      cos   normalise(float(ab), float(a2), float(b2))  spatial.h:1904-1972 -> the f32 normaliser
 */
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "device_index.h"

namespace usearch_b200 {

/* cos: the two reciprocal roots of cos_normalize_f32 are per-operand (qr, vr), computed once per row / column of
 * the tile; the per-pair remainder is the same two multiplies and the subtraction, in the operand order of the
 * call (`metric(query, stored)` for an index, `metric(stored, query)` for exact_search_t) */
template <uint32_t METRIC, bool SWAP>
__device__ __forceinline__ float i8_distance(int ab, int qa2, int vb2, float qr, float vr) {
    if constexpr (METRIC == METRIC_IP) return __fsub_rn(1.0f, __int2float_rn(ab));
    else if constexpr (METRIC == METRIC_L2SQ) return __int2float_rn(qa2 + vb2 - 2 * ab);
    else {
        if (qa2 == 0 && vb2 == 0) return 0.0f;
        if (ab == 0) return 1.0f;
        float const abf = __int2float_rn(ab);
        float const r = SWAP ? __fsub_rn(1.0f, __fmul_rn(__fmul_rn(abf, vr), qr)) : __fsub_rn(1.0f, __fmul_rn(__fmul_rn(abf, qr), vr));
        return r > 0 ? r : 0.f;
    }
}

__device__ __forceinline__ float i8_rnorm(int x2) { return __frcp_rn(__fsqrt_rn(__int2float_rn(x2))); }


} // namespace usearch_b200
