/*
 *  exact_kernel.cu — brute-force ("exact") many-to-many search on the GPU.
 *
 *  Two reference entry points end here:
 *    index_gt::search(exact = true) -> search_exact_      index.hpp:4251-4268
 *        every non-deleted slot in slot order, `top.insert(candidate, count)`;
 *    exact_search_t / usearch_exact_search                 index_plugins.hpp:2071-2164, c/lib.cpp:468-501
 *        distance matrix, then std::partial_sort per query; the metric is called as metric(dataset, query).
 *  Both are "the k smallest distances"; they differ in tie order. A sequence of sorted_buffer_gt::insert calls in
 *  ascending slot order converges to the k smallest under the TOTAL order (distance ascending, slot descending),
 *  which is what `top_insert_reg_keyed` maintains — in any insertion order, so the dataset can be cut into
 *  segments that are scanned by different CTAs and merged afterwards. std::partial_sort leaves ties unspecified;
 *  the same rule is used there (distances and, where no two distances are equal, labels match the reference).
 *
 *  Distances are computed by the very metric structs of the search kernel (metrics.cuh): one (query, vector)
 *  pair yields the same bits in both kernels.
 *
 *  Two scan kernels share the partial-list format and the merge:
 *
 *  exact_tiled_kernel (the default): the scan is FFMA/LDS-bound, not HBM-bound (1M x 768 f32 against 4096 queries
 *  is 3.1e12 multiply-adds but only 3 GB of vectors), so the work is register-tiled like an SGEMM whose inner
 *  product keeps the reference's summation order: a CTA owns 8 warps x QT queries (in shared memory) and one
 *  segment of the dataset; warp 0 streams tiles of TV vectors into a double-buffered stage with per-lane TMA bulk
 *  copies; every lane group (LPV lanes) reduces VT vectors of the tile against the QT queries of its warp, all
 *  QT x VT accumulator sets in registers: one stage read feeds QT pairs and one (broadcast) query read feeds VT x 8
 *  groups. The k-best lists live in global memory (L2): after the first few tiles an insertion is a rare event.
 *
 *  exact_scan_kernel (fallback when the tiled stage does not fit in 227 KB): one query per warp, list in registers. Its
 *  own stage (8 queries and 2 x 32/LPV rows) holds f32 rows up to 2400 dims; longer rows are read in place from global
 *  memory by the same kernel (STAGED = false), so exact search serves any length the index does.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "device_index.h"
#include "exact_args.h"
#include "frozen_index.h"
#include "metrics.cuh"
#include "warp_primitives.cuh"

namespace usearch_b200 {

constexpr int EXACT_WARPS = 8;


template <class M, class = void> struct has_finish_sw : std::false_type {};
template <class M> struct has_finish_sw<M, decltype((void)&M::finish_sw, void())> : std::true_type {};

/* reciprocal norms (metrics with NORMS): computed once per query and once per stored vector of a tile */
template <class M, bool = M::NORMS> struct rnorm_of { using type = float; static __device__ __forceinline__ type get(float) { return 0.f; } };
template <class M> struct rnorm_of<M, true> {
    using type = typename M::rn_t;
    static __device__ __forceinline__ type get(float x2) { return M::rnorm(x2); }
};

template <class M, bool SWAP>
__device__ __forceinline__ float finish_ordered(typename M::acc_t const& acc, typename M::qconst_t qc) {
    if constexpr (SWAP && has_finish_sw<M>::value) return M::finish_sw(acc, qc);
    else return M::finish(acc, qc);
}

/* a 16-byte chunk of a staged row (shared memory) or of a row read in place (global memory, read-only path) */
template <bool STAGED> __device__ __forceinline__ uint4 scan_chunk(uint4 const* p) {
    if constexpr (STAGED) return *p;
    else return __ldg(p);
}

/* STAGED = false: the query and the rows are read from global memory where they lie, for rows too long to stage 8 queries
 * and 2 x VPP rows in 227 KB. Each lane group walks the same chunks in the same order through the same metric calls,
 * so both variants give the same bits.
 * LISTED: the CTA serves work item a.items[blockIdx.x]; row j of its segment is slot a.rows[list_begin + j] (exact_args.h). */
template <class M, bool SWAP, bool STAGED, bool LISTED = false>
__global__ void __launch_bounds__(EXACT_WARPS * 32) exact_scan_kernel(__grid_constant__ device_index_t const ix,
                                                                      __grid_constant__ exact_args_of<LISTED> const a) {
    constexpr int LPV = M::LPV, VPP = 32 / LPV;
    extern __shared__ __align__(128) uint8_t smem[];
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane / LPV, sub = lane % LPV;
    uint32_t const chunks = ix.chunks16, bytes = (uint32_t)ix.vec_stride;
    uint32_t const bars = smem_u32(smem + a.off_bars), stage_addr = smem_u32(smem + a.off_stage);
    uint32_t qi = blockIdx.x * EXACT_WARPS + warp;
    bool has_query = qi < a.nq;
    uint32_t seg_lo = blockIdx.y * a.segment_len, seg_hi = min(ix.n, seg_lo + a.segment_len);
    uint32_t const* list = nullptr; /* LISTED: the slots of this item's rows */
    if constexpr (LISTED) {
        exact_item_t const it = a.items[blockIdx.x];
        qi = it.first + (uint32_t)warp;
        has_query = (uint32_t)warp < it.count;
        listed_segment(it, a.segments, blockIdx.y, VPP, seg_lo, seg_hi);
        list = a.rows + it.list_begin;
    }
    uint32_t const ntiles = seg_hi > seg_lo ? (seg_hi - seg_lo + VPP - 1) / VPP : 0;
    uint4 const* q4; /* a dead query slot reads query 0: prepare() shuffles across the whole warp */
    if constexpr (STAGED) {
        uint4* const q4s = reinterpret_cast<uint4*>(smem + (size_t)warp * bytes);
        q4 = q4s;
        if (threadIdx.x == 0) {
            mbar_init(bars, 1);
            mbar_init(bars + 8, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
        if (has_query) {
            uint4 const* src = reinterpret_cast<uint4 const*>(a.queries + (size_t)qi * a.query_stride);
            for (uint32_t j = lane; j < chunks; j += 32) q4s[j] = src[j];
        }
        __syncthreads();
    } else {
        q4 = reinterpret_cast<uint4 const*>(a.queries + (size_t)(has_query ? qi : 0u) * a.query_stride);
    }
    typename M::qconst_t qc = M::prepare(q4, chunks, lane);
    typename rnorm_of<M>::type q_rn = 0;
    if constexpr (M::NORMS) q_rn = rnorm_of<M>::get(qc.a2);

    auto issue = [&](uint32_t t) { /* thread 0 only */
        uint32_t const base = seg_lo + t * VPP, cnt = min((uint32_t)VPP, seg_hi - base), set = t & 1u;
        mbar_expect_tx(bars + 8u * set, cnt * bytes);
        for (uint32_t i = 0; i < cnt; ++i)
            bulk_copy_g2s(stage_addr + (set * VPP + i) * a.stage_stride,
                          ix.vectors + (size_t)(LISTED ? list[base + i] : base + i) * ix.vec_stride, bytes, bars + 8u * set);
    };
    if constexpr (STAGED)
        if (threadIdx.x == 0 && ntiles) issue(0);

    float td[TOP_E];
    uint32_t ts[TOP_E];
#pragma unroll
    for (int j = 0; j < TOP_E; ++j) { td[j] = 0.f; ts[j] = 0u; }
    uint32_t top_size = 0, phase = 0;
    float worst = 0.f;

    for (uint32_t t = 0; t < ntiles; ++t) {
        uint32_t const set = t & 1u, base = seg_lo + t * VPP, cnt = min((uint32_t)VPP, seg_hi - base);
        if constexpr (STAGED) {
            if (threadIdx.x == 0 && t + 1 < ntiles) issue(t + 1); /* the other set was released by the barrier below */
            mbar_wait(bars + 8u * set, (phase >> set) & 1u);
            phase ^= 1u << set;
        }
        bool const act = has_query && (uint32_t)g < cnt;
        uint32_t slot = base + (uint32_t)g;
        if constexpr (LISTED) slot = act ? list[slot] : 0u;
        typename M::acc_t acc;
        M::init(acc);
        if (act) {
            uint4 const* buf = STAGED ? reinterpret_cast<uint4 const*>(smem + a.off_stage + (size_t)(set * VPP + g) * a.stage_stride)
                                      : reinterpret_cast<uint4 const*>(ix.vectors + (size_t)slot * ix.vec_stride);
            uint32_t j = sub;
            for (; j + 3 * LPV < chunks; j += 4 * LPV) {
                uint4 b0 = scan_chunk<STAGED>(buf + j), b1 = scan_chunk<STAGED>(buf + j + LPV), b2 = scan_chunk<STAGED>(buf + j + 2 * LPV),
                      b3 = scan_chunk<STAGED>(buf + j + 3 * LPV);
                uint4 q0 = scan_chunk<STAGED>(q4 + j), q1 = scan_chunk<STAGED>(q4 + j + LPV), q2 = scan_chunk<STAGED>(q4 + j + 2 * LPV),
                      q3 = scan_chunk<STAGED>(q4 + j + 3 * LPV);
                M::step(acc, b0, q0);
                M::step(acc, b1, q1);
                M::step(acc, b2, q2);
                M::step(acc, b3, q3);
            }
            for (; j < chunks; j += LPV) M::step(acc, scan_chunk<STAGED>(buf + j), scan_chunk<STAGED>(q4 + j));
        }
        float d = finish_ordered<M, SWAP>(acc, qc);
        if constexpr (M::NORMS) {
            float const b2 = act ? __ldg(ix.norms + slot) : 0.f;
            auto const v_rn = rnorm_of<M>::get(b2);
            d = SWAP ? M::finalize_rn(d, b2, qc.a2, v_rn, q_rn) : M::finalize_rn(d, qc.a2, b2, q_rn, v_rn);
        }
        bool keep = act && sub == 0;
        if (keep && ix.deleted_bits) keep = !((ix.deleted_bits[slot >> 5] >> (slot & 31)) & 1u);
        /* candidates that can still enter: everything while the list is short, then d <= worst (an equal distance
         * with a larger slot number goes in front of the old one) */
        uint32_t todo = __ballot_sync(0xffffffffu, keep && (top_size < a.k || !(d > worst)));
        while (todo) {
            int const src_lane = __ffs(todo) - 1;
            todo &= todo - 1;
            float const cd = __shfl_sync(0xffffffffu, d, src_lane);
            uint32_t const cs = LISTED ? __shfl_sync(0xffffffffu, slot, src_lane) : base + (uint32_t)(src_lane / LPV);
            if (top_size < a.k || !(cd > worst)) {
                top_insert_reg_keyed(td, ts, top_size, a.k, cd, cs, lane);
                worst = top_back_reg(td, top_size);
            }
        }
        if constexpr (STAGED) __syncthreads(); /* every warp is done with this set before thread 0 refills it */
    }

    if (has_query) { /* partial result of this (query, segment) */
        size_t const row = ((size_t)qi * a.segments + blockIdx.y) * a.k;
#pragma unroll
        for (int j = 0; j < TOP_E; ++j) {
            uint32_t const i = (uint32_t)lane * TOP_E + (uint32_t)j;
            if (i < top_size) { a.part_d[row + i] = td[j]; a.part_s[row + i] = ts[j]; }
        }
        if (lane == 0) a.part_n[(size_t)qi * a.segments + blockIdx.y] = top_size;
    }
}

/* ---- register-tiled scan ------------------------------------------------------------------------------------- */

constexpr int TILED_WARPS = 8; /* two per scheduler: one warp alone leaves half of the issue slots idle (ncu) */

template <class M> struct exact_tile_t {
    static constexpr int QT = M::LPV == 4 ? 4 : 8;  /* queries per warp */
    static constexpr int VT = M::LPV == 4 ? 2 : 1;  /* vectors per lane group and tile */
    static constexpr int TV = (32 / M::LPV) * VT;   /* vectors per tile */
    static constexpr int QPC = TILED_WARPS * QT;    /* queries per CTA */
};

template <class M, bool SWAP, bool LISTED = false>
__global__ void __launch_bounds__(TILED_WARPS * 32, 1) exact_tiled_kernel(__grid_constant__ device_index_t const ix,
                                                                          __grid_constant__ exact_args_of<LISTED> const a) {
    using T = exact_tile_t<M>;
    constexpr int LPV = M::LPV, QT = T::QT, VT = T::VT, TV = T::TV, GROUPS = 32 / LPV;
    extern __shared__ __align__(128) uint8_t smem[];
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane / LPV, sub = lane % LPV;
    uint32_t const chunks = ix.chunks16, bytes = (uint32_t)ix.vec_stride;
    uint32_t const bars = smem_u32(smem + a.off_bars), stage_addr = smem_u32(smem + a.off_stage);
    uint32_t q0 = blockIdx.x * T::QPC + (uint32_t)warp * QT; /* first query of this warp */
    uint32_t q_end = 0;                                         /* LISTED: queries from q_end on are dead slots */
    uint32_t seg_lo = blockIdx.y * a.segment_len, seg_hi = min(ix.n, seg_lo + a.segment_len);
    uint32_t const* list = nullptr;
    if constexpr (LISTED) {
        exact_item_t const it = a.items[blockIdx.x];
        q0 = it.first + (uint32_t)warp * QT;
        q_end = it.first + it.count;
        listed_segment(it, a.segments, blockIdx.y, TV, seg_lo, seg_hi);
        list = a.rows + it.list_begin;
    }
    uint32_t const ntiles = seg_hi > seg_lo ? (seg_hi - seg_lo + TV - 1) / TV : 0;

    if (threadIdx.x == 0) {
        mbar_init(bars, 1);
        mbar_init(bars + 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    uint4 const* qrow[QT];
#pragma unroll
    for (int qi = 0; qi < QT; ++qi) {
        uint4* dst = reinterpret_cast<uint4*>(smem + a.off_queries + (size_t)(warp * QT + qi) * bytes);
        qrow[qi] = dst;
        bool const live = q0 + qi < (LISTED ? q_end : a.nq);
        uint4 const* src = reinterpret_cast<uint4 const*>(a.queries + (size_t)(live ? q0 + qi : 0) * a.query_stride);
        for (uint32_t j = lane; j < chunks; j += 32) dst[j] = live ? src[j] : make_uint4(0u, 0u, 0u, 0u);
    }
    __syncthreads();
    typename M::qconst_t qc[QT];
#pragma unroll
    for (int qi = 0; qi < QT; ++qi) qc[qi] = M::prepare(qrow[qi], chunks, lane);
    typename rnorm_of<M>::type q_rn[QT];
#pragma unroll
    for (int qi = 0; qi < QT; ++qi) {
        q_rn[qi] = 0;
        if constexpr (M::NORMS) q_rn[qi] = rnorm_of<M>::get(qc[qi].a2);
    }

    auto issue = [&](uint32_t t) { /* warp 0: lane i fetches vector i of the tile */
        uint32_t const base = seg_lo + t * TV, cnt = min((uint32_t)TV, seg_hi - base), set = t & 1u;
        if (lane == 0) mbar_expect_tx(bars + 8u * set, cnt * bytes);
        __syncwarp();
        for (uint32_t i = lane; i < cnt; i += 32)
            bulk_copy_g2s(stage_addr + (set * TV + i) * a.stage_stride,
                          ix.vectors + (size_t)(LISTED ? list[base + i] : base + i) * ix.vec_stride, bytes, bars + 8u * set);
    };
    if (warp == 0 && ntiles) issue(0);

    uint32_t sizes[QT];
    float worst[QT];
#pragma unroll
    for (int qi = 0; qi < QT; ++qi) { sizes[qi] = 0; worst[qi] = 0.f; }
    uint32_t phase = 0;

    for (uint32_t t = 0; t < ntiles; ++t) {
        uint32_t const set = t & 1u, base = seg_lo + t * TV, cnt = min((uint32_t)TV, seg_hi - base);
        if (warp == 0 && t + 1 < ntiles) issue(t + 1); /* the other set was released by the barrier below */
        mbar_wait(bars + 8u * set, (phase >> set) & 1u);
        phase ^= 1u << set;

        typename M::acc_t acc[QT][VT];
#pragma unroll
        for (int qi = 0; qi < QT; ++qi)
#pragma unroll
            for (int vt = 0; vt < VT; ++vt) M::init(acc[qi][vt]);
        uint4 const* vrow[VT];
#pragma unroll
        for (int vt = 0; vt < VT; ++vt) /* a short last tile reads stale stage rows: results are discarded below */
            vrow[vt] = reinterpret_cast<uint4 const*>(smem + a.off_stage + (size_t)(set * TV + vt * GROUPS + g) * a.stage_stride);
#pragma unroll 2
        for (uint32_t j = sub; j < chunks; j += LPV) {
            uint4 b[VT];
#pragma unroll
            for (int vt = 0; vt < VT; ++vt) b[vt] = vrow[vt][j];
#pragma unroll
            for (int qi = 0; qi < QT; ++qi) {
                uint4 const q = qrow[qi][j];
#pragma unroll
                for (int vt = 0; vt < VT; ++vt) M::step(acc[qi][vt], b[vt], q);
            }
        }

#pragma unroll
        for (int vt = 0; vt < VT; ++vt) {
            uint32_t const in_tile = (uint32_t)(vt * GROUPS + g),
                           slot = LISTED ? (in_tile < cnt ? list[base + in_tile] : 0u) : base + in_tile;
            bool usable = in_tile < cnt;
            float b2 = 0.f;
            if constexpr (M::NORMS) b2 = usable ? __ldg(ix.norms + slot) : 0.f;
            auto const v_rn = rnorm_of<M>::get(b2);
            if (usable && ix.deleted_bits) usable = !((ix.deleted_bits[slot >> 5] >> (slot & 31)) & 1u);
            usable = usable && sub == 0;
#pragma unroll
            for (int qi = 0; qi < QT; ++qi) {
                float d = finish_ordered<M, SWAP>(acc[qi][vt], qc[qi]);
                if constexpr (M::NORMS)
                    d = SWAP ? M::finalize_rn(d, b2, qc[qi].a2, v_rn, q_rn[qi]) : M::finalize_rn(d, qc[qi].a2, b2, q_rn[qi], v_rn);
                bool const live = q0 + qi < (LISTED ? q_end : a.nq);
                uint32_t todo = __ballot_sync(0xffffffffu, usable && live && (sizes[qi] < a.k || !(d > worst[qi])));
                if (todo) {
                    size_t const row = ((size_t)(q0 + qi) * a.segments + blockIdx.y) * a.k;
                    while (todo) {
                        int const src_lane = __ffs(todo) - 1;
                        todo &= todo - 1;
                        float const cd = __shfl_sync(0xffffffffu, d, src_lane);
                        uint32_t const cs = LISTED ? __shfl_sync(0xffffffffu, slot, src_lane) : base + (uint32_t)(vt * GROUPS + src_lane / LPV);
                        if (sizes[qi] < a.k || !(cd > worst[qi])) {
                            top_insert_global_keyed(a.part_d + row, a.part_s + row, sizes[qi], a.k, cd, cs, lane);
                            if (sizes[qi] == a.k) worst[qi] = reinterpret_cast<float volatile*>(a.part_d)[row + a.k - 1];
                        }
                    }
                }
            }
        }
        __syncthreads(); /* every warp is done with this set before warp 0 refills it */
    }

    if (lane == 0) {
#pragma unroll
        for (int qi = 0; qi < QT; ++qi)
            if (q0 + qi < (LISTED ? q_end : a.nq)) a.part_n[(size_t)(q0 + qi) * a.segments + blockIdx.y] = sizes[qi];
    }
}

/* one warp per query: merge the per-segment lists under (distance asc, slot desc), map slots to keys, pad.
 * A free search over a dataset in chunks (exact_free.cu) scans one chunk per launch: `row_offset` turns the chunk's rows
 * into dataset rows, and with `carry` the output row already holds the merged list of the chunks before (slots as keys),
 * which is merged as one more segment. The order is total, so any cut of the dataset gives the same list. */
__global__ void exact_merge_kernel(device_index_t ix, exact_args_t a, uint32_t row_offset, bool carry) {
    uint32_t const qi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    if (qi >= a.nq) return;
    float td[TOP_E];
    uint32_t ts[TOP_E];
#pragma unroll
    for (int j = 0; j < TOP_E; ++j) { td[j] = 0.f; ts[j] = 0u; }
    uint32_t top_size = 0;
    if (carry) {
        uint32_t const n = a.out_counts[qi];
        size_t const row = (size_t)qi * a.k;
        for (uint32_t i = 0; i < n; ++i)
            top_insert_reg_keyed(td, ts, top_size, a.k, a.out_dists[row + i], (uint32_t)a.out_keys[row + i], lane);
    }
    for (uint32_t seg = 0; seg < a.segments; ++seg) {
        uint32_t const n = a.part_n[(size_t)qi * a.segments + seg];
        size_t const row = ((size_t)qi * a.segments + seg) * a.k;
        for (uint32_t i = 0; i < n; ++i)
            top_insert_reg_keyed(td, ts, top_size, a.k, a.part_d[row + i], a.part_s[row + i] + row_offset, lane);
    }
    __syncwarp(); /* every lane has read the carried row before any lane overwrites it */
#pragma unroll
    for (int j = 0; j < TOP_E; ++j) {
        uint32_t const i = (uint32_t)lane * TOP_E + (uint32_t)j;
        if (i < a.k) {
            uint64_t key = 0;
            uint32_t bits = SNAN_BITS;
            if (i < top_size) {
                key = a.slots_as_keys ? (uint64_t)ts[j] : ix.keys[ts[j]];
                bits = __float_as_uint(td[j]);
            }
            a.out_keys[(size_t)qi * a.k + i] = key;
            reinterpret_cast<uint32_t*>(a.out_dists)[(size_t)qi * a.k + i] = bits;
        }
    }
    if (lane == 0) a.out_counts[qi] = top_size;
}

/* the same merge for count > 256: the merged list lives in global memory (L2) instead of registers */
__global__ void exact_merge_big_kernel(device_index_t ix, exact_args_t a, float* merged_d, uint32_t* merged_s, uint32_t row_offset,
                                       bool carry) {
    uint32_t const qi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    if (qi >= a.nq) return;
    float* md = merged_d + (size_t)qi * a.k;
    uint32_t* ms = merged_s + (size_t)qi * a.k;
    uint32_t top_size = 0;
    float worst = 0.f;
    if (carry) /* the chunks before, ascending like a segment's list; it cannot overflow the empty list */
        for (uint32_t i = 0, n = a.out_counts[qi]; i < n; ++i)
            top_insert_global_keyed(md, ms, top_size, a.k, a.out_dists[(size_t)qi * a.k + i], (uint32_t)a.out_keys[(size_t)qi * a.k + i], lane);
    if (top_size == a.k) worst = reinterpret_cast<float volatile*>(md)[a.k - 1];
    for (uint32_t seg = 0; seg < a.segments; ++seg) {
        uint32_t const n = a.part_n[(size_t)qi * a.segments + seg];
        size_t const row = ((size_t)qi * a.segments + seg) * a.k;
        for (uint32_t i = 0; i < n; ++i) {
            float const cd = a.part_d[row + i];
            if (top_size == a.k && cd > worst) break; /* the segment's list is ascending: nothing later can enter */
            top_insert_global_keyed(md, ms, top_size, a.k, cd, a.part_s[row + i] + row_offset, lane);
            if (top_size == a.k) worst = reinterpret_cast<float volatile*>(md)[a.k - 1];
        }
    }
    __syncwarp();
    for (uint32_t i = lane; i < a.k; i += 32) {
        uint64_t key = 0;
        uint32_t bits = SNAN_BITS;
        if (i < top_size) {
            uint32_t const slot = reinterpret_cast<uint32_t volatile*>(ms)[i];
            key = a.slots_as_keys ? (uint64_t)slot : ix.keys[slot];
            bits = __float_as_uint(reinterpret_cast<float volatile*>(md)[i]);
        }
        a.out_keys[(size_t)qi * a.k + i] = key;
        reinterpret_cast<uint32_t*>(a.out_dists)[(size_t)qi * a.k + i] = bits;
    }
    if (lane == 0) a.out_counts[qi] = top_size;
}

template <class M, bool STAGED> static cudaError_t exact_launch_scan_t(device_index_t const& ix, exact_listed_args_t const& a, bool swap, bool listed,
                                                                      dim3 grid, size_t smem, cudaStream_t stream) {
    if (listed) { /* index mode only: metric(query, stored) */
        cudaError_t e = cudaFuncSetAttribute(exact_scan_kernel<M, false, STAGED, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_scan_kernel<M, false, STAGED, true><<<grid, EXACT_WARPS * 32, smem, stream>>>(ix, a);
    } else if (swap) {
        cudaError_t e = cudaFuncSetAttribute(exact_scan_kernel<M, true, STAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_scan_kernel<M, true, STAGED><<<grid, EXACT_WARPS * 32, smem, stream>>>(ix, a);
    } else {
        cudaError_t e = cudaFuncSetAttribute(exact_scan_kernel<M, false, STAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_scan_kernel<M, false, STAGED><<<grid, EXACT_WARPS * 32, smem, stream>>>(ix, a);
    }
    return cudaGetLastError();
}

/* smem == 0: the staged scan does not fit, rows are read in place */
template <class M> static cudaError_t exact_launch_t(device_index_t const& ix, exact_listed_args_t const& a, bool swap, bool listed, dim3 grid,
                                                     size_t smem, cudaStream_t stream) {
    return smem ? exact_launch_scan_t<M, true>(ix, a, swap, listed, grid, smem, stream)
                : exact_launch_scan_t<M, false>(ix, a, swap, listed, grid, 0, stream);
}

template <class M> static cudaError_t exact_launch_tiled_t(device_index_t const& ix, exact_listed_args_t const& a, bool swap, bool listed, dim3 grid,
                                                           size_t smem, cudaStream_t stream) {
    if (listed) {
        cudaError_t e = cudaFuncSetAttribute(exact_tiled_kernel<M, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_tiled_kernel<M, false, true><<<grid, TILED_WARPS * 32, smem, stream>>>(ix, a);
    } else if (swap) {
        cudaError_t e = cudaFuncSetAttribute(exact_tiled_kernel<M, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_tiled_kernel<M, true><<<grid, TILED_WARPS * 32, smem, stream>>>(ix, a);
    } else {
        cudaError_t e = cudaFuncSetAttribute(exact_tiled_kernel<M, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        exact_tiled_kernel<M, false><<<grid, TILED_WARPS * 32, smem, stream>>>(ix, a);
    }
    return cudaGetLastError();
}

template <class M> static cudaError_t exact_launch_any_t(bool tiled, device_index_t const& ix, exact_listed_args_t const& a, bool swap, bool listed,
                                                         dim3 grid, size_t smem, cudaStream_t stream) {
    return tiled ? exact_launch_tiled_t<M>(ix, a, swap, listed, grid, smem, stream) : exact_launch_t<M>(ix, a, swap, listed, grid, smem, stream);
}

static int exact_lpv(device_index_t const& ix) {
    if (ix.scalar == SCALAR_F16 || ix.scalar == SCALAR_BF16) return 1;
    if (ix.scalar == SCALAR_B1) return 2;
    return 4;
}

/*
 *  Exact top-k of `nq` device-resident queries (index scalar kind, rows `query_stride` bytes apart, 16-byte aligned
 *  and readable up to vec_stride) against every vector of `ix`. `swap` = call the metric as metric(stored, query).
 *  Scratch for the per-segment partial lists is taken from `scratch` (grown on demand).
 *  `listed` (exact filtered search, swap = false): the CTAs serve its work items against their slot lists instead; with
 *  `listed->items == nullptr` nothing runs and `listed->qpc` receives the queries per item of the kernel that would.
 *  `row_offset` and `carry`: one chunk of a free search (exact_merge_kernel).
 */
template <class scratch_at>
static char const* exact_run(device_index_t const& ix, int sm_count, void const* d_queries, size_t nq, size_t query_stride, size_t k,
                             bool swap, bool slots_as_keys, exact_listed_t* listed, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                             scratch_at& scratch, cudaStream_t stream, uint32_t row_offset = 0, bool carry = false) {
    if (!nq || !k) return nullptr;
    /* count <= 256: k-best lists in registers (scan, IMMA, merge); beyond that the tiled kernel's global-memory lists and
     * exact_merge_big_kernel carry any count (search_exact_ takes any `wanted`, index.hpp:4251-4268) */
    bool const big_k = k > 32 * TOP_E;
    if (!ix.n) { /* nothing to scan: empty rows */
        if (cudaMemsetAsync(d_counts, 0, nq * 4, stream) != cudaSuccess) return "CUDA failure: memset";
        if (cudaMemsetAsync(d_keys, 0, nq * k * 8, stream) != cudaSuccess) return "CUDA failure: memset";
        if (cudaMemsetAsync(d_dists, 0xFF, nq * k * 4, stream) != cudaSuccess) return "CUDA failure: memset"; /* NaN */
        return nullptr;
    }
    int const lpv = exact_lpv(ix);
    exact_listed_args_t a; /* the listed fields stay null for a scan of every slot */
    a.queries = static_cast<uint8_t const*>(d_queries);
    a.query_stride = query_stride;
    a.nq = (uint32_t)nq;
    a.k = (uint32_t)k;
    a.slots_as_keys = slots_as_keys ? 1u : 0u;
    a.stage_stride = (uint32_t)((ix.vec_stride + 127) / 128 * 128) + 16u * (uint32_t)lpv;
    /* the register-tiled kernel when its stage fits; USEARCH_B200_EXACT=scan|tiled forces one (tests) */
    int const qt = lpv == 4 ? 4 : 8, tile_vectors = (32 / lpv) * (lpv == 4 ? 2 : 1), qpc_tiled = TILED_WARPS * qt;
    size_t const tiled_smem = ((size_t)qpc_tiled * ix.vec_stride + 16 + 127) / 128 * 128 + 2 * (size_t)tile_vectors * a.stage_stride;
    static int const forced = [] {
        char const* v = std::getenv("USEARCH_B200_EXACT");
        return !v ? 0 : (std::strcmp(v, "scan") == 0 ? 1 : (std::strcmp(v, "tiled") == 0 ? 2 : (std::strcmp(v, "imma") == 0 ? 3 : (std::strcmp(v, "wgmma") == 0 ? 4 : 0))));
    }();
    /* i8: integer sums are order independent, the tensor cores give the reference's bits (exact_imma.cu) */
    bool const imma = !big_k && ix.scalar == SCALAR_I8 && (forced == 0 || forced == 3 || forced == 4) &&
                      (ix.metric == METRIC_IP || ix.metric == METRIC_L2SQ || ix.metric == METRIC_COS);
    if ((forced == 3 || forced == 4) && !imma) return "The tensor-core exact-search kernels serve i8 vectors only";
    /* wgmma (exact_wgmma.cu) when the driver can encode tensor maps; mma.sync (exact_imma.cu) otherwise or when forced.
     * Its TMA tensor maps read contiguous slabs and cannot follow a slot list: listed scans take mma.sync. */
    bool const wgmma = !listed && imma && forced != 3 && exact_wgmma_usable(ix, a); /* count <= 24; larger counts stay on mma.sync */
    bool const tiled = !imma && (forced == 1 && !big_k ? false : tiled_smem <= 227 * 1024);
    if (big_k && !tiled) return "Exact search with count > 256 needs vectors that fit the tiled stage";
    if (forced == 2 && !tiled) return "Vectors too long for the tiled exact-search stage";
    int const vpp = wgmma ? exact_wgmma_tile_vectors() : (imma ? exact_imma_tile_vectors() : (tiled ? tile_vectors : 32 / lpv)); /* vectors per tile */
    uint32_t const qpc = wgmma ? (uint32_t)exact_wgmma_tile_queries()
                              : (imma ? (uint32_t)exact_imma_tile_queries() : (tiled ? (uint32_t)qpc_tiled : (uint32_t)EXACT_WARPS));
    uint32_t off = qpc * (uint32_t)ix.vec_stride;
    a.off_queries = 0;
    a.off_bars = off;
    off = (off + 16 + 127) / 128 * 128;
    a.off_stage = off;
    size_t smem = wgmma ? exact_wgmma_smem_bytes() : (imma ? exact_imma_smem_bytes() : off + 2 * (size_t)vpp * a.stage_stride);
    /* only the one-query-per-warp scan can outgrow its stage (the tiled one is not chosen then): it reads in place */
    bool const in_place = smem > 227 * 1024;
    if (in_place) smem = 0;
    if (listed && !listed->items) {
        listed->qpc = qpc;
        return nullptr;
    }
    bool const is_listed = listed != nullptr;
    uint32_t const groups = is_listed ? listed->n_items : (uint32_t)((nq + qpc - 1) / qpc);
    uint32_t const scanned = is_listed ? listed->total_rows : ix.n; /* rows the segments share out */
    /* cut the dataset so that the grid fills whole waves of the resident CTAs (1 per SM tiled, ~3 per SM staged, 4 per SM
     * in place: up to 64 registers) */
    uint32_t const resident = (uint32_t)sm_count * (wgmma ? 1u : (imma ? 2u : (tiled ? 1u : (in_place ? 4u : 3u))));
    uint32_t const max_segments =
        std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)(((uint64_t)scanned + 8 * (uint32_t)vpp - 1) / (8 * (uint32_t)vpp)), 65535u));
    uint32_t segments = 1;
    {
        double best = -1;
        uint32_t const lo = std::max<uint32_t>(1, (resident + groups - 1) / groups);
        for (uint32_t s = lo; s <= lo + 24; ++s) {
            uint32_t const c = std::min(s, max_segments);
            double const total = (double)groups * c, waves = std::ceil(total / resident);
            double const util = total / (waves * resident) - 0.002 * c; /* prefer fewer segments on a tie */
            if (util > best) { best = util; segments = c; }
        }
    }
    size_t const list_bytes = nq * k * 8;
    while (segments > 1 && list_bytes * segments > ((size_t)1 << 30)) --segments;
    if (is_listed) { /* every item cuts its own list into `segments` (listed_segment); some may come out empty */
        a.segments = segments;
        a.segment_len = 0;
        a.items = listed->items;
        a.rows = listed->rows;
    } else {
        uint32_t seg_len = (ix.n + segments - 1) / segments;
        seg_len = (seg_len + (uint32_t)vpp - 1) / (uint32_t)vpp * (uint32_t)vpp;
        segments = (ix.n + seg_len - 1) / seg_len;
        a.segments = segments;
        a.segment_len = seg_len;
    }
    size_t const rows = nq * segments;
    size_t const lists = rows * k * 8 + rows * 4;
    size_t const norms_at = (lists + 15) / 16 * 16;
    size_t const need = norms_at + (imma ? (nq + (size_t)scanned) * 4 : 0) + (big_k ? nq * k * 8 : 0) + 64;
    if (char const* e = scratch.reserve(need)) return e;
    a.part_d = reinterpret_cast<float*>(scratch.ptr);
    a.part_s = reinterpret_cast<uint32_t*>(scratch.ptr + rows * k * 4);
    a.part_n = reinterpret_cast<uint32_t*>(scratch.ptr + rows * k * 8);
    if (imma && ix.metric != METRIC_IP) {
        int* qn = reinterpret_cast<int*>(scratch.ptr + norms_at);
        int* vn = qn + nq;
        cudaError_t const ev = is_listed ? exact_imma_listed_self_dots(ix.vectors, ix.vec_stride, ix.chunks16, listed->rows, scanned, vn, stream)
                                         : exact_imma_self_dots(ix.vectors, ix.vec_stride, ix.chunks16, ix.n, vn, stream);
        if (exact_imma_self_dots(a.queries, query_stride, ix.chunks16, (uint32_t)nq, qn, stream) != cudaSuccess || ev != cudaSuccess)
            return "CUDA failure: i8 norms launch";
        a.query_norms = qn;
        a.vector_norms = vn;
    }
    a.out_keys = d_keys;
    a.out_dists = d_dists;
    a.out_counts = d_counts;
    dim3 const grid(groups, segments);
    cudaError_t e = cudaErrorInvalidValue;
    if (wgmma) e = exact_wgmma_launch(ix, a, swap, grid, stream);
    else if (imma) e = is_listed ? exact_imma_listed_launch(ix, a, grid, stream) : exact_imma_launch(ix, a, swap, grid, stream);
    else switch (ix.scalar) {
    case SCALAR_F32:
        if (ix.metric == METRIC_L2SQ) e = exact_launch_any_t<l2sq_f32_t>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_IP) e = exact_launch_any_t<ip_f32_t>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_COS) e = exact_launch_any_t<cos_f32_t>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        break;
    case SCALAR_F64:
        if (ix.metric == METRIC_L2SQ) e = exact_launch_any_t<l2sq_f64_t>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_IP) e = exact_launch_any_t<ip_f64_t>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_COS) e = exact_launch_any_t<cos_f64_t>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        break;
    case SCALAR_F16:
        if (ix.metric == METRIC_L2SQ) e = exact_launch_any_t<l2sq_half_t<f16_conv_t>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_IP) e = exact_launch_any_t<ip_half_t<f16_conv_t>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_COS) e = exact_launch_any_t<cos_half_t<f16_conv_t>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        break;
    case SCALAR_BF16:
        if (ix.metric == METRIC_L2SQ) e = exact_launch_any_t<l2sq_half_t<bf16_conv_t>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_IP) e = exact_launch_any_t<ip_half_t<bf16_conv_t>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_COS) e = exact_launch_any_t<cos_half_t<bf16_conv_t>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        break;
    case SCALAR_I8:
        if (ix.metric == METRIC_L2SQ) e = exact_launch_any_t<l2sq_i8_t<4>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_IP) e = exact_launch_any_t<ip_i8_t<4>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_COS) e = exact_launch_any_t<cos_i8_t<4>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        break;
    case SCALAR_B1:
        if (ix.metric == METRIC_HAMMING) e = exact_launch_any_t<hamming_b1_t<2>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_TANIMOTO || ix.metric == METRIC_JACCARD) e = exact_launch_any_t<tanimoto_b1_t<2>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        else if (ix.metric == METRIC_SORENSEN) e = exact_launch_any_t<sorensen_b1_t<2>>(tiled, ix, a, swap, is_listed, grid, smem, stream);
        break;
    default: break;
    }
    if (e != cudaSuccess) return "CUDA failure: exact scan launch";
    if (big_k) {
        float* merged_d = reinterpret_cast<float*>(scratch.ptr + norms_at);
        exact_merge_big_kernel<<<(unsigned)((nq * 32 + 255) / 256), 256, 0, stream>>>(
            ix, a, merged_d, reinterpret_cast<uint32_t*>(merged_d + nq * k), row_offset, carry);
    } else
        exact_merge_kernel<<<(unsigned)((nq * 32 + 255) / 256), 256, 0, stream>>>(ix, a, row_offset, carry);
    if (cudaGetLastError() != cudaSuccess) return "CUDA failure: exact merge launch";
    return nullptr;
}

char const* exact_search_device(device_index_t const& ix, int sm_count, void const* d_queries, size_t nq, size_t query_stride, size_t k,
                                bool swap, bool slots_as_keys, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                                device_buffer_t<uint8_t>& scratch, cudaStream_t stream) {
    return exact_run(ix, sm_count, d_queries, nq, query_stride, k, swap, slots_as_keys, nullptr, d_keys, d_dists, d_counts, scratch, stream);
}

char const* exact_search_chunk_device(device_index_t const& chunk, int sm_count, void const* d_queries, size_t nq, size_t query_stride,
                                      size_t k, uint32_t row_offset, bool carry, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                                      stream_buffer_t<uint8_t>& scratch, cudaStream_t stream) {
    return exact_run(chunk, sm_count, d_queries, nq, query_stride, k, true, true, nullptr, d_keys, d_dists, d_counts, scratch, stream,
                     row_offset, carry);
}

char const* exact_search_check(device_index_t const& shape, size_t k) {
    uint32_t qpc = 0;
    return exact_listed_queries_per_item(shape, k, &qpc);
}

char const* exact_listed_queries_per_item(device_index_t const& ix, size_t k, uint32_t* qpc) {
    device_buffer_t<uint8_t> unused;
    exact_listed_t plan_only;
    if (char const* e = exact_run(ix, 0, nullptr, 1, 0, k, false, false, &plan_only, nullptr, nullptr, nullptr, unused, nullptr)) return e;
    *qpc = plan_only.qpc;
    return nullptr;
}

char const* exact_listed_search_device(device_index_t const& ix, int sm_count, void const* d_queries, size_t nq, size_t k,
                                       exact_listed_t const& listed, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                                       device_buffer_t<uint8_t>& scratch, cudaStream_t stream) {
    exact_listed_t l = listed;
    return exact_run(ix, sm_count, d_queries, nq, ix.vec_stride, k, false, false, &l, d_keys, d_dists, d_counts, scratch, stream);
}

} // namespace usearch_b200
