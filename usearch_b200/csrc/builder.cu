/*
 *  builder.cu — GPU-assisted `add` (SURVEY.md §8f row N4): HNSW construction in BATCHES, the graph staying in the flat
 *  HBM layout of device_index.h the whole time.
 *
 *  What one insertion is in the reference (index_gt::add, index.hpp:2780-2880):
 *    level        choose_random_level_ (index.hpp:3895-3899): floor(-ln(U) / ln(M))
 *    descent      search_for_one_ from the entry point down to level+1                       (:3963-4003)
 *    per level    search_to_insert_ (:4010-4079): best-first with ef = expansion_add, candidates instead of results
 *                 form_links_to_closest_ (:3825-3846): refine_ (:4276-4318) keeps a candidate only if it is not closer to an
 *                   already kept neighbour than to the new member, at most M of them -> the new member's list
 *                 form_reverse_links_ (:3848-3893): the new member is appended to each chosen neighbour; a neighbour whose
 *                   list is full re-runs refine_ over its list plus the newcomer
 *    entry point  moves when the new member's level exceeds the current top                  (:2873-2876)
 *
 *  How a BATCH of new members goes through the same steps here (members of one batch do not see each other — measured to
 *  cost nothing at batches <= 1/32 of the current size, DESIGN.md §9):
 *    1. one launch of the search kernel in INSERT mode (search_kernel.cu): a work item per (member, level), each running
 *       descent + search_to_insert_ on its level -> candidate slots/distances, ascending;
 *    2. link_forward_kernel: a CTA per work item runs refine_ (the lazy sequential heuristic, evaluated for all kept
 *       neighbours of a step at once) and writes the member's list; the chosen (neighbour, member, distance) triples
 *       are emitted as pairs;
 *    3. the pairs are sorted by (level, neighbour) (cub radix sort) and cut into runs;
 *    4. link_reverse_kernel: a CTA per (level, neighbour) run appends the arrivals, or — when the list would overflow —
 *       measures the neighbour against its list, sorts list + arrivals and runs refine_ with the level's capacity.
 *  All distances come from the metric structs of the search kernel (metrics.cuh): what the reference would compute for the
 *  same pair, bit for bit. The result is not bit-identical to a reference build — neither is the reference's own
 *  multi-threaded build (SURVEY.md §3.3); the parity bar is DESIGN.md §9 (structure invariants, recall and work per query
 *  of the REFERENCE search on the GPU-built file).
 */
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "cuda_check.h"
#include "frozen_index.h"
#include "metrics.cuh"
#include "scalar_casts.h"
#include "warp_primitives.cuh"

namespace usearch_b200 {

namespace {

constexpr int LINK_THREADS = 256;         /* 8 warps work on one refine */
constexpr uint32_t LINK_CAND_MAX = 256;   /* candidates one refine can hold (expansion_add and list + arrivals are cut to it) */
constexpr int LINK_LOADS_IN_FLIGHT = 8;


uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }

struct link_args_t {
    /* forward: one task per (new member, level) */
    uint32_t ntasks = 0;
    uint32_t const* task_slot = nullptr;
    uint8_t const* task_level = nullptr;
    uint32_t const* cand_slots = nullptr; /* [ntasks x ef] ascending by distance */
    float const* cand_dists = nullptr;
    uint32_t const* cand_counts = nullptr;
    uint32_t ef = 0;
    /* pairs: slot p = task * m + rank holds (level << 32 | neighbour) and the distance; unused = ~0 */
    uint64_t* pair_keys = nullptr;
    float* pair_dists = nullptr;
    /* reverse: runs of equal keys in the sorted pairs */
    uint64_t const* sorted_keys = nullptr;
    uint32_t const* sorted_idx = nullptr;
    uint32_t npairs = 0;
    uint32_t const* heads = nullptr;
    uint32_t const* nheads = nullptr; /* device scalar */
    uint32_t* work_counter = nullptr;
    /* shared-memory carve-up (bytes): two vector buffers, then the candidate and kept lists */
    uint32_t off_cs = 0, off_cd = 0, off_kept = 0, off_keptd = 0;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, void const* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

/* the whole CTA requests one stored vector into a shared-memory buffer */
__device__ __forceinline__ void fetch_vector(device_index_t const& ix, uint32_t slot, uint32_t dst) {
    uint8_t const* src = ix.vectors + (size_t)slot * ix.vec_stride;
    for (uint32_t j = threadIdx.x; j < ix.chunks16; j += blockDim.x) cp_async16(dst + 16u * j, src + 16u * (size_t)j);
}

/* query constants of metric(query = stored vector `slot`, ...): the stored norm where the metric keeps norms */
template <class M>
__device__ __forceinline__ typename M::qconst_t query_constants(device_index_t const& ix, uint4 const* q4, uint32_t slot, int lane) {
    if constexpr (M::NORMS) {
        typename M::qconst_t qc;
        qc.a2 = __ldg(ix.norms + slot);
        return qc;
    } else
        return M::prepare(q4, ix.chunks16, lane);
}

/*
 *  Distances from the vector in shared memory (`q4`) to `n` stored vectors, the groups of LPV lanes of all warps of the
 *  CTA taking one vector each (the DIRECT scheme of search_kernel.cu: 16-byte chunks through registers). Each group leader
 *  either stores the distance (out != NULL) or reports whether it is below `threshold` (the refine_ test).
 */
template <class M>
__device__ __forceinline__ bool block_distances(device_index_t const& ix, uint4 const* q4, typename M::qconst_t qc,
                                                uint32_t const* slots, uint32_t n, float* out, float threshold) {
    constexpr int LPV = M::LPV, VPP = 32 / LPV;
    int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int const g = lane / LPV, sub = lane % LPV;
    uint32_t const chunks = ix.chunks16;
    bool below = false;
    for (uint32_t base = (uint32_t)warp * VPP; base < n; base += (uint32_t)nwarps * VPP) {
        uint32_t const c = base + g;
        bool const act = c < n;
        uint32_t const slot = act ? slots[c] : 0u;
        uint4 const* v = reinterpret_cast<uint4 const*>(ix.vectors + (size_t)slot * ix.vec_stride);
        typename M::acc_t acc;
        M::init(acc);
        for (uint32_t j0 = sub; j0 < chunks; j0 += LPV * LINK_LOADS_IN_FLIGHT) {
            uint4 r[LINK_LOADS_IN_FLIGHT];
#pragma unroll
            for (int u = 0; u < LINK_LOADS_IN_FLIGHT; ++u) {
                uint32_t const j = j0 + u * LPV;
                if (act && j < chunks) r[u] = __ldg(v + j); /* hot in L2: the search of this batch has just read them */
            }
#pragma unroll
            for (int u = 0; u < LINK_LOADS_IN_FLIGHT; ++u) {
                uint32_t const j = j0 + u * LPV;
                if (act && j < chunks) M::step(acc, r[u], q4[j]);
            }
        }
        float d = M::finish(acc, qc); /* shuffles inside the LPV group: every lane executes it */
        if constexpr (M::NORMS) d = M::finalize(d, qc, act ? __ldg(ix.norms + slot) : 1.f);
        if (act && sub == 0) {
            if (out) out[c] = d;
            below |= d < threshold;
        }
    }
    return below;
}

/*
 *  refine_ (index.hpp:4276-4318) by one CTA. `cs`/`cd` hold `ncand` candidates ascending by distance to the centre.
 *  Fewer candidates than `needed`: all are kept, unsorted in the reference, sorted here (the order inside a list has no
 *  meaning). Otherwise the first is kept, and candidate c is kept iff no already kept s has d(c, s) < d(c, centre);
 *  the sequential inner loop of the reference breaks at the first such s, here all kept s of a step are measured together.
 *  The vector of candidate c+1 is requested (cp.async) while candidate c is being measured.
 */
template <class M>
__device__ __forceinline__ uint32_t refine_block(device_index_t const& ix, uint8_t* smem, link_args_t const& a, uint32_t ncand,
                                                 uint32_t needed) {
    uint32_t const* cs = reinterpret_cast<uint32_t const*>(smem + a.off_cs);
    float const* cd = reinterpret_cast<float const*>(smem + a.off_cd);
    uint32_t* kept = reinterpret_cast<uint32_t*>(smem + a.off_kept);
    float* keptd = reinterpret_cast<float*>(smem + a.off_keptd);
    int const lane = threadIdx.x & 31;
    if (ncand < needed) {
        for (uint32_t i = threadIdx.x; i < ncand; i += blockDim.x) { kept[i] = cs[i]; keptd[i] = cd[i]; }
        __syncthreads();
        return ncand;
    }
    uint32_t const vbytes = (uint32_t)ix.vec_stride;
    uint32_t const buf0 = smem_u32(smem);
    if (threadIdx.x == 0) { kept[0] = cs[0]; keptd[0] = cd[0]; }
    uint32_t nkept = 1;
    if (ncand > 1) fetch_vector(ix, cs[1], buf0 + vbytes);
    cp_async_wait_all();
    __syncthreads();
    for (uint32_t c = 1; c < ncand && nkept < needed; ++c) {
        /* buffer c&1 holds candidate c (visible to everyone since the barrier that ended the previous step) */
        if (c + 1 < ncand) fetch_vector(ix, cs[c + 1], buf0 + ((c + 1) & 1u) * vbytes);
        uint4 const* q4 = reinterpret_cast<uint4 const*>(smem + (c & 1u) * vbytes);
        typename M::qconst_t const qc = query_constants<M>(ix, q4, cs[c], lane);
        bool const below = block_distances<M>(ix, q4, qc, kept, nkept, nullptr, cd[c]);
        cp_async_wait_all();
        /* written before the barrier so that every thread sees it in the next step; it only counts if accepted */
        if (threadIdx.x == 0) { kept[nkept] = cs[c]; keptd[nkept] = cd[c]; }
        int const bad = __syncthreads_or(below ? 1 : 0);
        if (!bad) nkept += 1;
    }
    __syncthreads();
    return nkept;
}

__device__ __forceinline__ uint32_t* list_row(device_index_t const& ix, uint32_t slot, uint32_t level, uint32_t& capacity,
                                              uint32_t& stride) {
    if (level == 0) {
        capacity = ix.m0;
        stride = ix.m0_stride;
        return const_cast<uint32_t*>(ix.nbr0) + (size_t)slot * ix.m0_stride;
    }
    capacity = ix.m;
    stride = ix.m_stride;
    return const_cast<uint32_t*>(ix.upper) + ((size_t)ix.upper_base[slot] + (level - 1u)) * ix.m_stride;
}

/* ---- step 2: form_links_to_closest_ for every (new member, level) ------------------------------------------- */

template <class M>
__global__ void __launch_bounds__(LINK_THREADS, 3) link_forward_kernel(__grid_constant__ device_index_t const ix,
                                                                    __grid_constant__ link_args_t const a) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint32_t task_shared;
    uint32_t* cs = reinterpret_cast<uint32_t*>(smem + a.off_cs);
    float* cd = reinterpret_cast<float*>(smem + a.off_cd);
    uint32_t const* kept = reinterpret_cast<uint32_t const*>(smem + a.off_kept);
    float const* keptd = reinterpret_cast<float const*>(smem + a.off_keptd);
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) task_shared = atomicAdd(a.work_counter, 1u);
        __syncthreads();
        uint32_t const t = task_shared;
        if (t >= a.ntasks) break;
        uint32_t const member = a.task_slot[t], level = a.task_level[t];
        uint32_t const ncand = min(min(a.cand_counts[t], a.ef), LINK_CAND_MAX);
        for (uint32_t i = threadIdx.x; i < ncand; i += blockDim.x) {
            cs[i] = a.cand_slots[(size_t)t * a.ef + i];
            cd[i] = a.cand_dists[(size_t)t * a.ef + i];
        }
        __syncthreads();
        uint32_t const nkept = refine_block<M>(ix, smem, a, ncand, ix.m); /* `config_.connectivity` on every level */
        uint32_t capacity, stride;
        uint32_t* row = list_row(ix, member, level, capacity, stride);
        for (uint32_t i = threadIdx.x; i < stride; i += blockDim.x) row[i] = i < nkept ? kept[i] : EMPTY_SLOT;
        for (uint32_t i = threadIdx.x; i < ix.m; i += blockDim.x) {
            a.pair_keys[(size_t)t * ix.m + i] = i < nkept ? (((uint64_t)level << 32) | kept[i]) : ~0ull;
            a.pair_dists[(size_t)t * ix.m + i] = i < nkept ? keptd[i] : 0.f;
        }
    }
}

/* ---- step 3: runs of equal (level, neighbour) in the sorted pairs ---------------------------------------------- */

__global__ void pair_heads_kernel(uint64_t const* sorted_keys, uint32_t npairs, uint32_t* heads, uint32_t* nheads) {
    uint32_t const p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npairs) return;
    uint64_t const key = sorted_keys[p];
    if (key == ~0ull) return;
    if (p == 0 || sorted_keys[p - 1] != key) heads[atomicAdd(nheads, 1u)] = p;
}

/* ---- step 4: form_reverse_links_ for every (level, neighbour) that was chosen by members of the batch ------------- */

template <class M>
__global__ void __launch_bounds__(LINK_THREADS, 3) link_reverse_kernel(__grid_constant__ device_index_t const ix,
                                                                    __grid_constant__ link_args_t const a) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint32_t task_shared, count_shared;
    uint32_t* cs = reinterpret_cast<uint32_t*>(smem + a.off_cs);
    float* cd = reinterpret_cast<float*>(smem + a.off_cd);
    uint32_t const* kept = reinterpret_cast<uint32_t const*>(smem + a.off_kept);
    int const lane = threadIdx.x & 31;
    uint32_t const nheads = *a.nheads;
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) { task_shared = atomicAdd(a.work_counter, 1u); count_shared = 0; }
        __syncthreads();
        uint32_t const h = task_shared;
        if (h >= nheads) break;
        uint32_t const p0 = a.heads[h];
        uint64_t const key = a.sorted_keys[p0];
        uint32_t const level = (uint32_t)(key >> 32), centre = (uint32_t)key;
        uint32_t capacity, stride;
        uint32_t* row = list_row(ix, centre, level, capacity, stride);
        /* members already listed: a dense prefix of the row */
        uint32_t mine = 0;
        for (uint32_t i = threadIdx.x; i < capacity; i += blockDim.x) mine += row[i] != EMPTY_SLOT ? 1u : 0u;
        if (mine) atomicAdd(&count_shared, mine);
        __syncthreads();
        uint32_t const listed = count_shared;
        /* arrivals: the run of equal keys that starts at p0 (cut to what one refine can hold) */
        uint32_t const room = LINK_CAND_MAX - min(listed, LINK_CAND_MAX);
        uint32_t run = 0;
        while (run < room && p0 + run < a.npairs && a.sorted_keys[p0 + run] == key) ++run; /* uniform */
        /* An arrival that the list already holds is not appended again: a reused slot can still be listed from its
         * previous life (the reference appends a second copy; the search kernel's visited test needs lists without
         * repeats). `arrival` keeps the positions in the run of the others, in run order. */
        uint32_t* const arrival = reinterpret_cast<uint32_t*>(smem + a.off_kept);
        for (uint32_t i = threadIdx.x; i < run; i += blockDim.x) {
            uint32_t const s = a.task_slot[a.sorted_idx[p0 + i] / ix.m];
            bool listed_already = false;
            for (uint32_t j = 0; j < listed && !listed_already; ++j) listed_already = row[j] == s;
            arrival[i] = listed_already ? EMPTY_SLOT : p0 + i;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t fresh = 0;
            for (uint32_t i = 0; i < run; ++i)
                if (arrival[i] != EMPTY_SLOT) arrival[fresh++] = arrival[i];
            count_shared = fresh;
        }
        __syncthreads();
        uint32_t const arrivals = count_shared;
        if (listed + arrivals <= capacity) { /* close_header.push_back(new_slot), index.hpp:3871-3874 */
            for (uint32_t i = threadIdx.x; i < arrivals; i += blockDim.x) {
                uint32_t const idx = a.sorted_idx[arrival[i]];
                row[listed + i] = a.task_slot[idx / ix.m];
            }
            continue;
        }
        /* refine_ over the list plus the arrivals (index.hpp:3876-3890) */
        for (uint32_t i = threadIdx.x; i < LINK_CAND_MAX; i += blockDim.x) {
            uint32_t s = EMPTY_SLOT;
            float d = __int_as_float(0x7f800000);
            if (i < listed) s = row[i];
            else if (i < listed + arrivals) {
                uint32_t const idx = a.sorted_idx[arrival[i - listed]];
                s = a.task_slot[idx / ix.m];
                d = a.pair_dists[idx];
            }
            cs[i] = s;
            cd[i] = d;
        }
        __syncthreads(); /* `arrival` shares its memory with the kept list of refine_block */
        fetch_vector(ix, centre, smem_u32(smem));
        cp_async_wait_all();
        __syncthreads();
        {
            uint4 const* q4 = reinterpret_cast<uint4 const*>(smem);
            typename M::qconst_t const qc = query_constants<M>(ix, q4, centre, lane);
            block_distances<M>(ix, q4, qc, cs, listed, cd, 0.f);
        }
        __syncthreads();
        /* ascending by distance: bitonic sort of the LINK_CAND_MAX padded entries, one per thread */
        static_assert(LINK_CAND_MAX == LINK_THREADS, "one candidate per thread in the sort");
        for (uint32_t size = 2; size <= LINK_CAND_MAX; size <<= 1) {
            for (uint32_t step = size >> 1; step > 0; step >>= 1) {
                uint32_t const i = threadIdx.x, j = i ^ step;
                if (j > i) {
                    bool const up = (i & size) == 0;
                    float const di = cd[i], dj = cd[j];
                    uint32_t const si = cs[i], sj = cs[j];
                    bool const swap = up ? (di > dj || (di == dj && si > sj)) : (di < dj || (di == dj && si < sj));
                    if (swap) { cd[i] = dj; cd[j] = di; cs[i] = sj; cs[j] = si; }
                }
                __syncthreads();
            }
        }
        uint32_t const nkept = refine_block<M>(ix, smem, a, listed + arrivals, capacity);
        for (uint32_t i = threadIdx.x; i < stride; i += blockDim.x) row[i] = i < nkept ? kept[i] : EMPTY_SLOT;
    }
}

/* ---- dispatch over the metric family (the one-lane-group-per-vector structs of metrics.cuh) -------------------------- */

#define BUILD_DISPATCH(FN, ...)                                                                     \
    switch (ix.scalar) {                                                                            \
    case SCALAR_F32:                                                                                \
        if (ix.metric == METRIC_L2SQ) return FN<l2sq_f32_t>(__VA_ARGS__);                           \
        if (ix.metric == METRIC_IP) return FN<ip_f32_t>(__VA_ARGS__);                               \
        if (ix.metric == METRIC_COS) return FN<cos_f32_t>(__VA_ARGS__);                             \
        break;                                                                                      \
    case SCALAR_F64:                                                                                \
        if (ix.metric == METRIC_L2SQ) return FN<l2sq_f64_t>(__VA_ARGS__);                           \
        if (ix.metric == METRIC_IP) return FN<ip_f64_t>(__VA_ARGS__);                               \
        if (ix.metric == METRIC_COS) return FN<cos_f64_t>(__VA_ARGS__);                             \
        break;                                                                                      \
    case SCALAR_F16:                                                                                \
        if (ix.metric == METRIC_L2SQ) return FN<l2sq_half_t<f16_conv_t>>(__VA_ARGS__);              \
        if (ix.metric == METRIC_IP) return FN<ip_half_t<f16_conv_t>>(__VA_ARGS__);                  \
        if (ix.metric == METRIC_COS) return FN<cos_half_t<f16_conv_t>>(__VA_ARGS__);                \
        break;                                                                                      \
    case SCALAR_BF16:                                                                               \
        if (ix.metric == METRIC_L2SQ) return FN<l2sq_half_t<bf16_conv_t>>(__VA_ARGS__);             \
        if (ix.metric == METRIC_IP) return FN<ip_half_t<bf16_conv_t>>(__VA_ARGS__);                 \
        if (ix.metric == METRIC_COS) return FN<cos_half_t<bf16_conv_t>>(__VA_ARGS__);               \
        break;                                                                                      \
    case SCALAR_I8:                                                                                 \
        if (ix.metric == METRIC_L2SQ) return FN<l2sq_i8_t<4>>(__VA_ARGS__);                         \
        if (ix.metric == METRIC_IP) return FN<ip_i8_t<4>>(__VA_ARGS__);                             \
        if (ix.metric == METRIC_COS) return FN<cos_i8_t<4>>(__VA_ARGS__);                           \
        break;                                                                                      \
    case SCALAR_B1:                                                                                 \
        if (ix.metric == METRIC_HAMMING) return FN<hamming_b1_t<2>>(__VA_ARGS__);                   \
        if (ix.metric == METRIC_TANIMOTO || ix.metric == METRIC_JACCARD) return FN<tanimoto_b1_t<2>>(__VA_ARGS__); \
        if (ix.metric == METRIC_SORENSEN) return FN<sorensen_b1_t<2>>(__VA_ARGS__);                 \
        break;                                                                                      \
    default: break;                                                                                 \
    }                                                                                               \
    return cudaErrorInvalidValue;

template <class M>
cudaError_t launch_forward_t(device_index_t const& ix, link_args_t const& a, int blocks, size_t smem, cudaStream_t s) {
    cudaError_t e = cudaFuncSetAttribute(link_forward_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    link_forward_kernel<M><<<blocks, LINK_THREADS, smem, s>>>(ix, a);
    return cudaGetLastError();
}
template <class M>
cudaError_t launch_reverse_t(device_index_t const& ix, link_args_t const& a, int blocks, size_t smem, cudaStream_t s) {
    cudaError_t e = cudaFuncSetAttribute(link_reverse_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    link_reverse_kernel<M><<<blocks, LINK_THREADS, smem, s>>>(ix, a);
    return cudaGetLastError();
}
cudaError_t launch_forward(device_index_t const& ix, link_args_t const& a, int blocks, size_t smem, cudaStream_t s) {
    BUILD_DISPATCH(launch_forward_t, ix, a, blocks, smem, s)
}
cudaError_t launch_reverse(device_index_t const& ix, link_args_t const& a, int blocks, size_t smem, cudaStream_t s) {
    BUILD_DISPATCH(launch_reverse_t, ix, a, blocks, smem, s)
}

/* ---- one pair: usearch_distance (c/lib.cpp:458-466) ---------------------------------------------------------------- */

template <class M> __global__ void pair_distance_kernel(device_index_t const ix, uint8_t const* query, float* out) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint4* q4 = reinterpret_cast<uint4*>(smem);
    int const lane = threadIdx.x;
    for (uint32_t j = lane; j < ix.chunks16; j += 32) q4[j] = reinterpret_cast<uint4 const*>(query)[j];
    __syncwarp();
    typename M::qconst_t const qc = M::prepare(q4, ix.chunks16, lane);
    constexpr int LPV = M::LPV;
    int const sub = lane % LPV;
    uint4 const* v = reinterpret_cast<uint4 const*>(ix.vectors);
    typename M::acc_t acc;
    M::init(acc);
    for (uint32_t j = sub; j < ix.chunks16; j += LPV) M::step(acc, v[j], q4[j]);
    float d = M::finish(acc, qc);
    if constexpr (M::NORMS) {
        typename M::qconst_t const sc = M::prepare(v, ix.chunks16, lane); /* the stored side's norm, same chain */
        d = M::finalize(d, qc, sc.a2);
    }
    if (lane == 0) *out = d;
}
template <class M> cudaError_t launch_pair_t(device_index_t const& ix, uint8_t const* query, float* out, cudaStream_t s) {
    pair_distance_kernel<M><<<1, 32, ix.vec_stride, s>>>(ix, query, out);
    return cudaGetLastError();
}
cudaError_t launch_pair(device_index_t const& ix, uint8_t const* query, float* out, cudaStream_t s) {
    BUILD_DISPATCH(launch_pair_t, ix, query, out, s)
}

/* ---- gathered pairs: metric(a.rows[slot_a[j]], b.rows[slot_b[j]]) for join and pairwise_distance ----------------- */

/* One warp per pair, every lane group of LPV lanes walking both rows as pair_distance_kernel does (the groups of a warp
 * compute the same value, so `prepare` can use the whole warp). cos takes the stored norms of both rows where the index
 * keeps them: the same chain as `prepare`, so the bits equal usearch_distance for the same two vectors. */
template <class M>
__global__ void pair_distances_kernel(device_index_t const a, device_index_t const b, uint32_t const* slot_a,
                                      uint32_t const* slot_b, uint32_t n, float* out) {
    constexpr int LPV = M::LPV;
    int const lane = threadIdx.x & 31, sub = lane % LPV;
    uint32_t const warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += warps) {
        uint32_t const sa = slot_a[j], sb = slot_b[j];
        uint4 const* qa = reinterpret_cast<uint4 const*>(a.vectors + (size_t)sa * a.vec_stride);
        uint4 const* vb = reinterpret_cast<uint4 const*>(b.vectors + (size_t)sb * b.vec_stride);
        typename M::qconst_t qc;
        if constexpr (M::NORMS) {
            if (a.norms) qc.a2 = __ldg(a.norms + sa);
            else qc = M::prepare(qa, a.chunks16, lane);
        } else
            qc = M::prepare(qa, a.chunks16, lane);
        typename M::acc_t acc;
        M::init(acc);
        for (uint32_t c = sub; c < a.chunks16; c += LPV) M::step(acc, __ldg(vb + c), __ldg(qa + c));
        float d = M::finish(acc, qc);
        if constexpr (M::NORMS) d = M::finalize(d, qc, b.norms ? __ldg(b.norms + sb) : M::prepare(vb, b.chunks16, lane).a2);
        if (lane == 0) out[j] = d;
    }
}
template <class M>
cudaError_t launch_pairs_t(device_index_t const& ix, device_index_t const& b, uint32_t const* slot_a, uint32_t const* slot_b,
                           uint32_t n, float* out, cudaStream_t s) {
    unsigned const blocks = (unsigned)std::min<uint32_t>((n + 7) / 8, 65535u * 4);
    pair_distances_kernel<M><<<blocks, 256, 0, s>>>(ix, b, slot_a, slot_b, n, out);
    return cudaGetLastError();
}
cudaError_t launch_pairs(device_index_t const& ix, device_index_t const& b, uint32_t const* slot_a, uint32_t const* slot_b,
                         uint32_t n, float* out, cudaStream_t s) {
    BUILD_DISPATCH(launch_pairs_t, ix, b, slot_a, slot_b, n, out, s)
}

/* ---- scalar casts on the device (index_plugins.hpp:1105-1224; the element conversions are scalar_casts.h) ------------- */

/* element i of a row in scalar kind `kind`, as the value the reference's cast_gt<from, *> sees */
__device__ __forceinline__ double load_scalar(uint8_t const* row, uint32_t kind, uint32_t i) {
    switch (kind) {
    case SCALAR_F32: return (double)reinterpret_cast<float const*>(row)[i];
    case SCALAR_F64: return reinterpret_cast<double const*>(row)[i];
    case SCALAR_F16: return (double)f16_bits_to_f32(reinterpret_cast<uint16_t const*>(row)[i]);
    case SCALAR_BF16: return (double)bf16_bits_to_f32(reinterpret_cast<uint16_t const*>(row)[i]);
    case SCALAR_I8: return (double)((float)reinterpret_cast<int8_t const*>(row)[i] / 127.f); /* cast_from_i8_gt */
    case SCALAR_B1: return (row[i >> 3] & (128u >> (i & 7u))) ? 1.0 : 0.0;                   /* cast_from_b1x8_gt */
    default: return 0.0;
    }
}

/* the same element as an f32, for f32 / f16 / bf16 targets: an f32 source is read as it is and an f64 narrowed as the host
 * narrows it, so that NaN payloads and signalling NaNs reach the half casts unchanged (an f64 round trip would quiet
 * them, and the device's own f64 -> f32 conversion returns a canonical NaN) */
__device__ __forceinline__ float load_f32(uint8_t const* row, uint32_t kind, uint32_t i) {
    switch (kind) {
    case SCALAR_F32: return reinterpret_cast<float const*>(row)[i];
    case SCALAR_F64: return f64_to_f32(reinterpret_cast<double const*>(row)[i]);
    case SCALAR_F16: return f16_bits_to_f32(reinterpret_cast<uint16_t const*>(row)[i]);
    case SCALAR_BF16: return bf16_bits_to_f32(reinterpret_cast<uint16_t const*>(row)[i]);
    default: return (float)load_scalar(row, kind, i); /* i8 and b1 values are finite */
    }
}

/* float targets and bits: one thread per element / per output byte */
__global__ void cast_elements_kernel(uint8_t const* src, size_t src_stride, uint32_t from, uint8_t* dst, size_t dst_stride,
                                     uint32_t to, uint32_t dims, size_t rows) {
    size_t const per_row = to == SCALAR_B1 ? (dims + 7) / 8 : dims;
    size_t const gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= rows * per_row) return;
    size_t const r = gid / per_row;
    uint32_t const i = (uint32_t)(gid - r * per_row);
    uint8_t const* in = src + r * src_stride;
    uint8_t* out = dst + r * dst_stride;
    if (to == SCALAR_B1) { /* cast_to_b1x8_gt: bit = value > 0, most significant bit first */
        uint32_t byte = 0;
        for (uint32_t b = 0; b < 8 && i * 8 + b < dims; ++b)
            if (load_scalar(in, from, i * 8 + b) > 0) byte |= 128u >> b;
        out[i] = (uint8_t)byte;
        return;
    }
    /* f64 sources are narrowed to f32 first: f16_bits_t(double) / bf16_bits_t(double), index_plugins.hpp:489, :553 */
    float const v = load_f32(in, from, i);
    if (to == SCALAR_F32) reinterpret_cast<float*>(out)[i] = v;
    else if (to == SCALAR_F16) reinterpret_cast<uint16_t*>(out)[i] = f32_to_f16_bits(v);
    else if (to == SCALAR_BF16) reinterpret_cast<uint16_t*>(out)[i] = f32_to_bf16_bits(v);
    else if (to == SCALAR_I8) reinterpret_cast<int8_t*>(out)[i] = v > 0 ? 1 : 0; /* b1 sources only: cast_from_b1x8_gt<i8_t> */
}

/* cast_to_i8_gt (index_plugins.hpp:1172-1191): x * 127 / |x| in f64, clamp, truncate; the magnitude is the SEQUENTIAL f64
 * sum of squares, so one thread walks a row (mul and add kept apart: the parity build of the reference does not contract) */
__global__ void cast_rows_to_i8_kernel(uint8_t const* src, size_t src_stride, uint32_t from, uint8_t* dst, size_t dst_stride,
                                       uint32_t dims, size_t rows) {
    size_t const r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    uint8_t const* in = src + r * src_stride;
    int8_t* out = reinterpret_cast<int8_t*>(dst + r * dst_stride);
    double magnitude = 0.0;
    for (uint32_t i = 0; i < dims; ++i) {
        double const x = load_scalar(in, from, i);
        magnitude = __dadd_rn(magnitude, __dmul_rn(x, x));
    }
    magnitude = __dsqrt_rn(magnitude);
    for (uint32_t i = 0; i < dims; ++i) {
        double v = __ddiv_rn(__dmul_rn(load_scalar(in, from, i), 127.0), magnitude);
        v = v > 127.0 ? 127.0 : (v < -127.0 ? -127.0 : v); /* NaN (zero vector) passes through, like usearch::clamp */
        out[i] = (int8_t)(int)v;
    }
}

/* cast_gt<*, f64> (index_plugins.hpp:1105-1224), one thread per element: f32, f16 and bf16 widen exactly, b1 gives 1.0 or
 * 0.0, and i8 is cast_from_i8_gt<f64>, a double division `(double)x / 127.0` (not the f32 quotient of load_scalar) */
__global__ void cast_elements_to_f64_kernel(uint8_t const* src, size_t src_stride, uint32_t from, uint8_t* dst, size_t dst_stride,
                                            uint32_t dims, size_t rows) {
    size_t const gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= rows * dims) return;
    size_t const r = gid / dims;
    uint32_t const i = (uint32_t)(gid - r * dims);
    uint8_t const* in = src + r * src_stride;
    double const v = from == SCALAR_I8 ? __ddiv_rn((double)reinterpret_cast<int8_t const*>(in)[i], 127.0) : load_scalar(in, from, i);
    reinterpret_cast<double*>(dst + r * dst_stride)[i] = v;
}

/* ---- removal and reuse: per-slot edits of `keys` / `deleted_bits`, rows scattered into reused slots ------------------ */

/* new_keys == NULL: index_dense_gt::remove (index_dense.hpp:1479-1513), the slot takes the free key and its deleted bit;
 * else the slot is reused under new_keys[i] and leaves the removed set */
__global__ void edit_slots_kernel(uint32_t const* slots, uint32_t n, uint64_t const* new_keys, uint64_t free_key, uint64_t* keys,
                                  uint32_t* deleted_bits) {
    uint32_t const i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t const s = slots[i];
    if (new_keys) {
        keys[s] = new_keys[i];
        atomicAnd(deleted_bits + (s >> 5), ~(1u << (s & 31)));
    } else {
        keys[s] = free_key;
        atomicOr(deleted_bits + (s >> 5), 1u << (s & 31));
    }
}

/* row i of `src` (already zero-padded to vec_stride) -> the row of slot slots[i] */
__global__ void scatter_rows_kernel(uint4 const* src, uint32_t const* slots, uint32_t n, uint32_t chunks16, uint4* vectors) {
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        uint4* dst = vectors + (size_t)slots[i] * chunks16;
        for (uint32_t j = threadIdx.x; j < chunks16; j += blockDim.x) dst[j] = src[(size_t)i * chunks16 + j];
    }
}

/* index_gt::isolate (index.hpp:3695-3728): one warp per list — the layer-0 rows of slots [0, n), then the upper rows in
 * use — drops every link to a removed slot, keeps the survivors in stored order and fills the tail with EMPTY_SLOT. The
 * dropped links are the reference's `pruned_edges`. Removed members keep their own links (the reference's comment at
 * index.hpp:3684-3690). */
__global__ void isolate_kernel(device_index_t const ix, uint32_t upper_rows, unsigned long long* pruned) {
    uint32_t const lane = threadIdx.x & 31, lt = (1u << lane) - 1;
    size_t const warps = (size_t)gridDim.x * (blockDim.x >> 5);
    size_t const rows = (size_t)ix.n + upper_rows;
    uint32_t dropped = 0;
    for (size_t r = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += warps) {
        bool const base = r < ix.n;
        uint32_t const width = base ? ix.m0 : ix.m;
        uint32_t* const row = const_cast<uint32_t*>(base ? ix.nbr0 + r * ix.m0_stride : ix.upper + (r - ix.n) * ix.m_stride);
        uint32_t kept = 0;
        for (uint32_t b = 0; b < width; b += 32) {
            uint32_t const s = b + lane < width ? row[b + lane] : EMPTY_SLOT;
            bool const gone = s != EMPTY_SLOT && ((ix.deleted_bits[s >> 5] >> (s & 31)) & 1u);
            bool const keep = s != EMPTY_SLOT && !gone;
            uint32_t const bal = __ballot_sync(0xffffffffu, keep);
            dropped += __popc(__ballot_sync(0xffffffffu, gone));
            __syncwarp(); /* every lane has read its entry before the survivors move down */
            if (keep) row[kept + __popc(bal & lt)] = s;
            kept += __popc(bal);
        }
        __syncwarp();
        for (uint32_t i = kept + lane; i < width; i += 32) row[i] = EMPTY_SLOT;
    }
    if (lane == 0 && dropped) atomicAdd(pruned, (unsigned long long)dropped);
}

uint64_t mix64(uint64_t x) { /* splitmix64 finaliser */
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

} // namespace

/* rows of `from` scalars -> rows of the index's scalar kind, zero-padded to dst_stride; both on the device */
char const* cast_rows_device(uint8_t const* src, size_t src_stride, uint32_t from, uint8_t* dst, size_t dst_stride, uint32_t to,
                             size_t dims, size_t rows, cudaStream_t s) {
    if (!rows) return nullptr;
    size_t const to_bytes = (dims * bits_per_scalar(to) + 7) / 8;
    if (dst_stride != to_bytes) CU(cudaMemsetAsync(dst, 0, rows * dst_stride, s));
    if (from == to) {
        CU(cudaMemcpy2DAsync(dst, dst_stride, src, src_stride, to_bytes, rows, cudaMemcpyDeviceToDevice, s));
        return nullptr;
    }
    if (!bits_per_scalar(from)) return "Unknown scalar kind!";
    if (to == SCALAR_I8 && from != SCALAR_B1) {
        cast_rows_to_i8_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, s>>>(src, src_stride, from, dst, dst_stride, (uint32_t)dims, rows);
    } else if (to == SCALAR_F64) {
        cast_elements_to_f64_kernel<<<(unsigned)((rows * dims + 255) / 256), 256, 0, s>>>(src, src_stride, from, dst, dst_stride, (uint32_t)dims, rows);
    } else if (to == SCALAR_F32 || to == SCALAR_F16 || to == SCALAR_BF16 || to == SCALAR_B1 || to == SCALAR_I8) {
        size_t const total = rows * (to == SCALAR_B1 ? (dims + 7) / 8 : dims);
        cast_elements_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(src, src_stride, from, dst, dst_stride, to, (uint32_t)dims, rows);
    } else
        return "Unsupported scalar kind";
    CU(cudaGetLastError());
    return nullptr;
}

/* metric(a, b) for one pair of vectors already in the index's scalar kind and padded to whole 16-byte chunks */
char const* pair_distance_device(device_index_t const& shape, uint8_t const* d_a, uint8_t const* d_b, float* d_out, cudaStream_t s) {
    device_index_t ix = shape;
    ix.vectors = d_b;
    ix.n = 1;
    CU(launch_pair(ix, d_a, d_out, s));
    return nullptr;
}

/* metric(a.rows[slot_a[j]], b.rows[slot_b[j]]) for j < n; a and b share metric, scalar kind and dimensions */
char const* pair_distances_device(device_index_t const& a, device_index_t const& b, uint32_t const* d_slot_a, uint32_t const* d_slot_b,
                                  size_t n, float* d_out, cudaStream_t s) {
    if (!n) return nullptr;
    if (n > 0xFFFFFFFFull) return "Too many pairs in one batch";
    CU(launch_pairs(a, b, d_slot_a, d_slot_b, (uint32_t)n, d_out, s));
    return nullptr;
}

__global__ void iota_u64_kernel(uint64_t* out, uint32_t n) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = i;
}

char const* iota_u64_device(uint64_t* d_out, size_t n, cudaStream_t s) {
    if (!n) return nullptr;
    iota_u64_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, 65535), 256, 0, s>>>(d_out, (uint32_t)n);
    CU(cudaGetLastError());
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------------------------------- */
/*  capacity                                                                                                                */
/* ---------------------------------------------------------------------------------------------------------------------- */

namespace {

template <typename T>
char const* regrow(device_buffer_t<T>& array, T const*& view, size_t old_count, size_t new_count, int fill_byte, cudaStream_t s) {
    device_buffer_t<T> fresh;
    if (char const* e = fresh.reserve(std::max<size_t>(new_count, 1))) return e;
    if (old_count) CU(cudaMemcpyAsync(fresh.ptr, view, old_count * sizeof(T), cudaMemcpyDeviceToDevice, s));
    if (new_count > old_count && fill_byte >= 0)
        CU(cudaMemsetAsync(fresh.ptr + old_count, fill_byte, (new_count - old_count) * sizeof(T), s));
    CU(cudaStreamSynchronize(s));
    array = std::move(fresh);
    view = array.ptr;
    return nullptr;
}

} // namespace

/* index_dense_gt::try_reserve (index_dense.hpp:907-945) for the HBM layout: room for `slots` members */
char const* frozen_index_t::reserve_slots(size_t slots) {
    if (char const* e = ensure_context()) return e;
    if (!configured()) return "Index is not initialized: call usearch_init with options or load a file first";
    if (slots >= 0xFFFFFFFFull) return "Too many entries for 32-bit slots";
    if (connectivity_base >= LINK_CAND_MAX || connectivity > connectivity_base)
        return "Connectivity too large for the GPU builder (a list plus one arrival must fit 256 candidates)";
    if (!loaded) { /* first reservation of an index made by usearch_init(options): the empty layout */
        device_index_t ix;
        ix.m = (uint32_t)connectivity;
        ix.m0 = (uint32_t)connectivity_base;
        ix.m_stride = round_up(ix.m, 4);
        ix.m0_stride = round_up(ix.m0, 4);
        ix.dims = (uint32_t)dimensions;
        ix.bytes_per_vector = (uint32_t)((dimensions * bits_per_scalar(scalar) + 7) / 8);
        ix.vec_stride = round_up(ix.bytes_per_vector, 16);
        ix.chunks16 = (uint32_t)(ix.vec_stride / 16);
        ix.metric = metric;
        ix.scalar = scalar;
        if (search_needs_shadow(ix)) ix.code_stride = search_code_stride(ix);
        d = ix;
        loaded = true;
    }
    if (slots <= capacity) return nullptr;
    size_t const old_cap = capacity;
    size_t const rows_old = upper_capacity;
    /* expected upper rows: n / (M - 1); keep a quarter more, the rest grows on demand */
    size_t const rows_new = std::max<size_t>(rows_old, slots / std::max<size_t>(connectivity - 1, 1) * 5 / 4 + 1024);
    if (char const* e = regrow(hbm.vectors, d.vectors, old_cap * d.vec_stride, slots * d.vec_stride, -1, stream)) return e;
    if (char const* e = regrow(hbm.keys, d.keys, old_cap, slots, -1, stream)) return e;
    if (char const* e = regrow(hbm.nbr0, d.nbr0, old_cap * d.m0_stride, slots * d.m0_stride, 0xFF, stream)) return e;
    if (char const* e = regrow(hbm.upper_base, d.upper_base, old_cap, slots, 0xFF, stream)) return e;
    if (rows_new > rows_old) {
        if (char const* e = regrow(hbm.upper, d.upper, rows_old * d.m_stride, rows_new * d.m_stride, 0xFF, stream)) return e;
        upper_capacity = rows_new;
    }
    if (d.deleted_bits)
        if (char const* e = regrow(hbm.deleted_bits, d.deleted_bits, (old_cap + 31) / 32, (slots + 31) / 32, 0, stream)) return e;
    if (search_needs_norms(metric, scalar))
        if (char const* e = regrow(hbm.norms, d.norms, old_cap, slots, -1, stream)) return e;
    if (d.code_stride) { /* the int8 shadow of cos / ip f32 (prefilter_bound.h) */
        if (char const* e = regrow(hbm.codes, d.codes, old_cap * d.code_stride, slots * d.code_stride, -1, stream)) return e;
        if (char const* e = regrow(hbm.shadow, d.shadow, old_cap, slots, -1, stream)) return e;
    }
    capacity = slots;
    hbm_bytes = capacity * (d.vec_stride + 8 + (size_t)d.m0_stride * 4 + 4 + (d.norms ? 4 : 0) +
                            (d.code_stride ? d.code_stride + sizeof(pf_record_t) : 0)) + upper_capacity * d.m_stride * 4 +
                (d.deleted_bits ? (capacity + 31) / 32 * 4 : 0);
    visited_zeroed_words = 0; /* the visits bitmaps are sized by capacity */
    return nullptr;
}

char const* frozen_index_t::reserve_upper_rows(size_t rows) {
    if (rows <= upper_capacity) return nullptr;
    size_t const rows_new = std::max(rows, upper_capacity * 2 + 1024);
    if (char const* e = regrow(hbm.upper, d.upper, upper_capacity * d.m_stride, rows_new * d.m_stride, 0xFF, stream)) return e;
    upper_capacity = rows_new;
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------------------------------- */
/*  add                                                                                                                     */
/* ---------------------------------------------------------------------------------------------------------------------- */

/* choose_random_level_ (index.hpp:3895-3899) with a counter-based generator: the level of the member in slot s is a pure
 * function of (s, seed), so a build is reproducible whatever the batch boundaries are */
int16_t frozen_index_t::draw_level(size_t slot) const {
    uint64_t const bits = mix64((uint64_t)slot ^ (level_seed * 0xD6E8FEB86659FD93ull));
    double const u = ((double)(bits >> 11) + 1.0) * (1.0 / 9007199254740992.0); /* (0, 1] */
    double const r = -std::log(u) * (1.0 / std::log((double)connectivity));
    return (int16_t)std::min<double>(r, 30.0);
}

/* `rows` caller vectors (host or device memory, any supported scalar kind) -> device rows of the index's scalar kind at
 * `dst`, zero-padded to vec_stride; cast on the device when the kinds differ */
char const* frozen_index_t::write_rows(void const* vectors, size_t rows, size_t stride, uint32_t kind, bool on_device, uint8_t* dst) {
    if (!rows) return nullptr;
    size_t const src_bytes = (dimensions * bits_per_scalar(kind) + 7) / 8;
    if (kind == scalar) {
        if (d.vec_stride != d.bytes_per_vector) CU(cudaMemsetAsync(dst, 0, rows * d.vec_stride, stream));
        CU(cudaMemcpy2DAsync(dst, d.vec_stride, vectors, stride, d.bytes_per_vector, rows,
                             on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream));
        return nullptr;
    }
    size_t const chunk_rows = std::max<size_t>(1, (256u << 20) / std::max<size_t>(src_bytes, 1));
    for (size_t lo = 0; lo < rows; lo += chunk_rows) {
        size_t const n = std::min(chunk_rows, rows - lo);
        uint8_t const* src = static_cast<uint8_t const*>(vectors) + lo * stride;
        size_t src_stride = stride;
        if (!on_device) {
            if (char const* e = cast_stage.reserve(n * src_bytes)) return e;
            CU(cudaMemcpy2DAsync(cast_stage.ptr, src_bytes, src, stride, src_bytes, n, cudaMemcpyHostToDevice, stream));
            src = cast_stage.ptr;
            src_stride = src_bytes;
        }
        if (char const* e = cast_rows_device(src, src_stride, kind, dst + lo * d.vec_stride, d.vec_stride, scalar, dimensions, n, stream))
            return e;
        CU(cudaStreamSynchronize(stream)); /* the staging buffer is reused by the next chunk */
    }
    return nullptr;
}

/* keys == NULL: mark `slots` removed; else give slot slots[i] the key keys[i] (host memory) and clear its deleted bit */
char const* frozen_index_t::set_slot_keys(uint32_t const* slots, size_t count, uint64_t const* keys) {
    if (!count) return nullptr;
    if (!d.deleted_bits) {
        size_t const words = (capacity + 31) / 32;
        if (char const* e = hbm.deleted_bits.reserve(words)) return e;
        CU(cudaMemsetAsync(hbm.deleted_bits.ptr, 0, words * 4, stream));
        d.deleted_bits = hbm.deleted_bits.ptr;
        hbm_bytes += words * 4;
    }
    if (char const* e = edit_slots.reserve(count)) return e;
    CU(cudaMemcpyAsync(edit_slots.ptr, slots, count * 4, cudaMemcpyHostToDevice, stream));
    if (keys) {
        if (char const* e = edit_keys.reserve(count)) return e;
        CU(cudaMemcpyAsync(edit_keys.ptr, keys, count * 8, cudaMemcpyHostToDevice, stream));
    }
    edit_slots_kernel<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(edit_slots.ptr, (uint32_t)count, keys ? edit_keys.ptr : nullptr,
                                                                           free_key, const_cast<uint64_t*>(d.keys),
                                                                           const_cast<uint32_t*>(d.deleted_bits));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(stream)); /* `slots` / `keys` are the caller's pageable memory */
    return nullptr;
}

/* Store `count` vectors (host or device memory, any supported scalar kind), assign keys and levels, and link them into the
 * graph batch by batch. With `reuse_removed`, the first of them take the oldest removed slots (index_dense_gt::add_,
 * index_dense.hpp:2020-2049, then index_gt::update, index.hpp:2911-2999) and only the rest are appended. */
char const* frozen_index_t::add_many(uint64_t const* new_keys, void const* vectors, size_t count, size_t stride, uint32_t kind,
                                     bool on_device) {
    if (!count) return nullptr;
    if (char const* e = ensure_context()) return e;
    keys_generation += 1;
    if (!configured()) return "Index is not initialized: call usearch_init with options or load a file first";
    if (!bits_per_scalar(kind)) return "Unknown scalar kind!";
    size_t const reused = reuse_removed ? std::min(count, free_slots.size()) : 0;
    size_t const appended = count - reused;
    size_t const first = size;
    if (first + appended >= 0xFFFFFFFFull) return "Too many entries for 32-bit slots";
    if (first + appended > capacity) {
        /* c/lib.cpp leaves growth to the caller ("Reserve capacity ahead of insertions!", index.hpp:2816); the Python binding
         * grows by powers of two (python/lib.cpp:203-208) — here the library does the same on its own */
        size_t want = std::max<size_t>(first + appended, capacity * 2);
        if (char const* e = reserve_slots(want)) return e;
    }
    std::vector<uint64_t> keys_copy;
    if (on_device) { /* the checks below read the keys on the host */
        keys_copy.resize(count);
        CU(cudaMemcpy(keys_copy.data(), new_keys, count * 8, cudaMemcpyDeviceToHost));
    }
    uint64_t const* const hk = on_device ? keys_copy.data() : new_keys;
    for (size_t i = 0; i < count; ++i)
        if (hk[i] == free_key) return "Key is reserved for removed entries";
    if (!multi) { /* index_dense.hpp:2014: "Duplicate keys not allowed in high-level wrappers" */
        build_key_map();
        for (size_t i = 0; i < count; ++i)
            if (key_map.contains(hk[i])) return "Duplicate keys not allowed in high-level wrappers";
        if (count > 1) { /* ... nor twice within one call: the reference would refuse the second `add` */
            std::vector<uint64_t> sorted(hk, hk + count);
            std::sort(sorted.begin(), sorted.end());
            if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) return "Duplicate keys not allowed in high-level wrappers";
        }
    }
    size_t const src_bytes = (dimensions * bits_per_scalar(kind) + 7) / 8;
    if (stride == 0) stride = src_bytes;
    uint8_t const* const appended_vectors = static_cast<uint8_t const*>(vectors) + reused * stride;

    /* reused slots: the new rows are staged, scattered into their slots, and their norms / int8 shadow recomputed */
    std::vector<uint32_t> reuse_slots(free_slots.begin(), free_slots.begin() + (ptrdiff_t)reused);
    if (reused) {
        if (char const* e = reuse_stage.reserve(reused * d.vec_stride)) return e;
        if (char const* e = write_rows(vectors, reused, stride, kind, on_device, reuse_stage.ptr)) return e;
        if (char const* e = edit_slots.reserve(reused)) return e;
        CU(cudaMemcpyAsync(edit_slots.ptr, reuse_slots.data(), reused * 4, cudaMemcpyHostToDevice, stream));
        scatter_rows_kernel<<<(unsigned)std::min<size_t>(reused, 65535), 128, 0, stream>>>(
            reinterpret_cast<uint4 const*>(reuse_stage.ptr), edit_slots.ptr, (uint32_t)reused, d.chunks16,
            reinterpret_cast<uint4*>(const_cast<uint8_t*>(d.vectors)));
        CU(cudaGetLastError());
        device_index_t part = d;
        part.n = (uint32_t)reused;
        if (d.norms) CU(search_compute_norms(part, const_cast<float*>(d.norms), stream, edit_slots.ptr));
        if (d.codes) /* after the norms: the records copy them */
            CU(search_compute_shadow(part, d.norms, const_cast<int8_t*>(d.codes), const_cast<pf_record_t*>(d.shadow), stream,
                                     edit_slots.ptr));
        CU(cudaStreamSynchronize(stream));
        free_slots.erase(free_slots.begin(), free_slots.begin() + (ptrdiff_t)reused);
    }

    /* appended: vectors -> slab rows [first, first + appended) */
    uint8_t* slab = const_cast<uint8_t*>(d.vectors) + first * d.vec_stride;
    if (appended) {
        if (char const* e = write_rows(appended_vectors, appended, stride, kind, on_device, slab)) {
            free_slots.insert(free_slots.begin(), reuse_slots.begin(), reuse_slots.end());
            return e;
        }
        CU(cudaMemcpyAsync(const_cast<uint64_t*>(d.keys) + first, new_keys + reused, appended * 8,
                           on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream));
        if (d.norms) {
            device_index_t part = d;
            part.vectors = slab;
            part.n = (uint32_t)appended;
            CU(search_compute_norms(part, const_cast<float*>(d.norms) + first, stream));
        }
        if (d.codes) { /* after the norms: the records copy them */
            device_index_t part = d;
            part.vectors = slab;
            part.n = (uint32_t)appended;
            CU(search_compute_shadow(part, d.norms ? d.norms + first : nullptr, const_cast<int8_t*>(d.codes) + first * d.code_stride,
                                     const_cast<pf_record_t*>(d.shadow) + first, stream));
        }
        CU(cudaStreamSynchronize(stream)); /* `vectors` / `new_keys` may be pageable host memory owned by the caller */
    }

    /* host-side bookkeeping of the appended members: keys, levels, rows in `upper` */
    host_keys.reserve(first + appended);
    levels.reserve(first + appended);
    std::vector<uint32_t> bases(appended);
    size_t rows = upper_rows;
    host_keys.insert(host_keys.end(), hk + reused, hk + count);
    for (size_t i = 0; i < appended; ++i) {
        int16_t const level = draw_level(first + i);
        levels.push_back(level);
        bases[i] = level ? (uint32_t)rows : EMPTY_SLOT;
        rows += (size_t)level;
    }
    if (rows >= 0xFFFFFFFFull) return "Too many upper-level rows";
    if (char const* e = reserve_upper_rows(rows)) return e;
    upper_rows = rows;
    if (appended) {
        CU(cudaMemcpyAsync(const_cast<uint32_t*>(d.upper_base) + first, bases.data(), appended * 4, cudaMemcpyHostToDevice, stream));
        CU(cudaStreamSynchronize(stream));
    }
    if (key_map.built)
        for (size_t i = 0; i < appended; ++i) key_map.insert(host_keys[first + i], (uint32_t)(first + i));
    size = first + appended; /* stored; `d.n` counts the members that are linked into the graph */

    /* link them, batch by batch: the reused slots first, then the appended ones */
    static size_t const batch_max = [] { char const* v = std::getenv("USEARCH_B200_BUILD_BATCH"); return v && std::atol(v) > 0 ? (size_t)std::atol(v) : (size_t)32768; }();
    static size_t const ratio = [] { char const* v = std::getenv("USEARCH_B200_BUILD_RATIO"); return v && std::atol(v) > 0 ? (size_t)std::atol(v) : (size_t)32; }();
    auto drop_unlinked = [&](size_t reused_linked) {
        /* reused slots that were not linked go back to the front of the queue and stay removed; members that were
         * stored but not linked are dropped again: the index stays what the graph says it is */
        free_slots.insert(free_slots.begin(), reuse_slots.begin() + (ptrdiff_t)reused_linked, reuse_slots.end());
        size_t rows_kept = 0;
        for (size_t i = 0; i < (size_t)d.n; ++i) rows_kept += (size_t)levels[i];
        size = d.n;
        host_keys.resize(size);
        levels.resize(size);
        upper_rows = rows_kept;
        key_map.clear();
        cudaMemsetAsync(const_cast<uint32_t*>(d.nbr0) + size * d.m0_stride, 0xFF, (first + appended - size) * d.m0_stride * 4, stream);
        if (upper_capacity > upper_rows)
            cudaMemsetAsync(const_cast<uint32_t*>(d.upper) + upper_rows * d.m_stride, 0xFF, (upper_capacity - upper_rows) * d.m_stride * 4, stream);
        cudaStreamSynchronize(stream);
    };
    for (size_t at = 0; at < reused;) {
        /* a reused member keeps its level (<= the top level) and its rows: it never ends a batch */
        size_t const batch = std::min<size_t>({reused - at, batch_max, std::max<size_t>((size_t)d.n / ratio, 1)});
        char const* e = link_batch(reuse_slots.data() + at, batch);
        if (!e) e = set_slot_keys(reuse_slots.data() + at, batch, hk + at);
        if (e) {
            drop_unlinked(at);
            return e;
        }
        build_key_map();
        for (size_t i = at; i < at + batch; ++i) {
            host_keys[reuse_slots[i]] = hk[i];
            key_map.insert(hk[i], reuse_slots[i]);
        }
        count_deleted -= batch;
        at += batch;
    }
    std::vector<uint32_t> batch_slots;
    size_t at = first;
    while (at < size) {
        if (d.n == 0) { /* the first member: entry point, no links (index.hpp:2836-2841) */
            d.entry_slot = (uint32_t)at;
            d.max_level = levels[at];
            d.n = 1;
            at += 1;
            continue;
        }
        size_t batch = std::min<size_t>({size - at, batch_max, std::max<size_t>((size_t)d.n / ratio, 1)});
        /* a member above the current top level ends its batch: the next batch descends from it */
        for (size_t i = 0; i < batch; ++i)
            if (levels[at + i] > d.max_level) { batch = i + 1; break; }
        batch_slots.resize(batch);
        for (size_t i = 0; i < batch; ++i) batch_slots[i] = (uint32_t)(at + i);
        if (char const* e = link_batch(batch_slots.data(), batch)) {
            drop_unlinked(reused);
            return e;
        }
        at += batch;
    }
    return nullptr;
}

/* steps 1-4 of the header comment for the members in `slots`: appended slots (>= d.n, in order), or reused slots whose
 * rows are rewritten on every level they own */
char const* frozen_index_t::link_batch(uint32_t const* slots, size_t count) {
    cudaStream_t const s = stream;
    uint32_t const top_level = (uint32_t)d.max_level;
    /* work items: level 0 of every member first (the long searches start first), then the upper levels */
    std::vector<uint32_t> t_slot;
    std::vector<uint8_t> t_level;
    t_slot.reserve(count + count / 8 + 8);
    t_level.reserve(count + count / 8 + 8);
    for (size_t i = 0; i < count; ++i) { t_slot.push_back(slots[i]); t_level.push_back(0); }
    int16_t new_top = d.max_level;
    uint32_t new_entry = d.entry_slot, new_n = d.n;
    for (size_t i = 0; i < count; ++i) {
        int16_t const level = levels[slots[i]];
        for (uint32_t l = 1; l <= std::min<uint32_t>((uint32_t)level, top_level); ++l) { t_slot.push_back(slots[i]); t_level.push_back((uint8_t)l); }
        if (level > new_top) { new_top = level; new_entry = slots[i]; }
        new_n = std::max(new_n, slots[i] + 1);
    }
    size_t const ntasks = t_slot.size();
    uint32_t const ef = (uint32_t)std::max<size_t>(expansion_add ? expansion_add : 128, 1);
    uint32_t const m = d.m;

    build_scratch_t& b = build;
    if (char const* e = b.task_slot.reserve(ntasks)) return e;
    if (char const* e = b.task_level.reserve(ntasks)) return e;
    if (char const* e = b.cand_slots.reserve(ntasks * ef)) return e;
    if (char const* e = b.cand_dists.reserve(ntasks * ef)) return e;
    if (char const* e = b.cand_counts.reserve(ntasks)) return e;
    if (char const* e = b.pair_keys.reserve(ntasks * m)) return e;
    if (char const* e = b.pair_keys_sorted.reserve(ntasks * m)) return e;
    if (char const* e = b.pair_idx.reserve(ntasks * m)) return e;
    if (char const* e = b.pair_idx_sorted.reserve(ntasks * m)) return e;
    if (char const* e = b.pair_dists.reserve(ntasks * m)) return e;
    if (char const* e = b.heads.reserve(ntasks * m)) return e;
    if (char const* e = b.counters.reserve(4)) return e;
    if (char const* e = status.reserve(ntasks)) return e;
    if (char const* e = h_status.reserve(ntasks)) return e;
    CU(cudaMemcpyAsync(b.task_slot.ptr, t_slot.data(), ntasks * 4, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(b.task_level.ptr, t_level.data(), ntasks, cudaMemcpyHostToDevice, s));
    if (b.iota_count < ntasks * m) { /* values of the pair sort: 0, 1, 2, ... (written once, a prefix is reused) */
        std::vector<uint32_t> iota(ntasks * m);
        for (size_t i = 0; i < iota.size(); ++i) iota[i] = (uint32_t)i;
        CU(cudaMemcpyAsync(b.pair_idx.ptr, iota.data(), iota.size() * 4, cudaMemcpyHostToDevice, s));
        CU(cudaStreamSynchronize(s));
        b.iota_count = iota.size();
    }

    /* 1. candidates: the search kernel in INSERT mode, scratch grown and the launch repeated on overflow */
    for (uint64_t scale = 1;; scale *= 8) {
        launch_plan_t pl;
        if (char const* e = plan(ef, (uint32_t)std::min<uint64_t>(scale, 1u << 30), pl, ef)) return e;
        int const blocks = (int)std::min<size_t>((size_t)pl.blocks, ntasks);
        search_args_t a;
        if (char const* e = prepare_launch(pl, (size_t)blocks, a, s)) return e;
        a.queries = d.vectors;
        a.query_stride = d.vec_stride;
        a.nq = (uint32_t)ntasks;
        a.query_list = b.task_slot.ptr;
        a.task_levels = b.task_level.ptr;
        a.k = ef;
        a.out_slots = b.cand_slots.ptr;
        a.out_dists = b.cand_dists.ptr;
        a.out_counts = b.cand_counts.ptr;
        a.status = status.ptr;
        CU(cudaMemsetAsync(work_counter.ptr, 0, 8, s));
        CU(search_launch(d, a, blocks, pl.smem_per_block, s));
        kernel_launches += 1;
        CU(cudaMemcpyAsync(h_status.ptr, status.ptr, ntasks * 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        bool failed = false;
        for (size_t i = 0; i < ntasks && !failed; ++i) failed = h_status.ptr[i] != STATUS_OK;
        if (!failed) break;
        if (pl.maxed) return "Search scratch overflow that full-size scratch could not fix";
    }

    /* 2. forward links + pairs */
    link_args_t la;
    la.ntasks = (uint32_t)ntasks;
    la.task_slot = b.task_slot.ptr;
    la.task_level = b.task_level.ptr;
    la.cand_slots = b.cand_slots.ptr;
    la.cand_dists = b.cand_dists.ptr;
    la.cand_counts = b.cand_counts.ptr;
    la.ef = ef;
    la.pair_keys = b.pair_keys.ptr;
    la.pair_dists = b.pair_dists.ptr;
    uint32_t off = 2 * (uint32_t)d.vec_stride;
    la.off_cs = off; off += LINK_CAND_MAX * 4;
    la.off_cd = off; off += LINK_CAND_MAX * 4;
    la.off_kept = off; off += LINK_CAND_MAX * 4;
    la.off_keptd = off; off += LINK_CAND_MAX * 4;
    size_t const smem = off;
    if (smem > 200 * 1024) return "Dimensionality too large for the on-chip state of the builder";
    int const per_sm = (int)std::max<size_t>(1, std::min<size_t>(2048 / LINK_THREADS, (228 * 1024) / (smem + 1024)));
    int const grid = per_sm * stream.sm_count;
    CU(cudaMemsetAsync(b.counters.ptr, 0, 16, s));
    la.work_counter = b.counters.ptr + 0;
    CU(launch_forward(d, la, (int)std::min<size_t>((size_t)grid, ntasks), smem, s));

    /* 3. sort the pairs by (level, neighbour), cut into runs */
    size_t const npairs = ntasks * m;
    int const key_bits = 32 + 8;
    size_t temp_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, b.pair_keys.ptr, b.pair_keys_sorted.ptr, b.pair_idx.ptr,
                                       b.pair_idx_sorted.ptr, (int)npairs, 0, key_bits, s));
    if (char const* e = b.sort_temp.reserve(temp_bytes)) return e;
    CU(cub::DeviceRadixSort::SortPairs(b.sort_temp.ptr, temp_bytes, b.pair_keys.ptr, b.pair_keys_sorted.ptr, b.pair_idx.ptr,
                                       b.pair_idx_sorted.ptr, (int)npairs, 0, key_bits, s));
    pair_heads_kernel<<<(unsigned)((npairs + 255) / 256), 256, 0, s>>>(b.pair_keys_sorted.ptr, (uint32_t)npairs, b.heads.ptr, b.counters.ptr + 1);
    CU(cudaGetLastError());

    /* 4. reverse links */
    la.sorted_keys = b.pair_keys_sorted.ptr;
    la.sorted_idx = b.pair_idx_sorted.ptr;
    la.npairs = (uint32_t)npairs;
    la.heads = b.heads.ptr;
    la.nheads = b.counters.ptr + 1;
    la.work_counter = b.counters.ptr + 2;
    CU(launch_reverse(d, la, grid, smem, s));
    kernel_launches += 3;
    CU(cudaStreamSynchronize(s));

    d.n = new_n;
    d.max_level = new_top;
    d.entry_slot = new_entry;
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------------------------------- */
/*  remove                                                                                                                  */
/* ---------------------------------------------------------------------------------------------------------------------- */

/* index_dense_gt::remove over many keys (index_dense.hpp:1515-1557): each entry keeps its node and its links, its key becomes
 * the free key (so searches skip it: `deleted_bits`), the key leaves the lookup table, and the slot joins `free_slots`.
 * With `compact`, links that lead to removed entries are then pruned (python/lib.cpp:1210-1227 -> isolate). */
char const* frozen_index_t::remove_many(uint64_t const* keys, size_t count, bool compact, size_t* removed, size_t* pruned) {
    *removed = 0;
    if (pruned) *pruned = 0;
    if (!loaded || !size) return nullptr;
    if (char const* e = ensure_context()) return e;
    keys_generation += 1;
    build_key_map();
    std::vector<uint32_t> slots;
    for (size_t i = 0; i < count; ++i) {
        size_t const before = slots.size();
        key_map.for_each(keys[i], [&](uint32_t slot, size_t cell) { slots.push_back(slot); key_map.erase_cell(cell); return true; });
        std::sort(slots.begin() + (ptrdiff_t)before, slots.end()); /* the entries of one key of a multi index: insertion order */
    }
    if (char const* e = set_slot_keys(slots.data(), slots.size(), nullptr)) {
        key_map.clear(); /* rebuilt from host_keys, which still hold the keys */
        return e;
    }
    for (uint32_t slot : slots) {
        host_keys[slot] = free_key;
        free_slots.push_back(slot);
    }
    count_deleted += slots.size();
    *removed = slots.size();
    if (!compact) return nullptr;
    return isolate(pruned);
}

char const* frozen_index_t::isolate(size_t* pruned) {
    if (pruned) *pruned = 0;
    if (!d.deleted_bits || !d.n) return nullptr; /* nothing was ever removed */
    if (char const* e = pruned_counter.reserve(1)) return e;
    CU(cudaMemsetAsync(pruned_counter.ptr, 0, 8, stream));
    size_t const rows = (size_t)d.n + upper_rows;
    unsigned const blocks = (unsigned)std::min<size_t>((rows + 7) / 8, (size_t)stream.sm_count * 8);
    isolate_kernel<<<blocks, 256, 0, stream>>>(d, (uint32_t)upper_rows, pruned_counter.ptr);
    CU(cudaGetLastError());
    unsigned long long total = 0;
    CU(cudaMemcpyAsync(&total, pruned_counter.ptr, 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    if (pruned) *pruned = (size_t)total;
    return nullptr;
}

} // namespace usearch_b200
