/*
 *  search_kernel.cu — the batched HNSW search() hot path as ONE persistent, warp-per-query kernel.
 *
 *  What a warp does for one query reproduces, decision for decision, the reference's
 *    index_gt::search            index.hpp:3016-3075
 *    search_for_one_             index.hpp:3963-4003   (greedy descent, levels max..1)
 *    search_to_find_in_base_     index.hpp:4175-4246   (best-first expansion, layer 0)
 *    sorted_buffer_gt::insert    index.hpp:928-939     (`top`, ascending, lower_bound position)
 *    max_heap_gt insert / pop    index.hpp:753-834     (`next`, same sift rules => same tie order)
 *    growing_hash_set_gt::set    index.hpp:1163-1175   (`visits`, exact set semantics)
 *    search_result_t::dump_to    index.hpp:2707-2722   (padding with key 0 / signalling NaN)
 *  so the returned labels are bit-identical to the CPU search at the same ef, ties included.
 *
 *  How the work is laid out on the GPU is new:
 *    - a persistent grid (a multiple of the SM count, one warp per CTA) pulls query ids from one
 *      atomic counter;
 *    - the per-query state lives on chip: the query itself (read ~D times), the head of the `next`
 *      heap (its deep levels spill to a per-warp slab in HBM) and the hop's candidate list in shared
 *      memory, `top` in registers (8 entries per lane, sorted, maintained with ballots and shuffles;
 *      shared memory beyond ef = 256);
 *    - `visits` is a per-warp bitmap over all slots in HBM/L2 driven with atomicOr (an open-addressing
 *      table driven with atomicCAS where the bitmaps would not fit the scratch budget), so that the 32
 *      lanes test-and-set a whole neighbour list at once;
 *    - the neighbour vectors of a hop are fetched together. STAGED kernels (vectors >= 256 B) issue
 *      one TMA bulk copy (cp.async.bulk, UBLKCP) per candidate vector into a shared-memory slot and
 *      wait on its mbarrier: eight whole vectors are in flight per warp without holding a single
 *      register, and LPV lanes then reduce each slot in the reference's summation order. DIRECT
 *      kernels (short vectors: binary codes) stream 16-byte chunks through registers instead;
 *    - only the accept/insert replay that follows is sequential, as the reference's inner loop is,
 *      and it only visits the candidates that can still pass the radius test.
 *  The same kernel, instantiated with INSERT = true, is search_to_insert_ (index.hpp:4010-4079) for the
 *  batched builder (builder.cu): a work item per (new member, level), best-first on that level's lists.
 */
#include <cuda_runtime.h>

#include <cstdlib>

#include "device_index.h"
#include "metrics.cuh"
#include "warp_primitives.cuh"

namespace usearch_b200 {

constexpr int THREADS = 32; /* one warp per CTA: warps never synchronise with each other */
constexpr int LOADS_IN_FLIGHT = 8;
constexpr int BATCH_LOADS = 4; /* 16-byte loads a lane keeps in flight across passes in measure_direct_batched */

__device__ __forceinline__ uint32_t hash_slot(uint32_t s) { return s * 0x9E3779B1u; }

/* ---- `next`: binary max-heap on -distance, stored as +distance with reversed compares ------ */

/*
 *  Same tree, same sift rules as max_heap_gt (index.hpp:664-835), therefore the same pop order on
 *  ties. Storage is 1-based: logical element i lives at physical index i+1, so the two children of
 *  physical node p are the ADJACENT pair (2p, 2p+1) — one 16-byte load fetches both. Physical
 *  indices below `smem_cap` are in shared memory, deeper ones spill to the warp's slab in HBM.
 */
struct heap_t {
    uint32_t smem_addr; /* shared-window address of physical index 0 (explicit ld/st.shared: never generic) */
    cand_t* spill;
    uint32_t smem_cap; /* even */
    static __device__ __forceinline__ cand_t lds(uint32_t addr) {
        cand_t c;
        asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=f"(c.d), "=r"(c.s) : "r"(addr));
        return c;
    }
    static __device__ __forceinline__ void sts(uint32_t addr, cand_t c) {
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "f"(c.d), "r"(c.s) : "memory");
    }
    __device__ __forceinline__ cand_t get(uint32_t p) const {
        if (p < smem_cap) return lds(smem_addr + 8u * p);
        return spill[p - smem_cap];
    }
    __device__ __forceinline__ void put(uint32_t p, cand_t c) const {
        if (p < smem_cap) sts(smem_addr + 8u * p, c);
        else spill[p - smem_cap] = c;
    }
    __device__ __forceinline__ cand_t root() const { return lds(smem_addr + 8u); }
    __device__ __forceinline__ void set_root(cand_t c) const { sts(smem_addr + 8u, c); }

    /* max_heap_gt::insert_reserved + shift_up (index.hpp:764-770, :808-811), by the whole warp: the
     * ancestors of the new leaf are known up front (p>>1, p>>2, ...), lane l fetches the one at level l;
     * the first ancestor that is NOT `less` than the element (parent.d <= c.d) stops the climb — the
     * sequential loop stops at exactly that ancestor — and everything below it moves down one step.
     * `size` is the number of elements before the push. */
    __device__ __forceinline__ void push(uint32_t size, cand_t c, int lane) const {
        uint32_t const p = size + 1;
        uint32_t const depth = 31u - (uint32_t)__clz(p);
        cand_t e{0.f, 0u};
        if ((uint32_t)lane < depth) e = get(p >> (lane + 1));
        uint32_t const stops = __ballot_sync(0xffffffffu, (uint32_t)lane < depth && !(e.d > c.d));
        uint32_t const stop = stops ? (uint32_t)__ffs(stops) - 1u : depth;
        if ((uint32_t)lane < stop) put(p >> lane, e);
        if (lane == 0) put(p >> stop, c);
        __syncwarp();
    }

    /* max_heap_gt::pop + shift_down (index.hpp:786-794, :819-834), lane 0 only. `size` is the size
     * before the pop (> 0). The root has already been read by the caller. */
    __device__ __forceinline__ void pop(uint32_t size) const {
        uint32_t const n = size - 1; /* elements that remain: physical 1..n */
        if (n == 0) return;
        cand_t const last = get(size);
        uint32_t p = 1;
        for (;;) {
            uint32_t const l = 2 * p, r = l + 1;
            if (l > n) break;
            cand_t le, re;
            if (r < smem_cap) { /* both children in shared memory: one 16-byte load */
                asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                             : "=f"(le.d), "=r"(le.s), "=f"(re.d), "=r"(re.s)
                             : "r"(smem_addr + 8u * l));
            } else {
                le = get(l);
                re = r <= n ? get(r) : le;
            }
            uint32_t best_i = p;
            float best = last.d;
            if (best > le.d) { best_i = l; best = le.d; }
            if (r <= n && best > re.d) best_i = r;
            if (best_i == p) break;
            put(p, best_i == l ? le : re);
            p = best_i;
        }
        put(p, last);
    }

    /*
     *  The same pop by the whole warp, for heaps whose internal nodes all sit in shared memory
     *  (size <= 2*32*WORDS and size < smem_cap). shift_down (index.hpp:819-834) keeps `best` = last.d, moves
     *  it to le.d if last.d > le.d, then to re.d if best > re.d. With le.d a number that sends the element
     *  right iff re.d < min(last.d, le.d), i.e. iff re.d < le.d and last.d > re.d; with le.d NaN the first
     *  test fails, best stays last.d, and it goes right iff last.d > re.d. So the child it can take is fixed
     *  by the two children alone: right iff (right exists && (re.d < le.d || le.d is NaN)), else left
     *  (heap_goes_right, search_order.h), and the element moves there iff last.d > child.d. The walk follows
     *  those choices from the root and stops at the first level where last.d > child.d fails:
     *    1. every lane evaluates the choice bit of up to WORDS internal nodes, one per 32-node word the heap reaches:
     *       one 16-byte load and one ballot each;
     *    2. all lanes walk the <= 9 levels on those bits in registers (no memory on the critical path);
     *    3. lane k fetches the path node of level k, a ballot finds the stop level, the path shifts up.
     *  Returns false (nothing done) when the heap is too large: the caller falls back to `pop`.
     *  WORDS = 8 (heaps up to 512 entries) or 16 (up to 1024: one more level of choice words). The prefiltered cos / ip
     *  f32 search takes 16, because its plan gives the heap a head of at least 512 entries; every other kernel keeps 8,
     *  whose smaller walk measured faster where heaps stay small (C1, l2sq 100K x 128: 1.53 against 1.57 ms per launch).
     */
    template <int WORDS> __device__ __forceinline__ bool pop_warp(uint32_t size, int lane) const {
        static_assert(WORDS == 8 || WORDS == 16, "choice words: 8 or 16");
        uint32_t const n = size - 1;
        if (n == 0) return true;
        if (size > 64u * WORDS || size >= smem_cap) return false;
        cand_t const last = lds(smem_addr + 8u * size);
        uint32_t const internal = n >> 1; /* nodes 1..internal have at least a left child */
        uint32_t w[WORDS];
#pragma unroll
        for (int r = 0; r < WORDS; ++r) {
            w[r] = 0u;
            if ((uint32_t)(r * 32) <= internal) {
                uint32_t const p = (uint32_t)(r * 32 + lane);
                bool right = false;
                if (p >= 1u && 2u * p + 1u <= n) {
                    cand_t le, re;
                    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                                 : "=f"(le.d), "=r"(le.s), "=f"(re.d), "=r"(re.s)
                                 : "r"(smem_addr + 16u * p));
                    right = heap_goes_right(le.d, re.d);
                }
                w[r] = __ballot_sync(0xffffffffu, right);
            }
        }
        /* walk: level k node p -> 2p + choice(p); the word holding choice(p) is static per level */
        uint32_t p = 1, mine = 1, parent = 1, depth = 0;
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            if (2u * p <= n) {
                uint32_t word;
                if (k <= 4) word = w[0];
                else if (k == 5) word = w[1];
                else if (k == 6) word = (p & 32u) ? w[3] : w[2];
                else if (k == 7) word = (p & 64u) ? ((p & 32u) ? w[7] : w[6]) : ((p & 32u) ? w[5] : w[4]);
                else if constexpr (WORDS == 8) word = 0u; /* level-8 nodes (256..511) have no children when size <= 512 */
                else /* level 8 (level-9 nodes, 512..1023, have no children when size <= 1024) */
                    word = (p & 128u) ? ((p & 64u) ? ((p & 32u) ? w[15] : w[14]) : ((p & 32u) ? w[13] : w[12]))
                                      : ((p & 64u) ? ((p & 32u) ? w[11] : w[10]) : ((p & 32u) ? w[9] : w[8]));
                uint32_t const child = 2u * p + ((word >> (p & 31u)) & 1u);
                if (lane == k + 1) { mine = child; parent = p; }
                p = child;
                depth = (uint32_t)k + 1u;
            }
        }
        /* lane k (1..depth) owns path node p_k and its parent p_{k-1} */
        cand_t e{0.f, 0u};
        bool const on_path = lane >= 1 && (uint32_t)lane <= depth;
        if (on_path) e = lds(smem_addr + 8u * mine);
        uint32_t const stays = __ballot_sync(0xffffffffu, on_path && !(last.d > e.d));
        uint32_t const moves = stays ? (uint32_t)__ffs(stays) - 2u : depth; /* levels 1..moves shift up */
        if (on_path && (uint32_t)lane <= moves) sts(smem_addr + 8u * parent, e);
        /* `last` lands on path node p_moves (the root when nothing moved) */
        uint32_t const landing = __shfl_sync(0xffffffffu, mine, (int)moves);
        if (lane == 0) sts(smem_addr + 8u * (moves ? landing : 1u), last);
        return true;
    }
};

/* ---- `top`: ascending sorted array, maintained by the whole warp ---------------------------- */

/* sorted_buffer_gt::insert(element, limit) (index.hpp:928-939). Uniform across the warp.
 * Lane l owns elements l, l+32, ...: every element is loaded once (the same loads feed the
 * lower_bound ballots), one barrier, then every element at or after the insertion point is
 * stored one place to the right. `has_nan` (uniform) says `top` may hold a NaN: the count of
 * smaller elements is lower_bound only while it does not, so then the position is probed as
 * libstdc++ probes it (search_order.h). */
__device__ __forceinline__ void top_insert(float* td, uint32_t* ts, uint32_t& size, uint32_t limit, float d, uint32_t s,
                                           bool& has_nan, int lane) {
    uint32_t pos = 0;
    if (!has_nan) {
        for (uint32_t b = 0; b < size; b += 32) {
            uint32_t i = b + lane;
            bool lt = i < size && td[i] < d;
            pos += __popc(__ballot_sync(0xffffffffu, lt));
        }
    } else
        pos = probe_lower_bound([td](uint32_t i) { return td[i]; }, size, d);
    if (pos == limit) return;
    has_nan = top_may_hold_nan(has_nan, d);
    bool full = size == limit;
    uint32_t hi = size - (full ? 1u : 0u);
    if (hi > pos) {
        for (int b = (int)((hi - 1) & ~31u); b >= (int)(pos & ~31u); b -= 32) {
            uint32_t i = (uint32_t)b + lane;
            bool mv = i >= pos && i < hi;
            float x = 0.f;
            uint32_t y = 0;
            if (mv) { x = td[i]; y = ts[i]; }
            __syncwarp();
            if (mv) { td[i + 1] = x; ts[i + 1] = y; }
            __syncwarp();
        }
    }
    if (lane == 0) { td[pos] = d; ts[pos] = s; }
    size += full ? 0u : 1u;
    __syncwarp();
}

/* ---- per-warp view of shared memory and scratch ---------------------------------------------- */

struct warp_ctx_t {
    uint4* q4;
    float* top_d;
    uint32_t* top_s;
    uint32_t* cand_s;
    float* cand_d;
    uint8_t* stage;      /* STAGED: VPP slots of stage_stride bytes */
    uint32_t stage_addr; /* shared-window address of `stage` */
    uint32_t bars_addr;  /* shared-window address of the VPP mbarriers */
    uint32_t phase;      /* one parity bit per slot, uniform across the warp */
    uint32_t t_wait;     /* introspection: cycles spent waiting for staged vectors */
    uint32_t t_code;     /* introspection: cycles spent waiting for the prefilter's int8 codes */
    uint32_t t_dot;      /* introspection: the prefilter's IMMA dot products and their conversion to `dot` */
    uint32_t t_bound;    /* introspection: the prefilter's bound, ballots and compaction */
    uint32_t t_conv;     /* introspection: the part of t_dot after the IMMAs: conversion to `dot` and its stores */
    uint32_t n_code_pass; /* introspection: the prefilter's code passes */
};

/* ---- distances of a whole candidate list ---------------------------------------------------- */

/*
 *  DIRECT, short vectors: a lane's share of a vector is CPL <= 2 chunks, so the loads of BATCH_LOADS / CPL PASSES (each pass = 32 / LPV
 *  candidates) are issued together before any of them is consumed: a whole list of 128 binary codes of 256 bits
 *  (BASELINE config C5: LPV 2, CPL 1) costs two memory round trips instead of eight (more loads in flight would spill: the caller keeps ~110 registers live).
 */
template <class M, int CPL>
__device__ __noinline__ void measure_direct_batched(device_index_t const& ix, warp_ctx_t& w, typename M::qconst_t qc,
                                                       uint32_t ncand, int lane) {
    constexpr int LPV = M::LPV, VPP = 32 / LPV, PB = BATCH_LOADS / CPL;
    int const g = lane / LPV, sub = lane % LPV;
    uint32_t const chunks = ix.chunks16;
    for (uint32_t base = 0; base < ncand; base += VPP * PB) {
        uint4 r[PB][CPL];
#pragma unroll
        for (int p = 0; p < PB; ++p) {
            uint32_t const c = base + (uint32_t)(p * VPP + g);
            uint32_t const slot = c < ncand ? w.cand_s[c] : 0u;
            uint4 const* v = reinterpret_cast<uint4 const*>(ix.vectors + (size_t)slot * ix.vec_stride);
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
                uint32_t const j = (uint32_t)(sub + i * LPV);
                if (c < ncand && j < chunks) r[p][i] = ldg_stream(v + j);
            }
        }
#pragma unroll
        for (int p = 0; p < PB; ++p) {
            uint32_t const c = base + (uint32_t)(p * VPP + g);
            if (base + (uint32_t)(p * VPP) >= ncand) break; /* uniform: no candidate in this pass */
            typename M::acc_t acc;
            M::init(acc);
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
                uint32_t const j = (uint32_t)(sub + i * LPV);
                if (c < ncand && j < chunks) M::step(acc, r[p][i], w.q4[j]);
            }
            float const d = M::finish(acc, qc); /* shuffles inside the lane group: executed by every lane */
            if (c < ncand && sub == 0) w.cand_d[c] = d;
        }
    }
    __syncwarp();
}

/* DIRECT: 16-byte chunks straight from HBM into registers, LOADS_IN_FLIGHT per lane. */
template <class M>
__device__ __noinline__ void measure_direct(device_index_t const& ix, warp_ctx_t& w, typename M::qconst_t qc,
                                               uint32_t ncand, int lane) {
    constexpr int LPV = M::LPV, VPP = 32 / LPV;
    int const g = lane / LPV, sub = lane % LPV;
    uint32_t const chunks = ix.chunks16;
    uint32_t const cpl = (chunks + LPV - 1) / LPV; /* chunks per lane */
    if (cpl == 1) return measure_direct_batched<M, 1>(ix, w, qc, ncand, lane);
    if (cpl == 2) return measure_direct_batched<M, 2>(ix, w, qc, ncand, lane);
    for (uint32_t base = 0; base < ncand; base += VPP) {
        uint32_t c = base + g;
        bool act = c < ncand;
        uint32_t slot = act ? w.cand_s[c] : 0u;
        uint4 const* v = reinterpret_cast<uint4 const*>(ix.vectors + (size_t)slot * ix.vec_stride);
        typename M::acc_t acc;
        M::init(acc);
        for (uint32_t j0 = sub; j0 < chunks; j0 += LPV * LOADS_IN_FLIGHT) {
            uint4 r[LOADS_IN_FLIGHT];
#pragma unroll
            for (int u = 0; u < LOADS_IN_FLIGHT; ++u) {
                uint32_t j = j0 + u * LPV;
                if (act && j < chunks) r[u] = ldg_stream(v + j);
            }
#pragma unroll
            for (int u = 0; u < LOADS_IN_FLIGHT; ++u) {
                uint32_t j = j0 + u * LPV;
                if (act && j < chunks) M::step(acc, r[u], w.q4[j]);
            }
        }
        float d = M::finish(acc, qc); /* warp-wide shuffles inside: executed by every lane */
        if (act && sub == 0) w.cand_d[c] = d;
    }
    __syncwarp();
}

/*
 *  STAGED: TMA bulk copies (cp.async.bulk, UBLKCP) land candidate vectors in shared-memory slots, LPV lanes
 *  then reduce each slot in the reference's summation order. A PASS = the next 32 / LPV candidates; pass p goes to slot set
 *  p mod nsets (nsets = 1: fetch-then-reduce; 2: the next pass lands during the math), one mbarrier per set.
 *  (Round 1 could also fetch a vector as two half-size segments for more resident warps; measured a wash, and the index
 *  arithmetic it needed — divisions by run-time constants in this loop — showed up as 5 % of the kernel's issue slots in
 *  ncu. Removed in round 2.)
 */
template <class M>
__device__ __forceinline__ void measure_staged(device_index_t const& ix, search_args_t const& a, warp_ctx_t& w,
                                               typename M::qconst_t qc, uint32_t ncand, int lane, uint32_t const* slots,
                                               float* out) {
    constexpr int LPV = M::LPV, VPP = 32 / LPV;
    int const g = lane / LPV, sub = lane % LPV;
    bool const two_sets = a.stage_sets > 1;
    uint32_t const npass = (ncand + VPP - 1) / VPP;
    uint32_t const bytes = ix.chunks16 * 16u;
    /* `cp.async.bulk` takes uniform-register operands, so the per-lane issue is serialised by the compiler with an ELECT
     * loop; lane 0 issuing all copies back to back measured 7 % slower end to end (round 1). */
    auto issue = [&](uint32_t pass) {
        uint32_t const base = pass * VPP, cnt = min((uint32_t)VPP, ncand - base), set = two_sets ? (pass & 1u) : 0u;
        uint32_t const my_slot = (uint32_t)lane < cnt ? slots[base + lane] : 0u;
        uint32_t const bar = w.bars_addr + 8u * set;
        if (lane == 0) mbar_expect_tx(bar, cnt * bytes);
        __syncwarp();
        if ((uint32_t)lane < cnt)
            bulk_copy_g2s(w.stage_addr + (set * VPP + lane) * a.stage_stride, ix.vectors + (size_t)my_slot * ix.vec_stride, bytes, bar);
    };
    issue(0);
    if (two_sets && npass > 1) issue(1);
    /* unit j of the vector: a 16-byte chunk, or a 32-bit word for the WORD metrics */
    using U = typename unit_of<M>::type;
    constexpr uint32_t UPC = unit_of<M>::UPC;
    uint32_t const u1 = ix.chunks16 * UPC;
    U const* const qu = reinterpret_cast<U const*>(w.q4);
    for (uint32_t pass = 0; pass < npass; ++pass) {
        uint32_t const base = pass * VPP, cnt = min((uint32_t)VPP, ncand - base), set = two_sets ? (pass & 1u) : 0u;
        U const* const buf = reinterpret_cast<U const*>(w.stage + (size_t)(set * VPP + g) * a.stage_stride);
        bool const act = (uint32_t)g < cnt;
        typename M::acc_t acc;
        M::init(acc);
        if (a.phase_cycles) { /* introspection only: attribute the wait for the slowest slot to `vector_wait` */
            long long t = clock64();
            if (act) mbar_wait(w.bars_addr + 8u * set, (w.phase >> set) & 1u);
            __syncwarp();
            w.t_wait += (uint32_t)(clock64() - t);
        }
        if (act) {
            if (!a.phase_cycles) mbar_wait(w.bars_addr + 8u * set, (w.phase >> set) & 1u);
            /* 4 steps per iteration, the next iteration's 8 shared-memory loads issued before this one's math */
            uint32_t j = (uint32_t)sub;
            if (j + 3 * LPV < u1) {
                U b0 = buf[j], b1 = buf[j + LPV], b2 = buf[j + 2 * LPV], b3 = buf[j + 3 * LPV];
                U q0 = qu[j], q1 = qu[j + LPV], q2 = qu[j + 2 * LPV], q3 = qu[j + 3 * LPV];
                j += 4 * LPV;
                for (; j + 3 * LPV < u1; j += 4 * LPV) {
                    U nb0 = buf[j], nb1 = buf[j + LPV], nb2 = buf[j + 2 * LPV], nb3 = buf[j + 3 * LPV];
                    U nq0 = qu[j], nq1 = qu[j + LPV], nq2 = qu[j + 2 * LPV], nq3 = qu[j + 3 * LPV];
                    M::step(acc, b0, q0);
                    M::step(acc, b1, q1);
                    M::step(acc, b2, q2);
                    M::step(acc, b3, q3);
                    b0 = nb0; b1 = nb1; b2 = nb2; b3 = nb3;
                    q0 = nq0; q1 = nq1; q2 = nq2; q3 = nq3;
                }
                M::step(acc, b0, q0);
                M::step(acc, b1, q1);
                M::step(acc, b2, q2);
                M::step(acc, b3, q3);
            }
            for (; j < u1; j += LPV) M::step(acc, buf[j], qu[j]);
        }
        float const d = M::finish(acc, qc); /* horizontal reduce (warp-wide shuffles: every lane) */
        if (act && sub == 0) out[base + g] = d;
        w.phase ^= 1u << set; /* one parity bit per set */
        __syncwarp();         /* every lane is done with this set before it is refilled */
        uint32_t const next = pass + (two_sets ? 2u : 1u);
        if (next < npass) issue(next);
    }
}

template <class M, bool STAGED>
__device__ __forceinline__ void measure_list(device_index_t const& ix, search_args_t const& a, warp_ctx_t& w,
                                             typename M::qconst_t qc, uint32_t ncand, int lane) {
    /* An empty list (the only member of the top level has one) must not touch the mbarriers: an `expect_tx` of zero bytes
     * completes a phase that no wait consumes, and every later wait of this warp is then one phase behind — it returns
     * before its copy has landed, or deadlocks (the round-1 golden-test hang: cluster(level = top) on a one-member top). */
    if (ncand == 0) return;
    float n0 = 0.f, n1 = 0.f;
    if constexpr (M::NORMS) { /* requested now, consumed after the last pass */
        if ((uint32_t)lane < ncand) n0 = __ldg(ix.norms + w.cand_s[lane]);
        if ((uint32_t)lane + 32 < ncand) n1 = __ldg(ix.norms + w.cand_s[lane + 32]);
    }
    if constexpr (STAGED) measure_staged<M>(ix, a, w, qc, ncand, lane, w.cand_s, w.cand_d);
    else measure_direct<M>(ix, w, qc, ncand, lane);
    if constexpr (M::NORMS) { /* one candidate per lane: a single f64 normalisation sequence per hop */
        if ((uint32_t)lane < ncand) w.cand_d[lane] = M::finalize(w.cand_d[lane], qc, n0);
        if ((uint32_t)lane + 32 < ncand) w.cand_d[lane + 32] = M::finalize(w.cand_d[lane + 32], qc, n1);
        for (uint32_t c = 64 + lane; c < ncand; c += 32) w.cand_d[c] = M::finalize(w.cand_d[c], qc, __ldg(ix.norms + w.cand_s[c]));
        __syncwarp();
    }
}

/*
 *  The layer-0 list of a hop that starts with `top` full (cos / ip f32 with a shadow). The reference drops a candidate
 *  with d >= radius without a trace: it is neither pushed nor inserted, and only `computed_distances` counts it. The
 *  radius only shrinks inside a hop, so a candidate whose lower bound (prefilter_bound.h) reaches the radius at the start
 *  of the hop is rejected at its turn too, and the accept replay never looks at it. So the survivors are compacted to
 *  the front of the list in stored order, measured exactly, and the replay that follows visits only them. Rejected
 *  candidates never touch their f32 row. Returns the number of survivors.
 *
 *    1. TMA bulk copies put the int8 codes of up to `code_pass` candidates into the stage area, records load meanwhile;
 *    2. the tensor cores form the exact integers D1 = q1.c and D2 = q2.c against the query's int8 split (split_query):
 *       mma.sync m16n8k32 s8, the codes of 16 candidates as A (one ldmatrix.x4 per 32-byte k-step), q1 and q2 as
 *       columns 0 and 1 of B (the other 6 are zero), s32 accumulators; `dot` = fl32(sa1 D1 + sa2 D2);
 *    3. one lane per candidate evaluates the bound; a ballot lists the survivors in stored order;
 *    4. the survivors' rows go through the STAGED pipeline, their distances land in `cand_d[0, ns)`.
 */
__device__ __forceinline__ pf_record_t ldg_record(pf_record_t const* p) {
    float4 const v = __ldg(reinterpret_cast<float4 const*>(p));
    return pf_record_t{v.x, v.y, v.z, v.w};
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double warp_max_f64(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

/* The B fragment of m16n8k32 s8 gives lane `sub` of column g the k-bytes 4 sub .. 4 sub + 3 and 16 + 4 sub .. 16 + 4 sub
 * + 3 of each 32-byte k-step. The split is stored with the words of a step in the order 0 4 1 5 2 6 3 7, so that one
 * 8-byte load fetches both. */
__device__ __forceinline__ uint32_t qsplit_word_place(uint32_t word) { return (word & ~7u) + (word & 3u) * 2u + ((word >> 2) & 1u); }

/* pf_split_query (prefilter_bound.h) by one warp: the same element steps, the maxima and the sum of squares across lanes.
 * `q1` and `q2` get `len` bytes each (zero beyond `n`) in the B-fragment order above. Uniform across the warp. */
__device__ __forceinline__ pf_query_split_t split_query(float const* qa, uint32_t n, uint8_t* q1, uint8_t* q2, uint32_t len,
                                                        int lane) {
    double mx1 = 0.0;
    bool finite = true;
    for (uint32_t i = (uint32_t)lane; i < n; i += 32) {
        double const x = fabs((double)qa[i]);
        finite = finite && x < INFINITY;
        mx1 = fmax(mx1, x);
    }
    mx1 = warp_max_f64(mx1);
    finite = __all_sync(0xffffffffu, finite);
    float const sa1 = pf_scale(mx1);
    bool const usable = finite && sa1 > 0.0f;
    double mx2 = 0.0;
    int8_t c1, c2;
    if (usable)
        for (uint32_t i = (uint32_t)lane; i < n; i += 32) mx2 = fmax(mx2, fabs(pf_split_step((double)qa[i], sa1, c1)));
    mx2 = warp_max_f64(mx2);
    float const sa2 = usable ? pf_scale(mx2) : 0.0f;
    double e2 = 0.0;
    for (uint32_t wd = (uint32_t)lane; wd < len / 4; wd += 32) {
        uint32_t p1 = 0, p2 = 0;
#pragma unroll
        for (uint32_t b = 0; b < 4; ++b) {
            uint32_t const i = 4 * wd + b;
            c1 = c2 = 0;
            if (usable && i < n) {
                double const r2 = pf_split_step(pf_split_step((double)qa[i], sa1, c1), sa2, c2);
                e2 += r2 * r2;
            }
            p1 |= (uint32_t)(uint8_t)c1 << (8 * b);
            p2 |= (uint32_t)(uint8_t)c2 << (8 * b);
        }
        reinterpret_cast<uint32_t*>(q1)[qsplit_word_place(wd)] = p1;
        reinterpret_cast<uint32_t*>(q2)[qsplit_word_place(wd)] = p2;
    }
    e2 = warp_sum_f64(e2);
    __syncwarp();
    return usable ? pf_query_split_t{sa1, sa2, pf_round_up_norm(e2)} : pf_query_split_t{0.0f, 0.0f, INFINITY};
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}

__device__ __forceinline__ void imma_16832(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

/*
 *  The prefilter's dot products for NT (1 or 2) tiles of 16 rows: D1 = q1.c and D2 = q2.c, exact in s32, and
 *  `dot` = fl32(sa1 D1 + sa2 D2) into out[i] for i < cnt. NT is a template parameter so that no IMMA or ldmatrix is
 *  predicated and no branch splits the k-loop. k outer, tiles inner: one B load per k-step serves every tile. Rows of the
 *  last tile beyond `cnt` hold stale bytes, and the k-bytes beyond `code_stride` of a row were never copied: the split is
 *  zero there, so they add 0 to D1 and D2, and the rows' results are dropped.
 *  Even k-steps accumulate into acc[0], odd ones into acc[1], so that every tile has two independent chains of IMMAs; the
 *  s32 sums are exact, so D1 and D2 do not depend on the split. Four fragment sets rotate so that the fragments of step
 *  k + 2 are requested before the IMMAs of step k issue: no ldmatrix is consumed within two k-steps of its issue.
 */
template <uint32_t NT>
__device__ __forceinline__ void prefilter_dots(uint32_t a_addr, uint32_t b_addr, uint32_t scs, uint32_t ksteps, double sa1,
                                               double sa2, float* out, uint32_t cnt, int lane, warp_ctx_t& w, bool prof) {
    int acc[2][NT][4] = {};
    uint32_t f0[NT][4], f1[NT][4], f2[NT][4], f3[NT][4], b0[2], b1[2], b2[2], b3[2];
    auto load = [&](uint32_t k, uint32_t(&A)[NT][4], uint32_t(&B)[2]) {
        B[0] = B[1] = 0u;
        if (lane < 8) asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(B[0]), "=r"(B[1]) : "r"(b_addr + 32u * k));
#pragma unroll
        for (uint32_t t = 0; t < NT; ++t) ldmatrix_x4(a_addr + t * 16u * scs + 32u * k, A[t][0], A[t][1], A[t][2], A[t][3]);
    };
    auto mma = [&](int (&C)[NT][4], uint32_t const(&A)[NT][4], uint32_t const(&B)[2]) {
#pragma unroll
        for (uint32_t t = 0; t < NT; ++t) imma_16832(C[t], A[t][0], A[t][1], A[t][2], A[t][3], B[0], B[1]);
    };
    static_assert(NT == 1 || NT == 2, "tiles per k-loop: 1 or 2");
    uint32_t k = 0;
    load(0, f0, b0);
    if (ksteps > 1) load(1, f1, b1);
    for (; k + 6 <= ksteps; k += 4) { /* f0, f1 hold steps k, k + 1 */
        load(k + 2, f2, b2);
        mma(acc[0], f0, b0);
        load(k + 3, f3, b3);
        mma(acc[1], f1, b1);
        load(k + 4, f0, b0);
        mma(acc[0], f2, b2);
        load(k + 5, f1, b1);
        mma(acc[1], f3, b3);
    }
    /* 1 to 5 steps remain, the first two of them loaded (uniform branches, once per pass) */
    if (k + 2 < ksteps) load(k + 2, f2, b2);
    if (k + 3 < ksteps) load(k + 3, f3, b3);
    mma(acc[0], f0, b0);
    if (k + 1 < ksteps) mma(acc[1], f1, b1);
    if (k + 4 < ksteps) load(k + 4, f0, b0);
    if (k + 2 < ksteps) mma(acc[0], f2, b2);
    if (k + 3 < ksteps) mma(acc[1], f3, b3);
    if (k + 4 < ksteps) mma(acc[0], f0, b0);
    /* C: lane 4 g holds columns 0 and 1 (D1, D2) of rows g and g + 8 */
    int d[NT][4];
#pragma unroll
    for (uint32_t t = 0; t < NT; ++t)
#pragma unroll
        for (int j = 0; j < 4; ++j) d[t][j] = acc[0][t][j] + acc[1][t][j];
    long long const t_conv = prof ? clock64() : 0; /* the IMMAs have retired: their sums are in registers */
    uint32_t const g = (uint32_t)lane >> 2, sub = (uint32_t)lane & 3;
#pragma unroll
    for (uint32_t t = 0; t < NT; ++t) {
        uint32_t const i = 16u * t + g;
        if (sub == 0 && i < cnt) out[i] = __double2float_rn(sa1 * (double)d[t][0] + sa2 * (double)d[t][1]);
        if (sub == 0 && i + 8 < cnt) out[i + 8] = __double2float_rn(sa1 * (double)d[t][2] + sa2 * (double)d[t][3]);
    }
    __syncwarp(); /* dots visible, and every lane is done with the stage area before it is refilled */
    if (prof) w.t_conv += (uint32_t)(clock64() - t_conv);
}

template <class M>
__device__ __forceinline__ uint32_t measure_prefiltered(device_index_t const& ix, search_args_t const& a, warp_ctx_t& w,
                                                     typename M::qconst_t qc, pf_query_bound_t const& qb,
                                                     pf_query_split_t const& sp, float radius, uint32_t ncand, int lane) {
    uint8_t* const smem = reinterpret_cast<uint8_t*>(w.q4); /* the query opens the warp's shared memory */
    float* const surv_b2 = reinterpret_cast<float*>(smem + a.off_surv_b2); /* cos: the survivors' stored squared norms */
    uint32_t const cs = ix.code_stride, scs = a.code_smem_stride, ksteps = a.qsplit_len / 32;
    uint32_t const bar = w.bars_addr; /* set 0's barrier */
    uint32_t const g = (uint32_t)lane >> 2, sub = (uint32_t)lane & 3;
    /* B: lanes 0-3 hold column 0 (q1), lanes 4-7 column 1 (q2); the other lanes' columns are zero */
    uint32_t const b_addr = smem_u32(smem + a.off_qsplit) + g * a.qsplit_len + 8u * sub;
    /* A: lane l gives the address of row l & 7 of matrix l >> 3: rows 0-7 / 8-15 of the tile, k-bytes 0-15 / 16-31 */
    uint32_t const a_addr = w.stage_addr + ((uint32_t)lane & 7u) * scs + (((uint32_t)lane >> 3) & 1u) * 8u * scs + ((uint32_t)lane >> 4) * 16u;
    double const sa1 = (double)sp.sa1, sa2 = (double)sp.sa2;
    uint32_t ns = 0;
    for (uint32_t base = 0; base < ncand; base += a.code_pass) {
        uint32_t const cnt = min(a.code_pass, ncand - base); /* code_pass <= 64 */
        if (lane == 0) mbar_expect_tx(bar, cnt * cs);
        __syncwarp();
        pf_record_t r0{}, r1{};
        uint32_t s0 = 0, s1 = 0; /* slots of candidates base + lane and base + lane + 32 */
        if ((uint32_t)lane < cnt) {
            s0 = w.cand_s[base + lane];
            bulk_copy_g2s(w.stage_addr + lane * scs, ix.codes + (size_t)s0 * cs, cs, bar);
            r0 = ldg_record(ix.shadow + s0);
        }
        if ((uint32_t)lane + 32 < cnt) {
            s1 = w.cand_s[base + lane + 32];
            bulk_copy_g2s(w.stage_addr + (lane + 32) * scs, ix.codes + (size_t)s1 * cs, cs, bar);
            r1 = ldg_record(ix.shadow + s1);
        }
        if (a.phase_cycles) { /* introspection only: the wait for the codes goes to `code_wait` */
            long long const t = clock64();
            mbar_wait(bar, w.phase & 1u);
            w.t_code += (uint32_t)(clock64() - t);
        } else
            mbar_wait(bar, w.phase & 1u);
        w.phase ^= 1u;
        long long const t_dot = a.phase_cycles ? clock64() : 0;
        bool const prof = a.phase_cycles != nullptr;
        /* tiles of this pass (code_pass <= 64): 3 or 4 tiles (64-candidate passes, never at 768-d) go as two passes over
         * the k-steps, of 2 tiles and of the rest, since the fragments of 3 or 4 tiles would push the kernel past 255
         * registers */
        uint32_t const ntiles = (cnt + 15) / 16;
        if (ntiles == 1) prefilter_dots<1>(a_addr, b_addr, scs, ksteps, sa1, sa2, w.cand_d + base, cnt, lane, w, prof);
        else prefilter_dots<2>(a_addr, b_addr, scs, ksteps, sa1, sa2, w.cand_d + base, min(cnt, 32u), lane, w, prof);
        if (ntiles == 3)
            prefilter_dots<1>(a_addr + 32u * scs, b_addr, scs, ksteps, sa1, sa2, w.cand_d + base + 32, cnt - 32, lane, w, prof);
        else if (ntiles == 4)
            prefilter_dots<2>(a_addr + 32u * scs, b_addr, scs, ksteps, sa1, sa2, w.cand_d + base + 32, cnt - 32, lane, w, prof);
        if (prof) w.n_code_pass += 1;
        long long const t_bound = a.phase_cycles ? clock64() : 0;
        if (a.phase_cycles) w.t_dot += (uint32_t)(t_bound - t_dot);
        uint32_t const lt = (1u << lane) - 1u;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            uint32_t const i = (uint32_t)lane + 32u * (uint32_t)h, c = base + i;
            if (32u * (uint32_t)h >= cnt) break; /* uniform */
            pf_record_t const r = h ? r1 : r0;
            bool keep = false;
            if (i < cnt) keep = !(M::pf_lower(w.cand_d[c], r, qb) >= (double)radius);
            uint32_t const bal = __ballot_sync(0xffffffffu, keep);
            if (keep) { /* in place: ns + rank <= c, and the slots of this pass are in registers */
                w.cand_s[ns + __popc(bal & lt)] = h ? s1 : s0;
                surv_b2[ns + __popc(bal & lt)] = r.b2;
            }
            ns += __popc(bal);
        }
        __syncwarp();
        if (a.phase_cycles) w.t_bound += (uint32_t)(clock64() - t_bound);
    }
    if (ns) {
        measure_staged<M>(ix, a, w, qc, ns, lane, w.cand_s, w.cand_d);
        __syncwarp();
        if constexpr (M::NORMS) {
            for (uint32_t j = lane; j < ns; j += 32) w.cand_d[j] = M::finalize(w.cand_d[j], qc, surv_b2[j]);
            __syncwarp();
        }
    }
    return ns;
}

/* The predicate of index_dense_gt::search_ (index_dense.hpp:2071-2083): not the free key, and — for a
 * filtered search — accepted by the caller's predicate, here a bitmap over slots. */
__device__ __forceinline__ bool slot_allowed(device_index_t const& ix, search_args_t const& a, uint32_t s) {
    if (ix.deleted_bits && ((ix.deleted_bits[s >> 5] >> (s & 31)) & 1u)) return false;
    if (a.allow_bits && !((a.allow_bits[s >> 5] >> (s & 31)) & 1u)) return false;
    return true;
}

/* the same predicate with the query's own bitmap row (grouped filtered search) */
__device__ __forceinline__ bool slot_allowed_row(device_index_t const& ix, uint32_t const* row, uint32_t s) {
    if (ix.deleted_bits && ((ix.deleted_bits[s >> 5] >> (s & 31)) & 1u)) return false;
    return (row[s >> 5] >> (s & 31)) & 1u;
}

/* ---- one query ------------------------------------------------------------------------------ */

template <class M, bool STAGED, bool INSERT, bool GROUPED>
__device__ __forceinline__ void search_one(device_index_t const& ix, search_args_t const& a, uint32_t qi, uint32_t out_row,
                                           int const bl_arg, warp_ctx_t& w, heap_t const& heap, uint32_t* visited, int lane) {
    uint32_t const k = a.k, ef = a.ef;
    /* INSERT mode: search_to_insert_ (index.hpp:4010-4079) on level `bl` — no predicate, slots out. A template
     * parameter, so that the plain search kernels compile to the code they had before the builder existed. */
    constexpr bool insert = INSERT;
    /* GROUPED: query qi's predicate is the bitmap row of its own group, resolved once here (by query id, never by work
     * item, so retries and rounds launched through `query_list` find the same row). A template parameter for the same
     * reason as INSERT. */
    uint32_t const* const group_row =
        GROUPED ? a.allow_bits + (size_t)(a.allow_groups[qi] - a.allow_group_base) * a.allow_words : nullptr;
    int const bl = INSERT ? bl_arg : 0;
    uint32_t const width = bl == 0 ? ix.m0 : ix.m; /* list capacity on the searched level */
    auto row_of = [&](uint32_t slot) -> uint32_t const* {
        if (bl == 0) return ix.nbr0 + (size_t)slot * ix.m0_stride;
        uint32_t const ub = __ldg(ix.upper_base + slot); /* a member reached on level bl has rows 1..level >= bl */
        return ix.upper + ((size_t)ub + (uint32_t)(bl - 1)) * ix.m_stride;
    };
    uint32_t top_size = 0, heap_size = 0, computed = 0, cycles = 0, status = STATUS_OK;
    bool top_nan = false; /* `top` may hold a NaN: its inserts probe as lower_bound does */
    uint32_t visited_total = 0;
    bool log_overflow_out = false;
    bool const prof = a.phase_cycles != nullptr;
    uint32_t pc0 = 0, pc1 = 0, pc2 = 0, pc4 = 0, pc5 = 0, n_push = 0, max_heap = 0, n_pref = 0, n_surv = 0;
    uint32_t pc4_full = 0, n_pf_hops = 0; /* distance math of the hops that start with `top` full; prefiltered hops */
    /* the layer-0 prefilter: plain searches of the f32 metrics that declare it, on an index that has the shadow */
    constexpr bool PF = prefilter_of<M>::value && STAGED && !INSERT;
    long long tp = prof ? clock64() : 0;
    w.t_wait = 0;
    w.t_code = 0;
    w.t_dot = 0;
    w.t_bound = 0;
    w.t_conv = 0;
    w.n_code_pass = 0;
#define PHASE(acc)                                  \
    if (prof) {                                     \
        long long now_ = clock64();                 \
        acc += (uint32_t)(now_ - tp);               \
        tp = now_;                                  \
    }
    float* const top_d = w.top_d; /* shared-memory `top`: only for ef > 32*TOP_E */
    uint32_t* const top_s = w.top_s;
    bool const topreg = ef <= 32u * TOP_E;
    float rtd[TOP_E];
    uint32_t rts[TOP_E];
#pragma unroll
    for (int c = 0; c < TOP_E; ++c) { rtd[c] = 0.f; rts[c] = 0u; }
    uint32_t* const cand_s = w.cand_s;
    float* const cand_d = w.cand_d;

    if (ix.n != 0 && k != 0) {
        /* stage the query, zero-padded to whole 16-byte chunks */
        {
            uint8_t const* src = a.queries + (size_t)qi * a.query_stride;
            uint32_t const bpv = ix.bytes_per_vector;
            bool wide = ((reinterpret_cast<size_t>(src) | a.query_stride) & 15) == 0 && a.query_stride >= (uint64_t)ix.chunks16 * 16;
            if (wide) {
                for (uint32_t j = lane; j < ix.chunks16; j += 32) w.q4[j] = reinterpret_cast<uint4 const*>(src)[j];
            } else {
                uint8_t* dst = reinterpret_cast<uint8_t*>(w.q4);
                for (uint32_t b = lane; b < ix.chunks16 * 16; b += 32) dst[b] = b < bpv ? src[b] : (uint8_t)0;
            }
        }
        /* visits.clear() */
        bool const bitmap = a.visited_bitmap_words != 0;
        bool const logged = bitmap && a.visit_log != nullptr; /* the bitmap is already all-zero */
        uint32_t* const vlog = logged ? a.visit_log + (size_t)blockIdx.x * a.visit_log_cap : nullptr;
        bool log_overflow = false;
        if (!logged) {
            uint32_t const fill = bitmap ? 0u : EMPTY_SLOT;
            uint4 const word = make_uint4(fill, fill, fill, fill);
            uint4* v4 = reinterpret_cast<uint4*>(visited);
            uint32_t const n4 = (bitmap ? a.visited_bitmap_words : a.visited_cap) / 4;
            for (uint32_t j = lane; j < n4; j += 32) v4[j] = word;
        }
        __threadfence_block();
        __syncwarp();
        typename M::qconst_t qc = M::prepare(w.q4, ix.chunks16, lane);
        pf_query_split_t pf_sp{0.f, 0.f, INFINITY}; /* the query's int8 split, the B operand of the prefilter */
        pf_query_bound_t pf_qb{};                   /* what the bound needs of the query alone */
        if constexpr (PF) {
            if (a.prefilter) {
                float const a2 = cos_f32_t::self_dot(w.q4, ix.chunks16, lane); /* as the reference accumulates it */
                uint8_t* const q1 = reinterpret_cast<uint8_t*>(w.q4) + a.off_qsplit;
                pf_sp = split_query(reinterpret_cast<float const*>(w.q4), ix.dims, q1, q1 + a.qsplit_len, a.qsplit_len, lane);
                pf_qb = pf_query_bound(a2, ix.dims, pf_sp.rho_a);
            }
        }
        uint32_t const vmask = a.visited_cap - 1;
        uint32_t visited_count = 0;

        /* ---- search_for_one_: greedy descent (index.hpp:3963-4003) ---- */
        uint32_t closest = ix.entry_slot;
        if (lane == 0) cand_s[0] = closest;
        __syncwarp();
        measure_list<M, STAGED>(ix, a, w, qc, 1, lane);
        computed += 1;
        float closest_d = cand_d[0];
        __syncwarp();
        bool const cluster = a.cluster_end_level >= 0; /* index_gt::cluster (index.hpp:3092-3125): descent only */
        int const end_level = cluster ? a.cluster_end_level : bl;
        for (int level = ix.max_level; level > end_level; --level) {
            bool changed;
            do {
                changed = false;
                uint32_t const ubase = ix.upper_base[closest];
                uint32_t const* row = ix.upper + ((size_t)ubase + (uint32_t)(level - 1)) * ix.m_stride;
                uint32_t n = 0;
                for (uint32_t b = 0; b < ix.m; b += 32) {
                    uint32_t i = b + lane;
                    uint32_t s = (i < ix.m && ubase != EMPTY_SLOT) ? row[i] : EMPTY_SLOT;
                    bool valid = s != EMPTY_SLOT;
                    uint32_t bal = __ballot_sync(0xffffffffu, valid);
                    if (valid) cand_s[n + __popc(bal & ((1u << lane) - 1))] = s;
                    n += __popc(bal);
                }
                __syncwarp();
                measure_list<M, STAGED>(ix, a, w, qc, n, lane);
                computed += n;
                /* sequential `if (d < closest_d)` scan == first occurrence of the strict minimum */
                for (uint32_t b = 0; b < n; b += 32) {
                    uint32_t i = b + lane;
                    float d = i < n ? cand_d[i] : 0.f;
                    bool better = i < n && d < closest_d;
                    float best = better ? d : __int_as_float(0x7f800000);
                    uint32_t best_i = better ? i : 0xFFFFFFFFu;
#pragma unroll
                    for (int o = 16; o; o >>= 1) { /* warp argmin with first-index tie-break */
                        float od = __shfl_xor_sync(0xffffffffu, best, o);
                        uint32_t oi = __shfl_xor_sync(0xffffffffu, best_i, o);
                        if (oi != 0xFFFFFFFFu && (best_i == 0xFFFFFFFFu || od < best || (od == best && oi < best_i))) {
                            best = od;
                            best_i = oi;
                        }
                    }
                    if (best_i != 0xFFFFFFFFu) {
                        closest_d = best;
                        closest = cand_s[best_i];
                        changed = true;
                    }
                }
                __syncwarp();
                cycles += 1;
            } while (changed);
        }

        if (prof && lane == 0) atomicAdd(a.phase_cycles + 20, (unsigned long long)w.t_wait); /* the descent's vector waits */
        /* ---- search_to_find_in_base_ (index.hpp:4175-4246) ---- */
        if (lane == 0) cand_s[0] = closest;
        __syncwarp();
        measure_list<M, STAGED>(ix, a, w, qc, 1, lane);
        computed += 1;
        float radius = cand_d[0];
        __syncwarp();
        if (lane == 0 && !cluster) {
            heap.set_root(cand_t{radius, closest});
            if (bitmap) atomicOr(&visited[closest >> 5], 1u << (closest & 31));
            else atomicCAS(&visited[hash_slot(closest) & vmask], EMPTY_SLOT, closest);
            if (logged) vlog[0] = closest;
        }
        heap_size = cluster ? 0 : 1;
        visited_count = cluster ? 0 : 1;
        uint32_t pre_node = EMPTY_SLOT, pre_s0 = EMPTY_SLOT, pre_s1 = EMPTY_SLOT; /* speculative row prefetch */
        /* DIRECT kernels (short vectors, binary codes) have registers to spare and hops so short that the list itself is
         * the critical path: they keep rows of up to 128 neighbours (M = 64, BASELINE config C5) in registers as well */
        constexpr bool WIDE = !STAGED;
        uint32_t pre_s2 = EMPTY_SLOT, pre_s3 = EMPTY_SLOT;
        PHASE(pc0)
        {
            /* cluster(): the closest member at that level is the whole answer, predicate ignored (index.hpp:3122) */
            /* search_to_update_ (index.hpp:4086-4168): a reused slot is searched from and expanded, but never
             * enters its own `top`. For an appended member no list reaches its slot, so the test never fires. */
            bool allowed = cluster || (insert ? closest != qi
                                                   : GROUPED ? slot_allowed_row(ix, group_row, closest) : slot_allowed(ix, a, closest));
            if (allowed) {
                if (topreg) {
                    if (lane == 0) { rtd[0] = radius; rts[0] = closest; }
                } else if (lane == 0) { top_d[0] = radius; top_s[0] = closest; }
                top_size = 1;
                top_nan = top_may_hold_nan(false, radius);
            }
        }
        __syncwarp();

        while (heap_size) {
            cand_t cur = heap.root();
            if (cur.d > radius && top_size == ef) break;
            /* the neighbour row is addressed by the root alone: fetch it while lane 0 sifts the heap */
            uint32_t const* row = row_of(cur.s);
            uint32_t s0, s1, s2 = EMPTY_SLOT, s3 = EMPTY_SLOT;
            if (cur.s == pre_node) { /* the row was prefetched during the previous hop */
                s0 = pre_s0;
                s1 = pre_s1;
                if constexpr (WIDE) { s2 = pre_s2; s3 = pre_s3; }
            } else {
                s0 = lane < (int)width ? __ldg(row + lane) : EMPTY_SLOT;
                s1 = lane + 32 < (int)width ? __ldg(row + lane + 32) : EMPTY_SLOT;
                if constexpr (WIDE) {
                    s2 = lane + 64 < (int)width ? __ldg(row + lane + 64) : EMPTY_SLOT;
                    s3 = lane + 96 < (int)width ? __ldg(row + lane + 96) : EMPTY_SLOT;
                }
            }
            __syncwarp(); /* every lane holds `cur` before lane 0 rearranges the heap */
            /* BITMAP visits: one atomicOr per neighbour, all in flight together (the frozen lists hold no
             * duplicates and no self-links: those can never be `fresh`, freeze drops them). They are issued
             * BEFORE the pop so that lane 0 sifts the heap while the atomics make their round trip to L2. */
            uint32_t o0 = 0xFFFFFFFFu, o1 = 0xFFFFFFFFu, o2 = 0xFFFFFFFFu, o3 = 0xFFFFFFFFu;
            if (bitmap) {
                if (s0 != EMPTY_SLOT) o0 = atomicOr(&visited[s0 >> 5], 1u << (s0 & 31));
                if (s1 != EMPTY_SLOT) o1 = atomicOr(&visited[s1 >> 5], 1u << (s1 & 31));
                if constexpr (WIDE) {
                    if (s2 != EMPTY_SLOT) o2 = atomicOr(&visited[s2 >> 5], 1u << (s2 & 31));
                    if (s3 != EMPTY_SLOT) o3 = atomicOr(&visited[s3 >> 5], 1u << (s3 & 31));
                }
            }
            if (!heap.template pop_warp<PF ? 16 : 8>(heap_size, lane)) {
                if (lane == 0) heap.pop(heap_size);
            }
            heap_size -= 1;
            cycles += 1;
            __syncwarp();
            /* Speculation: unless this hop finds something closer, the new root is expanded next.
             * Its neighbour row is requested now and only consumed one hop later. */
            if (heap_size) {
                pre_node = heap.root().s;
                uint32_t const* next_row = row_of(pre_node);
                pre_s0 = lane < (int)width ? __ldg(next_row + lane) : EMPTY_SLOT;
                pre_s1 = lane + 32 < (int)width ? __ldg(next_row + lane + 32) : EMPTY_SLOT;
                if constexpr (WIDE) {
                    pre_s2 = lane + 64 < (int)width ? __ldg(next_row + lane + 64) : EMPTY_SLOT;
                    pre_s3 = lane + 96 < (int)width ? __ldg(next_row + lane + 96) : EMPTY_SLOT;
                }
            } else
                pre_node = EMPTY_SLOT;
            PHASE(pc1)

            /* compact the unseen neighbours in stored order */
            uint32_t ncand = 0;
            if (bitmap) {
                bool f0 = s0 != EMPTY_SLOT && !((o0 >> (s0 & 31)) & 1u);
                bool f1 = s1 != EMPTY_SLOT && !((o1 >> (s1 & 31)) & 1u);
                uint32_t bal0 = __ballot_sync(0xffffffffu, f0), bal1 = __ballot_sync(0xffffffffu, f1);
                uint32_t const lt = (1u << lane) - 1;
                if (f0) cand_s[__popc(bal0 & lt)] = s0;
                ncand = __popc(bal0);
                if (f1) cand_s[ncand + __popc(bal1 & lt)] = s1;
                ncand += __popc(bal1);
                if (logged) { /* remember which bits this query set */
                    if (visited_count + width > a.visit_log_cap) log_overflow = true;
                    if (!log_overflow) {
                        if (f0) vlog[visited_count + __popc(bal0 & lt)] = s0;
                        if (f1) vlog[visited_count + __popc(bal0) + __popc(bal1 & lt)] = s1;
                    }
                }
                if constexpr (WIDE) { /* neighbours 64..127, already in registers */
                    bool const f2 = s2 != EMPTY_SLOT && !((o2 >> (s2 & 31)) & 1u);
                    bool const f3 = s3 != EMPTY_SLOT && !((o3 >> (s3 & 31)) & 1u);
                    uint32_t const bal2 = __ballot_sync(0xffffffffu, f2), bal3 = __ballot_sync(0xffffffffu, f3);
                    uint32_t const at2 = ncand + __popc(bal2 & lt), at3 = ncand + __popc(bal2) + __popc(bal3 & lt);
                    if (f2) cand_s[at2] = s2;
                    if (f3) cand_s[at3] = s3;
                    if (logged && !log_overflow) {
                        if (f2) vlog[visited_count + at2] = s2;
                        if (f3) vlog[visited_count + at3] = s3;
                    }
                    ncand += __popc(bal2) + __popc(bal3);
                }
                for (uint32_t b = WIDE ? 128 : 64; b < width; b += 32) {
                    uint32_t i = b + lane;
                    uint32_t s = i < width ? __ldg(row + i) : EMPTY_SLOT;
                    uint32_t o = s != EMPTY_SLOT ? atomicOr(&visited[s >> 5], 1u << (s & 31)) : 0xFFFFFFFFu;
                    bool f = s != EMPTY_SLOT && !((o >> (s & 31)) & 1u);
                    uint32_t bal = __ballot_sync(0xffffffffu, f);
                    if (f) cand_s[ncand + __popc(bal & lt)] = s;
                    if (logged && !log_overflow && f) vlog[visited_count + ncand + __popc(bal & lt)] = s;
                    ncand += __popc(bal);
                }
            } else {
                /* visits.reserve(): keep the table at most half full so probing terminates quickly */
                if ((visited_count + width) * 2 > a.visited_cap) { status = STATUS_VISITED_OVERFLOW; break; }
                for (uint32_t b = 0; b < width; b += 32) {
                    uint32_t i = b + lane;
                    uint32_t s = b == 0 ? s0 : (b == 32 ? s1 : (WIDE && b == 64 ? s2 : (WIDE && b == 96 ? s3 : (i < width ? __ldg(row + i) : EMPTY_SLOT))));
                    bool fresh = false;
                    if (s != EMPTY_SLOT) {
                        uint32_t h = hash_slot(s) & vmask;
                        for (;;) {
                            uint32_t old = atomicCAS(&visited[h], EMPTY_SLOT, s);
                            if (old == EMPTY_SLOT) { fresh = true; break; }
                            if (old == s) break;
                            h = (h + 1) & vmask;
                        }
                    }
                    uint32_t bal = __ballot_sync(0xffffffffu, fresh);
                    if (fresh) cand_s[ncand + __popc(bal & ((1u << lane) - 1))] = s;
                    ncand += __popc(bal);
                }
            }
            visited_count += ncand;
            __syncwarp();
            PHASE(pc2)
            if (ncand == 0) continue;

            bool measured = false;
            uint32_t nacc = ncand; /* the candidates the accept replay visits */
            uint32_t const waits0 = w.t_wait + w.t_code, pc4_0 = pc4; /* introspection */
            if constexpr (PF) {
                if (a.prefilter && top_size == ef) { /* `top` full: every candidate must beat the radius */
                    nacc = measure_prefiltered<M>(ix, a, w, qc, pf_qb, pf_sp, radius, ncand, lane);
                    n_pref += ncand;
                    n_surv += nacc;
                    n_pf_hops += 1;
                    measured = true;
                }
            }
            if (!measured) measure_list<M, STAGED>(ix, a, w, qc, ncand, lane);
            computed += ncand;
            PHASE(pc4)
            if (prof && top_size == ef) pc4_full += (pc4 - pc4_0) - (w.t_wait + w.t_code - waits0);

            /* The reference's sequential accept loop, replayed in stored order. `radius` only shrinks
             * and `top` only grows inside a hop, so a candidate that fails `|top|<ef || d<radius` at the
             * start of the hop fails it at its turn as well: only the others are visited. */
            for (uint32_t b = 0; b < nacc && status == STATUS_OK; b += 32) {
                uint32_t c = b + lane;
                bool maybe = c < nacc && (top_size < ef || cand_d[c] < radius);
                uint32_t todo = __ballot_sync(0xffffffffu, maybe);
                while (todo) {
                    uint32_t c2 = b + (__ffs(todo) - 1);
                    todo &= todo - 1;
                    float d = cand_d[c2];
                    if (top_size < ef || d < radius) {
                        uint32_t s = cand_s[c2];
                        if (heap_size + 2 >= a.heap_smem_cap + a.heap_spill_cap) { status = STATUS_HEAP_OVERFLOW; break; }
                        heap.push(heap_size, cand_t{d, s}, lane);
                        heap_size += 1;
                        if (prof) { n_push += 1; max_heap = max(max_heap, heap_size); }
                        bool allowed = insert ? s != qi : GROUPED ? slot_allowed_row(ix, group_row, s) : slot_allowed(ix, a, s);
                        if (allowed) {
                            if (topreg) {
                                top_insert_reg(rtd, rts, top_size, ef, d, s, top_nan, lane);
                                radius = top_back_reg(rtd, top_size);
                            } else {
                                top_insert(top_d, top_s, top_size, ef, d, s, top_nan, lane);
                                radius = top_d[top_size - 1];
                            }
                        }
                        __syncwarp();
                    }
                }
            }
            PHASE(pc5)
            if (status != STATUS_OK) break;
        }
        visited_total = visited_count;
        log_overflow_out = log_overflow;
    }

    /* leave the logged bitmap all-zero for the next query of this warp */
    if (ix.n != 0 && k != 0 && a.visited_bitmap_words != 0 && a.visit_log != nullptr) {
        __syncwarp();
        if (!log_overflow_out) {
            /* eight independent log reads in flight per lane: the loop is a chain of L2 round trips otherwise
             * (measured at 10M x 768: 6 % of the kernel in this loop before the unrolling) */
            uint32_t const* vlog = a.visit_log + (size_t)blockIdx.x * a.visit_log_cap;
            for (uint32_t i0 = 0; i0 < visited_total; i0 += 32 * 8) {
                uint32_t e[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    uint32_t const i = i0 + (uint32_t)(u * 32 + lane);
                    e[u] = i < visited_total ? vlog[i] : EMPTY_SLOT;
                }
#pragma unroll
                for (int u = 0; u < 8; ++u)
                    if (e[u] != EMPTY_SLOT) visited[e[u] >> 5] = 0u;
            }
        } else {
            uint4 const zero = make_uint4(0u, 0u, 0u, 0u);
            uint4* v4 = reinterpret_cast<uint4*>(visited);
            for (uint32_t j = lane; j < a.visited_bitmap_words / 4; j += 32) v4[j] = zero;
        }
        __threadfence_block();
    }

    /* ---- dump_to (index.hpp:2707-2722) ---- */
    __syncwarp();
    uint32_t count = top_size < k ? top_size : k;
    if (topreg) {
#pragma unroll
        for (int j = 0; j < TOP_E; ++j) {
            uint32_t const i = (uint32_t)lane * TOP_E + (uint32_t)j;
            if (i < k) {
                uint64_t key = 0;
                uint32_t bits = SNAN_BITS;
                if (i < count) {
                    key = insert ? (uint64_t)rts[j] : ix.keys[rts[j]];
                    bits = __float_as_uint(rtd[j]);
                }
                if (insert) a.out_slots[(size_t)out_row * k + i] = (uint32_t)key;
                else a.out_keys[(size_t)out_row * k + i] = key;
                reinterpret_cast<uint32_t*>(a.out_dists)[(size_t)out_row * k + i] = bits;
            }
        }
    } else {
        for (uint32_t i = lane; i < k; i += 32) {
            uint64_t key = 0;
            uint32_t bits = SNAN_BITS;
            if (i < count) {
                key = insert ? (uint64_t)top_s[i] : ix.keys[top_s[i]];
                bits = __float_as_uint(top_d[i]);
            }
            if (insert) a.out_slots[(size_t)out_row * k + i] = (uint32_t)key;
            else a.out_keys[(size_t)out_row * k + i] = key;
            reinterpret_cast<uint32_t*>(a.out_dists)[(size_t)out_row * k + i] = bits;
        }
    }
    if (lane == 0) {
        a.out_counts[out_row] = count;
        if (a.out_computed) a.out_computed[out_row] = computed;
        if (a.out_visited) a.out_visited[out_row] = cycles;
        a.status[out_row] = status;
    }
    __syncwarp();
    if (prof && lane == 0) {
        uint32_t pc6 = (uint32_t)(clock64() - tp);
        atomicAdd(a.phase_cycles + 0, (unsigned long long)pc0);
        atomicAdd(a.phase_cycles + 1, (unsigned long long)pc1);
        atomicAdd(a.phase_cycles + 2, (unsigned long long)pc2);
        atomicAdd(a.phase_cycles + 3, (unsigned long long)w.t_wait);
        atomicAdd(a.phase_cycles + 4, (unsigned long long)(pc4 - w.t_wait - w.t_code));
        atomicAdd(a.phase_cycles + 5, (unsigned long long)pc5);
        atomicAdd(a.phase_cycles + 6, (unsigned long long)pc6);
        atomicAdd(a.phase_cycles + 7, 1ull);
        atomicAdd(a.phase_cycles + 8, (unsigned long long)n_push);
        atomicAdd(a.phase_cycles + 9, (unsigned long long)max_heap);
        atomicMax(a.phase_cycles + 10, (unsigned long long)max_heap);
        atomicAdd(a.phase_cycles + 11, (unsigned long long)n_pref);
        atomicAdd(a.phase_cycles + 12, (unsigned long long)n_surv);
        atomicAdd(a.phase_cycles + 13, (unsigned long long)w.t_code);
        atomicAdd(a.phase_cycles + 14, (unsigned long long)w.t_dot);
        atomicAdd(a.phase_cycles + 15, (unsigned long long)w.t_bound);
        atomicAdd(a.phase_cycles + 16, (unsigned long long)w.t_conv);
        atomicAdd(a.phase_cycles + 17, (unsigned long long)w.n_code_pass);
        atomicAdd(a.phase_cycles + 18, (unsigned long long)n_pf_hops);
        atomicAdd(a.phase_cycles + 19, (unsigned long long)pc4_full);
    }
#undef PHASE
}

/* MIN_CTAS: resident CTAs (= warps) per SM the register allocation must allow: 8 for the staged f32 kernel (its 16
 * accumulators and the register-resident `top` want ~220 registers), 16 for everything else (see the dispatch below). */
template <class M, bool STAGED, int MIN_CTAS = (STAGED ? 8 : 16), bool INSERT = false, bool GROUPED = false>
__global__ void __launch_bounds__(THREADS, MIN_CTAS) hnsw_search_kernel(__grid_constant__ device_index_t const ix,
                                                              __grid_constant__ search_args_t const a) {
    extern __shared__ __align__(128) uint8_t smem[];
    int const lane = threadIdx.x;
    warp_ctx_t w;
    w.q4 = reinterpret_cast<uint4*>(smem);
    w.top_d = reinterpret_cast<float*>(smem + a.off_top_d);
    w.top_s = reinterpret_cast<uint32_t*>(smem + a.off_top_s);
    w.cand_s = reinterpret_cast<uint32_t*>(smem + a.off_cand_s);
    w.cand_d = reinterpret_cast<float*>(smem + a.off_cand_d);
    w.stage = smem + a.off_stage;
    w.stage_addr = smem_u32(w.stage);
    w.bars_addr = smem_u32(smem + a.off_bars);
    w.phase = 0;
    heap_t heap{smem_u32(smem + a.off_heap), a.heap_spill + (size_t)blockIdx.x * a.heap_spill_cap, a.heap_smem_cap};
    uint32_t* visited = a.visited + (size_t)blockIdx.x * (a.visited_bitmap_words ? a.visited_bitmap_words : a.visited_cap);
    if constexpr (STAGED) {
        mbar_init(w.bars_addr + 8u * lane, 1); /* 32 mbarriers: 2 sets x 8 slots (LPV 4) or 1 set x 32 slots (LPV 1) */
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
    }
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(a.work_counter, 1u);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= a.nq) break;
        uint32_t const qi = a.query_list ? a.query_list[item] : item;
        /* INSERT mode: one output row per work item (the same member is searched once per level) */
        uint32_t const out_row = INSERT ? item : qi;
        int const bl = INSERT ? (int)a.task_levels[item] : 0;
        search_one<M, STAGED, INSERT, GROUPED>(ix, a, qi, out_row, bl, w, heap, visited, lane);
    }
}

/* ---- results of a search in an empty index: no matches, rows padded like dump_to (index.hpp:2715-2720) ------------- */

__global__ void fill_empty_kernel(uint64_t* keys, uint32_t* dist_bits, uint32_t* counts, uint32_t* computed, uint32_t* visited,
                                  size_t nq, size_t k) {
    size_t const i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nq * k) { keys[i] = 0; dist_bits[i] = SNAN_BITS; }
    if (i < nq) {
        counts[i] = 0;
        if (computed) computed[i] = 0;
        if (visited) visited[i] = 0;
    }
}

cudaError_t search_fill_empty(uint64_t* keys, float* dists, uint32_t* counts, uint32_t* computed, uint32_t* visited, size_t nq,
                              size_t k, cudaStream_t stream) {
    size_t const total = nq * (k ? k : 1);
    fill_empty_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(keys, reinterpret_cast<uint32_t*>(dists), counts, computed,
                                                                           visited, nq, k);
    return cudaGetLastError();
}

/* ---- filtered search: allowed keys -> bitmap over slots -------------------------------------------- */

__global__ void allow_bits_kernel(uint64_t const* keys, uint32_t n, uint64_t const* allowed_sorted, uint32_t m, uint32_t* bits) {
    uint32_t const slot = blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (slot < n) {
        uint64_t const key = keys[slot];
        uint32_t lo = 0, hi = m;
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1;
            if (allowed_sorted[mid] < key) lo = mid + 1;
            else hi = mid;
        }
        hit = lo < m && allowed_sorted[lo] == key;
    }
    uint32_t const word = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && slot < n) bits[slot >> 5] = word;
}

cudaError_t search_build_allow_bits(device_index_t const& ix, uint64_t const* allowed_sorted, uint32_t m, uint32_t* bits,
                                    cudaStream_t stream) {
    if (!ix.n) return cudaSuccess;
    allow_bits_kernel<<<(ix.n + 255) / 256, 256, 0, stream>>>(ix.keys, ix.n, allowed_sorted, m, bits);
    return cudaGetLastError();
}

/* ---- freeze-time helper: squared norms in the metric's summation order -------------------------- */

template <class M> __global__ void norms_kernel(device_index_t ix, float* norms, uint32_t const* slots) {
    constexpr int LPV = M::LPV;
    uint32_t const lane = threadIdx.x & 31, group = (blockIdx.x * blockDim.x + threadIdx.x) / LPV;
    uint32_t const i = group < ix.n ? group : ix.n - 1; /* whole warps stay converged for the shuffles */
    uint32_t const slot = slots ? slots[i] : i;
    uint4 const* v = reinterpret_cast<uint4 const*>(ix.vectors + (size_t)slot * ix.vec_stride);
    float b2 = M::self_dot(v, ix.chunks16, (int)lane);
    if (group < ix.n && (lane % LPV) == 0) norms[slot] = b2;
}

bool search_needs_norms(uint32_t metric, uint32_t scalar) {
    return metric == METRIC_COS && (scalar == SCALAR_F32 || scalar == SCALAR_F16 || scalar == SCALAR_BF16);
}

cudaError_t search_compute_norms(device_index_t const& ix, float* norms, cudaStream_t stream, uint32_t const* slots) {
    if (!ix.n) return cudaSuccess;
    uint32_t const threads = 256;
    if (ix.scalar == SCALAR_F32) {
        uint32_t const per_block = threads / 4;
        norms_kernel<cos_f32_t><<<(ix.n + per_block - 1) / per_block, threads, 0, stream>>>(ix, norms, slots);
    } else if (ix.scalar == SCALAR_F16) {
        norms_kernel<cos_half_t<f16_conv_t>><<<(ix.n + threads - 1) / threads, threads, 0, stream>>>(ix, norms, slots);
    } else if (ix.scalar == SCALAR_BF16) {
        norms_kernel<cos_half_t<bf16_conv_t>><<<(ix.n + threads - 1) / threads, threads, 0, stream>>>(ix, norms, slots);
    } else
        return cudaErrorInvalidValue;
    return cudaGetLastError();
}

/* ---- the int8 shadow of cos / ip f32 rows (prefilter_bound.h): one warp per row -------------------------- */

__global__ void shadow_kernel(device_index_t ix, float const* norms, int8_t* codes, pf_record_t* records, uint32_t const* slots) {
    uint32_t const lane = threadIdx.x & 31, i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= ix.n) return; /* uniform per warp */
    uint32_t const row = slots ? slots[i] : i;
    float const* b = reinterpret_cast<float const*>(ix.vectors + (size_t)row * ix.vec_stride);
    double mx = 0.0;
    bool finite = true;
    for (uint32_t i = lane; i < ix.dims; i += 32) {
        double const x = fabs((double)b[i]);
        finite = finite && x < INFINITY;
        mx = fmax(mx, x);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    finite = __all_sync(0xffffffffu, finite);
    float const s = pf_scale(mx);
    bool const usable = finite && s > 0.0f;
    double e2 = 0.0, n2 = 0.0;
    int8_t* const c = codes + (size_t)row * ix.code_stride;
    for (uint32_t i = lane; i < ix.code_stride; i += 32) {
        int8_t q = 0;
        if (usable && i < ix.dims) {
            q = pf_code(b[i], s);
            double const e = (double)b[i] - (double)s * (double)q;
            e2 += e * e;
            n2 += (double)b[i] * (double)b[i];
        }
        c[i] = q;
    }
    e2 = warp_sum_f64(e2);
    n2 = warp_sum_f64(n2);
    if (lane == 0) {
        float const b2 = norms ? norms[row] : 0.f;
        records[row] = usable ? pf_record_t{s, pf_round_up_norm(e2), pf_round_up_norm(n2), b2}
                              : pf_record_t{0.f, INFINITY, INFINITY, b2};
    }
}

bool search_is_staged(device_index_t const& ix);
bool search_needs_shadow(device_index_t const& ix) {
    return ix.scalar == SCALAR_F32 && (ix.metric == METRIC_COS || ix.metric == METRIC_IP) && search_is_staged(ix);
}
uint32_t search_code_stride(device_index_t const& ix) { return (ix.dims + 15u) & ~15u; }

cudaError_t search_compute_shadow(device_index_t const& ix, float const* norms, int8_t* codes, pf_record_t* records,
                                  cudaStream_t stream, uint32_t const* slots) {
    if (!ix.n) return cudaSuccess;
    uint32_t const rows_per_block = 8;
    shadow_kernel<<<(ix.n + rows_per_block - 1) / rows_per_block, 32 * rows_per_block, 0, stream>>>(ix, norms, codes, records, slots);
    return cudaGetLastError();
}

/* ---- host-side dispatch --------------------------------------------------------------------- */

/*
 *  Which kernel serves which index:
 *    f32, vectors >= 256 B      STAGED, 4 lanes per vector, 8 resident warps per SM allowed by the register budget
 *    f64                        the f32 layout (4 lanes per vector, two doubles per 16-byte chunk): STAGED from 256 B,
 *                               DIRECT below; both compiled for 8 resident warps per SM
 *    f16 / bf16, >= 256 B       STAGED with the WORD metrics (4 lanes per vector split by accumulator) compiled for 16
 *                               resident warps per SM; one stage set up to 2 KB vectors (a quarter of the shared memory
 *                               per warp of one lane per vector in a single 32-slot set)
 *    i8, >= 256 B               STAGED compiled for 16 resident warps per SM, one stage set up to 2 KB: a hop moves few
 *                               bytes, so resident warps matter more than double buffering
 *    b1, and anything < 256 B   DIRECT (16-byte chunks through registers)
 *  Every one of them also exists as an INSERT-mode kernel for the builder, and as a GROUPED kernel for grouped filtered
 *  search.
 */
template <class M, bool STAGED, int MIN_CTAS>
static cudaError_t launch_k(device_index_t const& ix, search_args_t const& a, int blocks, size_t smem, cudaStream_t stream) {
    if (a.out_slots) { /* INSERT mode (builder.cu) */
        auto kernel = hnsw_search_kernel<M, STAGED, MIN_CTAS, true>;
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kernel<<<blocks, THREADS, smem, stream>>>(ix, a);
        return cudaGetLastError();
    }
    if (a.allow_groups) { /* grouped filtered search: a bitmap row per query's group */
        auto kernel = hnsw_search_kernel<M, STAGED, MIN_CTAS, false, true>;
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kernel<<<blocks, THREADS, smem, stream>>>(ix, a);
        return cudaGetLastError();
    }
    auto kernel = hnsw_search_kernel<M, STAGED, MIN_CTAS, false>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kernel<<<blocks, THREADS, smem, stream>>>(ix, a);
    return cudaGetLastError();
}

template <class M, bool STAGED, int MIN_CTAS> static cudaError_t occupancy_k(int* blocks_per_sm, size_t smem, bool grouped) {
    /* the INSERT twin needs no more registers; the GROUPED one is asked for itself */
    auto kernel = grouped ? hnsw_search_kernel<M, STAGED, MIN_CTAS, false, true> : hnsw_search_kernel<M, STAGED, MIN_CTAS, false>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, kernel, THREADS, smem);
}

/* OP is `launch_k` or `occupancy_k`; ARGS its run-time arguments in parentheses */
#define FOR_METRIC(OP, ARGS)                                                                                    \
    switch (ix.scalar) {                                                                                        \
    case SCALAR_F32:                                                                                            \
        if (ix.metric == METRIC_L2SQ) return staged ? OP<l2sq_f32_t, true, 8> ARGS : OP<l2sq_f32_t, false, 16> ARGS; \
        if (ix.metric == METRIC_IP) return staged ? OP<ip_f32_t, true, 8> ARGS : OP<ip_f32_t, false, 16> ARGS;  \
        if (ix.metric == METRIC_COS) return staged ? OP<cos_f32_t, true, 8> ARGS : OP<cos_f32_t, false, 16> ARGS; \
        break;                                                                                                  \
    case SCALAR_F64:                                                                                            \
        if (ix.metric == METRIC_L2SQ) return staged ? OP<l2sq_f64_t, true, 8> ARGS : OP<l2sq_f64_t, false, 8> ARGS; \
        if (ix.metric == METRIC_IP) return staged ? OP<ip_f64_t, true, 8> ARGS : OP<ip_f64_t, false, 8> ARGS;  \
        if (ix.metric == METRIC_COS) return staged ? OP<cos_f64_t, true, 8> ARGS : OP<cos_f64_t, false, 8> ARGS; \
        break;                                                                                                  \
    case SCALAR_F16:                                                                                            \
        if (ix.metric == METRIC_L2SQ) return staged ? OP<l2sq_halfw_t<f16_conv_t>, true, 16> ARGS : OP<l2sq_half_t<f16_conv_t>, false, 16> ARGS; \
        if (ix.metric == METRIC_IP) return staged ? OP<ip_halfw_t<f16_conv_t>, true, 16> ARGS : OP<ip_half_t<f16_conv_t>, false, 16> ARGS; \
        if (ix.metric == METRIC_COS) return staged ? OP<cos_halfw_t<f16_conv_t>, true, 16> ARGS : OP<cos_half_t<f16_conv_t>, false, 16> ARGS; \
        break;                                                                                                  \
    case SCALAR_BF16:                                                                                           \
        if (ix.metric == METRIC_L2SQ) return staged ? OP<l2sq_halfw_t<bf16_conv_t>, true, 16> ARGS : OP<l2sq_half_t<bf16_conv_t>, false, 16> ARGS; \
        if (ix.metric == METRIC_IP) return staged ? OP<ip_halfw_t<bf16_conv_t>, true, 16> ARGS : OP<ip_half_t<bf16_conv_t>, false, 16> ARGS; \
        if (ix.metric == METRIC_COS) return staged ? OP<cos_halfw_t<bf16_conv_t>, true, 16> ARGS : OP<cos_half_t<bf16_conv_t>, false, 16> ARGS; \
        break;                                                                                                  \
    case SCALAR_I8:                                                                                             \
        if (ix.metric == METRIC_L2SQ) return staged ? OP<l2sq_i8_t<4>, true, 16> ARGS : OP<l2sq_i8_t<4>, false, 16> ARGS; \
        if (ix.metric == METRIC_IP) return staged ? OP<ip_i8_t<4>, true, 16> ARGS : OP<ip_i8_t<4>, false, 16> ARGS; \
        if (ix.metric == METRIC_COS) return staged ? OP<cos_i8_t<4>, true, 16> ARGS : OP<cos_i8_t<4>, false, 16> ARGS; \
        break;                                                                                                  \
    case SCALAR_B1:                                                                                             \
        if (ix.metric == METRIC_HAMMING) return OP<hamming_b1_t<2>, false, 16> ARGS;                            \
        if (ix.metric == METRIC_TANIMOTO || ix.metric == METRIC_JACCARD) return OP<tanimoto_b1_t<2>, false, 16> ARGS; \
        if (ix.metric == METRIC_SORENSEN) return OP<sorensen_b1_t<2>, false, 16> ARGS;                          \
        break;                                                                                                  \
    default: break;                                                                                             \
    }                                                                                                           \
    return cudaErrorInvalidValue;

/* vectors of at least this many bytes are fetched with TMA bulk copies into shared memory */
constexpr uint32_t STAGED_MIN_BYTES = 256;

bool search_is_staged(device_index_t const& ix) { return ix.scalar != SCALAR_B1 && ix.vec_stride >= STAGED_MIN_BYTES; }
static bool is_half(device_index_t const& ix) { return ix.scalar == SCALAR_F16 || ix.scalar == SCALAR_BF16; }
int search_lanes_per_vector(device_index_t const&) { return 4; } /* every STAGED metric splits a vector over 4 lanes */
/* bytes added to a 128-byte-rounded slot so that the lane groups of a pass hit disjoint banks: 16*LPV for 16-byte
 * units (each lane of a group reads its own chunk), 16 for word units (a group reads one chunk) */
uint32_t search_stage_pad(device_index_t const& ix) { return is_half(ix) ? 16u : 64u; }
int search_stage_slots(device_index_t const& ix) { return search_is_staged(ix) ? 8 : 0; }
/* resident warps per SM the compiled kernel's registers allow (its MIN_CTAS): what the plan may count on */
int search_max_warps_per_sm(device_index_t const& ix) {
    if (ix.scalar == SCALAR_F64) return 8; /* both f64 kernels: 16 warps per SM would spill their f64 accumulators */
    if (!search_is_staged(ix)) return 24;
    return ix.scalar == SCALAR_F32 ? 8 : 16;
}
/* one stage set (no double buffering, more resident warps) for the short staged vectors of the 16-warp kernels */
bool search_single_stage_set(device_index_t const& ix) {
    return search_is_staged(ix) && ix.scalar != SCALAR_F32 && ix.scalar != SCALAR_F64 && ix.vec_stride <= 2048;
}

cudaError_t search_launch(device_index_t const& ix, search_args_t const& a, int blocks, size_t smem, cudaStream_t stream) {
    bool const staged = search_is_staged(ix);
    FOR_METRIC(launch_k, (ix, a, blocks, smem, stream))
}

cudaError_t search_occupancy(device_index_t const& ix, int* blocks_per_sm, size_t smem, bool grouped) {
    bool const staged = search_is_staged(ix);
    FOR_METRIC(occupancy_k, (blocks_per_sm, smem, grouped))
}

bool search_supported(uint32_t metric, uint32_t scalar) {
    switch (scalar) {
    case SCALAR_F32:
    case SCALAR_F64:
    case SCALAR_F16:
    case SCALAR_BF16:
    case SCALAR_I8: return metric == METRIC_L2SQ || metric == METRIC_IP || metric == METRIC_COS;
    case SCALAR_B1:
        return metric == METRIC_HAMMING || metric == METRIC_TANIMOTO || metric == METRIC_JACCARD || metric == METRIC_SORENSEN;
    default: return false;
    }
}

int search_warps_per_block() { return 1; }

} // namespace usearch_b200
