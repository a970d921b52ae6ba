/*
 *  device_index.h — the frozen, flat structure-of-arrays HNSW index as it lives in HBM, and the
 *  arguments of one batched search launch. Plain structs, passed to kernels by value.
 *
 *  The layout replaces the reference's per-node byte tapes and pointer tables
 *  (index.hpp:2116-2195 `node_t`/`neighbors_ref_t`, index.hpp:2280 `nodes_`,
 *  index_dense.hpp:452-460 `vectors_lookup_`) with arrays indexed by slot:
 *
 *    vectors      [n x vec_stride] bytes   row = one vector, zero-padded to a multiple of 16 B so
 *                                          that every lane issues aligned 128-bit loads
 *    keys         [n] u64                  slot -> user key (only read for the k results)
 *    nbr0         [n x m0_stride] u32      layer-0 neighbour slots in stored order; unused tail =
 *                                          0xFFFFFFFF, so no separate count word is needed:
 *                                          one hop reads exactly 4*m0_stride bytes
 *    upper_base   [n] u32                  first row of the node in `upper`, 0xFFFFFFFF if level 0
 *    upper        [rows x m_stride] u32    rows level 1..L of every multi-level node, back to back
 *    norms        [n] f32                  cos/f32 only: squared norm of every vector, accumulated by
 *                                          the exact fma chain the metric would use per distance
 *    codes        [n x code_stride] i8     cos/ip f32 served by the STAGED kernel: the int8 shadow of every vector
 *                                          (prefilter_bound.h), code_stride = round_up(dims, 16), zero padding
 *    shadow       [n] 16-byte records      the same indexes: scale, residual bound, norm bound, squared norm
 *    deleted_bits [ceil(n/32)] u32         bit set when keys[slot] == free_key; NULL when the
 *                                          index holds no removed entries (the common case), which
 *                                          removes the per-candidate key read of
 *                                          index_dense.hpp:2071-2077 from the hot loop
 */
#pragma once
#include <cstddef>
#include <cstdint>

namespace usearch_b200 {

struct pf_record_t; /* prefilter_bound.h */

constexpr uint32_t EMPTY_SLOT = 0xFFFFFFFFu;
constexpr uint32_t SNAN_BITS = 0x7FA00000u; /* numeric_limits<float>::signaling_NaN, index.hpp:2715-2720 */

/* enum values of the reference's serialised head (index_plugins.hpp:113-159) */
enum : uint32_t {
    METRIC_IP = 'i', METRIC_COS = 'c', METRIC_L2SQ = 'e', METRIC_HAMMING = 'b',
    METRIC_TANIMOTO = 't', METRIC_SORENSEN = 's', METRIC_JACCARD = 'j',
};
enum : uint32_t { SCALAR_B1 = 1, SCALAR_BF16 = 4, SCALAR_F64 = 10, SCALAR_F32 = 11, SCALAR_F16 = 12, SCALAR_I8 = 23 };

struct device_index_t {
    uint8_t const* vectors = nullptr;
    uint64_t const* keys = nullptr;
    uint32_t const* nbr0 = nullptr;
    uint32_t const* upper_base = nullptr;
    uint32_t const* upper = nullptr;
    uint32_t const* deleted_bits = nullptr;
    float const* norms = nullptr; /* [n] ||v||^2 in the metric's own summation order (cos f32), else NULL */
    int8_t const* codes = nullptr;        /* [n x code_stride] int8 shadow (cos / ip f32, STAGED), else NULL */
    pf_record_t const* shadow = nullptr; /* [n] its records */
    uint32_t code_stride = 0;             /* bytes */
    uint64_t vec_stride = 0; /* bytes */
    uint32_t n = 0;
    uint32_t m0 = 0, m0_stride = 0; /* connectivity_base and its row stride (u32 units, multiple of 4) */
    uint32_t m = 0, m_stride = 0;   /* connectivity and its row stride */
    uint32_t entry_slot = 0;
    int32_t max_level = 0;
    uint32_t dims = 0;
    uint32_t bytes_per_vector = 0;
    uint32_t chunks16 = 0; /* vec_stride / 16 */
    uint32_t metric = 0, scalar = 0;
};

struct cand_t { /* candidate_t, index.hpp:2097-2101: ordered by distance only */
    float d;
    uint32_t s;
};

/* status codes written per query */
enum : uint32_t { STATUS_OK = 0, STATUS_VISITED_OVERFLOW = 1, STATUS_HEAP_OVERFLOW = 2 };

struct search_args_t {
    /* queries, already in the index's scalar kind */
    uint8_t const* queries = nullptr;
    uint64_t query_stride = 0;
    uint32_t nq = 0;
    uint32_t const* query_list = nullptr; /* optional indirection (retries): work item i -> query id */
    uint32_t k = 0, ef = 0;
    int32_t cluster_end_level = -1; /* >= 0: index_gt::cluster — stop the descent above this level, report the closest member */
    /* INSERT mode (GPU-assisted add, builder.cu): work item i runs search_to_insert_ (index.hpp:4010-4079) for the stored
     * vector of slot query_list[i] on level task_levels[i]: greedy descent down to that level, then the best-first loop over
     * that level's lists with no predicate. Results are SLOTS, one row per WORK ITEM: out_slots/out_dists [nq x k], out_counts [nq]. */
    uint8_t const* task_levels = nullptr;
    uint32_t* out_slots = nullptr;
    /* outputs, dense [nq x k] / [nq] indexed by query id */
    uint64_t* out_keys = nullptr;
    float* out_dists = nullptr;
    uint32_t* out_counts = nullptr;
    uint32_t* out_computed = nullptr; /* may be NULL */
    uint32_t* out_visited = nullptr;  /* may be NULL */
    uint32_t* status = nullptr;
    /* optional device-side predicate (filtered_search): one bit per slot, set = allowed. Applied exactly
     * where the reference applies its predicate (index.hpp:4201, :4236-4240): a rejected member still
     * enters `next` and is expanded, it just never enters `top`. */
    uint32_t const* allow_bits = nullptr;
    /* scheduling + scratch */
    uint32_t* work_counter = nullptr;
    uint32_t* visited = nullptr; /* [warps x visited_cap] */
    uint32_t visited_cap = 0;    /* HASH mode: table entries per warp, power of two */
    /* BITMAP mode (visited_bitmap_words != 0): `visited` holds one bit per slot, words per warp
     * (multiple of 4); one atomicOr per neighbour answers "seen before?" in a single round trip */
    uint32_t visited_bitmap_words = 0;
    /* Large bitmaps are not wiped per query: every slot whose bit gets set is appended to a per-warp log and
     * exactly those words are zeroed when the query ends (the bitmap is all-zero between queries). A log that
     * overflows falls back to a full wipe of that query's bitmap. NULL = wipe at the start of every query. */
    uint32_t* visit_log = nullptr; /* [warps x visit_log_cap] */
    uint32_t visit_log_cap = 0;
    cand_t* heap_spill = nullptr; /* [warps x heap_spill_cap] */
    uint32_t heap_spill_cap = 0;
    uint32_t heap_smem_cap = 0;
    /* per-warp shared memory carve-up (bytes) */
    uint32_t smem_per_warp = 0, off_top_d = 0, off_top_s = 0, off_cand_s = 0, off_cand_d = 0, off_heap = 0;
    /* STAGED kernels: mbarriers and the slots TMA bulk copies land in (stride = 64 mod 128 bytes, so
     * that the 4-lane groups of a quarter-warp read disjoint banks) */
    uint32_t off_bars = 0, off_stage = 0, stage_stride = 0;
    uint32_t stage_sets = 1; /* 2 = double buffered: 2 x (32/LPV) slots, the next pass lands during the math */
    /* layer-0 prefilter (cos / ip f32 with a shadow): once `top` is full, a hop first bulk-copies the int8 codes of its
     * candidates into the stage area (`code_pass` per pass, `code_smem_stride` bytes apart), multiplies them on the
     * tensor cores with the query's int8 split (off_qsplit: q1 then q2, `qsplit_len` bytes each), rejects those whose
     * lower bound proves d >= radius, and measures only the survivors, compacted in `cand_s` (cos: their stored
     * squared norms in surv_b2) */
    uint32_t prefilter = 0, code_pass = 0, code_smem_stride = 0, off_surv_b2 = 0;
    uint32_t off_qsplit = 0, qsplit_len = 0;
    /* optional introspection: PHASE_COUNTERS counters summed over all queries (lane 0 clock64 deltas and counts), in
     * the order of include/usearch_b200.h (usearch_b200_profile_phases, usearch_b200_profile_phases_n) */
    unsigned long long* phase_cycles = nullptr;
    /* grouped filtered search (GROUPED kernels only): `allow_bits` holds one row of `allow_words` words per group of the
     * launch, and query qi tests row allow_groups[qi] - allow_group_base. Appended last, so that the parameter offsets the
     * other kernels read stay where they were. */
    uint32_t const* allow_groups = nullptr;
    uint32_t allow_group_base = 0;
    uint32_t allow_words = 0;
};
constexpr uint32_t PHASE_COUNTERS = 21;

} // namespace usearch_b200
