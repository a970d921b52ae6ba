/*
 *  grouped_filter.cu — filtered search where every query brings its own key set: query i is searched as
 *  filtered_search(queries[i], k, set_keys[offsets[g] .. offsets[g + 1]]) with g = groups[i], all in one launch.
 *
 *  Each set becomes one bitmap row over slots (ceil(size / 32) words), the row allow_bits_kernel would build for it: one
 *  thread per (set, key) entry walks the key -> slot table (device_keys.h) and sets the bit of every slot it finds, so the
 *  cost is O(total keys), never O(slots x sets). The GROUPED search kernels test row groups[qi] where the single-set
 *  kernels test their one bitmap. When the rows of all sets do not fit the `group_bitmap_mb` budget, the sets are served
 *  in rounds of consecutive set ids, each round's queries a contiguous slice of the query ids sorted by set.
 *
 *  The exact form (search_exact_ over only the allowed slots) turns every set into an ascending, duplicate-free list of
 *  its live slots: one thread per entry counts the key's cells in the table, a scan places them, a second pass writes one
 *  (set << 32 | slot) word per cell, and a radix sort plus a unique leave the lists back to back. The queries, sorted by
 *  set and gathered, then run through the LISTED exact kernels, whose CTAs never mix sets (exact_kernel.cu).
 *
 *  Excluded sets (query i searches every live entry whose key is NOT in its set) reuse both: on the graph each row starts
 *  all ones and loses the set's slots; the exact form runs the unfiltered scan at count k + e (e = the live slots of the
 *  set, from its slot list) and drops the set's slots from each row.
 *
 *  All four modes enter through key_set_search_host / key_set_search_device, which share the checks, the empty-index
 *  answer and the key table, and keep their scratch in frozen_index_t::key_set_scratch.
 */
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>

#include "cuda_check.h"
#include "device_keys.h"
#include "exact_args.h"
#include "frozen_index.h"

namespace usearch_b200 {

namespace {

char const* const ERR_SHARDED = "Grouped filtered search does not serve a sharded handle: it holds one shard of its index";
char const* const ERR_NO_SETS = "A batch of queries needs at least one key set";
char const* const ERR_GROUP = "A query's key set index is out of range";
char const* const ERR_OFFSETS = "Key set offsets must start at 0 and never decrease";
char const* const ERR_NO_GROUPS = "Without a set index per query, there must be exactly one key set";

enum : uint32_t { BAD_GROUP = 1, BAD_OFFSETS = 2 };

unsigned grid_for(size_t items, int sm_count) { return (unsigned)std::max<size_t>(1, std::min<size_t>((items + 255) / 256, (size_t)sm_count * 16)); }

/* the bits a radix sort needs for values below `values` (at least 1) */
int bits_for(size_t values) {
    int bits = 1;
    while (bits < 32 && (values - 1) >> bits) ++bits;
    return bits;
}

/* the first i of [lo, hi) with !less(i), for a `less` that holds on a prefix of the range (hi when it holds on all) */
template <typename Less> __device__ __forceinline__ uint32_t lower_bound(uint32_t lo, uint32_t hi, Less less) {
    while (lo < hi) {
        uint32_t const mid = (lo + hi) >> 1;
        if (less(mid)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

/* the set g of [g0, g1) holding CSR entry e: offsets[g] <= e < offsets[g + 1], for offsets[g0] <= e < offsets[g1] */
__device__ __forceinline__ uint32_t set_of_entry(uint64_t const* offsets, uint32_t g0, uint32_t g1, uint64_t e) {
    return lower_bound(g0 + 1, g1, [&](uint32_t g) { return offsets[g] <= e; }) - 1;
}

__global__ void grouped_validate_kernel(uint32_t const* groups, size_t nq, uint64_t const* offsets, size_t group_count, uint32_t* flag) {
    size_t const n = max(nq, group_count);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        if (i < nq && groups[i] >= group_count) atomicOr(flag, (uint32_t)BAD_GROUP);
        if (i < group_count && offsets[i + 1] < offsets[i]) atomicOr(flag, (uint32_t)BAD_OFFSETS);
        if (i == 0 && offsets[0] != 0) atomicOr(flag, (uint32_t)BAD_OFFSETS);
    }
}

/* what each mode accepts beyond the CSR rules all share */
struct key_set_rules_t {
    uint64_t max_sets;    /* refused from this many sets on */
    bool groups_optional; /* `groups` may be NULL when there is one set: every query uses set 0 */
    uint64_t max_entries; /* keys in all the sets */
};
constexpr key_set_rules_t GRAPH_SETS{0xFFFFFFFFull, false, UINT64_MAX};
constexpr key_set_rules_t EXCLUDED_GRAPH_SETS{0xFFFFFFFFull, true, UINT64_MAX};
constexpr key_set_rules_t EXACT_SETS{0x7FFFFFFFull, true, 0x7FFFFFFFull}; /* both exact forms */
key_set_rules_t const& rules_of(bool excluded, bool exact) { return exact ? EXACT_SETS : excluded ? EXCLUDED_GRAPH_SETS : GRAPH_SETS; }

/* the sets of a host entry, checked before anything is uploaded (the offsets size the upload) */
char const* check_key_sets_host(key_sets_t const& sets, size_t nq, key_set_rules_t const& rules) {
    if (sets.count == 0) return ERR_NO_SETS;
    if (!sets.groups && !(rules.groups_optional && sets.count == 1)) return ERR_NO_GROUPS;
    if (sets.offsets[0] != 0) return ERR_OFFSETS;
    for (size_t g = 0; g < sets.count; ++g)
        if (sets.offsets[g + 1] < sets.offsets[g]) return ERR_OFFSETS;
    if (sets.groups)
        for (size_t i = 0; i < nq; ++i)
            if (sets.groups[i] >= sets.count) return ERR_GROUP;
    return nullptr;
}

/* the sets of a device entry, checked on the device before any output is written: one launch, one read-back, which also
 * brings back the number of keys in all the sets */
char const* check_key_sets_device(frozen_index_t& ix, key_sets_t const& sets, size_t nq, key_set_rules_t const& rules, uint64_t* entries,
                                  cudaStream_t s) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    if (sets.count == 0) return ERR_NO_SETS;
    if (sets.count >= rules.max_sets) return "Too many key sets in one call";
    if (!sets.groups && !(rules.groups_optional && sets.count == 1)) return ERR_NO_GROUPS;
    if (char const* e = x.flag.reserve(1)) return e;
    CU(cudaMemsetAsync(x.flag.ptr, 0, 4, s));
    grouped_validate_kernel<<<grid_for(std::max(nq, sets.count), ix.stream.sm_count), 256, 0, s>>>(sets.groups, sets.groups ? nq : 0, sets.offsets,
                                                                                                   sets.count, x.flag.ptr);
    CU(cudaGetLastError());
    ix.kernel_launches += 1;
    uint32_t flag = 0;
    CU(cudaMemcpyAsync(&flag, x.flag.ptr, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(entries, sets.offsets + sets.count, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (flag & BAD_GROUP) return ERR_GROUP;
    if (flag & BAD_OFFSETS) return ERR_OFFSETS;
    if (*entries > rules.max_entries) return "Too many keys in one call's sets";
    return nullptr;
}

/* a host entry's sets to the device: `groups` (when given) to x.groups, `offsets` to x.offsets, the keys to key_stage */
char const* upload_key_sets(frozen_index_t& ix, key_sets_t const& sets, size_t nq) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    if (char const* e = x.groups.reserve(nq)) return e;
    if (char const* e = x.offsets.reserve(sets.count + 1)) return e;
    if (char const* e = ix.stage_keys(sets.keys, sets.offsets[sets.count])) return e;
    if (sets.groups) CU(cudaMemcpyAsync(x.groups.ptr, sets.groups, nq * 4, cudaMemcpyHostToDevice, ix.stream));
    CU(cudaMemcpyAsync(x.offsets.ptr, sets.offsets, (sets.count + 1) * 8, cudaMemcpyHostToDevice, ix.stream));
    return nullptr;
}

/* rows[(g - g0) * words ..] |= the slots of every key of set g, for g0 <= g < g1; the rows start zeroed. The free key
 * allows the removed slots, as allow_bits_kernel's search of keys[] does (the deleted bits reject them first anyway). */
__global__ void grouped_bits_kernel(key_cell_t const* cells, uint64_t mask, uint64_t const* offsets, uint64_t const* set_keys, uint32_t g0,
                                    uint32_t g1, uint64_t free_key, uint32_t const* deleted_bits, uint32_t size, uint32_t words,
                                    uint32_t* rows) {
    uint64_t const begin = offsets[g0], end = offsets[g1];
    for (uint64_t e = begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < end; e += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t* const row = rows + (size_t)(set_of_entry(offsets, g0, g1, e) - g0) * words;
        uint64_t const key = set_keys[e];
        if (key == free_key) {
            if (deleted_bits)
                for (uint32_t w = 0; w < words; ++w) {
                    uint32_t bits = deleted_bits[w];
                    if (w == words - 1 && (size & 31)) bits &= (1u << (size & 31)) - 1u;
                    if (bits) atomicOr(row + w, bits);
                }
            continue;
        }
        key_table_for_each(cells, mask, key, [&](uint32_t s) { atomicOr(row + (s >> 5), 1u << (s & 31)); });
    }
}

/* excluded sets: rows[(g - g0) * words ..] &= ~(the slots of every key of set g); the rows start all ones. The table holds
 * no cell of the free key, and the deleted bits reject removed slots before any row is read, so the free key needs no case. */
__global__ void excluded_bits_kernel(key_cell_t const* cells, uint64_t mask, uint64_t const* offsets, uint64_t const* set_keys, uint32_t g0,
                                     uint32_t g1, uint32_t words, uint32_t* rows) {
    uint64_t const begin = offsets[g0], end = offsets[g1];
    for (uint64_t e = begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < end; e += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t* const row = rows + (size_t)(set_of_entry(offsets, g0, g1, e) - g0) * words;
        key_table_for_each(cells, mask, set_keys[e], [&](uint32_t s) { atomicAnd(row + (s >> 5), ~(1u << (s & 31))); });
    }
}

__global__ void iota_u32_kernel(uint32_t* out, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) out[i] = (uint32_t)i;
}

/* bounds[r] = the first position of `sorted` holding a value >= r * per_round, for r <= rounds */
__global__ void round_bounds_kernel(uint32_t const* sorted, uint32_t nq, uint32_t per_round, uint32_t rounds, uint32_t* bounds) {
    uint32_t const r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r > rounds) return;
    uint64_t const first = (uint64_t)r * per_round;
    bounds[r] = lower_bound(0, nq, [&](uint32_t p) { return sorted[p] < first; });
}

/* x.order = the query ids 0 .. nq - 1 stably sorted by key[id] over bits [0, end_bit), x.sorted = their keys. Nothing waits. */
char const* sort_queries(frozen_index_t& ix, uint32_t const* key, size_t nq, int end_bit, cudaStream_t s) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    if (char const* e = x.ids.reserve(nq)) return e;
    if (char const* e = x.order.reserve(nq)) return e;
    if (char const* e = x.sorted.reserve(nq)) return e;
    iota_u32_kernel<<<grid_for(nq, ix.stream.sm_count), 256, 0, s>>>(x.ids.ptr, nq);
    CU(cudaGetLastError());
    size_t temp_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, key, x.sorted.ptr, x.ids.ptr, x.order.ptr, (int)nq, 0, end_bit, s));
    if (char const* e = x.temp.reserve(std::max<size_t>(temp_bytes, 1))) return e;
    CU(cub::DeviceRadixSort::SortPairs(x.temp.ptr, temp_bytes, key, x.sorted.ptr, x.ids.ptr, x.order.ptr, (int)nq, 0, end_bit, s));
    return nullptr;
}

/* ---- exact filtered search ---- */

/* counts[e] = the live slots under set_keys[e]; the table holds no slot of the free key, so removed slots never count. The
 * counts are 64-bit so that their scan sums in 64 bits (cub takes the sum's type from its input). */
__global__ void listed_count_kernel(key_cell_t const* cells, uint64_t mask, uint64_t const* set_keys, size_t entries, uint64_t* counts) {
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < entries; e += (size_t)gridDim.x * blockDim.x) {
        uint64_t c = 0;
        key_table_for_each(cells, mask, set_keys[e], [&](uint32_t) { ++c; });
        counts[e] = c;
    }
}

/* words[at[e] ..] = (set << 32) | slot for every slot under set_keys[e] */
__global__ void listed_write_kernel(key_cell_t const* cells, uint64_t mask, uint64_t const* offsets, uint32_t sets, uint64_t const* set_keys,
                                    size_t entries, uint64_t const* at, uint64_t* words) {
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < entries; e += (size_t)gridDim.x * blockDim.x) {
        uint64_t const set = set_of_entry(offsets, 0, sets, e);
        uint64_t p = at[e];
        key_table_for_each(cells, mask, set_keys[e], [&](uint32_t s) { words[p++] = set << 32 | s; });
    }
}

/* rows[i] = the slot of unique word i, and slot 0 past the last one up to `bound` (every row a listed scan may size its
 * self-dots by is a real slot); list_at[g] = the first word of set g or later, for g <= sets */
__global__ void listed_rows_kernel(uint64_t const* words, uint32_t const* unique_count, uint32_t bound, uint32_t sets, uint32_t* rows,
                                   uint32_t* list_at) {
    uint32_t const n = *unique_count;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < bound; i += gridDim.x * blockDim.x) rows[i] = i < n ? (uint32_t)words[i] : 0u;
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g <= sets; g += gridDim.x * blockDim.x)
        list_at[g] = lower_bound(0, n, [&](uint32_t i) { return (words[i] >> 32) < g; });
}

/* query_at[g] = the first position of `sorted` (set ids of the queries, ascending) holding g or more; per_set[g] = the
 * work items set g needs at `qpc` queries per item (per_set[sets] = 0, so an exclusive scan ends at the item count) */
__global__ void listed_item_counts_kernel(uint32_t const* sorted, uint32_t nq, uint32_t sets, uint32_t qpc, uint32_t* query_at, uint32_t* per_set) {
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g <= sets; g += gridDim.x * blockDim.x) {
        auto first = [&](uint32_t v) { return lower_bound(0, nq, [&](uint32_t p) { return sorted[p] < v; }); };
        uint32_t const a = first(g);
        query_at[g] = a;
        per_set[g] = g < sets ? (first(g + 1) - a + qpc - 1) / qpc : 0u;
    }
}

__global__ void listed_items_kernel(uint32_t const* query_at, uint32_t const* item_at, uint32_t const* list_at, uint32_t sets, uint32_t qpc,
                                    exact_item_t* items) {
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < sets; g += gridDim.x * blockDim.x) {
        uint32_t const q0 = query_at[g], q1 = query_at[g + 1];
        uint32_t at = item_at[g];
        for (uint32_t q = q0; q < q1; q += qpc) items[at++] = exact_item_t{q, min(qpc, q1 - q), list_at[g], list_at[g + 1] - list_at[g]};
    }
}

/* row p of `out` (vec_stride bytes, zero padded) = the first `bytes` of caller row order[p] */
__global__ void listed_gather_queries_kernel(uint8_t const* queries, size_t stride, uint32_t const* order, uint32_t nq, uint32_t bytes,
                                             uint32_t vec_stride, uint8_t* out) {
    for (uint32_t p = blockIdx.x; p < nq; p += gridDim.x) {
        uint8_t const* src = queries + (size_t)order[p] * stride;
        uint8_t* dst = out + (size_t)p * vec_stride;
        for (uint32_t b = threadIdx.x; b < vec_stride; b += blockDim.x) dst[b] = b < bytes ? src[b] : (uint8_t)0;
    }
}

/* the merged rows, in set order, back to the caller's order; computed_distances = the length of the query's list */
__global__ void listed_scatter_kernel(uint32_t const* order, uint32_t const* sorted, uint32_t const* list_at, uint32_t nq, uint32_t k,
                                      uint64_t const* keys, float const* dists, uint32_t const* counts, uint64_t* out_keys, float* out_dists,
                                      uint32_t* out_counts, uint32_t* out_computed, uint32_t* out_visited) {
    for (uint32_t p = blockIdx.x; p < nq; p += gridDim.x) {
        uint32_t const i = order[p];
        for (uint32_t j = threadIdx.x; j < k; j += blockDim.x) {
            out_keys[(size_t)i * k + j] = keys[(size_t)p * k + j];
            out_dists[(size_t)i * k + j] = dists[(size_t)p * k + j];
        }
        if (threadIdx.x == 0) {
            out_counts[i] = counts[p];
            if (out_computed) out_computed[i] = list_at[sorted[p] + 1] - list_at[sorted[p]];
            if (out_visited) out_visited[i] = 0;
        }
    }
}

/* ---- exact excluded search ---- */

/* bucket[i] = the least b with 2^b >= min(k + e, cap), e = the live slots of query i's set: the count its scan runs at is
 * min(2^b, cap) */
__global__ void excluded_bucket_kernel(uint32_t const* groups, uint32_t const* list_at, uint32_t nq, uint64_t k, uint64_t cap, uint32_t* bucket) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += gridDim.x * blockDim.x) {
        uint32_t const g = groups[i];
        uint64_t const want = min(k + (list_at[g + 1] - list_at[g]), cap);
        uint32_t b = 0;
        while (b < 63 && (1ull << b) < want) ++b;
        bucket[i] = b;
    }
}

/* one warp per query of a bucket: row p of the unfiltered scan (`width` slots, ascending under the scan's order) keeps its
 * first k slots that are not in the query's sorted excluded list, as keys, in caller row order[p]; the rest of the row is
 * padded. computed_distances = the live entries less the excluded ones. */
__global__ void excluded_drop_kernel(uint32_t const* order, uint32_t const* groups, uint32_t const* list_at, uint32_t const* rows, uint32_t nq,
                                     uint32_t width, uint32_t k, uint64_t const* slots, float const* dists, uint32_t const* counts,
                                     uint64_t const* keys, uint32_t live, uint64_t* out_keys, float* out_dists, uint32_t* out_counts,
                                     uint32_t* out_computed, uint32_t* out_visited) {
    uint32_t const p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint32_t const lane = threadIdx.x & 31;
    if (p >= nq) return;
    uint32_t const i = order[p], g = groups[i];
    uint32_t const* const list = rows + list_at[g];
    uint32_t const e = list_at[g + 1] - list_at[g], n = counts[p];
    uint32_t* const out_bits = reinterpret_cast<uint32_t*>(out_dists) + (size_t)i * k;
    uint32_t kept = 0;
    for (uint32_t j0 = 0; j0 < n && kept < k; j0 += 32) {
        uint32_t const j = j0 + lane;
        uint32_t slot = 0;
        bool keep = false;
        if (j < n) {
            slot = (uint32_t)slots[(size_t)p * width + j];
            uint32_t const at = lower_bound(0, e, [&](uint32_t m) { return list[m] < slot; });
            keep = at == e || list[at] != slot;
        }
        uint32_t const ballot = __ballot_sync(0xFFFFFFFFu, keep);
        uint32_t const at = kept + __popc(ballot & ((1u << lane) - 1u));
        if (keep && at < k) {
            out_keys[(size_t)i * k + at] = keys[slot];
            out_bits[at] = reinterpret_cast<uint32_t const*>(dists)[(size_t)p * width + j];
        }
        kept += __popc(ballot);
    }
    kept = min(kept, k);
    for (uint32_t j = kept + lane; j < k; j += 32) {
        out_keys[(size_t)i * k + j] = 0;
        out_bits[j] = SNAN_BITS;
    }
    if (lane == 0) {
        out_counts[i] = kept;
        if (out_computed) out_computed[i] = live - e;
        if (out_visited) out_visited[i] = 0;
    }
}

/* ---- the three searches, past the shared checks: `sets.groups` is never NULL and the key table is current ---- */

/* graph: rows that allow the sets' slots, or (`excluded`) rows that allow every slot but them */
char const* rows_search(frozen_index_t& ix, void const* d_queries, size_t nq, size_t stride, size_t k, key_sets_t const& sets, bool excluded,
                        device_results_t const& out, cudaStream_t s) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    uint32_t const words = (uint32_t)((ix.size + 31) / 32);
    size_t const budget = (size_t)std::max(ix.tune.group_bitmap_mb, 0) << 20;
    size_t const per_round = std::min<size_t>(std::max<size_t>(budget / ((size_t)words * 4), 1), sets.count);
    size_t const rounds = (sets.count + per_round - 1) / per_round;
    if (char const* e = x.bits.reserve(per_round * words)) return e;

    launch_plan_t pl;
    if (char const* e = ix.plan((uint32_t)k, 0, pl, 0, true)) return e;
    int const wpb = search_warps_per_block();
    if (char const* e = ix.h_status.reserve(nq)) return e;
    if (char const* e = ix.status.reserve(nq)) return e;
    /* the retry of a round scans every query id: the words of the other rounds' queries must read STATUS_OK */
    CU(cudaMemsetAsync(ix.status.ptr, 0, nq * 4, s));
    if (ix.profile_phases)
        if (char const* e = ix.phase_cycles.reserve(PHASE_COUNTERS)) return e;

    /* the sets [g0, g1) into rows, then their queries: `items` work items, through `list` when it is not NULL */
    auto round = [&](uint32_t g0, uint32_t g1, uint32_t const* list, size_t items) -> char const* {
        /* allowed sets: rows of zeros that gain their slots; excluded sets: rows of ones that lose theirs */
        CU(cudaMemsetAsync(x.bits.ptr, excluded ? 0xFF : 0, (size_t)(g1 - g0) * words * 4, s));
        if (excluded)
            excluded_bits_kernel<<<ix.stream.sm_count * 16, 256, 0, s>>>(ix.key_table.cells.ptr, ix.key_table.mask, sets.offsets, sets.keys, g0,
                                                                         g1, words, x.bits.ptr);
        else
            grouped_bits_kernel<<<ix.stream.sm_count * 16, 256, 0, s>>>(ix.key_table.cells.ptr, ix.key_table.mask, sets.offsets, sets.keys, g0,
                                                                        g1, ix.free_key, ix.d.deleted_bits, (uint32_t)ix.size, words,
                                                                        x.bits.ptr);
        CU(cudaGetLastError());
        ix.kernel_launches += 1;
        int const blocks = (int)std::min<size_t>((size_t)pl.blocks, (items + wpb - 1) / wpb);
        search_args_t a;
        if (char const* e = ix.prepare_launch(pl, (size_t)blocks * wpb, a, s)) return e;
        a.queries = static_cast<uint8_t const*>(d_queries);
        a.query_stride = stride;
        a.nq = (uint32_t)items;
        a.query_list = list;
        a.k = (uint32_t)k;
        a.out_keys = out.keys;
        a.out_dists = out.dists;
        a.out_counts = out.counts;
        a.out_computed = out.computed;
        a.out_visited = out.visited;
        a.status = ix.status.ptr;
        a.allow_bits = x.bits.ptr;
        a.allow_groups = sets.groups;
        a.allow_group_base = g0;
        a.allow_words = words;
        if (ix.profile_phases) a.phase_cycles = ix.phase_cycles.ptr;
        CU(cudaMemsetAsync(ix.work_counter.ptr, 0, 8, s));
        CU(cudaEventRecord(ix.ev_begin, s));
        CU(search_launch(ix.d, a, blocks, pl.smem_per_block, s));
        CU(cudaEventRecord(ix.ev_end, s));
        ix.kernel_launches += 1;
        CU(cudaMemcpyAsync(ix.h_status.ptr, ix.status.ptr, nq * 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        CU(cudaEventElapsedTime(&ix.last_kernel_ms, ix.ev_begin, ix.ev_end));
        search_args_t every = a; /* the failed queries of this round, by query id */
        every.nq = (uint32_t)nq;
        return ix.retry_overflowed(every, pl.maxed, s);
    };
    if (rounds == 1) return round(0, (uint32_t)sets.count, nullptr, nq);

    /* query ids sorted by set: round r serves the contiguous slice of ids whose sets lie in its range */
    if (char const* e = x.bounds.reserve(rounds + 1)) return e;
    if (char const* e = sort_queries(ix, sets.groups, nq, bits_for(sets.count), s)) return e;
    round_bounds_kernel<<<(unsigned)((rounds + 1 + 255) / 256), 256, 0, s>>>(x.sorted.ptr, (uint32_t)nq, (uint32_t)per_round, (uint32_t)rounds,
                                                                             x.bounds.ptr);
    CU(cudaGetLastError());
    ix.kernel_launches += 3;
    std::vector<uint32_t> bounds(rounds + 1);
    CU(cudaMemcpyAsync(bounds.data(), x.bounds.ptr, (rounds + 1) * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    for (size_t r = 0; r < rounds; ++r) {
        if (bounds[r + 1] == bounds[r]) continue; /* no query asks for these sets */
        uint32_t const g0 = (uint32_t)(r * per_round), g1 = (uint32_t)std::min(sets.count, (r + 1) * per_round);
        if (char const* e = round(g0, g1, x.order.ptr + bounds[r], bounds[r + 1] - bounds[r])) return e;
    }
    return nullptr;
}

/* the slot-list build, step 1: the live slots of every entry, placed by an exclusive scan into x.entry_at (one extra zero
 * count: its place, entry_at[n_entries], is the cell total). Nothing waits. */
char const* listed_place_cells(frozen_index_t& ix, uint64_t const* set_keys, size_t n_entries, cudaStream_t s) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    size_t temp_bytes = 0;
    if (char const* e = x.entry_counts.reserve(n_entries + 1)) return e;
    if (char const* e = x.entry_at.reserve(n_entries + 1)) return e;
    if (char const* e = x.scalars.reserve(4)) return e;
    CU(cudaMemsetAsync(x.entry_counts.ptr + n_entries, 0, 8, s));
    if (n_entries)
        listed_count_kernel<<<grid_for(n_entries, ix.stream.sm_count), 256, 0, s>>>(ix.key_table.cells.ptr, ix.key_table.mask, set_keys,
                                                                                    n_entries, x.entry_counts.ptr);
    CU(cudaGetLastError());
    CU(cub::DeviceScan::ExclusiveSum(nullptr, temp_bytes, x.entry_counts.ptr, x.entry_at.ptr, (int)(n_entries + 1), s));
    if (char const* e = x.temp.reserve(std::max<size_t>(temp_bytes, 1))) return e;
    CU(cub::DeviceScan::ExclusiveSum(x.temp.ptr, temp_bytes, x.entry_counts.ptr, x.entry_at.ptr, (int)(n_entries + 1), s));
    return nullptr;
}

/* the slot-list build, step 2, once the host knows the cell total (at most INT_MAX): (set << 32 | slot) words, sorted over
 * the bits in use and deduplicated, leave set g's ascending, duplicate-free slots at x.rows[x.list_at[g] .. x.list_at[g + 1]) */
char const* listed_build_lists(frozen_index_t& ix, uint64_t const* offsets, uint32_t sets, uint64_t const* set_keys, size_t n_entries,
                               uint64_t cells, cudaStream_t s) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    auto temp_for = [&](size_t bytes) { return x.temp.reserve(std::max<size_t>(bytes, 1)); };
    size_t temp_bytes = 0;
    int const n_cells = (int)cells;
    int end_bit = 32;
    while (end_bit < 64 && ((uint64_t)(sets - 1) >> (end_bit - 32))) ++end_bit;
    if (char const* e = x.words.reserve(std::max<size_t>(cells, 1))) return e;
    if (char const* e = x.words_sorted.reserve(std::max<size_t>(cells, 1))) return e;
    if (char const* e = x.rows.reserve(std::max<size_t>(cells, 1))) return e;
    if (char const* e = x.list_at.reserve((size_t)sets + 1)) return e;
    CU(cudaMemsetAsync(x.scalars.ptr, 0, 16, s));
    if (n_cells) {
        listed_write_kernel<<<grid_for(n_entries, ix.stream.sm_count), 256, 0, s>>>(ix.key_table.cells.ptr, ix.key_table.mask, offsets, sets,
                                                                                    set_keys, n_entries, x.entry_at.ptr, x.words.ptr);
        CU(cudaGetLastError());
        CU(cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, x.words.ptr, x.words_sorted.ptr, n_cells, 0, end_bit, s));
        if (char const* e = temp_for(temp_bytes)) return e;
        CU(cub::DeviceRadixSort::SortKeys(x.temp.ptr, temp_bytes, x.words.ptr, x.words_sorted.ptr, n_cells, 0, end_bit, s));
        CU(cub::DeviceSelect::Unique(nullptr, temp_bytes, x.words_sorted.ptr, x.words.ptr, x.scalars.ptr, n_cells, s));
        if (char const* e = temp_for(temp_bytes)) return e;
        CU(cub::DeviceSelect::Unique(x.temp.ptr, temp_bytes, x.words_sorted.ptr, x.words.ptr, x.scalars.ptr, n_cells, s));
        ix.kernel_launches += 3;
    }
    listed_rows_kernel<<<grid_for(std::max<size_t>(cells, (size_t)sets + 1), ix.stream.sm_count), 256, 0, s>>>(
        x.words.ptr, x.scalars.ptr, (uint32_t)cells, sets, x.rows.ptr, x.list_at.ptr);
    CU(cudaGetLastError());
    return nullptr;
}

/* exact, allowed sets: search_exact_ over the live slots of each query's set, `entries` keys in all the sets, `qpc` queries
 * per work item of the LISTED kernel */
char const* listed_exact_search(frozen_index_t& ix, void const* d_queries, size_t nq, size_t stride, size_t k, key_sets_t const& sets,
                                uint64_t entries, uint32_t qpc, device_results_t const& out, cudaStream_t s) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    uint32_t const n_sets = (uint32_t)sets.count;
    size_t const n_entries = (size_t)entries;
    auto temp_for = [&](size_t bytes) { return x.temp.reserve(std::max<size_t>(bytes, 1)); };
    size_t temp_bytes = 0;

    /* 1. the live slots of every entry, placed by an exclusive scan */
    if (char const* e = listed_place_cells(ix, sets.keys, n_entries, s)) return e;
    /* 2. the queries sorted by set, cut into work items of at most qpc queries that never mix sets (counted here, written
     * once the lists are placed) */
    if (char const* e = x.query_at.reserve(sets.count + 1)) return e;
    if (char const* e = x.per_set.reserve(sets.count + 1)) return e;
    if (char const* e = x.item_at.reserve(sets.count + 1)) return e;
    if (char const* e = x.items.reserve(nq)) return e;
    if (char const* e = sort_queries(ix, sets.groups, nq, bits_for(sets.count), s)) return e;
    listed_item_counts_kernel<<<grid_for(sets.count + 1, ix.stream.sm_count), 256, 0, s>>>(x.sorted.ptr, (uint32_t)nq, n_sets, qpc,
                                                                                           x.query_at.ptr, x.per_set.ptr);
    CU(cudaGetLastError());
    CU(cub::DeviceScan::ExclusiveSum(nullptr, temp_bytes, x.per_set.ptr, x.item_at.ptr, (int)(sets.count + 1), s));
    if (char const* e = temp_for(temp_bytes)) return e;
    CU(cub::DeviceScan::ExclusiveSum(x.temp.ptr, temp_bytes, x.per_set.ptr, x.item_at.ptr, (int)(sets.count + 1), s));
    /* one read-back: the cell total sizes the lists and the item count the grid. The total is an exact 64-bit sum (the
     * counts are 64-bit), so a multi index whose sets name more than INT_MAX cells is refused here, before the sort (whose
     * item count is an int) or any write to the lists. */
    uint64_t cells = 0;
    uint32_t n_items = 0;
    CU(cudaMemcpyAsync(&cells, x.entry_at.ptr + n_entries, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&n_items, x.item_at.ptr + sets.count, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (cells > 0x7FFFFFFFull) return "Too many listed rows in one call";

    /* 3. (set << 32 | slot) words, sorted over the bits in use and deduplicated: per-set ascending slot lists */
    if (char const* e = listed_build_lists(ix, sets.offsets, n_sets, sets.keys, n_entries, cells, s)) return e;

    listed_items_kernel<<<grid_for(sets.count, ix.stream.sm_count), 256, 0, s>>>(x.query_at.ptr, x.item_at.ptr, x.list_at.ptr, n_sets, qpc,
                                                                                 x.items.ptr);
    CU(cudaGetLastError());
    ix.kernel_launches += 8;

    /* 4. the gathered batch through the listed scans and the unchanged merge, then back to the caller's order */
    size_t const vs = ix.d.vec_stride;
    if (char const* e = x.queries.reserve(nq * vs)) return e;
    if (char const* e = x.keys.reserve(nq * k)) return e;
    if (char const* e = x.dists.reserve(nq * k)) return e;
    if (char const* e = x.counts.reserve(nq)) return e;
    listed_gather_queries_kernel<<<(unsigned)std::min<size_t>(nq, 65535), 128, 0, s>>>(static_cast<uint8_t const*>(d_queries), stride,
                                                                                       x.order.ptr, (uint32_t)nq, (uint32_t)ix.d.bytes_per_vector,
                                                                                       (uint32_t)vs, x.queries.ptr);
    CU(cudaGetLastError());
    exact_listed_t listed;
    listed.items = x.items.ptr;
    listed.n_items = n_items;
    listed.rows = x.rows.ptr;
    listed.total_rows = (uint32_t)cells; /* the lists' rows, duplicates still counted: the planner's bound */
    CU(cudaEventRecord(ix.ev_begin, s));
    if (char const* e = exact_listed_search_device(ix.d, ix.stream.sm_count, x.queries.ptr, nq, k, listed, x.keys.ptr, x.dists.ptr,
                                                   x.counts.ptr, x.exact, s))
        return e;
    CU(cudaEventRecord(ix.ev_end, s));
    listed_scatter_kernel<<<(unsigned)std::min<size_t>(nq, 65535), 128, 0, s>>>(x.order.ptr, x.sorted.ptr, x.list_at.ptr, (uint32_t)nq,
                                                                                (uint32_t)k, x.keys.ptr, x.dists.ptr, x.counts.ptr, out.keys,
                                                                                out.dists, out.counts, out.computed, out.visited);
    CU(cudaGetLastError());
    ix.kernel_launches += 4;
    CU(cudaStreamSynchronize(s));
    CU(cudaEventElapsedTime(&ix.last_kernel_ms, ix.ev_begin, ix.ev_end));
    return nullptr;
}

/* exact, excluded sets: search_exact_ over the live slots outside each query's set. The scan order (distance ascending,
 * slot descending) is total, so the k best entries outside a set of e live slots are what remains of the unfiltered
 * top-(k + e) once the set's slots are dropped. The sets become slot lists (the exact filtered search's build); the
 * queries are bucketed by k + e rounded up to a power of two, and each bucket runs the unfiltered scan once at its count,
 * with slots for keys, then the drop. */
char const* excluded_exact_search(frozen_index_t& ix, void const* d_queries, size_t nq, size_t stride, size_t k, key_sets_t const& sets,
                                  uint64_t entries, device_results_t const& out, cudaStream_t s) {
    frozen_index_t::key_set_scratch_t& x = ix.key_set_scratch;
    size_t const n_entries = (size_t)entries;

    /* 1. the sets' live slots as sorted lists */
    if (char const* e = listed_place_cells(ix, sets.keys, n_entries, s)) return e;
    uint64_t cells = 0;
    CU(cudaMemcpyAsync(&cells, x.entry_at.ptr + n_entries, 8, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (cells > 0x7FFFFFFFull) return "Too many listed rows in one call";
    if (char const* e = listed_build_lists(ix, sets.offsets, (uint32_t)sets.count, sets.keys, n_entries, cells, s)) return e;

    /* 2. the queries bucketed by the count their scan needs, in query order within a bucket (the sort is stable). No count
     * past max(k, live) is needed: that many rows hold every live entry. */
    uint64_t const live = ix.size - ix.count_deleted, cap = std::max<uint64_t>(k, live);
    int constexpr BUCKETS = 64;
    if (char const* e = x.buckets.reserve(nq)) return e;
    if (char const* e = x.bounds.reserve(BUCKETS + 1)) return e;
    excluded_bucket_kernel<<<grid_for(nq, ix.stream.sm_count), 256, 0, s>>>(sets.groups, x.list_at.ptr, (uint32_t)nq, k, cap, x.buckets.ptr);
    CU(cudaGetLastError());
    if (char const* e = sort_queries(ix, x.buckets.ptr, nq, 6, s)) return e;
    round_bounds_kernel<<<1, 256, 0, s>>>(x.sorted.ptr, (uint32_t)nq, 1, BUCKETS, x.bounds.ptr);
    CU(cudaGetLastError());
    ix.kernel_launches += 4;
    std::vector<uint32_t> at(BUCKETS + 1);
    CU(cudaMemcpyAsync(at.data(), x.bounds.ptr, (BUCKETS + 1) * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    auto count_of = [&](int b) { return std::min<uint64_t>(1ull << b, cap); };
    uint64_t widest = 0;
    size_t rows = 0;
    for (int b = 0; b < BUCKETS; ++b)
        if (at[b + 1] > at[b]) {
            widest = count_of(b);
            rows = std::max<size_t>(rows, (size_t)(at[b + 1] - at[b]) * widest);
        }
    /* count > 256 past the tiled stage is refused here, before any output is written */
    if (char const* e = exact_search_check(ix.d, widest)) return e;

    /* 3. the batch gathered in bucket order; per bucket the unfiltered scan at its count, then the drop into caller order */
    size_t const vs = ix.d.vec_stride;
    if (char const* e = x.queries.reserve(nq * vs)) return e;
    if (char const* e = x.keys.reserve(rows)) return e;
    if (char const* e = x.dists.reserve(rows)) return e;
    if (char const* e = x.counts.reserve(nq)) return e;
    listed_gather_queries_kernel<<<(unsigned)std::min<size_t>(nq, 65535), 128, 0, s>>>(static_cast<uint8_t const*>(d_queries), stride,
                                                                                       x.order.ptr, (uint32_t)nq, (uint32_t)ix.d.bytes_per_vector,
                                                                                       (uint32_t)vs, x.queries.ptr);
    CU(cudaGetLastError());
    ix.kernel_launches += 1;
    CU(cudaEventRecord(ix.ev_begin, s));
    for (int b = 0; b < BUCKETS; ++b) {
        uint32_t const q0 = at[b], n_b = at[b + 1] - at[b];
        if (!n_b) continue;
        uint64_t const width = count_of(b);
        if (char const* e = exact_search_device(ix.d, ix.stream.sm_count, x.queries.ptr + (size_t)q0 * vs, n_b, vs, width, false, true,
                                                x.keys.ptr, x.dists.ptr, x.counts.ptr, x.exact, s))
            return e;
        excluded_drop_kernel<<<(n_b + 7) / 8, 256, 0, s>>>(x.order.ptr + q0, sets.groups, x.list_at.ptr, x.rows.ptr, n_b, (uint32_t)width,
                                                           (uint32_t)k, x.keys.ptr, x.dists.ptr, x.counts.ptr, ix.d.keys, (uint32_t)live,
                                                           out.keys, out.dists, out.counts, out.computed, out.visited);
        CU(cudaGetLastError());
        ix.kernel_launches += 3;
    }
    CU(cudaEventRecord(ix.ev_end, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaEventElapsedTime(&ix.last_kernel_ms, ix.ev_begin, ix.ev_end));
    return nullptr;
}

} // namespace

size_t frozen_index_t::key_set_scratch_t::bytes() const {
    return bits.capacity * 4 + flag.capacity * 4 + groups.capacity * 4 + offsets.capacity * 8 + ids.capacity * 4 + order.capacity * 4 +
           sorted.capacity * 4 + bounds.capacity * 4 + temp.capacity + entry_counts.capacity * 8 + entry_at.capacity * 8 +
           words.capacity * 8 + words_sorted.capacity * 8 + rows.capacity * 4 + list_at.capacity * 4 + query_at.capacity * 4 +
           per_set.capacity * 4 + item_at.capacity * 4 + items.capacity * sizeof(exact_item_t) + scalars.capacity * 4 +
           buckets.capacity * 4 + queries.capacity + keys.capacity * 8 + dists.capacity * 4 + counts.capacity * 4 + exact.capacity;
}

char const* frozen_index_t::key_set_search_device(void const* d_queries, size_t nq, size_t stride, size_t k, key_sets_t const& sets,
                                                  bool excluded, bool exact, device_results_t const& out, cudaStream_t s) {
    if (shards) return ERR_SHARDED;
    if (char const* e = ensure_context()) return e;
    if (nq == 0 || k == 0) return nullptr;
    if (nq > 0x7FFFFFFFull) return "Too many queries in one batch";
    uint64_t entries = 0;
    if (char const* e = check_key_sets_device(*this, sets, nq, rules_of(excluded, exact), &entries, s)) return e;
    if (!loaded || d.n == 0) { /* no matches, no error (index.hpp:3036-3037) */
        CU(search_fill_empty(out.keys, out.dists, out.counts, out.computed, out.visited, nq, k, s));
        CU(cudaStreamSynchronize(s));
        return nullptr;
    }
    /* the exact forms' refusals at this count, before the key table is built */
    uint32_t qpc = 0;
    if (exact)
        if (char const* e = excluded ? exact_search_check(d, k) : exact_listed_queries_per_item(d, k, &qpc)) return e;
    key_sets_t in = sets;
    if (!in.groups) { /* one set: every query uses set 0 */
        if (char const* e = key_set_scratch.groups.reserve(nq)) return e;
        CU(cudaMemsetAsync(key_set_scratch.groups.ptr, 0, nq * 4, s));
        in.groups = key_set_scratch.groups.ptr;
    }
    if (char const* e = ensure_key_table(s)) return e;
    if (!exact) return rows_search(*this, d_queries, nq, stride, k, in, excluded, out, s);
    if (!excluded) return listed_exact_search(*this, d_queries, nq, stride, k, in, entries, qpc, out, s);
    return excluded_exact_search(*this, d_queries, nq, stride, k, in, entries, out, s);
}

/* host queries of any kind, host sets and host outputs: the sets checked here, then uploaded and run through the device path */
char const* frozen_index_t::key_set_search_host(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                                                key_sets_t const& sets, bool excluded, bool exact, host_results_t const& out, size_t* total) {
    std::lock_guard<std::mutex> lock(mutex);
    if (shards) return ERR_SHARDED;
    if (nq == 0 || k == 0) return nullptr;
    if (char const* e = check_key_sets_host(sets, nq, rules_of(excluded, exact))) return e;
    if (!loaded || d.n == 0) return answer_empty(nq, k, out);
    return search_round_trip(q, nq, stride, query_scalar, k, out, total,
                             [&](void const* dq, size_t vs, device_results_t const& r) -> char const* {
        if (char const* e = upload_key_sets(*this, sets, nq)) return e;
        key_sets_t const uploaded{sets.groups ? key_set_scratch.groups.ptr : nullptr, key_set_scratch.offsets.ptr, sets.count, key_stage.ptr};
        return key_set_search_device(dq, nq, vs, k, uploaded, excluded, exact, r, stream);
    });
}

} // namespace usearch_b200
