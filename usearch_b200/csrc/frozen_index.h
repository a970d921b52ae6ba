/*
 *  frozen_index.h — host-side owner of one HNSW index frozen into HBM, plus the scratch, streams
 *  and staging buffers its searches use. This is the object behind the opaque `usearch_index_t`
 *  of include/usearch_b200.h; it plays the role `index_dense_gt` plays behind the reference's
 *  handle (c/lib.cpp:136-182) for the search path only.
 */
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "cuda_buffers.h"
#include "device_index.h"
#include "device_keys.h"
#include "key_map.h"

namespace usearch_b200 {

struct exact_item_t; /* exact_args.h: one CTA row of a listed exact scan */

/* kernel entry points (search_kernel.cu) */
cudaError_t search_launch(device_index_t const& ix, search_args_t const& a, int blocks, size_t smem, cudaStream_t stream);
cudaError_t search_occupancy(device_index_t const& ix, int* blocks_per_sm, size_t smem, bool grouped = false);
bool search_supported(uint32_t metric, uint32_t scalar);
int search_warps_per_block();
bool search_is_staged(device_index_t const& ix);
int search_stage_slots(device_index_t const& ix);
int search_lanes_per_vector(device_index_t const& ix);
uint32_t search_stage_pad(device_index_t const& ix);
int search_max_warps_per_sm(device_index_t const& ix);
bool search_single_stage_set(device_index_t const& ix);
bool search_needs_norms(uint32_t metric, uint32_t scalar);
/* `slots` (optional, ix.n entries): recompute only those rows of the full arrays instead of rows 0 .. ix.n-1 */
cudaError_t search_compute_norms(device_index_t const& ix, float* norms, cudaStream_t stream, uint32_t const* slots = nullptr);
bool search_needs_shadow(device_index_t const& ix);
uint32_t search_code_stride(device_index_t const& ix);
cudaError_t search_compute_shadow(device_index_t const& ix, float const* norms, int8_t* codes, pf_record_t* records,
                                  cudaStream_t stream, uint32_t const* slots = nullptr);
cudaError_t search_fill_empty(uint64_t* keys, float* dists, uint32_t* counts, uint32_t* computed, uint32_t* visited, size_t nq,
                              size_t k, cudaStream_t stream);
cudaError_t search_build_allow_bits(device_index_t const& ix, uint64_t const* allowed_sorted, uint32_t m, uint32_t* bits,
                                    cudaStream_t stream);

/* `visits` is a per-warp bitmap whenever all the bitmaps fit this budget (else an open-addressing table);
 * bitmaps above BITMAP_WIPE_MAX_SLOTS are cleaned through a log of the bits each query set */
constexpr uint64_t BITMAP_SCRATCH_BUDGET = 12ull << 30;
constexpr uint64_t BITMAP_WIPE_MAX_SLOTS = 1ull << 20;

struct launch_plan_t {
    uint32_t ef = 0;
    uint32_t visited_cap = 0, visited_bitmap_words = 0, visit_log_cap = 0, heap_spill_cap = 0, heap_smem_cap = 0;
    bool maxed = false; /* growing the scratch any further cannot help */
    size_t visited_words_per_warp() const { return visited_bitmap_words ? visited_bitmap_words : visited_cap; }
    uint32_t smem_per_warp = 0, off_top_d = 0, off_top_s = 0, off_cand_s = 0, off_cand_d = 0, off_heap = 0;
    uint32_t off_bars = 0, off_stage = 0, stage_stride = 0, stage_sets = 1;
    uint32_t off_surv_b2 = 0, code_pass = 0, code_smem_stride = 0; /* prefilter */
    uint32_t off_qsplit = 0, qsplit_len = 0;
    bool prefilter = false; /* the layout above has room for the prefilter and the knobs let it run */
    int blocks = 0;
    uint32_t warps_per_sm_target = 0;
    size_t smem_per_block = 0;
    size_t warps() const { return (size_t)blocks * (size_t)search_warps_per_block(); }
};

/* device scratch of the batched builder (builder.cu) */
struct build_scratch_t {
    device_buffer_t<uint32_t> task_slot, cand_slots, cand_counts, pair_idx, pair_idx_sorted, heads, counters;
    device_buffer_t<uint8_t> task_level, sort_temp;
    device_buffer_t<float> cand_dists, pair_dists;
    device_buffer_t<uint64_t> pair_keys, pair_keys_sorted;
    size_t iota_count = 0;
};

struct shard_group_t; /* shards.cu */

/* what search_device filters by: a bitmap over slots (filtered search), the last level of the greedy descent (cluster) */
struct search_filter_t {
    uint32_t const* allow_bits = nullptr;
    int cluster_end_level = -1;
};

/* the host outputs of one search batch: rows of k keys / distances `keys_stride` / `dists_stride` bytes apart; counts,
 * computed and visited (one per query) may be NULL */
struct host_results_t {
    uint64_t* keys;
    size_t keys_stride;
    float* dists;
    size_t dists_stride;
    size_t* counts = nullptr;
    uint64_t* computed = nullptr;
    uint64_t* visited = nullptr;
};
/* the dense device outputs search_round_trip hands its device call; computed / visited are NULL unless the host caller
 * asked for them */
struct device_results_t {
    uint64_t* keys;
    float* dists;
    uint32_t* counts;
    uint32_t* computed;
    uint32_t* visited;
};
/* the key sets of a key-set search, as CSR: set g holds keys[offsets[g] .. offsets[g + 1]), query i uses set groups[i].
 * `groups` may be NULL with one set (every query uses set 0) except in the allowed graph form. */
struct key_sets_t {
    uint32_t const* groups;
    uint64_t const* offsets; /* count + 1 */
    size_t count;
    uint64_t const* keys;
};
/* the device call of a host search: queries in the index's kind, rows `stride` bytes apart, outputs in `out` */
using device_search_t = std::function<char const*(void const* d_queries, size_t stride, device_results_t const& out)>;
/* index_gt::search on an empty index: no matches, no error (index.hpp:3036-3037); every row key 0 and a signalling NaN */
char const* answer_empty(size_t nq, size_t k, host_results_t const& out);

struct frozen_index_t {
    /* configuration (usearch_init_options_t) */
    uint32_t metric = 0, scalar = 0; /* reference char codes */
    size_t dimensions = 0, connectivity = 0, connectivity_base = 0;
    size_t expansion_add = 128, expansion_search = 64; /* index.hpp:1340-1350 defaults */
    bool multi = false;
    uint64_t free_key = UINT64_MAX; /* index_dense.hpp:513 */

    /* population */
    size_t size = 0, count_deleted = 0;
    std::vector<int16_t> levels;     /* kept on the host: re-serialisation and the builder's work lists */
    std::vector<uint64_t> host_keys; /* host copy of `keys` (slot -> key): lookups by key never touch the device */
    key_map_t key_map;
    /* removed slots awaiting reuse, oldest first: the reference's `free_keys_` ring (index.hpp:1308-1330) pushes at the
     * head and pops from the tail. `remove` appends in removal order; a load refills it in ascending slot order. */
    std::deque<uint32_t> free_slots;
    bool reuse_removed = false; /* add() fills `free_slots` before appending (off: every add appends, as before) */
    size_t capacity = 0;                      /* slots the HBM arrays have room for */
    size_t upper_capacity = 0, upper_rows = 0; /* rows of `upper`: allocated / in use */
    uint64_t level_seed = 0;
    bool configured() const { return metric && scalar && dimensions && connectivity; }
    void build_key_map() { if (!key_map.built) key_map.rebuild(host_keys, free_key, capacity); }
    /* bumped by every call that can change the key -> slot relation (add, remove, rename, clear, load): a device key
     * table built at another generation is stale */
    uint64_t keys_generation = 0;

    /* device */
    cuda_stream_t stream; /* the handle's device (`stream.device`), its SM count and the handle's own stream */
    device_index_t d;     /* views of the arrays in `hbm` */
    size_t hbm_bytes = 0;
    bool loaded = false;
    struct hbm_arrays_t {
        device_buffer_t<uint8_t> vectors;
        device_buffer_t<uint64_t> keys;
        device_buffer_t<uint32_t> nbr0, upper_base, upper, deleted_bits;
        device_buffer_t<float> norms;
        device_buffer_t<int8_t> codes;
        device_buffer_t<pf_record_t> shadow;
    } hbm;

    /* tuning knobs of the search launch: environment at construction (USEARCH_B200_STAGE_SETS, _WARPS_PER_SM,
     * _PREFILTER, _HEAP_HEAD), changeable per handle with usearch_b200_tune (bench sweeps, tests) */
    struct tune_t {
        int stage_sets = env_int("USEARCH_B200_STAGE_SETS", 0);     /* 0 = planned, 1 or 2 = forced */
        int warps_per_sm = env_int("USEARCH_B200_WARPS_PER_SM", 0); /* 0 = as many as fit, else an upper bound */
        int prefilter = env_int("USEARCH_B200_PREFILTER", 1);       /* 0 = measure every layer-0 candidate exactly */
        int heap_head = env_int("USEARCH_B200_HEAP_HEAD", 0);       /* 0 = as planned, else an upper bound on the heap
                                                                       entries kept in shared memory (even, >= 2) */
        int get_chunk_rows = env_int("USEARCH_B200_GET_CHUNK_ROWS", 0); /* rows per chunk of get_many; 0 = 64 MB of output */
        int group_bitmap_mb = env_int("USEARCH_B200_GROUP_BITMAP_MB", 1024); /* grouped filtered search: bitmap rows per
                                                                               round fill at most this many MB (at least one row) */
        static int env_int(char const* name, int fallback) {
            char const* v = std::getenv(name);
            return v ? std::atoi(v) : fallback;
        }
    } tune;

    /* per-handle execution context */
    std::mutex mutex;
    cuda_event_t ev_begin, ev_end;
    device_buffer_t<uint32_t> visited, visit_log, work_counter, status, counts, computed, cycles, retry_list;
    size_t visited_zeroed_words = 0; /* the first this-many words of `visited` are known to be zero (logged bitmaps) */
    device_buffer_t<cand_t> heap_spill;
    device_buffer_t<uint8_t> queries;
    device_buffer_t<uint64_t> allowed_keys; /* filtered search: sorted allowed keys and the bitmap built from them */
    device_buffer_t<uint32_t> allow_bits;
    device_buffer_t<uint64_t> key_stage; /* the keys of a host entry (allowed keys, set keys), uploaded as given */
    device_buffer_t<uint64_t> out_keys;
    device_buffer_t<float> out_dists;
    pinned_buffer_t<uint8_t> h_queries;
    pinned_buffer_t<uint64_t> h_keys;
    pinned_buffer_t<float> h_dists;
    pinned_buffer_t<uint32_t> h_counts, h_computed, h_cycles, h_status;
    device_buffer_t<unsigned long long> phase_cycles; /* introspection, enabled by usearch_b200_profile_phases */
    bool profile_phases = false;
    uint64_t kernel_launches = 0;
    float last_kernel_ms = 0.f;

    ~frozen_index_t() { leave_shards(); } /* the NCCL communicator before the stream and buffers it uses */
    void release_device();
    char const* ensure_context();
    char const* counts_reserve_all(size_t nq);

    /* v2 blob -> HBM (index_dense.hpp:1084-1188, index.hpp:3322-3382) */
    char const* load_blob(uint8_t const* blob, size_t length);
    size_t serialized_length() const;
    char const* save_blob(uint8_t* out, size_t length) const;

    /* mutation (builder.cu): GPU-assisted add, capacity, tombstones */
    build_scratch_t build;
    device_buffer_t<uint8_t> cast_stage; /* raw caller rows awaiting a scalar cast on the device */
    char const* reserve_slots(size_t slots);
    char const* reserve_upper_rows(size_t rows);
    int16_t draw_level(size_t slot) const;
    char const* add_many(uint64_t const* keys, void const* vectors, size_t count, size_t stride, uint32_t scalar_kind, bool on_device);
    char const* link_batch(uint32_t const* slots, size_t count);
    /* remove / reuse: the slots of one call and the keys they take, uploaded once; reused rows staged before the scatter */
    device_buffer_t<uint32_t> edit_slots;
    device_buffer_t<uint64_t> edit_keys;
    device_buffer_t<uint8_t> reuse_stage;
    device_buffer_t<unsigned long long> pruned_counter;
    char const* write_rows(void const* vectors, size_t rows, size_t stride, uint32_t kind, bool on_device, uint8_t* dst);
    char const* set_slot_keys(uint32_t const* slots, size_t count, uint64_t const* keys);
    char const* remove_many(uint64_t const* keys, size_t count, bool compact, size_t* removed, size_t* pruned);
    char const* isolate(size_t* pruned);
    char const* rename_key(uint64_t from, uint64_t to, size_t* renamed);
    char const* get_vectors(uint64_t key, size_t max_count, void* out, uint32_t out_scalar, size_t* found);

    /* surface.cu: reading the index back out */
    char const* get_many(uint64_t const* keys, size_t n, size_t max_per_key, void* out, size_t out_stride, uint32_t out_scalar,
                         size_t* counts, size_t* rows);
    size_t export_keys(size_t offset, size_t limit, uint64_t* out) const;
    char const* export_keys_at(size_t const* offsets, size_t n, uint64_t* out) const;
    char const* copy_into(frozen_index_t& copy);
    char const* graph_levels(std::vector<uint64_t>& nodes, std::vector<uint64_t>& edges);

    /* join.cu: the reference's stable-marriage `join` of this index (a) with `other` (b), replayed as its one-thread run.
     * Pairs (a key, b key) come out in the reference's export order; stats as join_result_t. */
    char const* join(frozen_index_t& other, size_t max_proposals, bool exact, std::vector<uint64_t>& a_keys,
                     std::vector<uint64_t>& b_keys, size_t stats[4]);
    float last_join_ms[3] = {0.f, 0.f, 0.f}; /* wall clock of the last join called on this handle: search | pairs | replay */
    /* distance_between(left[i], right[i]).min for every i; a missing key gives FLT_MAX */
    char const* pairwise_distances(uint64_t const* left, uint64_t const* right, size_t n, float* out);

    /* sharded search (shards.cu): this handle is shard `rank` of `world`, one process per GPU */
    shard_group_t* shards = nullptr;
    char const* join_shards(int rank, int world, void const* unique_id128);
    void leave_shards();
    char const* sharded_search_device(void const* d_queries, size_t nq, size_t stride, size_t k, uint64_t* d_keys, float* d_dists,
                                      uint32_t* d_counts, uint32_t* d_computed, uint32_t* d_cycles, cudaStream_t stream);
    char const* sharded_search_host(void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                                    host_results_t const& out, size_t* total);

    /* device_keys.cu: lookups by key from device memory, through a key -> slot table in HBM built on first use */
    struct key_table_t {
        device_buffer_t<key_cell_t> cells;
        uint64_t mask = 0, generation = 0;
    } key_table;
    device_buffer_t<uint32_t> lookup_slots; /* get_many_device: the slot of every output row */
    device_buffer_t<uint8_t> lookup_gathered, lookup_casted, allowed_sort_temp;
    char const* ensure_key_table(cudaStream_t s);
    char const* count_many_device(uint64_t const* keys, size_t n, uint32_t* counts, cudaStream_t s);
    char const* get_many_device(uint64_t const* keys, size_t n, size_t max_per_key, void* out, size_t out_stride, uint32_t out_scalar,
                                uint32_t* counts, cudaStream_t s);
    char const* filtered_search_device(void const* d_queries, size_t nq, size_t stride, size_t k, uint64_t const* allowed,
                                       size_t allowed_count, uint64_t* d_keys, float* d_dists, uint32_t* d_counts, uint32_t* d_computed,
                                       uint32_t* d_visited, cudaStream_t s);
    char const* filtered_search_host(void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t k, uint64_t const* allowed,
                                     size_t allowed_count, host_results_t const& out, size_t* total);

    /* grouped_filter.cu: key-set searches, each query under its own set of a CSR list (key_sets_t). Query i searches the
     * live entries whose key is in set groups[i], or (`excluded`) whose key is not, through the graph or (`exact`) by brute
     * force: one bitmap row per set from the key table for the graph, one slot list per set for the exact forms. */
    struct key_set_scratch_t {
        device_buffer_t<uint32_t> bits;           /* graph: the rows of one round, as many as `group_bitmap_mb` allows */
        device_buffer_t<uint32_t> flag, groups;   /* the device checks' flag; `groups` of a host entry, or zeros for one set */
        device_buffer_t<uint64_t> offsets;        /* a host entry's `offsets` (its keys go to `key_stage`) */
        device_buffer_t<uint32_t> ids, order, sorted, bounds; /* query ids sorted by set or bucket, and the bounds of the runs */
        device_buffer_t<uint8_t> temp;            /* cub's */
        device_buffer_t<uint32_t> rows, list_at, query_at, per_set, item_at, scalars, counts, buckets; /* exact: slot lists, items */
        device_buffer_t<uint64_t> entry_counts, entry_at, words, words_sorted, keys;
        device_buffer_t<exact_item_t> items;
        device_buffer_t<uint8_t> queries, exact;
        device_buffer_t<float> dists;
        size_t bytes() const;
    } key_set_scratch; /* all of it counted by memory_usage and freed by clear */
    char const* key_set_search_device(void const* d_queries, size_t nq, size_t stride, size_t k, key_sets_t const& sets, bool excluded,
                                      bool exact, device_results_t const& out, cudaStream_t s);
    /* the same from host queries of any kind, host sets and host outputs */
    char const* key_set_search_host(void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t k, key_sets_t const& sets,
                                    bool excluded, bool exact, host_results_t const& out, size_t* total);

    /* searches */
    /* grouped: plan for the GROUPED kernel (its occupancy) */
    char const* plan(uint32_t k, uint32_t visited_cap_override, launch_plan_t& plan, uint32_t ef_override = 0,
                     bool grouped = false) const;
    char const* prepare_launch(launch_plan_t const& pl, size_t warps, search_args_t& a, cudaStream_t s);
    char const* search_device(void const* d_queries, size_t nq, size_t stride, size_t k, uint64_t* d_keys, float* d_dists,
                              uint32_t* d_counts, uint32_t* d_computed, uint32_t* d_cycles, cudaStream_t stream, bool defer = false,
                              search_filter_t const& filter = {});
    /* deferred launches (usearch_b200_search_many_enqueue): status words and arguments kept until search_finish */
    struct pending_search_t { uint32_t* status; search_args_t args; bool maxed; cudaStream_t stream; };
    std::vector<pending_search_t> pending;
    std::vector<device_buffer_t<uint32_t>> pending_status; /* pending[i] writes to pending_status[i]; the rest are free */
    char const* search_finish();
    char const* retry_overflowed(search_args_t const& a, bool maxed, cudaStream_t stream);
    /* usearch_search from many host threads: callers that arrive while a launch is in flight are gathered and served by
     * ONE launch (a leader runs the batch, the others wait for their rows) — the reference serves them from distinct
     * thread contexts in parallel (index.hpp:3033-3039, index_dense.hpp:1984-2000) */
    struct single_request_t {
        void const* query; uint32_t scalar; size_t count; uint64_t* keys; float* dists; size_t found; char const* error; bool done;
    };
    std::mutex gather_mutex;
    std::condition_variable gather_cv;
    std::vector<single_request_t*> gather_queue;
    bool gather_leader = false;
    uint64_t gathered_batches = 0, gathered_queries = 0;
    char const* search_single(void const* query, uint32_t query_scalar, size_t count, uint64_t* keys, float* dists, size_t* found);
    char const* upload_queries(void const* queries, size_t nq, size_t stride, uint32_t query_scalar);
    char const* stage_keys(uint64_t const* keys, size_t n);
    /* every host search entry, once it has its lock and its checks passed on a non-empty index: the queries up, `search`
     * on the device, the rows down into `out`; *total = the sum of counts */
    char const* search_round_trip(void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                                  host_results_t const& out, size_t* total, device_search_t const& search);
    device_buffer_t<uint8_t> exact_scratch;
    char const* exact_host(void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t k, host_results_t const& out,
                           size_t* total);
    char const* search_host(void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t k, host_results_t const& out,
                            size_t* total);
    char const* cluster_host(void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t level, uint64_t* keys,
                             float* dists, uint64_t* computed, uint64_t* visited);
};

/* exact_kernel.cu */
char const* exact_search_device(device_index_t const& ix, int sm_count, void const* d_queries, size_t nq, size_t query_stride, size_t k,
                                bool swap, bool slots_as_keys, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                                device_buffer_t<uint8_t>& scratch, cudaStream_t stream);
/* exact filtered search (grouped_filter.cu): `n_items` CTA rows of queries sorted by set, each against its set's slot list
 * (exact_item_t, exact_args.h), over `total_rows` listed slots; the queries are gathered into rows of vec_stride bytes */
struct exact_listed_t {
    exact_item_t const* items = nullptr;
    uint32_t n_items = 0;
    uint32_t const* rows = nullptr;
    uint32_t total_rows = 0;
    uint32_t qpc = 0; /* queries per item of the kernel chosen for (ix, k) */
};
char const* exact_listed_queries_per_item(device_index_t const& ix, size_t k, uint32_t* qpc);
char const* exact_listed_search_device(device_index_t const& ix, int sm_count, void const* d_queries, size_t nq, size_t k,
                                       exact_listed_t const& listed, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                                       device_buffer_t<uint8_t>& scratch, cudaStream_t stream);
/* one chunk of a free search (exact_free.cu): metric(row, query), keys are dataset rows `row_offset + chunk row`; with `carry`
 * the outputs already hold the merged top-k of the chunks before and are merged with this one */
char const* exact_search_chunk_device(device_index_t const& chunk, int sm_count, void const* d_queries, size_t nq, size_t query_stride,
                                      size_t k, uint32_t row_offset, bool carry, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                                      stream_buffer_t<uint8_t>& scratch, cudaStream_t stream);
/* the refusals exact_search_device would return for this shape (metric, scalar kind, row length) and count, nothing launched */
char const* exact_search_check(device_index_t const& shape, size_t k);

/* exact_free.cu: usearch_exact_search over host rows (any count of them), and its twin over device rows */
char const* exact_search_free(void const* dataset, size_t dataset_count, size_t dataset_stride, void const* queries,
                              size_t queries_count, size_t queries_stride, uint32_t scalar, size_t dimensions, uint32_t metric,
                              size_t count, size_t threads, uint64_t* keys, size_t keys_stride, float* distances, size_t distances_stride);
char const* exact_search_free_device(void const* dataset, size_t dataset_count, size_t dataset_stride, void const* queries,
                                     size_t queries_count, size_t queries_stride, uint32_t scalar, size_t dimensions, uint32_t metric,
                                     size_t count, uint64_t* keys, size_t keys_stride, float* distances, size_t distances_stride,
                                     cudaStream_t stream);

/* shards.cu */
char const* shards_unique_id(void* out128);
size_t shards_payload_bytes(size_t nq, size_t k);
char const* shards_merge_host(void const* payloads, int world, size_t nq, size_t k, uint64_t* keys, float* dists, uint32_t* counts);

/* indexes.cu: several handles on one device searched as one, the reference's `Indexes` run on one thread. The group
 * borrows its members (never frees them); one handle may be merged more than once. */
struct index_group_t;
index_group_t* index_group_create();
void index_group_free(index_group_t* group);
void index_group_merge(index_group_t& group, frozen_index_t* member);
size_t index_group_size(index_group_t& group);
float const* index_group_last_ms(index_group_t& group); /* searches | merge kernel of the last search, CUDA events */
char const* index_group_search(index_group_t& group, void const* queries, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                               bool exact, uint64_t* keys, float* dists, size_t* counts, uint64_t* computed, uint64_t* visited,
                               size_t* total);
/* merge_into of host rows: keys / dists [shards][nq][k], counts [shards][nq] -> [nq][k] and counts [nq] */
char const* indexes_merge_host(uint64_t const* keys, float const* dists, uint32_t const* counts, size_t shards, size_t nq, size_t k,
                               uint64_t* out_keys, float* out_dists, uint32_t* out_counts);

/* builder.cu: scalar casts and single-pair distances on the device */
char const* cast_rows_device(uint8_t const* src, size_t src_stride, uint32_t from, uint8_t* dst, size_t dst_stride, uint32_t to,
                             size_t dims, size_t rows, cudaStream_t stream);
char const* pair_distance_device(device_index_t const& shape, uint8_t const* d_a, uint8_t const* d_b, float* d_out, cudaStream_t stream);
/* metric(a.rows[slot_a[j]], b.rows[slot_b[j]]) for j < n, one launch; a and b share metric, scalar kind and dimensions */
char const* pair_distances_device(device_index_t const& a, device_index_t const& b, uint32_t const* d_slot_a, uint32_t const* d_slot_b,
                                  size_t n, float* d_out, cudaStream_t stream);
char const* iota_u64_device(uint64_t* d_out, size_t n, cudaStream_t stream);

char const* pair_distance_host(void const* a, void const* b, uint32_t scalar, size_t dimensions, uint32_t metric, float* result);
int default_device(); /* USEARCH_B200_DEVICE, else LOCAL_RANK (one process per GPU under torchrun), else 0 */

size_t bits_per_scalar(uint32_t scalar);

} // namespace usearch_b200
