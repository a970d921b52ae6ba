/*
 *  usearch_b200.h — C ABI of the B200-native batched HNSW search backend.
 *
 *  The library (usearch_b200/libusearch_b200.so) is a drop-in for the SEARCH path of the
 *  reference's C ABI. Every `usearch_*` symbol below has the name, argument order, argument
 *  meaning and error convention of the declaration it replaces in the reference header
 *  `c/usearch.h` (cited per function as usearch.h:LINE, implementation c/lib.cpp:LINE), so that
 *  Go (golang/lib.go:29-33), C# (NativeMethods.cs:16) and C callers bind it unchanged.
 *
 *  Division of labour (DESIGN.md §2): the graph is BUILT by the host path (the reference itself,
 *  or any writer of the v2 `.usearch` format), serialised, and handed to this library through
 *  `usearch_load[_buffer]` / `usearch_view[_buffer]`, which freeze it into a flat SoA layout in
 *  HBM. From then on every `usearch_search` / `usearch_search_many` runs on the GPU. Mutating
 *  entry points are exported so that existing bindings link, and report
 *  "Index is frozen in GPU memory ..." through `error` (the reference's own convention for an
 *  immutable `view`, index.hpp:2787-2788).
 *
 *  Error convention (usearch.h:24-28): `*error` receives a pointer to a static, NUL-terminated
 *  message that must not be freed; it is left untouched on success. Nothing throws across the ABI.
 *
 *  `usearch_b200_*` symbols are additive: the batch entry the reference lacks (SURVEY.md
 *  finding 2; python/lib.cpp:286-308 loops single-query calls on a thread pool instead), a
 *  device-pointer variant for callers that already hold queries in HBM, and introspection.
 */
#ifndef USEARCH_B200_H
#define USEARCH_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- types: identical to usearch.h:20-110 ------------------------------------------------ */

typedef void* usearch_index_t;
typedef uint64_t usearch_key_t;
typedef float usearch_distance_t;
typedef char const* usearch_error_t;
typedef usearch_distance_t (*usearch_metric_t)(void const*, void const*);

typedef enum usearch_metric_kind_t { /* usearch.h:40-52 */
    usearch_metric_unknown_k = 0,
    usearch_metric_cos_k = 1,
    usearch_metric_ip_k = 2,
    usearch_metric_l2sq_k = 3,
    usearch_metric_haversine_k = 4,
    usearch_metric_divergence_k = 5,
    usearch_metric_pearson_k = 6,
    usearch_metric_jaccard_k = 7,
    usearch_metric_hamming_k = 8,
    usearch_metric_tanimoto_k = 9,
    usearch_metric_sorensen_k = 10,
} usearch_metric_kind_t;

typedef enum usearch_scalar_kind_t { /* usearch.h:54-62 */
    usearch_scalar_unknown_k = 0,
    usearch_scalar_f32_k = 1,
    usearch_scalar_f64_k = 2,
    usearch_scalar_f16_k = 3,
    usearch_scalar_i8_k = 4,
    usearch_scalar_b1_k = 5,
    usearch_scalar_bf16_k = 6,
} usearch_scalar_kind_t;

typedef struct usearch_init_options_t { /* usearch.h:64-110, same field order */
    usearch_metric_kind_t metric_kind;
    usearch_metric_t metric; /* custom host callbacks cannot run on the device: must be NULL */
    usearch_scalar_kind_t quantization;
    size_t dimensions;
    size_t connectivity;
    size_t expansion_add;
    size_t expansion_search;
    bool multi;
} usearch_init_options_t;

/* ---- lifecycle & introspection ----------------------------------------------------------- */

char const* usearch_version(void);                                                      /* usearch.h:116 */
usearch_index_t usearch_init(usearch_init_options_t* options, usearch_error_t* error);  /* usearch.h:124; NULL options = empty index awaiting load (c/lib.cpp:142-147) */
void usearch_free(usearch_index_t index, usearch_error_t* error);                       /* usearch.h:131 */
size_t usearch_memory_usage(usearch_index_t index, usearch_error_t* error);             /* usearch.h:139; bytes of HBM held */
char const* usearch_hardware_acceleration(usearch_index_t index, usearch_error_t* error); /* usearch.h:147; "sm_90a" */
size_t usearch_serialized_length(usearch_index_t index, usearch_error_t* error);        /* usearch.h:154 */

/* ---- the hand-off: v2 `.usearch` blob → HBM (index_dense.hpp:1084-1188, index.hpp:3322-3382) */

void usearch_save(usearch_index_t index, char const* path, usearch_error_t* error);     /* usearch.h:162 */
void usearch_load(usearch_index_t index, char const* path, usearch_error_t* error);     /* usearch.h:170 */
void usearch_view(usearch_index_t index, char const* path, usearch_error_t* error);     /* usearch.h:178; same as load: the device copy never aliases the file */
void usearch_metadata(char const* path, usearch_init_options_t* options, usearch_error_t* error); /* usearch.h:186 */
void usearch_save_buffer(usearch_index_t index, void* buffer, size_t length, usearch_error_t* error);        /* usearch.h:195 */
void usearch_load_buffer(usearch_index_t index, void const* buffer, size_t length, usearch_error_t* error);  /* usearch.h:204 */
void usearch_view_buffer(usearch_index_t index, void const* buffer, size_t length, usearch_error_t* error);  /* usearch.h:214 */
void usearch_metadata_buffer(void const* buffer, size_t length, usearch_init_options_t* options, usearch_error_t* error); /* usearch.h:223 */

size_t usearch_size(usearch_index_t index, usearch_error_t* error);          /* usearch.h:231 */
size_t usearch_capacity(usearch_index_t index, usearch_error_t* error);      /* usearch.h:238 */
size_t usearch_dimensions(usearch_index_t index, usearch_error_t* error);    /* usearch.h:245 */
size_t usearch_connectivity(usearch_index_t index, usearch_error_t* error);  /* usearch.h:252 */
void usearch_reserve(usearch_index_t index, size_t capacity, usearch_error_t* error); /* usearch.h:260, c/lib.cpp:365-370: room for `capacity` members in HBM */
size_t usearch_expansion_add(usearch_index_t index, usearch_error_t* error);          /* usearch.h:268 */
size_t usearch_expansion_search(usearch_index_t index, usearch_error_t* error);       /* usearch.h:276 */
void usearch_change_expansion_add(usearch_index_t index, size_t expansion, usearch_error_t* error);    /* usearch.h:284 */
void usearch_change_expansion_search(usearch_index_t index, size_t expansion, usearch_error_t* error); /* usearch.h:292 */
void usearch_change_threads_add(usearch_index_t index, size_t threads, usearch_error_t* error);        /* usearch.h:300; accepted, ignored */
void usearch_change_threads_search(usearch_index_t index, size_t threads, usearch_error_t* error);     /* usearch.h:308; accepted, ignored */
void usearch_change_metric_kind(usearch_index_t index, usearch_metric_kind_t kind, usearch_error_t* error); /* usearch.h:316 */
void usearch_change_metric(usearch_index_t index, usearch_metric_t metric, void* state, usearch_metric_kind_t kind, usearch_error_t* error); /* usearch.h:327; host callbacks rejected */

/* ---- the hot path ------------------------------------------------------------------------ */

/* usearch.h:371-374, c/lib.cpp:398-411. Returns the number of matches; ALWAYS writes `count`
 * output slots, padding with key 0 / signalling-NaN distance (index.hpp:2707-2722). The query
 * may be of any scalar kind; it is cast to the index's kind with the reference's rules
 * (index_plugins.hpp:1105-1224). */
size_t usearch_search(usearch_index_t index, void const* query_vector, usearch_scalar_kind_t query_kind, size_t count,
                      usearch_key_t* keys, usearch_distance_t* distances, usearch_error_t* error);

/* usearch.h:391-395. Host callbacks cannot run on the device: reports an error unless `filter` is NULL. */
size_t usearch_filtered_search(usearch_index_t index, void const* query_vector, usearch_scalar_kind_t query_kind,
                               size_t count, int (*filter)(usearch_key_t key, void* filter_state), void* filter_state,
                               usearch_key_t* keys, usearch_distance_t* distances, usearch_error_t* error);

/* NEW (additive). One call = one batch = one persistent-kernel launch. Strides are in BYTES,
 * in the style of usearch_exact_search (usearch.h:467-474). `counts` receives the per-query
 * number of matches. Replaces the thread-pool loop in python/lib.cpp:261-319 (`search_typed`)
 * and cpp/bench.cpp:352-377. Buffers are HOST memory; copies are part of the call. Returns the
 * sum of counts. */
size_t usearch_search_many(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                           usearch_scalar_kind_t query_kind, size_t count,              //
                           usearch_key_t* keys, size_t keys_stride,                     //
                           usearch_distance_t* distances, size_t distances_stride,      //
                           size_t* counts, usearch_error_t* error);

/* ---- mutation and lookups by key ---------------------------------------------------------------- */

/* usearch.h:338, c/lib.cpp:378-386 -> index_gt::add (index.hpp:2780-2880). The member is linked into the graph on the GPU
 * by the batched builder (csrc/builder.cu) — a batch of one here; usearch_b200_add_many below is the throughput entry.
 * Capacity grows on demand (the reference's C layer reports "Reserve capacity ahead of insertions!" instead). Removed
 * entries keep their slot (tombstone, skipped by searches) until an add reuses it: see usearch_b200_change_reuse_removed. */
void usearch_add(usearch_index_t index, usearch_key_t key, void const* vector, usearch_scalar_kind_t vector_kind, usearch_error_t* error); /* usearch.h:338 */
bool usearch_contains(usearch_index_t index, usearch_key_t key, usearch_error_t* error);   /* usearch.h:349 */
size_t usearch_count(usearch_index_t index, usearch_key_t key, usearch_error_t* error);    /* usearch.h:358 */
size_t usearch_get(usearch_index_t index, usearch_key_t key, size_t count, void* vector, usearch_scalar_kind_t vector_kind, usearch_error_t* error); /* usearch.h:407 */
size_t usearch_remove(usearch_index_t index, usearch_key_t key, usearch_error_t* error);   /* usearch.h:418 */
size_t usearch_rename(usearch_index_t index, usearch_key_t from, usearch_key_t to, usearch_error_t* error); /* usearch.h:428 */
usearch_distance_t usearch_distance(void const* vector_first, void const* vector_second, usearch_scalar_kind_t scalar_kind,
                                    size_t dimensions, usearch_metric_kind_t metric_kind, usearch_error_t* error); /* usearch.h:441 */
void usearch_exact_search(void const* dataset, size_t dataset_size, size_t dataset_stride, void const* queries,
                          size_t queries_size, size_t queries_stride, usearch_scalar_kind_t scalar_kind, size_t dimensions,
                          usearch_metric_kind_t metric_kind, size_t count, size_t threads, usearch_key_t* keys,
                          size_t keys_stride, usearch_distance_t* distances, size_t distances_stride,
                          usearch_error_t* error); /* usearch.h:467; runs on the GPU; any vector length (rows too long for the scan's shared-memory stage are read in place); count > 256 needs vectors that fit the tiled stage (about 3.5 KB). The dataset may exceed GPU memory: it is scanned in chunks of rows, copied by `threads` host threads (0 = up to 8) into pinned staging buffers whose uploads overlap the scan; the result does not depend on the cut. Returns when the outputs are written. */
/* NEW (additive). usearch_exact_search with `dataset`, `queries`, `keys` and `distances` in DEVICE memory on one GPU,
 * strides in bytes (0 = dense outputs), enqueued on `cuda_stream` (a cudaStream_t; NULL = the default stream). The call
 * does not wait for the stream: the outputs are ready in stream order, and the scratch it takes is released in stream
 * order. Rows are scanned in place when the dataset is 16-byte aligned and dense with rows of whole 16-byte chunks;
 * otherwise they are repacked chunk by chunk. Refusals (the same messages as usearch_exact_search) come before anything is
 * enqueued, so the outputs are then left untouched. */
void usearch_b200_exact_search_device(void const* dataset, size_t dataset_size, size_t dataset_stride, void const* queries,
                                      size_t queries_size, size_t queries_stride, usearch_scalar_kind_t scalar_kind, size_t dimensions,
                                      usearch_metric_kind_t metric_kind, size_t count, usearch_key_t* keys, size_t keys_stride,
                                      usearch_distance_t* distances, size_t distances_stride, void* cuda_stream, usearch_error_t* error);
void usearch_clear(usearch_index_t index, usearch_error_t* error); /* usearch.h:481 */

/* NEW (additive). GPU-assisted construction (SURVEY.md §8f N4): `count` keys and vectors in one call. The vectors (any
 * supported scalar kind, rows `vectors_stride` bytes apart, 0 = dense) are copied into HBM, cast on the device if needed, and
 * linked batch by batch: one INSERT-mode launch of the search kernel per batch produces every member's candidates on every
 * level (search_to_insert_, index.hpp:4010-4079), two more kernels select forward and reverse links with the reference's
 * heuristic (refine_, index.hpp:4276-4318). Replaces the thread-pool loop of python/lib.cpp:171-258 (`add_typed_to_index`). */
void usearch_b200_add_many(usearch_index_t index, usearch_key_t const* keys, void const* vectors, size_t count,
                           size_t vectors_stride, usearch_scalar_kind_t vector_kind, usearch_error_t* error);
/* The same with `keys` and `vectors` in DEVICE memory on the index's GPU. */
void usearch_b200_add_many_device(usearch_index_t index, usearch_key_t const* keys, void const* vectors, size_t count,
                                  size_t vectors_stride, usearch_scalar_kind_t vector_kind, usearch_error_t* error);

/* NEW (additive). Removal of many keys (python/lib.cpp:1210-1227 `remove_many`): every entry under each key becomes a
 * tombstone and its slot joins a FIFO of removed slots (usearch_remove is this call with one key). Returns the number of
 * entries removed. With `compact`, every link that leads to a removed entry is then erased on the GPU, on every level
 * (index_dense_gt::isolate, index_dense.hpp:1709-1720); `pruned_edges` (may be NULL) receives the number of links erased.
 * Removed entries keep their own links. */
size_t usearch_b200_remove_many(usearch_index_t index, usearch_key_t const* keys, size_t count, bool compact,
                                size_t* pruned_edges, usearch_error_t* error);
/* NEW (additive). usearch_count for `count` keys at once (host only): counts[i] = entries stored under keys[i]; returns
 * their sum. */
size_t usearch_b200_count_many(usearch_index_t index, usearch_key_t const* keys, size_t count, size_t* counts,
                               usearch_error_t* error);
/* NEW (additive). Slot reuse, off by default. When on, every add gives its i-th new entry the oldest removed slot while any
 * is left (index_dense_gt::add_, index_dense.hpp:2020-2049) and appends the rest: the entry keeps the slot's level and
 * rows, its lists are rebuilt by the INSERT search with its own slot kept out of its results (index_gt::update,
 * index.hpp:2911-2999). Links that other entries still hold to the slot stay, as in the reference. When off, every add
 * appends and removed slots are never reused. */
void usearch_b200_change_reuse_removed(usearch_index_t index, bool reuse, usearch_error_t* error);
bool usearch_b200_reuse_removed(usearch_index_t index);

/* NEW (additive). Semantic join (index_dense_gt::join, index_dense.hpp:1762-1786; stable marriages, index.hpp:4345-4543) of
 * `a` with `b`, with the decisions of the reference's run on one thread. The side with fewer slots (removed entries
 * count) proposes; proposals are searches of the other index (approximate, or brute force with `exact`) with expansion
 * max(expansion_search(a), expansion_search(b)). `max_proposals` 0 means log(men) + 1, clamped to the men; at most 65535.
 * Removed entries take part, as in the reference, and are exported under the free key, so the number of pairs can exceed
 * usearch_size. Writes the engaged pairs (a key, b key) in the reference's export order into `a_keys_out` /
 * `b_keys_out`, each holding `capacity` keys; min(usearch_capacity(a), usearch_capacity(b)) is always enough. Returns the
 * number of pairs, or 0 and an error when they do not fit. `stats4_out` (may be NULL) receives intersection_size,
 * engagements, visited_members and computed_distances. Both handles must be on one device, not sharded, and share metric,
 * scalar kind and dimensions. */
size_t usearch_b200_join(usearch_index_t a, usearch_index_t b, size_t max_proposals, bool exact, usearch_key_t* a_keys_out,
                         usearch_key_t* b_keys_out, size_t capacity, size_t* stats4_out, usearch_error_t* error);
/* NEW (additive). Wall-clock milliseconds of the last usearch_b200_join called with `index` as `a`: proposal searches
 * (launches and copies back), pair distances, and the host replay without the columns it waited for. */
void usearch_b200_last_join_ms(usearch_index_t index, float* out3);
/* NEW (additive). out[i] = the distance between the vectors stored under left_keys[i] and right_keys[i], FLT_MAX where a
 * key is missing, one GPU launch. With one vector per key this is distance_between(left, right).min
 * (index_dense.hpp:808-862) bit for bit. A multi index takes the minimum over EVERY pair of their vectors; the reference
 * pairs only the first vector under the left key with each vector under the right key (its loop does not rewind the
 * right range), so the two differ when the left key holds several vectors. */
void usearch_b200_pairwise_distances(usearch_index_t index, usearch_key_t const* left_keys, usearch_key_t const* right_keys, size_t n,
                                     usearch_distance_t* out, usearch_error_t* error);

/* ---- additive: reading the index back out (index_dense_gt's get / export_keys / copy / stats) ---------------------- */

/* NEW (additive). index_dense_gt::get for `count` keys in one call (python/lib.cpp:971-1003). Each key gets
 * min(usearch_count(key), max_per_key) rows, in ascending slot order (the rows usearch_get would give). The rows are
 * packed in key order into `vectors`, `vectors_stride` bytes apart (0 = dense), cast to `kind` with the rules of
 * usearch_get. A key that is missing gets no row. `counts[i]` receives the rows of key i. Returns the number of rows.
 * The slots are resolved on the host; one gather kernel, a cast kernel when `kind` differs from the stored kind, and one
 * copy back run per chunk of rows, and the device and pinned scratch stay bounded (the "get_chunk_rows" knob). */
size_t usearch_b200_get_many(usearch_index_t index, usearch_key_t const* keys, size_t count, size_t max_per_key, void* vectors,
                             size_t vectors_stride, usearch_scalar_kind_t kind, size_t* counts, usearch_error_t* error);
/* NEW (additive). index_dense_gt::export_keys (index_dense.hpp:1595-1608): the live keys from the `offset`-th on, at most
 * `limit` of them, in ascending slot order (the reference walks its hash table instead). Returns the number written. */
size_t usearch_b200_export_keys(usearch_index_t index, size_t offset, size_t limit, usearch_key_t* keys, usearch_error_t* error);
/* keys[i] = the offsets[i]-th live key in the same order, for `count` offsets in any order; an offset past the last live
 * key is an error */
void usearch_b200_export_keys_at(usearch_index_t index, size_t const* offsets, size_t count, usearch_key_t* keys,
                                 usearch_error_t* error);
/* NEW (additive). index_dense_gt::copy (index_dense.hpp:1615-1650): a new, independent handle on the same device holding
 * a copy of every array and of all host state (configuration, free-slot queue, knobs). Free it with usearch_free. The
 * same further calls on both give identical results and identical files. A sharded handle is refused. */
usearch_index_t usearch_b200_copy(usearch_index_t index, usearch_error_t* error);
/* NEW (additive). index_gt::stats (index.hpp:3133-3225). `per_level4` receives, for each level 0 .. max_level (at most
 * `levels_capacity` of them), nodes | edges | max_edges | allocated_bytes as stats(stats_per_level, max_level) gives
 * them; `total4` (may be NULL) receives stats(). Edges are the entries the device lists hold, counted in one launch;
 * allocated_bytes follows the reference's node layout, not HBM use. Returns max_level + 1, or 0 for an empty index. */
size_t usearch_b200_levels_stats(usearch_index_t index, size_t* per_level4, size_t levels_capacity, size_t* total4,
                                 usearch_error_t* error);
/* Whether the index keeps several entries per key. */
bool usearch_b200_multi(usearch_index_t index);

/* ---- additive: sharded search, one process per GPU (SURVEY.md §8e) ------------------------------------------------ */

/* The reference's `Indexes` (python/lib.cpp:74-107, :321-402) searches every query in every shard and merges by distance. Here
 * each process holds one shard on its GPU. Rank 0 obtains a 128-byte id (an ncclUniqueId), the host side hands it to every
 * rank over its own control plane (torch.distributed, MPI, a file), every rank joins. A sharded search = this shard's batched
 * search + ONE NCCL all-gather of the packed per-shard rows + a k-way merge kernel ordered by (distance, shard, position);
 * every rank receives the merged rows. Collective: all ranks must call with the same queries and count. */
void usearch_b200_shards_unique_id(void* unique_id128, usearch_error_t* error);
void usearch_b200_shards_join(usearch_index_t index, int rank, int world, void const* unique_id128, usearch_error_t* error);
/* Host buffers. Returns the sum of counts over the merged rows, whether or not `counts` is NULL. */
size_t usearch_b200_sharded_search_many(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                                        usearch_scalar_kind_t query_kind, size_t count, usearch_key_t* keys,
                                        usearch_distance_t* distances, size_t* counts, usearch_error_t* error);
/* device pointers, queries already in the index's scalar kind (see usearch_b200_search_many_device). With a `cuda_stream` the
 * all-gather and the merge are only ENQUEUED on it (the outputs are ready in stream order); with NULL the call uses the handle's
 * own stream and returns when the merged rows are complete. */
void usearch_b200_sharded_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                             size_t queries_stride, size_t count, usearch_key_t* keys,
                                             usearch_distance_t* distances, uint32_t* counts, uint32_t* computed_distances,
                                             uint32_t* visited_members, void* cuda_stream, usearch_error_t* error);
/* The merge on its own (search_result_t::merge_into, index.hpp:2650-2670, made deterministic), for callers that hold several
 * shards in one process: `payloads` = `world` blocks of usearch_b200_shards_payload_bytes(queries_count, count) bytes in HOST
 * memory, each `keys u64[nq*count] | distances f32[nq*count] | counts u32[nq]` (16-byte padded). */
size_t usearch_b200_shards_payload_bytes(size_t queries_count, size_t count);
void usearch_b200_merge_topk(void const* payloads, int world, size_t queries_count, size_t count, usearch_key_t* keys,
                             usearch_distance_t* distances, uint32_t* counts, usearch_error_t* error);

/* ---- additive: several indexes on one GPU searched as one (the reference's `Indexes`) ----------------------------- */

/* A group of index handles, the reference's `Indexes` (python/lib.cpp:74-107, :321-402). The group borrows its members:
 * they must outlive it, and it never frees them. The same handle may be merged more than once. A search gives what the
 * reference's `Indexes.search` gives on one thread: every member searched in merge order (with its own expansion_search),
 * each result folded into the query's row by search_result_t::merge_into (index.hpp:2650-2670). On data without NaN
 * that is (distance ascending, later insertion first): a later member wins a tie. Members must share dimensions and
 * device and must not be sharded handles. The call locks every distinct member for its duration, in ascending address
 * order. */
typedef void* usearch_b200_indexes_t;
usearch_b200_indexes_t usearch_b200_indexes_init(usearch_error_t* error);
void usearch_b200_indexes_free(usearch_b200_indexes_t indexes);
void usearch_b200_indexes_merge(usearch_b200_indexes_t indexes, usearch_index_t index, usearch_error_t* error);
/* the members' sizes summed (a handle merged twice counts twice, as in the reference) */
size_t usearch_b200_indexes_size(usearch_b200_indexes_t indexes, usearch_error_t* error);
/* Host buffers: `keys` / `distances` dense [queries_count x count], rows padded past counts[i] with key 0 and a signalling
 * NaN. `computed_distances` / `visited_members` (may be NULL) receive per query the sums over members. A group without
 * members answers with empty rows and no error. Returns the number of matches over all queries. */
size_t usearch_b200_indexes_search_many(usearch_b200_indexes_t indexes, void const* queries, size_t queries_count,
                                        size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count, bool exact,
                                        usearch_key_t* keys, usearch_distance_t* distances, size_t* counts,
                                        uint64_t* computed_distances, uint64_t* visited_members, usearch_error_t* error);
/* Milliseconds of the last search, from CUDA events on the group's stream: member searches (queries upload included) |
 * the merge kernel. */
void usearch_b200_indexes_last_ms(usearch_b200_indexes_t indexes, float* out2);
/* The merge kernel on host rows: `keys` / `distances` [shards x queries_count x count] and `counts` [shards x
 * queries_count] (each clamped to count), folded shard by shard as usearch_b200_indexes_search_many folds them. */
void usearch_b200_merge_into(usearch_key_t const* keys, usearch_distance_t const* distances, uint32_t const* counts, size_t shards,
                             size_t queries_count, size_t count, usearch_key_t* merged_keys, usearch_distance_t* merged_distances,
                             uint32_t* merged_counts, usearch_error_t* error);

/* ---- additive, device-resident variants ---------------------------------------------------- */

/* All pointers are DEVICE pointers on the index's GPU; `queries` must already be in the index's
 * scalar kind, rows `queries_stride` bytes apart (a multiple of 16 or equal to bytes-per-vector).
 * `keys`/`distances` are dense [queries_count x count]; `counts`, `computed_distances` and
 * `visited_members` (the reference's per-query counters, index.hpp:2605-2609; may be NULL) are
 * uint32 [queries_count]. `cuda_stream` is a cudaStream_t (NULL = the handle's own stream). Nothing is copied; the call
 * returns when the batch is complete (it waits for the kernel to read the per-query status words and retries scratch
 * overflows). For launches that do not wait, see usearch_b200_search_many_enqueue / _finish below. */
void usearch_b200_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                     size_t queries_stride, size_t count, usearch_key_t* keys,
                                     usearch_distance_t* distances, uint32_t* counts, uint32_t* computed_distances,
                                     uint32_t* visited_members, void* cuda_stream, usearch_error_t* error);

/* Lookups by key from DEVICE memory, for keys that a device pipeline produced (e.g. the keys of
 * usearch_b200_search_many_device). They follow usearch_b200_search_many_device: all pointers are DEVICE pointers on the
 * index's GPU, the work runs on `cuda_stream` (NULL = the handle's own stream) and the call returns when the outputs are
 * complete. count and get probe a key -> slot table in HBM (16 bytes per cell, at least twice as many cells as live
 * entries), built on the first such lookup after the keys changed and counted by usearch_memory_usage from then on. */

/* counts[i] = entries stored under keys[i] (usearch_b200_count_many). */
void usearch_b200_count_many_device(usearch_index_t index, usearch_key_t const* keys, size_t count, uint32_t* counts,
                                    void* cuda_stream, usearch_error_t* error);
/* usearch_b200_get_many with DEVICE keys and outputs. Key i owns rows i*max_per_key .. i*max_per_key+max_per_key-1 of
 * `vectors` (`vectors_stride` bytes apart, 0 = packed), cast to `kind`; counts[i] = the rows written for key i, and rows
 * past counts[i] are zero. A key's rows are its min(count, max_per_key) lowest slots (its oldest entries) in ascending
 * order: what usearch_b200_get_many returns whenever max_per_key >= the key's count, or the index holds no removed
 * entries. */
void usearch_b200_get_many_device(usearch_index_t index, usearch_key_t const* keys, size_t count, size_t max_per_key,
                                  void* vectors, size_t vectors_stride, usearch_scalar_kind_t kind, uint32_t* counts,
                                  void* cuda_stream, usearch_error_t* error);
/* usearch_b200_filtered_search_many with DEVICE queries (in the index's kind), DEVICE allowed keys and DEVICE outputs,
 * laid out as in usearch_b200_search_many_device. The allowed keys are sorted on the device; the result equals the host
 * call's with the same keys. */
void usearch_b200_filtered_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                              size_t queries_stride, size_t count, usearch_key_t const* allowed_keys,
                                              size_t allowed_count, usearch_key_t* keys, usearch_distance_t* distances,
                                              uint32_t* counts, uint32_t* computed_distances, uint32_t* visited_members,
                                              void* cuda_stream, usearch_error_t* error);

/* Grouped filtered search: one batch in which every query has its own allowed key set. The sets are given as CSR:
 * set g holds set_keys[offsets[g] .. offsets[g + 1]] (`sets_count` + 1 offsets, the first 0, never decreasing; a set may
 * be empty, repeat keys or name keys the index lacks), and query i uses set groups[i] < sets_count. Row i equals
 * usearch_b200_filtered_search_many(queries[i], count, that set): keys, distances, counts and both counters. Every set
 * becomes a bitmap row over slots; the rows of as many sets as the "group_bitmap_mb" knob allows (default 1024 MB) are
 * served per launch. A group id out of range, bad offsets or no sets for a non-empty batch are refused before any output
 * is written; so is a sharded handle. Buffers are HOST memory; queries may be of any kind (cast on the device). Returns
 * the sum of counts. */
size_t usearch_b200_grouped_filtered_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                 size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                 uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                 usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                 size_t* counts, uint64_t* computed_distances, uint64_t* visited_members,
                                                 usearch_error_t* error);
/* The same with DEVICE queries (in the index's kind), DEVICE groups, offsets, set keys and outputs, laid out as in
 * usearch_b200_search_many_device, on `cuda_stream` (NULL = the handle's stream). The arguments are checked on the device
 * before the search; the call returns when the outputs are complete. */
void usearch_b200_grouped_filtered_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                      size_t queries_stride, size_t count, uint32_t const* groups,
                                                      uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                      usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                      uint32_t* computed_distances, uint32_t* visited_members, void* cuda_stream,
                                                      usearch_error_t* error);

/* Exact filtered search: usearch_b200_grouped_filtered_search_many's sets and rows, but every query scans exactly the live
 * entries whose key is in its set, as the reference's filtered_search(..., exact = true) does (index_dense.hpp:774-779,
 * index.hpp:4251-4268): keys, distances and counts equal it, ties in the order of search(exact = true). A removed entry
 * never counts, even when the free key is in the set; on a multi index every entry of a key counts. computed_distances[i]
 * receives the number of entries query i measured (the live entries of its set). `groups` may be NULL when sets_count is 1:
 * every query uses set 0. Each set becomes an ascending list of its slots, so the cost follows the sets' sizes, never
 * slots x sets. Refusals as in usearch_b200_grouped_filtered_search_many. Buffers are HOST memory; queries may be of any
 * kind. Returns the sum of counts. */
size_t usearch_b200_grouped_filtered_exact_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                       size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                       uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                       usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                       size_t* counts, uint64_t* computed_distances, usearch_error_t* error);
/* The same with DEVICE queries (in the index's kind; any stride), DEVICE groups, offsets, set keys and outputs, on
 * `cuda_stream` (NULL = the handle's stream). The arguments are checked on the device before the search; the call returns
 * when the outputs are complete. */
void usearch_b200_grouped_filtered_exact_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                            size_t queries_stride, size_t count, uint32_t const* groups,
                                                            uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                            usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                            uint32_t* computed_distances, void* cuda_stream, usearch_error_t* error);

/* Excluded search: the sets of usearch_b200_grouped_filtered_search_many name keys a query must NOT return. Row i equals
 * the reference's filtered_search(queries[i], count, key not in set groups[i]) (index_dense.hpp:774-779): keys,
 * distances, counts and both counters. A removed entry is never returned; a free key, a key the index lacks or a repeated
 * key in a set changes nothing; on a multi index excluding a key excludes every entry under it; an empty set gives the
 * plain search's row. `groups` may be NULL when sets_count is 1: every query uses set 0. Each set becomes a bitmap row
 * that allows every slot but the set's, served in rounds under the "group_bitmap_mb" knob. Refusals as in
 * usearch_b200_grouped_filtered_search_many, before any output is written. Buffers are HOST memory; queries may be of
 * any kind. Returns the sum of counts. */
size_t usearch_b200_grouped_excluded_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                 size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                 uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                 usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                 size_t* counts, uint64_t* computed_distances, uint64_t* visited_members,
                                                 usearch_error_t* error);
/* The same with DEVICE queries (in the index's kind), DEVICE groups, offsets, set keys and outputs, on `cuda_stream`
 * (NULL = the handle's stream). The call returns when the outputs are complete. */
void usearch_b200_grouped_excluded_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                      size_t queries_stride, size_t count, uint32_t const* groups,
                                                      uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                      usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                      uint32_t* computed_distances, uint32_t* visited_members, void* cuda_stream,
                                                      usearch_error_t* error);
/* Exact excluded search: every query scans exactly the live entries whose key is not in its set, as the reference's
 * filtered_search(..., exact = true) does (index.hpp:4251-4268): keys, distances and counts equal it, and
 * computed_distances[i] = the live entries less the e live entries under the set's keys. It runs the unfiltered exact
 * search at count k + e rounded up to a power of two (one launch per such count) and drops the set's entries, so
 * k + e > 256 is refused, with exact search's message, for vectors too long for its tiled stage. Refusals and buffers as
 * in usearch_b200_grouped_filtered_exact_search_many. */
size_t usearch_b200_grouped_excluded_exact_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                       size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                       uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                       usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                       size_t* counts, uint64_t* computed_distances, usearch_error_t* error);
void usearch_b200_grouped_excluded_exact_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                            size_t queries_stride, size_t count, uint32_t const* groups,
                                                            uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                            usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                            uint32_t* computed_distances, void* cuda_stream, usearch_error_t* error);

/* The asynchronous pair. `enqueue` = the same arguments as usearch_b200_search_many_device, but it ONLY enqueues the
 * kernel on `cuda_stream` and returns; any number of batches may be in flight. `finish` waits for them, inspects the
 * per-query status words and re-runs, with larger scratch, the rare queries whose scratch overflowed; the outputs of
 * every enqueued batch are final when it returns. */
void usearch_b200_search_many_enqueue(usearch_index_t index, void const* queries, size_t queries_count,
                                      size_t queries_stride, size_t count, usearch_key_t* keys,
                                      usearch_distance_t* distances, uint32_t* counts, uint32_t* computed_distances,
                                      uint32_t* visited_members, void* cuda_stream, usearch_error_t* error);
void usearch_b200_search_many_finish(usearch_index_t index, usearch_error_t* error);

/* Like usearch_search_many (host buffers) but also returns the reference's two counters. */
size_t usearch_b200_search_many_stats(usearch_index_t index, void const* queries, size_t queries_count,
                                      size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                      usearch_key_t* keys, usearch_distance_t* distances, size_t* counts,
                                      uint64_t* computed_distances, uint64_t* visited_members, usearch_error_t* error);

/* Introspection for tests / bench: CUDA device ordinal, kernel launches issued so far by this
 * handle, duration in milliseconds of the most recent search kernel (CUDA events on its stream). */
/* Device-side counterpart of usearch_filtered_search (usearch.h:391-395) for the one predicate family that
 * can run on a GPU: "the key is in this set". `allowed_keys` (host memory, any order, may be empty) is turned
 * into a bitmap over slots; the predicate is applied where the reference applies its callback
 * (index_dense.hpp:2078-2083, index.hpp:4201/4236): rejected members are still traversed, never returned. The keys are
 * sorted on the device, as usearch_b200_filtered_search_many_device sorts them, so more than INT_MAX of them are refused
 * with its error. Returns the sum of counts. */
size_t usearch_b200_filtered_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                         size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                         usearch_key_t const* allowed_keys, size_t allowed_count, usearch_key_t* keys,
                                         usearch_distance_t* distances, size_t* counts, uint64_t* computed_distances,
                                         uint64_t* visited_members, usearch_error_t* error);

/* `index_dense_gt::cluster(vector, level)` (index_dense.hpp:788-793, index.hpp:3092-3125) for a batch: the closest
 * member on graph level `level` for every query (greedy descent only). Outputs hold one entry per query;
 * computed_distances / visited_members may be NULL. */
void usearch_b200_cluster_many(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                               usearch_scalar_kind_t query_kind, size_t level, usearch_key_t* keys,
                               usearch_distance_t* distances, uint64_t* computed_distances, uint64_t* visited_members,
                               usearch_error_t* error);

/* `search(exact = true)` of the reference's C++ / Python surface (index.hpp:3047-3051, search_exact_ :4251-4268) for a
 * batch: brute force over every non-removed member of the frozen index, ties resolved exactly like the reference's
 * sequence of sorted inserts (equal distances: larger slot first). Any count; beyond 256 the lists live in L2 instead of registers.
 * Returns the sum of counts, whether or not `counts` is NULL. */
size_t usearch_b200_exact_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                      size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                      usearch_key_t* keys, usearch_distance_t* distances, size_t* counts,
                                      usearch_error_t* error);

/* Phase introspection of the search kernel: enable != 0 turns on (and zeroes) sixteen device-side
 * counters summed over all queries since; `counters16` (may be NULL) first receives the current values:
 * cycles of setup+descent | heap pop | row + visited test | vector wait | distance math | accept replay |
 * output, then queries | heap pushes | sum of per-query max heap size | max heap size | candidates prefiltered (layer-0
 * candidates of cos / ip f32 judged on their int8 shadow) | survivors (those of them whose f32 row was read) | cycles
 * of code wait (the prefilter waiting for its int8 codes; not part of distance math) | cycles of the prefilter's dot
 * products (the tensor-core dots and their conversion; part of distance math) | cycles of the prefilter's bound (the
 * bound, its ballots and the survivors' compaction; part of distance math). */
void usearch_b200_profile_phases(usearch_index_t index, int enable, uint64_t* counters16);
/* The same counters, the first `count` of them into `counters` (may be NULL; words beyond those the kernel keeps are
 * zeroed). Words 0-15 are those of usearch_b200_profile_phases; then cycles of the conversion of the prefilter's dot
 * products to `dot` and their stores, after the tensor cores have finished (part of the dot products' cycles) | the
 * prefilter's code passes | hops measured through the prefilter | cycles of distance math in hops that start with
 * `top` full | cycles of vector wait in the upper-level descent (part of setup+descent; distance math, which is layer-0
 * time less every vector wait, subtracts them as well). Returns the number of counters the kernel keeps. */
size_t usearch_b200_profile_phases_n(usearch_index_t index, int enable, uint64_t* counters, size_t count);
/* Tuning knobs of the search launch for this handle ("stage_sets", "warps_per_sm", "prefilter" = 0 | 1: judge layer-0
 * candidates of cos / ip f32 on their int8 shadow first, on by default; "heap_head" = an upper bound on the candidate-heap
 * entries kept in shared memory, rounded down to an even number >= 2, the rest go to HBM; 0 = as planned), and
 * "get_chunk_rows" = rows per chunk of usearch_b200_get_many (0 = 64 MB of output), and "group_bitmap_mb" = the MB of
 * key-set bitmap rows one launch of usearch_b200_grouped_filtered_search_many may use (default 1024, at least one row
 * is always used); results never depend on them.
 * Returns 0, or -1 for an unknown knob. */
int usearch_b200_tune(usearch_index_t index, char const* knob, int value);
/* The launch plan a search of `count` neighbours gets under the current knobs, for a loaded index. `out16` receives:
 * stage sets | warps per SM (target) | blocks | shared memory per warp (bytes) | heap entries in shared memory | heap
 * entries in HBM per warp | visits (0 = hash table, 1 = bitmap, 2 = bitmap cleaned through a log) | hash table entries |
 * prefilter candidates per code pass | prefilter code row stride in shared memory (bytes) | bytes of each int8 query
 * split level | prefilter effective (0 | 1) | stage area (bytes) | 3 reserved.
 * Returns 0, or -1 with `error` set to the planner's message when no plan fits. */
int usearch_b200_launch_plan(usearch_index_t index, size_t count, uint64_t* out16, usearch_error_t* error);
int usearch_b200_device(usearch_index_t index);
uint64_t usearch_b200_kernel_launches(usearch_index_t index);
float usearch_b200_last_kernel_ms(usearch_index_t index);
size_t usearch_b200_bytes_per_vector(usearch_index_t index);
size_t usearch_b200_max_level(usearch_index_t index);

#ifdef __cplusplus
}
#endif
#endif /* USEARCH_B200_H */
