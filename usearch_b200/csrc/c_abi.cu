/*
 *  c_abi.cu — the `extern "C"` boundary declared in include/usearch_b200.h.
 *
 *  Each function keeps the name, arguments and error behaviour of the reference entry point it
 *  replaces (c/lib.cpp:125-507); only the search path does work, on the GPU. No torch types, no
 *  C++ types and no exceptions cross this boundary.
 */
#include <sys/mman.h>
#include <sys/stat.h>
#include <fcntl.h>
#include <unistd.h>

#include <cstdio>
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "../../include/usearch_b200.h"
#include "frozen_index.h"

using namespace usearch_b200;

namespace {

uint32_t metric_to_char(usearch_metric_kind_t kind) { /* c/lib.cpp:26-40 */
    switch (kind) {
    case usearch_metric_ip_k: return METRIC_IP;
    case usearch_metric_l2sq_k: return METRIC_L2SQ;
    case usearch_metric_cos_k: return METRIC_COS;
    case usearch_metric_haversine_k: return 'h';
    case usearch_metric_divergence_k: return 'd';
    case usearch_metric_pearson_k: return 'p';
    case usearch_metric_jaccard_k: return METRIC_JACCARD;
    case usearch_metric_hamming_k: return METRIC_HAMMING;
    case usearch_metric_tanimoto_k: return METRIC_TANIMOTO;
    case usearch_metric_sorensen_k: return METRIC_SORENSEN;
    default: return 0;
    }
}
usearch_metric_kind_t metric_to_c(uint32_t c) { /* c/lib.cpp:42-56 */
    switch (c) {
    case METRIC_IP: return usearch_metric_ip_k;
    case METRIC_L2SQ: return usearch_metric_l2sq_k;
    case METRIC_COS: return usearch_metric_cos_k;
    case 'h': return usearch_metric_haversine_k;
    case 'd': return usearch_metric_divergence_k;
    case 'p': return usearch_metric_pearson_k;
    case METRIC_JACCARD: return usearch_metric_jaccard_k;
    case METRIC_HAMMING: return usearch_metric_hamming_k;
    case METRIC_TANIMOTO: return usearch_metric_tanimoto_k;
    case METRIC_SORENSEN: return usearch_metric_sorensen_k;
    default: return usearch_metric_unknown_k;
    }
}
uint32_t scalar_to_char(usearch_scalar_kind_t kind) { /* c/lib.cpp:57-67 */
    switch (kind) {
    case usearch_scalar_f32_k: return SCALAR_F32;
    case usearch_scalar_f64_k: return SCALAR_F64;
    case usearch_scalar_f16_k: return SCALAR_F16;
    case usearch_scalar_bf16_k: return SCALAR_BF16;
    case usearch_scalar_i8_k: return SCALAR_I8;
    case usearch_scalar_b1_k: return SCALAR_B1;
    default: return 0;
    }
}
usearch_scalar_kind_t scalar_to_c(uint32_t c) { /* c/lib.cpp:69-79 */
    switch (c) {
    case SCALAR_F32: return usearch_scalar_f32_k;
    case SCALAR_F64: return usearch_scalar_f64_k;
    case SCALAR_F16: return usearch_scalar_f16_k;
    case SCALAR_BF16: return usearch_scalar_bf16_k;
    case SCALAR_I8: return usearch_scalar_i8_k;
    case SCALAR_B1: return usearch_scalar_b1_k;
    default: return usearch_scalar_unknown_k;
    }
}

frozen_index_t* as_index(usearch_index_t h) { return reinterpret_cast<frozen_index_t*>(h); }

/* nothing may propagate through the C boundary: host containers can throw std::bad_alloc */
template <class F> char const* guarded(F&& f) {
    try {
        return f();
    } catch (std::bad_alloc const&) {
        return "Out of memory!";
    } catch (...) {
        return "Unexpected failure inside the library";
    }
}

void set_error(usearch_error_t* error, char const* message) {
    if (error && message) *error = message;
}

/* a search entry on host buffers: `run(query scalar, &total)` under `guarded`; returns the sum of counts, 0 on an error */
template <class F> size_t host_search(usearch_scalar_kind_t query_kind, usearch_error_t* error, F&& run) {
    uint32_t const qs = scalar_to_char(query_kind);
    if (!qs) { set_error(error, "Unknown scalar kind!"); return 0; }
    size_t total = 0;
    if (char const* e = guarded([&] { return run(qs, &total); })) {
        set_error(error, e);
        return 0;
    }
    return total;
}

/* an entry on device buffers: `run(ix, stream)` under the handle's lock and `guarded`, with its context, on the caller's
 * stream (NULL = the handle's own) */
template <class F> void device_search(usearch_index_t index, void* cuda_stream, usearch_error_t* error, F&& run) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, guarded([&]() -> char const* {
        if (char const* e = ix->ensure_context()) return e;
        return run(ix, cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ix->stream);
    }));
}

/* read-only mapping of a file, handed to load_blob */
struct mapped_file_t {
    void* ptr = nullptr;
    size_t length = 0;
    int fd = -1;
    char const* open(char const* path) {
        fd = ::open(path, O_RDONLY);
        if (fd < 0) return "Can't open file";
        struct stat st;
        if (fstat(fd, &st) != 0) return "Can't stat file";
        length = (size_t)st.st_size;
        ptr = mmap(nullptr, length, PROT_READ, MAP_PRIVATE, fd, 0);
        if (ptr == MAP_FAILED) { ptr = nullptr; return "Can't memory-map file"; }
        return nullptr;
    }
    ~mapped_file_t() {
        if (ptr) munmap(ptr, length);
        if (fd >= 0) ::close(fd);
    }
};

char const* metadata_from(uint8_t const* blob, size_t length, usearch_init_options_t* options) {
    /* index_dense.hpp:253-369 metadata sniffers: skip the matrix, read the 64-byte head */
    if (length < 8 + 64) return "File is corrupted and lacks a header";
    uint32_t rows, cols;
    std::memcpy(&rows, blob, 4);
    std::memcpy(&cols, blob + 4, 4);
    size_t offset = 8 + (size_t)rows * cols;
    if (length < offset + 64) return "File is corrupted and lacks a header";
    uint8_t const* p = blob + offset;
    if (std::memcmp(p, "usearch", 7) != 0) return "Magic header mismatch - the file isn't an index";
    uint64_t dims;
    std::memcpy(&dims, p + 33, 8);
    options->metric_kind = metric_to_c(p[13]);
    options->quantization = scalar_to_c(p[14]);
    options->dimensions = dims;
    options->multi = p[41] != 0;
    options->connectivity = 0;
    options->expansion_add = 0;
    options->expansion_search = 0;
    options->metric = nullptr;
    return nullptr;
}

} // namespace

extern "C" {

char const* usearch_version(void) { return "2.21.0+b200"; }

usearch_index_t usearch_init(usearch_init_options_t* options, usearch_error_t* error) {
    frozen_index_t* index = new (std::nothrow) frozen_index_t();
    if (!index) {
        set_error(error, "Out of memory!");
        return nullptr;
    }
    index->stream.device = default_device();
    if (!options) return index; /* c/lib.cpp:142-147: empty index awaiting `load` */
    if (options->metric) {
        set_error(error, "Custom host metrics cannot run on the device");
        delete index;
        return nullptr;
    }
    index->metric = metric_to_char(options->metric_kind);
    index->scalar = scalar_to_char(options->quantization);
    if (!index->metric || !index->scalar || !search_supported(index->metric, index->scalar)) {
        set_error(error, "Unknown metric kind!");
        delete index;
        return nullptr;
    }
    index->dimensions = options->dimensions;
    index->connectivity = options->connectivity ? options->connectivity : 16; /* index.hpp:1340 */
    index->connectivity_base = index->connectivity * 2;                        /* index.hpp:1368 */
    if (options->expansion_add) index->expansion_add = options->expansion_add;
    if (options->expansion_search) index->expansion_search = options->expansion_search;
    index->multi = options->multi;
    return index;
}

void usearch_free(usearch_index_t index, usearch_error_t*) { delete as_index(index); }

size_t usearch_memory_usage(usearch_index_t index, usearch_error_t*) { /* the device key table and the key-set searches'
                                                                        scratch count once they exist */
    frozen_index_t const* ix = as_index(index);
    return ix->hbm_bytes + ix->key_table.cells.capacity * sizeof(key_cell_t) + ix->key_set_scratch.bytes();
}

char const* usearch_hardware_acceleration(usearch_index_t, usearch_error_t*) { return "sm_90a"; }

size_t usearch_serialized_length(usearch_index_t index, usearch_error_t*) { return as_index(index)->serialized_length(); }

void usearch_save_buffer(usearch_index_t index, void* buffer, size_t length, usearch_error_t* error) {
    set_error(error, guarded([&] { return as_index(index)->save_blob(static_cast<uint8_t*>(buffer), length); }));
}

void usearch_load_buffer(usearch_index_t index, void const* buffer, size_t length, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, guarded([&] { return ix->load_blob(static_cast<uint8_t const*>(buffer), length); }));
}

void usearch_view_buffer(usearch_index_t index, void const* buffer, size_t length, usearch_error_t* error) {
    usearch_load_buffer(index, buffer, length, error);
}

void usearch_metadata_buffer(void const* buffer, size_t length, usearch_init_options_t* options, usearch_error_t* error) {
    set_error(error, metadata_from(static_cast<uint8_t const*>(buffer), length, options));
}

void usearch_load(usearch_index_t index, char const* path, usearch_error_t* error) {
    mapped_file_t file;
    if (char const* e = file.open(path)) return set_error(error, e);
    usearch_load_buffer(index, file.ptr, file.length, error);
}

void usearch_view(usearch_index_t index, char const* path, usearch_error_t* error) { usearch_load(index, path, error); }

void usearch_metadata(char const* path, usearch_init_options_t* options, usearch_error_t* error) {
    mapped_file_t file;
    if (char const* e = file.open(path)) return set_error(error, e);
    set_error(error, metadata_from(static_cast<uint8_t const*>(file.ptr), file.length, options));
}

void usearch_save(usearch_index_t index, char const* path, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    size_t length = ix->serialized_length();
    int fd = ::open(path, O_RDWR | O_CREAT | O_TRUNC, 0644);
    if (fd < 0) return set_error(error, "Can't open file");
    if (ftruncate(fd, (off_t)length) != 0) { ::close(fd); return set_error(error, "Can't resize file"); }
    void* ptr = mmap(nullptr, length, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (ptr == MAP_FAILED) { ::close(fd); return set_error(error, "Can't memory-map file"); }
    set_error(error, ix->save_blob(static_cast<uint8_t*>(ptr), length));
    munmap(ptr, length);
    ::close(fd);
}

size_t usearch_size(usearch_index_t index, usearch_error_t*) { return as_index(index)->size - as_index(index)->count_deleted; }
size_t usearch_capacity(usearch_index_t index, usearch_error_t*) { return std::max(as_index(index)->capacity, as_index(index)->size); }
size_t usearch_dimensions(usearch_index_t index, usearch_error_t*) { return as_index(index)->dimensions; }
size_t usearch_connectivity(usearch_index_t index, usearch_error_t*) { return as_index(index)->connectivity; }
void usearch_reserve(usearch_index_t index, size_t capacity, usearch_error_t* error) { /* c/lib.cpp:365-370 */
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, guarded([&] { return ix->reserve_slots(capacity); }));
}
size_t usearch_expansion_add(usearch_index_t index, usearch_error_t*) { return as_index(index)->expansion_add; }
size_t usearch_expansion_search(usearch_index_t index, usearch_error_t*) { return as_index(index)->expansion_search; }
void usearch_change_expansion_add(usearch_index_t index, size_t expansion, usearch_error_t*) { as_index(index)->expansion_add = expansion; }
void usearch_change_expansion_search(usearch_index_t index, size_t expansion, usearch_error_t*) {
    /* under the lock: a join reads and temporarily replaces it for the whole call */
    std::lock_guard<std::mutex> lock(as_index(index)->mutex);
    as_index(index)->expansion_search = expansion;
}
void usearch_change_threads_add(usearch_index_t, size_t, usearch_error_t*) {}
void usearch_change_threads_search(usearch_index_t, size_t, usearch_error_t*) {}

void usearch_change_metric_kind(usearch_index_t index, usearch_metric_kind_t kind, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    uint32_t m = metric_to_char(kind);
    if (!m || !search_supported(m, ix->scalar)) return set_error(error, "Unknown metric kind!");
    std::lock_guard<std::mutex> lock(ix->mutex);
    if (ix->loaded && search_needs_norms(m, ix->scalar) && !ix->d.norms)
        return set_error(error, "Changing a frozen index to this metric needs a reload");
    ix->metric = m;
    ix->d.metric = m;
}

void usearch_change_metric(usearch_index_t, usearch_metric_t, void*, usearch_metric_kind_t, usearch_error_t* error) {
    set_error(error, "Custom host metrics cannot run on the device");
}

size_t usearch_search(usearch_index_t index, void const* query, usearch_scalar_kind_t query_kind, size_t count,
                      usearch_key_t* keys, usearch_distance_t* distances, usearch_error_t* error) {
    /* concurrent single-query callers are coalesced into one launch (frozen_index_t::search_single) */
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->search_single(query, qs, count, keys, distances, total);
    });
}

/* usearch.h:391-395, c/lib.cpp:413-429. A host callback cannot run inside the kernel; it is evaluated on the host once per
 * live key (the reference evaluates it lazily, per candidate: the same answers for a pure predicate) and the resulting key
 * set is applied on the device where the reference applies the callback (index_dense.hpp:2078-2083, index.hpp:4201/4236). */
size_t usearch_filtered_search(usearch_index_t index, void const* query, usearch_scalar_kind_t query_kind, size_t count,
                               int (*filter)(usearch_key_t, void*), void* filter_state, usearch_key_t* keys,
                               usearch_distance_t* distances, usearch_error_t* error) {
    if (!filter) return usearch_search(index, query, query_kind, count, keys, distances, error);
    frozen_index_t* ix = as_index(index);
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        std::vector<uint64_t> allowed;
        {
            std::lock_guard<std::mutex> lock(ix->mutex);
            for (uint64_t key : ix->host_keys)
                if (key != ix->free_key && filter(key, filter_state)) allowed.push_back(key);
        }
        return ix->filtered_search_host(query, 1, 0, qs, count, allowed.data(), allowed.size(), host_results_t{keys, count * 8, distances, count * 4},
                                        total);
    });
}

size_t usearch_search_many(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                           usearch_scalar_kind_t query_kind, size_t count, usearch_key_t* keys, size_t keys_stride,
                           usearch_distance_t* distances, size_t distances_stride, size_t* counts, usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->search_host(queries, queries_count, queries_stride, qs, count,
                                            host_results_t{keys, keys_stride, distances, distances_stride, counts}, total);
    });
}

size_t usearch_b200_search_many_stats(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                                      usearch_scalar_kind_t query_kind, size_t count, usearch_key_t* keys,
                                      usearch_distance_t* distances, size_t* counts, uint64_t* computed_distances,
                                      uint64_t* visited_members, usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->search_host(queries, queries_count, queries_stride, qs, count,
                                            host_results_t{keys, count * 8, distances, count * 4, counts, computed_distances, visited_members},
                                            total);
    });
}

size_t usearch_b200_filtered_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                         size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                         usearch_key_t const* allowed_keys, size_t allowed_count, usearch_key_t* keys,
                                         usearch_distance_t* distances, size_t* counts, uint64_t* computed_distances,
                                         uint64_t* visited_members, usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->filtered_search_host(queries, queries_count, queries_stride, qs, count, allowed_keys, allowed_count,
                                                     host_results_t{keys, count * 8, distances, count * 4, counts, computed_distances,
                                                                    visited_members},
                                                     total);
    });
}

void usearch_b200_search_many_device(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                                     size_t count, usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                     uint32_t* computed_distances, uint32_t* visited_members, void* cuda_stream,
                                     usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        return ix->search_device(queries, queries_count, queries_stride, count, keys, distances, counts, computed_distances, visited_members, s);
    });
}

/* lookups by key from device memory (device_keys.cu), on the caller's stream like usearch_b200_search_many_device */
void usearch_b200_count_many_device(usearch_index_t index, usearch_key_t const* keys, size_t count, uint32_t* counts,
                                    void* cuda_stream, usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) { return ix->count_many_device(keys, count, counts, s); });
}

void usearch_b200_get_many_device(usearch_index_t index, usearch_key_t const* keys, size_t count, size_t max_per_key,
                                  void* vectors, size_t vectors_stride, usearch_scalar_kind_t kind, uint32_t* counts,
                                  void* cuda_stream, usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) -> char const* {
        uint32_t const vs = scalar_to_char(kind);
        if (!vs) return "Unknown scalar kind!";
        return ix->get_many_device(keys, count, max_per_key, vectors, vectors_stride, vs, counts, s);
    });
}

void usearch_b200_filtered_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                              size_t queries_stride, size_t count, usearch_key_t const* allowed_keys,
                                              size_t allowed_count, usearch_key_t* keys, usearch_distance_t* distances,
                                              uint32_t* counts, uint32_t* computed_distances, uint32_t* visited_members,
                                              void* cuda_stream, usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        return ix->filtered_search_device(queries, queries_count, queries_stride, count, allowed_keys, allowed_count, keys, distances,
                                          counts, computed_distances, visited_members, s);
    });
}

/* grouped filtered search (grouped_filter.cu): query i filtered by key set groups[i] of a CSR list of sets */
size_t usearch_b200_grouped_filtered_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                 size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                 uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                 usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                 size_t* counts, uint64_t* computed_distances, uint64_t* visited_members,
                                                 usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->key_set_search_host(queries, queries_count, queries_stride, qs, count,
                                                    key_sets_t{groups, offsets, sets_count, set_keys}, false, false,
                                                    host_results_t{keys, count * 8, distances, count * 4, counts, computed_distances,
                                                                   visited_members},
                                                    total);
    });
}

void usearch_b200_grouped_filtered_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                      size_t queries_stride, size_t count, uint32_t const* groups,
                                                      uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                      usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                      uint32_t* computed_distances, uint32_t* visited_members, void* cuda_stream,
                                                      usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        return ix->key_set_search_device(queries, queries_count, queries_stride, count, key_sets_t{groups, offsets, sets_count, set_keys},
                                         false, false, device_results_t{keys, distances, counts, computed_distances, visited_members}, s);
    });
}

/* exact filtered search (grouped_filter.cu): search_exact_ over only the live slots of each query's key set */
size_t usearch_b200_grouped_filtered_exact_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                       size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                       uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                       usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                       size_t* counts, uint64_t* computed_distances, usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->key_set_search_host(queries, queries_count, queries_stride, qs, count,
                                                    key_sets_t{groups, offsets, sets_count, set_keys}, false, true,
                                                    host_results_t{keys, count * 8, distances, count * 4, counts, computed_distances}, total);
    });
}

void usearch_b200_grouped_filtered_exact_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                            size_t queries_stride, size_t count, uint32_t const* groups,
                                                            uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                            usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                            uint32_t* computed_distances, void* cuda_stream, usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        return ix->key_set_search_device(queries, queries_count, queries_stride, count, key_sets_t{groups, offsets, sets_count, set_keys},
                                         false, true, device_results_t{keys, distances, counts, computed_distances, nullptr}, s);
    });
}

/* excluded search (grouped_filter.cu): query i searches the live entries whose key is not in set groups[i] */
size_t usearch_b200_grouped_excluded_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                 size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                 uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                 usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                 size_t* counts, uint64_t* computed_distances, uint64_t* visited_members,
                                                 usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->key_set_search_host(queries, queries_count, queries_stride, qs, count,
                                                    key_sets_t{groups, offsets, sets_count, set_keys}, true, false,
                                                    host_results_t{keys, count * 8, distances, count * 4, counts, computed_distances,
                                                                   visited_members},
                                                    total);
    });
}

void usearch_b200_grouped_excluded_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                      size_t queries_stride, size_t count, uint32_t const* groups,
                                                      uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                      usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                      uint32_t* computed_distances, uint32_t* visited_members, void* cuda_stream,
                                                      usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        return ix->key_set_search_device(queries, queries_count, queries_stride, count, key_sets_t{groups, offsets, sets_count, set_keys},
                                         true, false, device_results_t{keys, distances, counts, computed_distances, visited_members}, s);
    });
}

size_t usearch_b200_grouped_excluded_exact_search_many(usearch_index_t index, void const* queries, size_t queries_count,
                                                       size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count,
                                                       uint32_t const* groups, uint64_t const* offsets, size_t sets_count,
                                                       usearch_key_t const* set_keys, usearch_key_t* keys, usearch_distance_t* distances,
                                                       size_t* counts, uint64_t* computed_distances, usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->key_set_search_host(queries, queries_count, queries_stride, qs, count,
                                                    key_sets_t{groups, offsets, sets_count, set_keys}, true, true,
                                                    host_results_t{keys, count * 8, distances, count * 4, counts, computed_distances}, total);
    });
}

void usearch_b200_grouped_excluded_exact_search_many_device(usearch_index_t index, void const* queries, size_t queries_count,
                                                            size_t queries_stride, size_t count, uint32_t const* groups,
                                                            uint64_t const* offsets, size_t sets_count, usearch_key_t const* set_keys,
                                                            usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                                            uint32_t* computed_distances, void* cuda_stream, usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        return ix->key_set_search_device(queries, queries_count, queries_stride, count, key_sets_t{groups, offsets, sets_count, set_keys},
                                         true, true, device_results_t{keys, distances, counts, computed_distances, nullptr}, s);
    });
}

/* the asynchronous pair: enqueue any number of batches (kernel launches only, nothing waits), then finish once */
void usearch_b200_search_many_enqueue(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                                      size_t count, usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                      uint32_t* computed_distances, uint32_t* visited_members, void* cuda_stream,
                                      usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        return ix->search_device(queries, queries_count, queries_stride, count, keys, distances, counts, computed_distances, visited_members, s,
                                 true);
    });
}

void usearch_b200_search_many_finish(usearch_index_t index, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, ix->search_finish());
}

/* c/lib.cpp:378-386 -> index_dense_gt::add (index_dense.hpp:760-765, :2002-2050). One member per call goes through the same
 * batched builder as usearch_b200_add_many (a batch of one): correct, but the throughput entry is the batch call. */
void usearch_add(usearch_index_t index, usearch_key_t key, void const* vector, usearch_scalar_kind_t kind, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    uint32_t const vs = scalar_to_char(kind);
    if (!vs) return set_error(error, "Unknown scalar kind!");
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, guarded([&] { return ix->add_many(&key, vector, 1, 0, vs, false); }));
}

void usearch_b200_add_many(usearch_index_t index, usearch_key_t const* keys, void const* vectors, size_t count, size_t vectors_stride,
                           usearch_scalar_kind_t kind, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    uint32_t const vs = scalar_to_char(kind);
    if (!vs) return set_error(error, "Unknown scalar kind!");
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, guarded([&] { return ix->add_many(keys, vectors, count, vectors_stride, vs, false); }));
}

void usearch_b200_add_many_device(usearch_index_t index, usearch_key_t const* keys, void const* vectors, size_t count,
                                  size_t vectors_stride, usearch_scalar_kind_t kind, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    uint32_t const vs = scalar_to_char(kind);
    if (!vs) return set_error(error, "Unknown scalar kind!");
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, guarded([&] { return ix->add_many(keys, vectors, count, vectors_stride, vs, true); }));
}

bool usearch_contains(usearch_index_t index, usearch_key_t key, usearch_error_t*) { /* c/lib.cpp:388-391 */
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    ix->build_key_map();
    return ix->key_map.contains(key);
}

size_t usearch_count(usearch_index_t index, usearch_key_t key, usearch_error_t*) { /* c/lib.cpp:393-396 */
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    ix->build_key_map();
    return ix->key_map.count(key);
}

size_t usearch_get(usearch_index_t index, usearch_key_t key, size_t count, void* vectors, usearch_scalar_kind_t kind,
                   usearch_error_t* error) { /* c/lib.cpp:431-437 */
    frozen_index_t* ix = as_index(index);
    uint32_t const vs = scalar_to_char(kind);
    if (!vs) { set_error(error, "Unknown scalar kind!"); return 0; }
    std::lock_guard<std::mutex> lock(ix->mutex);
    size_t found = 0;
    set_error(error, guarded([&] { return ix->get_vectors(key, count, vectors, vs, &found); }));
    return found;
}

size_t usearch_b200_get_many(usearch_index_t index, usearch_key_t const* keys, size_t count, size_t max_per_key, void* vectors,
                             size_t vectors_stride, usearch_scalar_kind_t kind, size_t* counts, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    uint32_t const vs = scalar_to_char(kind);
    if (!vs) { set_error(error, "Unknown scalar kind!"); return 0; }
    std::lock_guard<std::mutex> lock(ix->mutex);
    size_t rows = 0;
    set_error(error, guarded([&] { return ix->get_many(keys, count, max_per_key, vectors, vectors_stride, vs, counts, &rows); }));
    return rows;
}

size_t usearch_b200_export_keys(usearch_index_t index, size_t offset, size_t limit, usearch_key_t* keys, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    size_t written = 0;
    set_error(error, guarded([&]() -> char const* {
        if (char const* e = ix->ensure_context()) return e;
        written = ix->export_keys(offset, limit, keys);
        return nullptr;
    }));
    return written;
}

void usearch_b200_export_keys_at(usearch_index_t index, size_t const* offsets, size_t count, usearch_key_t* keys, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, guarded([&]() -> char const* {
        if (char const* e = ix->ensure_context()) return e;
        return ix->export_keys_at(offsets, count, keys);
    }));
}

usearch_index_t usearch_b200_copy(usearch_index_t index, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    frozen_index_t* copy = nullptr;
    std::lock_guard<std::mutex> lock(ix->mutex);
    char const* e = guarded([&]() -> char const* {
        copy = new frozen_index_t();
        return ix->copy_into(*copy);
    });
    if (e) {
        delete copy;
        set_error(error, e);
        return nullptr;
    }
    return copy;
}

size_t usearch_b200_levels_stats(usearch_index_t index, size_t* per_level4, size_t levels_capacity, size_t* total4, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    std::vector<uint64_t> nodes, edges;
    if (char const* e = guarded([&] { return ix->graph_levels(nodes, edges); })) {
        set_error(error, e);
        return 0;
    }
    /* node_bytes_ (index.hpp:2116-2195): a 10-byte head (key, level), then {u32 count, M0 slots} and {u32 count, M slots} per
     * upper level */
    size_t const m = ix->connectivity, m0 = ix->connectivity_base, head = 10, nb = 4 + 4 * m, nb0 = 4 + 4 * m0;
    size_t total[4] = {0, 0, 0, 0};
    for (size_t l = 0; l < nodes.size(); ++l) { /* stats(): every level of every node */
        total[0] = l ? total[0] : nodes[0];
        total[1] += edges[l];
        total[2] += nodes[l] * (l ? m : m0);
        total[3] += nodes[l] * (l ? nb : nb0 + head);
    }
    if (total4) std::memcpy(total4, total, sizeof(total));
    /* stats(stats_per_level, max_level): levels 0 .. max_level, the head counted on level 0 only */
    size_t const levels = nodes.empty() ? 0 : (size_t)ix->d.max_level + 1;
    for (size_t l = 0; l < std::min(levels, levels_capacity); ++l) {
        size_t const nl = l < nodes.size() ? nodes[l] : 0;
        per_level4[4 * l + 0] = nl;
        per_level4[4 * l + 1] = l < edges.size() ? edges[l] : 0;
        per_level4[4 * l + 2] = nl * (l ? m : m0);
        per_level4[4 * l + 3] = nl * (l ? nb : nb0 + head);
    }
    return levels;
}

bool usearch_b200_multi(usearch_index_t index) { return as_index(index)->multi; }

size_t usearch_remove(usearch_index_t index, usearch_key_t key, usearch_error_t* error) { /* c/lib.cpp:439-446 */
    return usearch_b200_remove_many(index, &key, 1, false, nullptr, error);
}

size_t usearch_b200_remove_many(usearch_index_t index, usearch_key_t const* keys, size_t count, bool compact,
                                size_t* pruned_edges, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    size_t removed = 0;
    set_error(error, guarded([&] { return ix->remove_many(keys, count, compact, &removed, pruned_edges); }));
    return removed;
}

size_t usearch_b200_count_many(usearch_index_t index, usearch_key_t const* keys, size_t count, size_t* counts, usearch_error_t*) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    ix->build_key_map();
    size_t total = 0;
    for (size_t i = 0; i < count; ++i) {
        size_t const c = ix->key_map.count(keys[i]);
        if (counts) counts[i] = c;
        total += c;
    }
    return total;
}

void usearch_b200_change_reuse_removed(usearch_index_t index, bool reuse, usearch_error_t*) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    ix->reuse_removed = reuse;
}

bool usearch_b200_reuse_removed(usearch_index_t index) { return as_index(index)->reuse_removed; }

size_t usearch_b200_join(usearch_index_t a, usearch_index_t b, size_t max_proposals, bool exact, usearch_key_t* a_keys_out,
                         usearch_key_t* b_keys_out, size_t capacity, size_t* stats4_out, usearch_error_t* error) {
    std::vector<uint64_t> ak, bk;
    size_t stats[4] = {0, 0, 0, 0};
    char const* e = guarded([&] { return as_index(a)->join(*as_index(b), max_proposals, exact, ak, bk, stats); });
    if (e) { set_error(error, e); return 0; }
    if (ak.size() > capacity) { set_error(error, "Output arrays too small for the engaged pairs: size them to min(capacity(a), capacity(b))"); return 0; }
    if (!ak.empty()) {
        std::memcpy(a_keys_out, ak.data(), ak.size() * sizeof(uint64_t));
        std::memcpy(b_keys_out, bk.data(), bk.size() * sizeof(uint64_t));
    }
    if (stats4_out) std::memcpy(stats4_out, stats, sizeof(stats));
    return ak.size();
}

void usearch_b200_last_join_ms(usearch_index_t index, float* out3) { std::memcpy(out3, as_index(index)->last_join_ms, 3 * sizeof(float)); }

void usearch_b200_pairwise_distances(usearch_index_t index, usearch_key_t const* left_keys, usearch_key_t const* right_keys, size_t n,
                                     usearch_distance_t* out, usearch_error_t* error) {
    set_error(error, guarded([&] { return as_index(index)->pairwise_distances(left_keys, right_keys, n, out); }));
}

size_t usearch_rename(usearch_index_t index, usearch_key_t from, usearch_key_t to, usearch_error_t* error) { /* c/lib.cpp:448-455 */
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    size_t renamed = 0;
    set_error(error, guarded([&] { return ix->rename_key(from, to, &renamed); }));
    return renamed;
}

/* c/lib.cpp:458-466: one distance between two caller vectors, through the metric structs the search kernels use */
usearch_distance_t usearch_distance(void const* a, void const* b, usearch_scalar_kind_t kind, size_t dimensions,
                                    usearch_metric_kind_t metric_kind, usearch_error_t* error) {
    uint32_t const m = metric_to_char(metric_kind), sc = scalar_to_char(kind);
    if (!m || !sc || !search_supported(m, sc)) { set_error(error, "Unknown metric kind!"); return 0; }
    float result = 0;
    set_error(error, pair_distance_host(a, b, sc, dimensions, m, &result));
    return result;
}

void usearch_exact_search(void const* dataset, size_t dataset_size, size_t dataset_stride, void const* queries, size_t queries_size,
                          size_t queries_stride, usearch_scalar_kind_t scalar_kind, size_t dimensions, usearch_metric_kind_t metric_kind,
                          size_t count, size_t threads, usearch_key_t* keys, size_t keys_stride, usearch_distance_t* distances,
                          size_t distances_stride, usearch_error_t* error) {
    uint32_t const m = metric_to_char(metric_kind), s = scalar_to_char(scalar_kind);
    if (!m || !s) return set_error(error, "Unknown metric kind!");
    set_error(error, guarded([&] {
        return exact_search_free(dataset, dataset_size, dataset_stride, queries, queries_size, queries_stride, s, dimensions, m, count, threads,
                                 keys, keys_stride, distances, distances_stride);
    }));
}

/* usearch_exact_search over device matrices, in the caller's stream (exact_free.cu) */
void usearch_b200_exact_search_device(void const* dataset, size_t dataset_size, size_t dataset_stride, void const* queries,
                                      size_t queries_size, size_t queries_stride, usearch_scalar_kind_t scalar_kind, size_t dimensions,
                                      usearch_metric_kind_t metric_kind, size_t count, usearch_key_t* keys, size_t keys_stride,
                                      usearch_distance_t* distances, size_t distances_stride, void* cuda_stream, usearch_error_t* error) {
    uint32_t const m = metric_to_char(metric_kind), s = scalar_to_char(scalar_kind);
    if (!m || !s) return set_error(error, "Unknown metric kind!");
    set_error(error, guarded([&] {
        return exact_search_free_device(dataset, dataset_size, dataset_stride, queries, queries_size, queries_stride, s, dimensions, m, count,
                                        keys, keys_stride, distances, distances_stride, static_cast<cudaStream_t>(cuda_stream));
    }));
}

/* index_dense_gt::cluster(vector, level) (index_dense.hpp:788-793 -> cluster_ :2088-2109 -> index.hpp:3092-3125) for a
 * batch: the greedy descent of the search kernel stopped at `level`; one (key, distance) per query. */
void usearch_b200_cluster_many(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                               usearch_scalar_kind_t query_kind, size_t level, usearch_key_t* keys, usearch_distance_t* distances,
                               uint64_t* computed_distances, uint64_t* visited_members, usearch_error_t* error) {
    host_search(query_kind, error, [&](uint32_t qs, size_t*) {
        return as_index(index)->cluster_host(queries, queries_count, queries_stride, qs, level, keys, distances, computed_distances,
                                             visited_members);
    });
}

size_t usearch_b200_exact_search_many(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                                      usearch_scalar_kind_t query_kind, size_t count, usearch_key_t* keys, usearch_distance_t* distances,
                                      size_t* counts, usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->exact_host(queries, queries_count, queries_stride, qs, count,
                                           host_results_t{keys, count * 8, distances, count * 4, counts}, total);
    });
}

/* ---- sharded search: one process per GPU, one shard per process (python/lib.cpp:321-402 `Indexes`) ------------------ */

void usearch_b200_shards_unique_id(void* unique_id128, usearch_error_t* error) { set_error(error, shards_unique_id(unique_id128)); }

void usearch_b200_shards_join(usearch_index_t index, int rank, int world, void const* unique_id128, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    set_error(error, ix->join_shards(rank, world, unique_id128));
}

size_t usearch_b200_sharded_search_many(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                                        usearch_scalar_kind_t query_kind, size_t count, usearch_key_t* keys,
                                        usearch_distance_t* distances, size_t* counts, usearch_error_t* error) {
    return host_search(query_kind, error, [&](uint32_t qs, size_t* total) {
        return as_index(index)->sharded_search_host(queries, queries_count, queries_stride, qs, count,
                                                    host_results_t{keys, count * 8, distances, count * 4, counts}, total);
    });
}

void usearch_b200_sharded_search_many_device(usearch_index_t index, void const* queries, size_t queries_count, size_t queries_stride,
                                             size_t count, usearch_key_t* keys, usearch_distance_t* distances, uint32_t* counts,
                                             uint32_t* computed_distances, uint32_t* visited_members, void* cuda_stream,
                                             usearch_error_t* error) {
    device_search(index, cuda_stream, error, [&](frozen_index_t* ix, cudaStream_t s) {
        char const* e = ix->sharded_search_device(queries, queries_count, queries_stride, count, keys, distances, counts,
                                                  computed_distances, visited_members, s);
        /* on the handle's own stream the caller has nothing to order its next use of the outputs with: finish before returning */
        if (!e && !cuda_stream && cudaStreamSynchronize(s) != cudaSuccess) e = "CUDA failure: synchronize";
        return e;
    });
}

size_t usearch_b200_shards_payload_bytes(size_t queries_count, size_t count) { return shards_payload_bytes(queries_count, count); }

void usearch_b200_merge_topk(void const* payloads, int world, size_t queries_count, size_t count, usearch_key_t* keys,
                             usearch_distance_t* distances, uint32_t* counts, usearch_error_t* error) {
    set_error(error, shards_merge_host(payloads, world, queries_count, count, keys, distances, counts));
}

/* ---- several indexes on one GPU searched as one (python/lib.cpp:74-107, :321-402 `Indexes`) ----------------------- */

usearch_b200_indexes_t usearch_b200_indexes_init(usearch_error_t* error) {
    index_group_t* group = nullptr;
    set_error(error, guarded([&]() -> char const* { group = index_group_create(); return nullptr; }));
    return group;
}

void usearch_b200_indexes_free(usearch_b200_indexes_t indexes) { index_group_free(static_cast<index_group_t*>(indexes)); }

void usearch_b200_indexes_merge(usearch_b200_indexes_t indexes, usearch_index_t index, usearch_error_t* error) {
    if (!index) return set_error(error, "No index to merge");
    set_error(error, guarded([&]() -> char const* {
        index_group_merge(*static_cast<index_group_t*>(indexes), as_index(index));
        return nullptr;
    }));
}

size_t usearch_b200_indexes_size(usearch_b200_indexes_t indexes, usearch_error_t*) {
    return index_group_size(*static_cast<index_group_t*>(indexes));
}

size_t usearch_b200_indexes_search_many(usearch_b200_indexes_t indexes, void const* queries, size_t queries_count,
                                        size_t queries_stride, usearch_scalar_kind_t query_kind, size_t count, bool exact,
                                        usearch_key_t* keys, usearch_distance_t* distances, size_t* counts,
                                        uint64_t* computed_distances, uint64_t* visited_members, usearch_error_t* error) {
    uint32_t qs = scalar_to_char(query_kind);
    if (!qs) { set_error(error, "Unknown scalar kind!"); return 0; }
    size_t total = 0;
    if (char const* e = guarded([&] {
            return index_group_search(*static_cast<index_group_t*>(indexes), queries, queries_count, queries_stride, qs, count, exact,
                                      keys, distances, counts, computed_distances, visited_members, &total);
        })) {
        set_error(error, e);
        return 0;
    }
    return total;
}

void usearch_b200_indexes_last_ms(usearch_b200_indexes_t indexes, float* out2) {
    std::memcpy(out2, index_group_last_ms(*static_cast<index_group_t*>(indexes)), 2 * sizeof(float));
}

void usearch_b200_merge_into(usearch_key_t const* keys, usearch_distance_t const* distances, uint32_t const* counts, size_t shards,
                             size_t queries_count, size_t count, usearch_key_t* merged_keys, usearch_distance_t* merged_distances,
                             uint32_t* merged_counts, usearch_error_t* error) {
    set_error(error, guarded([&] {
        return indexes_merge_host(keys, distances, counts, shards, queries_count, count, merged_keys, merged_distances, merged_counts);
    }));
}

void usearch_clear(usearch_index_t index, usearch_error_t*) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    ix->release_device();
}

size_t usearch_b200_profile_phases_n(usearch_index_t index, int enable, uint64_t* counters, size_t count) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    size_t const bytes = sizeof(uint64_t) * PHASE_COUNTERS;
    if (counters && count) {
        size_t const n = std::min<size_t>(count, PHASE_COUNTERS);
        std::memset(counters, 0, sizeof(uint64_t) * count);
        if (ix->phase_cycles.ptr) cudaMemcpy(counters, ix->phase_cycles.ptr, sizeof(uint64_t) * n, cudaMemcpyDeviceToHost);
    }
    ix->profile_phases = enable != 0;
    if (ix->profile_phases && !ix->phase_cycles.reserve(PHASE_COUNTERS)) cudaMemset(ix->phase_cycles.ptr, 0, bytes);
    return PHASE_COUNTERS;
}

void usearch_b200_profile_phases(usearch_index_t index, int enable, uint64_t* counters16) {
    usearch_b200_profile_phases_n(index, enable, counters16, 16);
}

int usearch_b200_tune(usearch_index_t index, char const* knob, int value) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    if (!std::strcmp(knob, "stage_sets")) ix->tune.stage_sets = value;
    else if (!std::strcmp(knob, "warps_per_sm")) ix->tune.warps_per_sm = value;
    else if (!std::strcmp(knob, "prefilter")) ix->tune.prefilter = value;
    else if (!std::strcmp(knob, "heap_head")) ix->tune.heap_head = value;
    else if (!std::strcmp(knob, "get_chunk_rows")) ix->tune.get_chunk_rows = value;
    else if (!std::strcmp(knob, "group_bitmap_mb")) ix->tune.group_bitmap_mb = value;
    else return -1;
    return 0;
}

int usearch_b200_launch_plan(usearch_index_t index, size_t count, uint64_t* out16, usearch_error_t* error) {
    frozen_index_t* ix = as_index(index);
    std::lock_guard<std::mutex> lock(ix->mutex);
    char const* e = ix->ensure_context();
    if (!e && (!ix->loaded || ix->d.n == 0)) e = "An empty index has no launch plan";
    launch_plan_t pl;
    if (!e) e = ix->plan((uint32_t)count, 0, pl);
    set_error(error, e);
    if (e) return -1;
    uint64_t const visits = pl.visited_bitmap_words ? (pl.visit_log_cap ? 2u : 1u) : 0u;
    uint64_t const v[16] = {pl.stage_sets, pl.warps_per_sm_target, (uint64_t)pl.blocks, pl.smem_per_warp,
                            pl.heap_smem_cap, pl.heap_spill_cap, visits, pl.visited_cap,
                            pl.code_pass, pl.code_smem_stride, pl.qsplit_len, pl.prefilter ? 1u : 0u,
                            pl.off_heap - pl.off_stage};
    std::memcpy(out16, v, sizeof(v));
    return 0;
}

int usearch_b200_device(usearch_index_t index) { return as_index(index)->stream.device; }
uint64_t usearch_b200_kernel_launches(usearch_index_t index) { return as_index(index)->kernel_launches; }
float usearch_b200_last_kernel_ms(usearch_index_t index) { return as_index(index)->last_kernel_ms; }
size_t usearch_b200_bytes_per_vector(usearch_index_t index) { return as_index(index)->d.bytes_per_vector; }
size_t usearch_b200_max_level(usearch_index_t index) { return (size_t)as_index(index)->d.max_level; }

} // extern "C"
