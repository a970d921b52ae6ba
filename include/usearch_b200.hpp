/*
 *  usearch_b200.hpp — C++11 host-side mirror of the reference's search surface over the C ABI.
 *
 *  The reference's C++ users instantiate `unum::usearch::index_dense_gt<>` (include/usearch/index_dense.hpp)
 *  and call `search(T const*, wanted)` which returns a `search_result_t` (index.hpp:2595-2742) exposing
 *  `count`, `visited_members`, `computed_distances`, `error`, `operator[]`, `dump_to`, `merge_into`, `contains`.
 *  This header offers the same names and semantics for an index frozen in GPU memory, so call sites written
 *  against the reference read the same:
 *
 *      auto state = usearch_b200::index_dense_t::make("index.usearch");       // index_dense.hpp:681-687
 *      auto result = state.index.search(query, 10);                            // index_dense.hpp:767-772
 *      result.dump_to(keys, distances);                                         // index.hpp:2707-2722
 *      auto batch = state.index.search_many(queries, nq, 10);                  // the batch entry the reference lacks
 *
 *  Header-only, no CUDA or torch types: it only calls the `extern "C"` functions of usearch_b200.h and links
 *  against libusearch_b200.so.
 */
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <limits>
#include <type_traits>
#include <utility>
#include <vector>

#include "usearch_b200.h"

namespace usearch_b200 {

using vector_key_t = usearch_key_t;
using distance_t = usearch_distance_t;

/* scalar tags with the reference's names (index_plugins.hpp:85-108) */
struct f16_bits_t { std::uint16_t bits; };
struct bf16_bits_t { std::uint16_t bits; };
enum b1x8_t : unsigned char {};
using f32_t = float;
using f64_t = double;
using i8_t = std::int8_t;

template <typename scalar_at> inline usearch_scalar_kind_t scalar_kind() noexcept {
    return std::is_same<scalar_at, f32_t>::value    ? usearch_scalar_f32_k
           : std::is_same<scalar_at, f64_t>::value  ? usearch_scalar_f64_k
           : std::is_same<scalar_at, f16_bits_t>::value  ? usearch_scalar_f16_k
           : std::is_same<scalar_at, bf16_bits_t>::value ? usearch_scalar_bf16_k
           : std::is_same<scalar_at, i8_t>::value   ? usearch_scalar_i8_k
           : std::is_same<scalar_at, b1x8_t>::value ? usearch_scalar_b1_k
                                                    : usearch_scalar_unknown_k;
}

/* error_t (index.hpp:407-461): a static C string, falsy when empty */
class error_t {
    char const* message_ = nullptr;

  public:
    error_t() noexcept = default;
    error_t(char const* message) noexcept : message_(message) {}
    explicit operator bool() const noexcept { return message_ != nullptr; }
    char const* what() const noexcept { return message_; }
    char const* release() noexcept { char const* m = message_; message_ = nullptr; return m; }
};

/* metric_punned_t (index_plugins.hpp:1678-2015), builtin metrics only: custom function pointers cannot run
 * on a device and are rejected by `usearch_init`. */
struct metric_punned_t {
    std::size_t dimensions_ = 0;
    usearch_metric_kind_t metric_kind_ = usearch_metric_unknown_k;
    usearch_scalar_kind_t scalar_kind_ = usearch_scalar_unknown_k;

    metric_punned_t() = default;
    metric_punned_t(std::size_t dimensions, usearch_metric_kind_t metric_kind = usearch_metric_l2sq_k,
                    usearch_scalar_kind_t scalar_kind = usearch_scalar_f32_k) noexcept
        : dimensions_(dimensions), metric_kind_(metric_kind), scalar_kind_(scalar_kind) {}
    static metric_punned_t builtin(std::size_t dimensions, usearch_metric_kind_t metric_kind = usearch_metric_l2sq_k,
                                   usearch_scalar_kind_t scalar_kind = usearch_scalar_f32_k) noexcept {
        return metric_punned_t(dimensions, metric_kind, scalar_kind);
    }
    std::size_t dimensions() const noexcept { return dimensions_; }
    usearch_metric_kind_t metric_kind() const noexcept { return metric_kind_; }
    usearch_scalar_kind_t scalar_kind() const noexcept { return scalar_kind_; }
    std::size_t bytes_per_vector() const noexcept { /* index_plugins.hpp:1853-1855 */
        std::size_t bits = scalar_kind_ == usearch_scalar_b1_k ? 1 : scalar_kind_ == usearch_scalar_i8_k ? 8
                           : (scalar_kind_ == usearch_scalar_f16_k || scalar_kind_ == usearch_scalar_bf16_k) ? 16
                           : scalar_kind_ == usearch_scalar_f64_k ? 64 : 32;
        return (dimensions_ * bits + 7) / 8;
    }
    char const* isa_name() const noexcept { return "sm_90a"; }
    bool missing() const noexcept { return metric_kind_ == usearch_metric_unknown_k; }
};

struct index_dense_config_t { /* index_dense.hpp:102-159, the fields that reach this backend */
    std::size_t connectivity = 16;
    std::size_t expansion_add = 128;
    std::size_t expansion_search = 64;
    bool multi = false;
};

struct index_dense_state_result_t;

class index_dense_t {
    usearch_index_t handle_ = nullptr;

  public:
    struct match_t { /* index.hpp match_t: {member.key, distance} */
        struct { vector_key_t key; } member;
        distance_t distance;
    };

    /* search_result_t (index.hpp:2595-2742). Owns its rows (the reference borrows a thread context instead). */
    class search_result_t {
        friend class index_dense_t;
        std::vector<vector_key_t> keys_;
        std::vector<distance_t> distances_;

      public:
        std::size_t count = 0;
        std::size_t visited_members = 0;
        std::size_t computed_distances = 0;
        error_t error{};

        explicit operator bool() const noexcept { return !error; }
        search_result_t failed(error_t message) noexcept { error = message; return std::move(*this); }
        operator std::size_t() const noexcept { return count; }
        std::size_t size() const noexcept { return count; }
        bool empty() const noexcept { return !count; }
        match_t at(std::size_t i) const noexcept { return match_t{{keys_[i]}, distances_[i]}; }
        match_t operator[](std::size_t i) const noexcept { return at(i); }
        match_t front() const noexcept { return at(0); }
        match_t back() const noexcept { return at(count - 1); }
        bool contains(vector_key_t key) const noexcept {
            for (std::size_t i = 0; i != count; ++i)
                if (keys_[i] == key) return true;
            return false;
        }
        /* index.hpp:2707-2722: unused slots receive key 0 and a signalling NaN */
        std::size_t dump_to(vector_key_t* keys, distance_t* distances, std::size_t capacity) const noexcept {
            std::size_t n = count < capacity ? count : capacity, i = 0;
            for (; i != n; ++i) keys[i] = keys_[i], distances[i] = distances_[i];
            for (; i != capacity; ++i) keys[i] = 0, distances[i] = std::numeric_limits<distance_t>::signaling_NaN();
            return n;
        }
        std::size_t dump_to(vector_key_t* keys, distance_t* distances) const noexcept { return dump_to(keys, distances, count); }
        /* index.hpp:2650-2670: insertion-merge by lower_bound on distance, the worst beyond max_count is dropped */
        std::size_t merge_into(vector_key_t* keys, distance_t* distances, std::size_t old_count, std::size_t max_count) const noexcept {
            std::size_t merged = old_count;
            for (std::size_t i = 0; i != count; ++i) {
                std::size_t offset = 0;
                while (offset < merged && distances[offset] < distances_[i]) ++offset;
                if (offset == max_count) continue;
                std::size_t worse = merged - offset - (max_count == merged);
                std::memmove(keys + offset + 1, keys + offset, worse * sizeof(vector_key_t));
                std::memmove(distances + offset + 1, distances + offset, worse * sizeof(distance_t));
                keys[offset] = keys_[i];
                distances[offset] = distances_[i];
                merged += merged != max_count;
            }
            return merged;
        }
    };

    /* rows of one batched call: the outputs python/lib.cpp:437-441 allocates */
    struct batch_result_t {
        std::vector<vector_key_t> keys;     /* [nq x wanted] */
        std::vector<distance_t> distances;  /* [nq x wanted] */
        std::vector<std::size_t> counts;    /* [nq] */
        std::size_t visited_members = 0, computed_distances = 0;
        error_t error{};
        explicit operator bool() const noexcept { return !error; }
    };

    using state_result_t = index_dense_state_result_t; /* index_dense.hpp:620-640, defined below the class */

    index_dense_t() = default;
    index_dense_t(index_dense_t&& other) noexcept : handle_(other.handle_) { other.handle_ = nullptr; }
    index_dense_t& operator=(index_dense_t&& other) noexcept { std::swap(handle_, other.handle_); return *this; }
    index_dense_t(index_dense_t const&) = delete;
    index_dense_t& operator=(index_dense_t const&) = delete;
    ~index_dense_t() { if (handle_) usearch_free(handle_, nullptr); }

    static state_result_t make(metric_punned_t metric, index_dense_config_t config = {}); /* index_dense.hpp:644-673 */
    static state_result_t make(char const* path, bool view = false);                        /* index_dense.hpp:681-687 */

    error_t load(char const* path) { usearch_error_t e = nullptr; usearch_load(handle_, path, &e); return e; }
    error_t view(char const* path) { usearch_error_t e = nullptr; usearch_view(handle_, path, &e); return e; }
    error_t load_from_buffer(void const* buffer, std::size_t length) { usearch_error_t e = nullptr; usearch_load_buffer(handle_, buffer, length, &e); return e; }
    error_t save(char const* path) const { usearch_error_t e = nullptr; usearch_save(handle_, path, &e); return e; }
    std::size_t serialized_length() const { return usearch_serialized_length(handle_, nullptr); }

    std::size_t size() const { return usearch_size(handle_, nullptr); }
    std::size_t capacity() const { return usearch_capacity(handle_, nullptr); }
    std::size_t dimensions() const { return usearch_dimensions(handle_, nullptr); }
    std::size_t connectivity() const { return usearch_connectivity(handle_, nullptr); }
    std::size_t expansion_search() const { return usearch_expansion_search(handle_, nullptr); }
    void change_expansion_search(std::size_t n) { usearch_change_expansion_search(handle_, n, nullptr); }
    std::size_t memory_usage() const { return usearch_memory_usage(handle_, nullptr); }
    std::size_t max_level() const { return usearch_b200_max_level(handle_); }
    usearch_index_t native_handle() const noexcept { return handle_; }

    /* index_dense.hpp:767-772 — `thread` is accepted and ignored; `exact` scans every member (index.hpp:4251-4268) */
    template <typename scalar_at>
    search_result_t search(scalar_at const* vector, std::size_t wanted, std::size_t /*thread*/ = 0, bool exact = false) const {
        search_result_t result;
        if (!wanted) return result;
        result.keys_.resize(wanted);
        result.distances_.resize(wanted);
        std::size_t count = 0;
        std::uint64_t computed = 0, visited = 0;
        usearch_error_t error = nullptr;
        if (exact) {
            usearch_b200_exact_search_many(handle_, vector, 1, 0, scalar_kind<scalar_at>(), wanted, result.keys_.data(),
                                           result.distances_.data(), &count, &error);
            if (error) return result.failed(error);
            result.count = count;
            result.computed_distances = size();
            return result;
        }
        usearch_b200_search_many_stats(handle_, vector, 1, 0, scalar_kind<scalar_at>(), wanted, result.keys_.data(),
                                       result.distances_.data(), &count, &computed, &visited, &error);
        if (error) return result.failed(error);
        result.count = count;
        result.computed_distances = computed;
        result.visited_members = visited;
        return result;
    }

    /* ---- mutation and lookups by key: add_result_t / labeling_result_t of the reference, trimmed (index.hpp:2548-2562,
     *      index_dense.hpp:525-540) ---- */
    struct add_result_t {
        error_t error{};
        std::size_t new_size = 0;
        explicit operator bool() const noexcept { return !error; }
    };
    struct labeling_result_t {
        error_t error{};
        std::size_t completed = 0;
        explicit operator bool() const noexcept { return !error; }
    };
    error_t reserve(std::size_t capacity) { usearch_error_t e = nullptr; usearch_reserve(handle_, capacity, &e); return e; }
    bool try_reserve(std::size_t capacity) { return !reserve(capacity); }
    /* index_dense.hpp:760-765 — `thread` and `copy_vector` are accepted and ignored (the index always owns a copy in HBM) */
    template <typename scalar_at> add_result_t add(vector_key_t key, scalar_at const* vector, std::size_t /*thread*/ = 0, bool /*copy*/ = true) {
        add_result_t result;
        usearch_error_t error = nullptr;
        usearch_add(handle_, key, vector, scalar_kind<scalar_at>(), &error);
        result.error = error;
        result.new_size = size();
        return result;
    }
    /* the batch driver of python/lib.cpp:171-258 as one call: the graph is linked on the GPU */
    template <typename scalar_at>
    add_result_t add_many(vector_key_t const* keys, scalar_at const* vectors, std::size_t count, std::size_t stride_bytes = 0) {
        add_result_t result;
        usearch_error_t error = nullptr;
        usearch_b200_add_many(handle_, keys, vectors, count, stride_bytes, scalar_kind<scalar_at>(), &error);
        result.error = error;
        result.new_size = size();
        return result;
    }
    bool contains(vector_key_t key) const { return usearch_contains(handle_, key, nullptr); }
    std::size_t count(vector_key_t key) const { return usearch_count(handle_, key, nullptr); }
    template <typename scalar_at> std::size_t get(vector_key_t key, scalar_at* vectors, std::size_t vectors_limit = 1) const {
        usearch_error_t error = nullptr;
        return usearch_get(handle_, key, vectors_limit, vectors, scalar_kind<scalar_at>(), &error);
    }
    /* get for `count` keys in one call: up to `vectors_per_key` rows per key, packed in key order into `vectors`, with
     * counts[i] the rows of key i (may be NULL); returns the number of rows */
    template <typename scalar_at>
    std::size_t get(vector_key_t const* keys, std::size_t count, scalar_at* vectors, std::size_t* counts,
                    std::size_t vectors_per_key = 1) const {
        std::vector<std::size_t> own(counts ? 0 : count);
        usearch_error_t error = nullptr;
        return usearch_b200_get_many(handle_, keys, count, vectors_per_key, vectors, 0, scalar_kind<scalar_at>(),
                                     counts ? counts : own.data(), &error);
    }
    /* lookups by key from DEVICE memory (usearch_b200_count_many_device, _get_many_device, _filtered_search_many_device):
     * every pointer is a device pointer on the index's GPU, `cuda_stream` a cudaStream_t (NULL = the handle's stream) */
    error_t count_device(vector_key_t const* keys, std::size_t count, std::uint32_t* counts, void* cuda_stream = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_count_many_device(handle_, keys, count, counts, cuda_stream, &e);
        return e;
    }
    /* key i owns rows i * vectors_per_key .. of `vectors`, its oldest entries first; rows past counts[i] are zero */
    template <typename scalar_at>
    error_t get_device(vector_key_t const* keys, std::size_t count, scalar_at* vectors, std::uint32_t* counts,
                       std::size_t vectors_per_key = 1, std::size_t stride_bytes = 0, void* cuda_stream = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_get_many_device(handle_, keys, count, vectors_per_key, vectors, stride_bytes, scalar_kind<scalar_at>(), counts,
                                     cuda_stream, &e);
        return e;
    }
    error_t filtered_search_device(void const* queries, std::size_t queries_count, std::size_t queries_stride, std::size_t wanted,
                                   vector_key_t const* allowed_keys, std::size_t allowed_count, vector_key_t* keys,
                                   distance_t* distances, std::uint32_t* counts, std::uint32_t* computed_distances = nullptr,
                                   std::uint32_t* visited_members = nullptr, void* cuda_stream = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_filtered_search_many_device(handle_, queries, queries_count, queries_stride, wanted, allowed_keys, allowed_count,
                                                 keys, distances, counts, computed_distances, visited_members, cuda_stream, &e);
        return e;
    }
    /* query i filtered by set groups[i]: set g is set_keys[offsets[g] .. offsets[g + 1]] (usearch_b200_grouped_filtered_search_many) */
    template <typename scalar_at>
    error_t grouped_filtered_search(scalar_at const* queries, std::size_t queries_count, std::size_t queries_stride, std::size_t wanted, std::uint32_t const* groups, std::uint64_t const* offsets, std::size_t sets_count,
                                    vector_key_t const* set_keys, vector_key_t* keys, distance_t* distances, std::size_t* counts,
                                    std::uint64_t* computed_distances = nullptr, std::uint64_t* visited_members = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_filtered_search_many(handle_, queries, queries_count, queries_stride, scalar_kind<scalar_at>(), wanted, groups, offsets,
                                                  sets_count, set_keys, keys, distances, counts, computed_distances, visited_members, &e);
        return e;
    }
    error_t grouped_filtered_search_device(void const* queries, std::size_t queries_count, std::size_t queries_stride, std::size_t wanted,
                                           std::uint32_t const* groups, std::uint64_t const* offsets, std::size_t sets_count,
                                           vector_key_t const* set_keys, vector_key_t* keys, distance_t* distances, std::uint32_t* counts,
                                           std::uint32_t* computed_distances = nullptr, std::uint32_t* visited_members = nullptr,
                                           void* cuda_stream = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_filtered_search_many_device(handle_, queries, queries_count, queries_stride, wanted, groups, offsets,
                                                         sets_count, set_keys, keys, distances, counts, computed_distances,
                                                         visited_members, cuda_stream, &e);
        return e;
    }
    /* the exact forms: every query scans exactly the live entries of its set (usearch_b200_grouped_filtered_exact_search_many);
     * `groups` may be NULL with one set */
    template <typename scalar_at>
    error_t grouped_filtered_exact_search(scalar_at const* queries, std::size_t queries_count, std::size_t queries_stride,
                                          std::size_t wanted, std::uint32_t const* groups, std::uint64_t const* offsets,
                                          std::size_t sets_count, vector_key_t const* set_keys, vector_key_t* keys,
                                          distance_t* distances, std::size_t* counts,
                                          std::uint64_t* computed_distances = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_filtered_exact_search_many(handle_, queries, queries_count, queries_stride, scalar_kind<scalar_at>(), wanted,
                                                        groups, offsets, sets_count, set_keys, keys, distances, counts,
                                                        computed_distances, &e);
        return e;
    }
    error_t grouped_filtered_exact_search_device(void const* queries, std::size_t queries_count, std::size_t queries_stride,
                                                 std::size_t wanted, std::uint32_t const* groups, std::uint64_t const* offsets,
                                                 std::size_t sets_count, vector_key_t const* set_keys, vector_key_t* keys,
                                                 distance_t* distances, std::uint32_t* counts,
                                                 std::uint32_t* computed_distances = nullptr, void* cuda_stream = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_filtered_exact_search_many_device(handle_, queries, queries_count, queries_stride, wanted, groups, offsets,
                                                               sets_count, set_keys, keys, distances, counts, computed_distances,
                                                               cuda_stream, &e);
        return e;
    }
    /* query i searches every live entry whose key is NOT in set groups[i] (usearch_b200_grouped_excluded_search_many);
     * `groups` may be NULL with one set */
    template <typename scalar_at>
    error_t grouped_excluded_search(scalar_at const* queries, std::size_t queries_count, std::size_t queries_stride, std::size_t wanted,
                                    std::uint32_t const* groups, std::uint64_t const* offsets, std::size_t sets_count,
                                    vector_key_t const* set_keys, vector_key_t* keys, distance_t* distances, std::size_t* counts,
                                    std::uint64_t* computed_distances = nullptr, std::uint64_t* visited_members = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_excluded_search_many(handle_, queries, queries_count, queries_stride, scalar_kind<scalar_at>(), wanted, groups, offsets,
                                                  sets_count, set_keys, keys, distances, counts, computed_distances, visited_members, &e);
        return e;
    }
    error_t grouped_excluded_search_device(void const* queries, std::size_t queries_count, std::size_t queries_stride, std::size_t wanted,
                                           std::uint32_t const* groups, std::uint64_t const* offsets, std::size_t sets_count,
                                           vector_key_t const* set_keys, vector_key_t* keys, distance_t* distances, std::uint32_t* counts,
                                           std::uint32_t* computed_distances = nullptr, std::uint32_t* visited_members = nullptr,
                                           void* cuda_stream = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_excluded_search_many_device(handle_, queries, queries_count, queries_stride, wanted, groups, offsets,
                                                         sets_count, set_keys, keys, distances, counts, computed_distances,
                                                         visited_members, cuda_stream, &e);
        return e;
    }
    template <typename scalar_at>
    error_t grouped_excluded_exact_search(scalar_at const* queries, std::size_t queries_count, std::size_t queries_stride,
                                          std::size_t wanted, std::uint32_t const* groups, std::uint64_t const* offsets,
                                          std::size_t sets_count, vector_key_t const* set_keys, vector_key_t* keys,
                                          distance_t* distances, std::size_t* counts,
                                          std::uint64_t* computed_distances = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_excluded_exact_search_many(handle_, queries, queries_count, queries_stride, scalar_kind<scalar_at>(), wanted,
                                                        groups, offsets, sets_count, set_keys, keys, distances, counts,
                                                        computed_distances, &e);
        return e;
    }
    error_t grouped_excluded_exact_search_device(void const* queries, std::size_t queries_count, std::size_t queries_stride,
                                                 std::size_t wanted, std::uint32_t const* groups, std::uint64_t const* offsets,
                                                 std::size_t sets_count, vector_key_t const* set_keys, vector_key_t* keys,
                                                 distance_t* distances, std::uint32_t* counts,
                                                 std::uint32_t* computed_distances = nullptr, void* cuda_stream = nullptr) const {
        usearch_error_t e = nullptr;
        usearch_b200_grouped_excluded_exact_search_many_device(handle_, queries, queries_count, queries_stride, wanted, groups, offsets,
                                                               sets_count, set_keys, keys, distances, counts, computed_distances,
                                                               cuda_stream, &e);
        return e;
    }
    /* index_dense.hpp:774-779. `exact`: predicate(key) is called once per live entry on the host and the entries it accepts
     * are scanned on the device; otherwise the predicate goes to usearch_filtered_search, which cannot run a host callback
     * on the device and reports so. `thread` is accepted and ignored. */
    template <typename scalar_at, typename predicate_at>
    search_result_t filtered_search(scalar_at const* vector, std::size_t wanted, predicate_at&& predicate, std::size_t /*thread*/ = 0,
                                    bool exact = false) const {
        search_result_t result;
        if (!wanted) return result;
        result.keys_.resize(wanted);
        result.distances_.resize(wanted);
        usearch_error_t error = nullptr;
        if (!exact) {
            /* the predicate's own constness is kept: `state` only carries its address back to the call */
            typedef typename std::remove_reference<predicate_at>::type predicate_t;
            struct trampoline_t {
                static int call(vector_key_t key, void* state) { return (*static_cast<predicate_t*>(state))(key) ? 1 : 0; }
            };
            void* const state = const_cast<void*>(static_cast<void const*>(&predicate));
            result.count = usearch_filtered_search(handle_, vector, scalar_kind<scalar_at>(), wanted, &trampoline_t::call, state,
                                                   result.keys_.data(), result.distances_.data(), &error);
            if (error) return result.failed(error);
            return result;
        }
        std::vector<vector_key_t> live(size()), allowed;
        live.resize(usearch_b200_export_keys(handle_, 0, live.size(), live.data(), &error));
        if (error) return result.failed(error);
        for (vector_key_t key : live)
            if (predicate(key)) allowed.push_back(key);
        std::uint64_t const offsets[2] = {0, allowed.size()};
        std::size_t count = 0;
        std::uint64_t computed = 0;
        usearch_b200_grouped_filtered_exact_search_many(handle_, vector, 1, 0, scalar_kind<scalar_at>(), wanted, nullptr, offsets, 1,
                                                        allowed.data(), result.keys_.data(), result.distances_.data(), &count, &computed,
                                                        &error);
        if (error) return result.failed(error);
        result.count = count;
        result.computed_distances = computed;
        return result;
    }
    /* index_dense.hpp:1595-1608, the live keys in slot order */
    void export_keys(vector_key_t* keys, std::size_t offset, std::size_t limit) const {
        usearch_b200_export_keys(handle_, offset, limit, keys, nullptr);
    }
    bool multi() const { return usearch_b200_multi(handle_); }
    /* index_dense.hpp:1615-1650: an independent index with the same contents */
    state_result_t copy() const;

    /* stats_t and the three stats functions of index_gt (index.hpp:3133-3225) */
    struct stats_t {
        std::size_t nodes = 0, edges = 0, max_edges = 0, allocated_bytes = 0;
    };
    stats_t stats() const {
        stats_t total;
        usearch_b200_levels_stats(handle_, nullptr, 0, &total.nodes, nullptr);
        return total;
    }
    /* levels 0 .. max_level into stats_per_level, the head of a node counted on level 0 only; returns their sum */
    stats_t stats(stats_t* stats_per_level, std::size_t max_level) const {
        std::vector<stats_t> levels(usearch_b200_levels_stats(handle_, nullptr, 0, nullptr, nullptr));
        usearch_b200_levels_stats(handle_, &levels.data()->nodes, levels.size(), nullptr, nullptr);
        stats_t total;
        for (std::size_t l = 0; l <= max_level; ++l) {
            stats_t const s = l < levels.size() ? levels[l] : stats_t();
            stats_per_level[l] = s;
            total.nodes += s.nodes, total.edges += s.edges, total.max_edges += s.max_edges, total.allocated_bytes += s.allocated_bytes;
        }
        return total;
    }
    /* the nodes on `level` and above, the 10-byte head of a node (key and level) counted on every level */
    stats_t stats(std::size_t level) const {
        std::vector<stats_t> levels(level + 1);
        stats(levels.data(), level);
        stats_t s = levels[level];
        if (level) s.allocated_bytes += 10 * s.nodes;
        return s;
    }

    labeling_result_t remove(vector_key_t key) {
        labeling_result_t result;
        usearch_error_t error = nullptr;
        result.completed = usearch_remove(handle_, key, &error);
        result.error = error;
        return result;
    }
    labeling_result_t rename(vector_key_t from, vector_key_t to) {
        labeling_result_t result;
        usearch_error_t error = nullptr;
        result.completed = usearch_rename(handle_, from, to, &error);
        result.error = error;
        return result;
    }

    /* cluster_result_t (index.hpp:2744-2755) and index_dense_gt::cluster(vector, level) (index_dense.hpp:788-793) */
    struct cluster_result_t {
        error_t error{};
        std::size_t visited_members = 0;
        std::size_t computed_distances = 0;
        struct match_t { struct member_t { vector_key_t key; } member; distance_t distance; } cluster{};
        explicit operator bool() const noexcept { return !error; }
    };
    template <typename scalar_at> cluster_result_t cluster(scalar_at const* vector, std::size_t level, std::size_t /*thread*/ = 0) const {
        cluster_result_t result;
        std::uint64_t computed = 0, visited = 0;
        usearch_error_t error = nullptr;
        usearch_b200_cluster_many(handle_, vector, 1, 0, scalar_kind<scalar_at>(), level, &result.cluster.member.key,
                                  &result.cluster.distance, &computed, &visited, &error);
        result.error = error;
        result.computed_distances = computed;
        result.visited_members = visited;
        return result;
    }

    /* the batch driver of python/lib.cpp:261-319 as one call */
    template <typename scalar_at>
    batch_result_t search_many(scalar_at const* vectors, std::size_t queries, std::size_t wanted, std::size_t stride_bytes = 0) const {
        batch_result_t batch;
        if (!wanted || !queries) return batch;
        if (!stride_bytes) stride_bytes = (dimensions() * (scalar_kind<scalar_at>() == usearch_scalar_b1_k ? 1 : sizeof(scalar_at) * 8) + 7) / 8;
        batch.keys.resize(queries * wanted);
        batch.distances.resize(queries * wanted);
        batch.counts.resize(queries);
        std::vector<std::uint64_t> computed(queries), visited(queries);
        usearch_error_t error = nullptr;
        usearch_b200_search_many_stats(handle_, vectors, queries, stride_bytes, scalar_kind<scalar_at>(), wanted, batch.keys.data(),
                                       batch.distances.data(), batch.counts.data(), computed.data(), visited.data(), &error);
        batch.error = error;
        for (std::size_t i = 0; i != queries; ++i) batch.computed_distances += computed[i], batch.visited_members += visited[i];
        return batch;
    }

    /* join_result_t (index.hpp:1577-1590) and index_dense_gt::join (index_dense.hpp:1762-1786): every engaged pair is
     * written as man_to_woman[key of this] = key of women, woman_to_man[key of women] = key of this, in the reference's
     * export order, into any map-like pair of outputs (`operator[]` on keys). The one-thread run of the reference. */
    struct join_result_t {
        error_t error{};
        std::size_t intersection_size = 0;
        std::size_t engagements = 0;
        std::size_t visited_members = 0;
        std::size_t computed_distances = 0;
        explicit operator bool() const noexcept { return !error; }
    };
    template <typename man_to_woman_at, typename woman_to_man_at>
    join_result_t join(index_dense_t const& women, std::size_t max_proposals, bool exact, man_to_woman_at&& man_to_woman,
                       woman_to_man_at&& woman_to_man) const {
        join_result_t result;
        std::size_t const slots = capacity() < women.capacity() ? capacity() : women.capacity();
        std::vector<vector_key_t> a(slots), b(slots);
        std::size_t stats[4] = {0, 0, 0, 0};
        usearch_error_t error = nullptr;
        std::size_t const pairs = usearch_b200_join(handle_, women.handle_, max_proposals, exact, a.data(), b.data(), slots, stats, &error);
        result.error = error;
        if (error) return result;
        for (std::size_t i = 0; i != pairs; ++i) {
            man_to_woman[a[i]] = b[i];
            woman_to_man[b[i]] = a[i];
        }
        result.intersection_size = stats[0];
        result.engagements = stats[1];
        result.visited_members = stats[2];
        result.computed_distances = stats[3];
        return result;
    }
};

struct index_dense_state_result_t {
    index_dense_t index;
    error_t error{};
    explicit operator bool() const noexcept { return !error; }
};

inline index_dense_t::state_result_t index_dense_t::make(metric_punned_t metric, index_dense_config_t config) {
    state_result_t state;
    usearch_init_options_t options;
    std::memset(&options, 0, sizeof(options));
    options.metric_kind = metric.metric_kind();
    options.quantization = metric.scalar_kind();
    options.dimensions = metric.dimensions();
    options.connectivity = config.connectivity;
    options.expansion_add = config.expansion_add;
    options.expansion_search = config.expansion_search;
    options.multi = config.multi;
    usearch_error_t error = nullptr;
    state.index.handle_ = usearch_init(&options, &error);
    state.error = error;
    return state;
}

inline index_dense_t::state_result_t index_dense_t::copy() const {
    state_result_t state;
    usearch_error_t error = nullptr;
    state.index.handle_ = usearch_b200_copy(handle_, &error);
    state.error = error;
    return state;
}

/* usearch_exact_search: brute force over a raw host matrix, keys are dataset row numbers (exact_search_t,
 * index_plugins.hpp:2071-2164). Strides in bytes; the dataset may exceed GPU memory. `threads` host threads stage it. */
template <typename scalar_at>
inline error_t exact_search(scalar_at const* dataset, std::size_t dataset_size, std::size_t dataset_stride, scalar_at const* queries,
                            std::size_t queries_size, std::size_t queries_stride, std::size_t dimensions, usearch_metric_kind_t metric,
                            std::size_t wanted, vector_key_t* keys, std::size_t keys_stride, distance_t* distances,
                            std::size_t distances_stride, std::size_t threads = 0) {
    usearch_error_t e = nullptr;
    usearch_exact_search(dataset, dataset_size, dataset_stride, queries, queries_size, queries_stride, scalar_kind<scalar_at>(), dimensions,
                         metric, wanted, threads, keys, keys_stride, distances, distances_stride, &e);
    return e;
}

/* the same over DEVICE arrays, enqueued on `cuda_stream` (a cudaStream_t; nullptr = the default stream) without waiting */
inline error_t exact_search_device(void const* dataset, std::size_t dataset_size, std::size_t dataset_stride, void const* queries,
                                   std::size_t queries_size, std::size_t queries_stride, usearch_scalar_kind_t scalar,
                                   std::size_t dimensions, usearch_metric_kind_t metric, std::size_t wanted, vector_key_t* keys,
                                   std::size_t keys_stride, distance_t* distances, std::size_t distances_stride,
                                   void* cuda_stream = nullptr) {
    usearch_error_t e = nullptr;
    usearch_b200_exact_search_device(dataset, dataset_size, dataset_stride, queries, queries_size, queries_stride, scalar, dimensions,
                                     metric, wanted, keys, keys_stride, distances, distances_stride, cuda_stream, &e);
    return e;
}

/* metadata is taken from the file */
inline index_dense_t::state_result_t index_dense_t::make(char const* path, bool view) {
    state_result_t state;
    usearch_error_t error = nullptr;
    state.index.handle_ = usearch_init(nullptr, &error);
    if (!error) (view ? usearch_view : usearch_load)(state.index.handle_, path, &error);
    state.error = error;
    return state;
}

} // namespace usearch_b200
