// The reference's f64 index (`index_dense_gt` with scalar_kind_t::f64_k) for the f64 tests and the f64 fixture
// generator. Compiled at test time against the reference headers where they lie (tests/f64_reference.py), never copied.
// `pinned` swaps the metric for tests/native/f64_pinned.h; otherwise the reference's own SimSIMD dispatch runs.
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include <usearch/index_dense.hpp>

#include "f64_pinned.h"

using namespace unum::usearch;
using index_t = index_dense_gt<std::uint64_t, std::uint32_t>;

namespace {

float pin_l2sq(std::size_t a, std::size_t b, std::size_t n) {
    return pinned_l2sq_f64(reinterpret_cast<double const*>(a), reinterpret_cast<double const*>(b), n);
}
float pin_ip(std::size_t a, std::size_t b, std::size_t n) {
    return pinned_ip_f64(reinterpret_cast<double const*>(a), reinterpret_cast<double const*>(b), n);
}
float pin_cos(std::size_t a, std::size_t b, std::size_t n) {
    return pinned_cos_f64(reinterpret_cast<double const*>(a), reinterpret_cast<double const*>(b), n);
}

metric_punned_t make_metric(metric_kind_t m, std::size_t dims, int pinned) {
    if (!pinned) return metric_punned_t::builtin(dims, m, scalar_kind_t::f64_k);
    std::uintptr_t fn = m == metric_kind_t::l2sq_k ? reinterpret_cast<std::uintptr_t>(&pin_l2sq)
                        : m == metric_kind_t::ip_k ? reinterpret_cast<std::uintptr_t>(&pin_ip)
                        : m == metric_kind_t::cos_k ? reinterpret_cast<std::uintptr_t>(&pin_cos)
                                                    : 0;
    if (!fn) return metric_punned_t{};
    return metric_punned_t::stateless(dims, fn, metric_punned_signature_t::array_array_size_k, m, scalar_kind_t::f64_k);
}

bool reserve(index_t& index, std::size_t members, std::size_t threads) {
    index_limits_t limits(std::max(index.capacity(), members), std::max<std::size_t>(threads, 1));
    return index.try_reserve(limits);
}

// scalar kinds by their reference enum values (index_plugins.hpp:113-159)
template <typename fn_at> bool with_kind(int kind, byte_t const* p, fn_at&& fn) {
    switch (static_cast<scalar_kind_t>(kind)) {
    case scalar_kind_t::f64_k: fn(reinterpret_cast<f64_t const*>(p)); return true;
    case scalar_kind_t::f32_k: fn(reinterpret_cast<f32_t const*>(p)); return true;
    case scalar_kind_t::f16_k: fn(reinterpret_cast<f16_t const*>(p)); return true;
    case scalar_kind_t::bf16_k: fn(reinterpret_cast<bf16_t const*>(p)); return true;
    case scalar_kind_t::i8_k: fn(reinterpret_cast<i8_t const*>(p)); return true;
    case scalar_kind_t::b1x8_k: fn(reinterpret_cast<b1x8_t const*>(p)); return true;
    default: return false;
    }
}

} // namespace

extern "C" {

void* f64_make(int metric_char, std::size_t dims, std::size_t connectivity, std::size_t expansion_add, std::size_t expansion_search) {
    index_dense_config_t config;
    config.connectivity = connectivity;
    config.connectivity_base = connectivity * 2;
    config.expansion_add = expansion_add;
    config.expansion_search = expansion_search;
    config.enable_key_lookups = true;
    auto state = index_t::make(metric_punned_t::builtin(dims, static_cast<metric_kind_t>(metric_char), scalar_kind_t::f64_k), config);
    if (!state) return nullptr;
    return new index_t(std::move(state.index));
}

void f64_free(void* h) { delete static_cast<index_t*>(h); }
char const* f64_isa_name(void* h) { return static_cast<index_t*>(h)->metric().isa_name(); }
std::size_t f64_size(void* h) { return static_cast<index_t*>(h)->size(); }
void f64_change_expansion_search(void* h, std::size_t ef) { static_cast<index_t*>(h)->change_expansion_search(ef); }

int f64_pin(void* h, int pinned) {
    auto* index = static_cast<index_t*>(h);
    metric_punned_t const& old = index->metric();
    metric_punned_t metric = make_metric(old.metric_kind(), old.dimensions(), pinned);
    if (metric.missing()) return -1;
    index->change_metric(metric);
    return 0;
}

// rows of `kind` scalars; threads > 1 adds them concurrently as the reference's batch add does
std::size_t f64_add(void* h, std::uint64_t const* keys, void const* rows, int kind, std::size_t n, std::size_t stride, std::size_t threads) {
    auto* index = static_cast<index_t*>(h);
    threads = std::max<std::size_t>(threads, 1);
    if (!reserve(*index, index->size() + n, threads)) return 0;
    std::atomic<std::size_t> done{0}, cursor{0};
    auto work = [&](std::size_t thread) {
        for (std::size_t i; (i = cursor.fetch_add(1)) < n;)
            with_kind(kind, static_cast<byte_t const*>(rows) + i * stride, [&](auto const* v) {
                if (index->add(keys[i], v, thread)) done.fetch_add(1);
            });
    };
    if (threads == 1) work(0);
    else {
        std::vector<std::thread> pool;
        for (std::size_t t = 0; t < threads; ++t) pool.emplace_back(work, t);
        for (auto& t : pool) t.join();
    }
    return done.load();
}

std::size_t f64_remove(void* h, std::uint64_t key) { return static_cast<index_t*>(h)->remove(key).completed; }

// index_dense_gt::isolate (index_dense.hpp:1709-1720): drops every link to a removed entry
void f64_isolate(void* h) { static_cast<index_t*>(h)->isolate(); }

std::size_t f64_serialized_length(void* h) { return static_cast<index_t*>(h)->serialized_length(); }

int f64_save(void* h, void* buffer, std::size_t length) {
    return static_cast<index_t*>(h)->save(memory_mapped_file_t(static_cast<byte_t*>(buffer), length)) ? 0 : -1;
}

int f64_view(void* h, void const* buffer, std::size_t length) {
    memory_mapped_file_t map(static_cast<byte_t*>(const_cast<void*>(buffer)), length);
    return static_cast<index_t*>(h)->view(std::move(map)) ? 0 : -1;
}

// allowed == nullptr: plain search; otherwise filtered_search with "key is in the sorted array `allowed`"
int f64_search(void* h, void const* queries, int kind, std::size_t nq, std::size_t stride, std::size_t wanted, int exact,
               std::uint64_t const* allowed, std::size_t allowed_count, std::uint64_t* keys, float* distances, std::uint64_t* counts,
               std::uint64_t* computed, std::uint64_t* visited) {
    auto* index = static_cast<index_t*>(h);
    if (!reserve(*index, index->size(), 1)) return -1;
    auto predicate = [=](std::uint64_t key) noexcept { return std::binary_search(allowed, allowed + allowed_count, key); };
    for (std::size_t i = 0; i != nq; ++i) {
        bool ok = with_kind(kind, static_cast<byte_t const*>(queries) + i * stride, [&](auto const* q) {
            auto result = allowed ? index->filtered_search(q, wanted, predicate, 0) : index->search(q, wanted, 0, exact != 0);
            counts[i] = result.dump_to(keys + i * wanted, distances + i * wanted, wanted);
            computed[i] = result.computed_distances;
            visited[i] = result.visited_members;
        });
        if (!ok) return -2;
    }
    return 0;
}

int f64_cluster(void* h, double const* queries, std::size_t nq, std::size_t level, std::uint64_t* keys, float* distances,
                std::uint64_t* computed, std::uint64_t* visited) {
    auto* index = static_cast<index_t*>(h);
    if (!reserve(*index, index->size(), 1)) return -1;
    for (std::size_t i = 0; i != nq; ++i) {
        auto result = index->cluster(queries + i * index->dimensions(), level, 0);
        if (!result) return -2;
        keys[i] = result.cluster.member.key;
        distances[i] = result.cluster.distance;
        computed[i] = result.computed_distances;
        visited[i] = result.visited_members;
    }
    return 0;
}

// index_dense_gt::get into `kind` scalars (index_dense.hpp:781-786)
std::size_t f64_get(void* h, std::uint64_t key, int kind, void* out) {
    auto* index = static_cast<index_t*>(h);
    switch (static_cast<scalar_kind_t>(kind)) {
    case scalar_kind_t::f64_k: return index->get(key, static_cast<f64_t*>(out));
    case scalar_kind_t::f32_k: return index->get(key, static_cast<f32_t*>(out));
    case scalar_kind_t::f16_k: return index->get(key, static_cast<f16_t*>(out));
    case scalar_kind_t::bf16_k: return index->get(key, static_cast<bf16_t*>(out));
    case scalar_kind_t::i8_k: return index->get(key, static_cast<i8_t*>(out));
    case scalar_kind_t::b1x8_k: return index->get(key, static_cast<b1x8_t*>(out));
    default: return 0;
    }
}

// exact_search_t over raw f64 matrices (index_plugins.hpp:2071-2164), keys = dataset row numbers
int f64_exact_search(double const* dataset, std::size_t n, double const* queries, std::size_t nq, int metric_char, std::size_t dims,
                     std::size_t wanted, int pinned, std::uint64_t* keys, float* distances) {
    metric_punned_t metric = make_metric(static_cast<metric_kind_t>(metric_char), dims, pinned);
    if (metric.missing()) return -1;
    exact_search_t search;
    exact_search_results_t result = search(reinterpret_cast<byte_t const*>(dataset), n, dims * 8, reinterpret_cast<byte_t const*>(queries),
                                           nq, dims * 8, wanted, metric);
    if (!result) return -3;
    for (std::size_t q = 0; q != nq; ++q) {
        auto row = result.at(q);
        for (std::size_t i = 0; i != wanted; ++i) keys[q * wanted + i] = row[i].offset, distances[q * wanted + i] = row[i].distance;
    }
    return 0;
}

float f64_distance(int metric_char, std::size_t dims, int pinned, double const* a, double const* b) {
    metric_punned_t metric = make_metric(static_cast<metric_kind_t>(metric_char), dims, pinned);
    return metric(reinterpret_cast<byte_t const*>(a), reinterpret_cast<byte_t const*>(b));
}

} // extern "C"
