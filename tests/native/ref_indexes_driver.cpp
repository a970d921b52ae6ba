// The reference's `Indexes.search` (python/lib.cpp:321-402) over saved graphs, for the `Indexes` tests. Compiled at test
// time against the reference headers where they lie (tests/indexes_reference.py), never copied. `pinned` swaps every
// metric for oracle/metrics_pinned.h, as the oracle does.
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

#include <usearch/index_dense.hpp>

#include "metrics_pinned.h"

using namespace unum::usearch;
using index_t = index_dense_gt<std::uint64_t, std::uint32_t>;

namespace {

template <typename fn_at> std::uintptr_t fn_addr(fn_at fn) { return reinterpret_cast<std::uintptr_t>(fn); }
#define PIN3(name, type)                                                                                     \
    float pin_##name(std::size_t a, std::size_t b, std::size_t n) {                                          \
        return pinned_##name(reinterpret_cast<type const*>(a), reinterpret_cast<type const*>(b), n);         \
    }
PIN3(l2sq_f32, float)
PIN3(ip_f32, float)
PIN3(cos_f32, float)
PIN3(l2sq_f16, std::uint16_t)
PIN3(ip_f16, std::uint16_t)
PIN3(cos_f16, std::uint16_t)
PIN3(l2sq_i8, std::int8_t)
PIN3(ip_i8, std::int8_t)
PIN3(cos_i8, std::int8_t)
PIN3(hamming_b1, std::uint8_t)

std::uintptr_t pinned_for(metric_kind_t m, scalar_kind_t s) {
    if (s == scalar_kind_t::f32_k && m == metric_kind_t::l2sq_k) return fn_addr(&pin_l2sq_f32);
    if (s == scalar_kind_t::f32_k && m == metric_kind_t::ip_k) return fn_addr(&pin_ip_f32);
    if (s == scalar_kind_t::f32_k && m == metric_kind_t::cos_k) return fn_addr(&pin_cos_f32);
    if (s == scalar_kind_t::f16_k && m == metric_kind_t::l2sq_k) return fn_addr(&pin_l2sq_f16);
    if (s == scalar_kind_t::f16_k && m == metric_kind_t::ip_k) return fn_addr(&pin_ip_f16);
    if (s == scalar_kind_t::f16_k && m == metric_kind_t::cos_k) return fn_addr(&pin_cos_f16);
    if (s == scalar_kind_t::i8_k && m == metric_kind_t::l2sq_k) return fn_addr(&pin_l2sq_i8);
    if (s == scalar_kind_t::i8_k && m == metric_kind_t::ip_k) return fn_addr(&pin_ip_i8);
    if (s == scalar_kind_t::i8_k && m == metric_kind_t::cos_k) return fn_addr(&pin_cos_i8);
    if (s == scalar_kind_t::b1x8_k && m == metric_kind_t::hamming_k) return fn_addr(&pin_hamming_b1);
    return 0;
}

char const* load(index_t& index, void const* blob, std::size_t length, bool pinned, std::size_t expansion) {
    auto loaded = index.load(memory_mapped_file_t(static_cast<byte_t*>(const_cast<void*>(blob)), length));
    if (!loaded) return loaded.error.release();
    if (pinned) {
        metric_punned_t const& old = index.metric();
        std::uintptr_t fn = pinned_for(old.metric_kind(), old.scalar_kind());
        if (!fn) return "No pinned metric for this metric / scalar kind";
        index.change_metric(metric_punned_t::stateless(old.dimensions(), fn, metric_punned_signature_t::array_array_size_k,
                                                       old.metric_kind(), old.scalar_kind()));
    }
    index.change_expansion_search(expansion);
    return nullptr;
}

} // namespace

// `blobs` are loaded once each; the group's members are blobs[order[0]], blobs[order[1]], ... (an index may be a member
// more than once, as in the reference). Then the loop of python/lib.cpp:350-390 on one thread: members in order, every
// query searched with `index_dense_gt::search` (which casts the queries from `query_scalar` for itself) and folded into
// its row with `search_result_t::merge_into`, rows starting at count 0. Rows are first filled with dump_to's padding (key
// 0, signalling NaN); `computed` / `visited` receive the per-query sums over members.
extern "C" char const* ref_indexes_search_blobs(void const* const* blobs, std::size_t const* lengths, std::size_t blob_count,
                                                std::size_t const* order, std::size_t members, std::size_t expansion, int pinned,
                                                void const* queries, std::size_t nq, std::size_t stride, int query_scalar,
                                                std::size_t wanted, int exact, std::uint64_t* keys, float* distances,
                                                std::uint64_t* counts, std::uint64_t* computed, std::uint64_t* visited) {
#if defined(__FAST_MATH__)
    if (pinned) return "The pinned metric is only exact without -ffast-math";
#endif
    std::vector<index_t> loaded(blob_count);
    for (std::size_t i = 0; i != blob_count; ++i) {
        if (char const* e = load(loaded[i], blobs[i], lengths[i], pinned != 0, expansion)) return e;
        if (!loaded[i].try_reserve(index_limits_t(loaded[i].size(), 1))) return "Out of memory!";
    }
    for (std::size_t i = 0; i != nq * wanted; ++i) keys[i] = 0, distances[i] = std::numeric_limits<float>::signaling_NaN();
    for (std::size_t i = 0; i != nq; ++i) counts[i] = computed[i] = visited[i] = 0;
    auto const* base = static_cast<byte_t const*>(queries);
    for (std::size_t m = 0; m != members; ++m) {
        index_t& index = loaded[order[m]];
        for (std::size_t i = 0; i != nq; ++i) {
            byte_t const* q = base + i * stride;
            char const* error = nullptr;
            auto fold = [&](index_t::search_result_t&& result) {
                if (!result) {
                    error = result.error.release();
                    return;
                }
                counts[i] = result.merge_into(keys + i * wanted, distances + i * wanted, counts[i], wanted);
                computed[i] += result.computed_distances;
                visited[i] += result.visited_members;
            };
            switch (static_cast<scalar_kind_t>(query_scalar)) {
            case scalar_kind_t::f32_k: fold(index.search(reinterpret_cast<f32_t const*>(q), wanted, 0, exact != 0)); break;
            case scalar_kind_t::f16_k: fold(index.search(reinterpret_cast<f16_t const*>(q), wanted, 0, exact != 0)); break;
            case scalar_kind_t::i8_k: fold(index.search(reinterpret_cast<i8_t const*>(q), wanted, 0, exact != 0)); break;
            case scalar_kind_t::b1x8_k: fold(index.search(reinterpret_cast<b1x8_t const*>(q), wanted, 0, exact != 0)); break;
            default: return "Unsupported query scalar kind";
            }
            if (error) return error;
        }
    }
    return nullptr;
}
