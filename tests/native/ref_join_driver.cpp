// The reference's own `index_dense_gt::join` (index_dense.hpp:1762-1786 -> index.hpp:4345-4543) over two saved graphs,
// for the join tests and tools/join_bench.py. Compiled at test time against the reference headers where they lie
// (tests/join_reference.py), never copied. `pinned` swaps both metrics for oracle/metrics_pinned.h, as the oracle does.
#include <cstdint>
#include <cstring>
#include <unordered_map>

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

char const* load(index_t& index, void const* blob, std::size_t length, bool pinned, std::size_t threads) {
    auto loaded = index.load(memory_mapped_file_t(static_cast<byte_t*>(const_cast<void*>(blob)), length));
    if (!loaded) return loaded.error.release();
    if (pinned) {
        metric_punned_t const& old = index.metric();
        std::uintptr_t fn = pinned_for(old.metric_kind(), old.scalar_kind());
        if (!fn) return "No pinned metric for this metric / scalar kind";
        index.change_metric(metric_punned_t::stateless(old.dimensions(), fn, metric_punned_signature_t::array_array_size_k,
                                                       old.metric_kind(), old.scalar_kind()));
    }
    if (!index.try_reserve(index_limits_t(index.size(), threads))) return "Out of memory!";
    return nullptr;
}

} // namespace

// a.join(b) as python/lib.cpp:780-799 drives it, on `threads` threads; `expansion` 0 = max(expansion_search of both).
// Writes the a -> b mapping (`*pairs` entries, any order) and join_result_t's four counters.
extern "C" char const* ref_join_blobs(void const* a_blob, std::size_t a_len, void const* b_blob, std::size_t b_len,
                                      std::size_t max_proposals, std::size_t expansion, int exact, std::size_t threads, int pinned,
                                      std::uint64_t* a_keys, std::uint64_t* b_keys, std::size_t* pairs, std::size_t* stats4) {
#if defined(__FAST_MATH__)
    if (pinned) return "The pinned metric is only exact without -ffast-math";
#endif
    if (threads == 0) threads = 1;
    index_t a, b;
    if (char const* e = load(a, a_blob, a_len, pinned != 0, threads)) return e;
    if (char const* e = load(b, b_blob, b_len, pinned != 0, threads)) return e;
    index_join_config_t config;
    config.max_proposals = max_proposals;
    config.exact = exact != 0;
    config.expansion = expansion ? expansion : (std::max)(a.expansion_search(), b.expansion_search());
    std::unordered_map<std::uint64_t, std::uint64_t> a_to_b;
    dummy_key_to_key_mapping_t b_to_a;
    executor_stl_t executor{threads};
    join_result_t result = a.join(b, config, a_to_b, b_to_a, executor);
    if (!result) return result.error.release();
    std::size_t i = 0;
    for (auto const& kv : a_to_b) a_keys[i] = kv.first, b_keys[i] = kv.second, ++i;
    *pairs = i;
    stats4[0] = result.intersection_size;
    stats4[1] = result.engagements;
    stats4[2] = result.visited_members;
    stats4[3] = result.computed_distances;
    return nullptr;
}
