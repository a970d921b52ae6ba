// What the reference itself reports for a saved graph: its three `stats` functions (index.hpp:3133-3225), `export_keys`
// (index_dense.hpp:1595-1608) and `get`, for the tests of the index surface model (tests/surface_reference.py). Also
// builds the graphs those tests need with the reference's own add / remove / isolate / slot reuse. Compiled at test time
// against the reference headers where they lie, never copied.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include <usearch/index_dense.hpp>

using namespace unum::usearch;
using index_t = index_dense_gt<std::uint64_t, std::uint32_t>;

namespace {

char const* save(index_t const& index, std::uint8_t** blob, std::size_t* length) {
    *length = index.serialized_length();
    *blob = static_cast<std::uint8_t*>(std::malloc(*length));
    if (!*blob) return "Out of memory!";
    auto saved = index.save(memory_mapped_file_t(reinterpret_cast<byte_t*>(*blob), *length));
    if (!saved) return saved.error.release();
    return nullptr;
}

} // namespace

extern "C" {

void ref_surface_free(void* p) { std::free(p); }

// A cos f32 graph of `n` random vectors of `dims`, on one thread, then: 0 = a multi index holding every key twice;
// 1 = every third key removed; 2 = the same, then isolate(); 3 = the same, then n / 4 new keys added, which take the
// removed slots first.
char const* ref_surface_scenario(int which, std::size_t n, std::size_t dims, std::uint8_t** blob, std::size_t* length) {
    index_dense_config_t config(16);
    config.multi = which == 0;
    auto made = index_t::make(metric_punned_t::builtin(dims, metric_kind_t::cos_k, scalar_kind_t::f32_k), config);
    if (!made) return made.error.release();
    index_t& index = made.index;
    if (!index.try_reserve(index_limits_t(2 * n, 1))) return "Out of memory!";
    std::mt19937 rng(7);
    std::normal_distribution<float> normal;
    std::vector<float> v(dims);
    auto add = [&](std::uint64_t key) -> char const* {
        for (float& x : v) x = normal(rng);
        auto added = index.add(key, v.data());
        return added ? nullptr : added.error.release();
    };
    for (std::size_t i = 0; i != n; ++i)
        if (char const* e = add(i)) return e;
    if (which == 0)
        for (std::size_t i = 0; i != n; i += 2)
            if (char const* e = add(i)) return e;
    if (which >= 1) {
        for (std::size_t i = 0; i < n; i += 3)
            if (!index.remove(i)) return "remove failed";
        if (which == 2) index.isolate();
        if (which == 3)
            for (std::size_t i = 0; i != n / 4; ++i)
                if (char const* e = add(1000000 + i)) return e;
    }
    return save(index, blob, length);
}

// Loads `blob` and reports: total4 = stats(); level4[l] = stats(l) for l = 0 .. max_level + 1; per_level4 =
// stats(per_level, max_level) per level, its return value in per_level_total4; keys = export_keys over size() keys.
char const* ref_surface_describe(void const* blob, std::size_t length, std::size_t* max_level, std::size_t* total4,
                                 std::size_t* level4, std::size_t* per_level4, std::size_t* per_level_total4, std::size_t levels_cap,
                                 std::uint64_t* keys, std::size_t keys_cap, std::size_t* nkeys) {
    index_t index;
    auto loaded = index.load(memory_mapped_file_t(static_cast<byte_t*>(const_cast<void*>(blob)), length));
    if (!loaded) return loaded.error.release();
    using stats_t = index_t::stats_t;
    auto put = [](std::size_t* out, stats_t const& s) { out[0] = s.nodes, out[1] = s.edges, out[2] = s.max_edges, out[3] = s.allocated_bytes; };
    std::size_t const top = index.max_level();
    *max_level = top;
    if (top + 2 > levels_cap) return "Too many levels for the output";
    put(total4, index.stats());
    for (std::size_t l = 0; l <= top + 1; ++l) put(level4 + 4 * l, index.stats(l));
    std::vector<stats_t> per(top + 1);
    put(per_level_total4, index.stats(per.data(), top));
    for (std::size_t l = 0; l <= top; ++l) put(per_level4 + 4 * l, per[l]);
    *nkeys = index.size();
    if (*nkeys > keys_cap) return "Too many keys for the output";
    index.export_keys(keys, 0, *nkeys);
    return nullptr;
}

// index.get(key, rows, count(key)) in the stored kind: the rows the reference keeps under `key` (its own order)
char const* ref_surface_get(void const* blob, std::size_t length, std::uint64_t const* keys, std::size_t n, std::uint8_t* rows,
                            std::size_t rows_cap, std::size_t* counts) {
    index_t index;
    auto loaded = index.load(memory_mapped_file_t(static_cast<byte_t*>(const_cast<void*>(blob)), length));
    if (!loaded) return loaded.error.release();
    std::size_t const bpv = index.bytes_per_vector();
    std::size_t at = 0;
    for (std::size_t i = 0; i != n; ++i) {
        std::size_t const c = index.count(keys[i]);
        if (at + c > rows_cap) return "Too many rows for the output";
        std::uint8_t* out = rows + at * bpv;
        switch (index.scalar_kind()) {
        case scalar_kind_t::f32_k: counts[i] = index.get(keys[i], reinterpret_cast<f32_t*>(out), c); break;
        case scalar_kind_t::f64_k: counts[i] = index.get(keys[i], reinterpret_cast<f64_t*>(out), c); break;
        case scalar_kind_t::f16_k: counts[i] = index.get(keys[i], reinterpret_cast<f16_t*>(out), c); break;
        case scalar_kind_t::i8_k: counts[i] = index.get(keys[i], reinterpret_cast<i8_t*>(out), c); break;
        case scalar_kind_t::b1x8_k: counts[i] = index.get(keys[i], reinterpret_cast<b1x8_t*>(out), c); break;
        default: return "Unsupported scalar kind";
        }
        at += counts[i];
    }
    return nullptr;
}

} // extern "C"
