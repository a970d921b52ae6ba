/*
 *  key_map.h — key -> slot(s) lookup on the host (plain C++11, no CUDA): what index_dense_gt::slot_lookup_ does for the
 *  reference (index_dense.hpp:462-500). Unit-tested natively in tests/native/test_key_map.cpp.
 */
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>

#include "device_index.h"

#ifdef __CUDACC__
#define USEARCH_B200_HOST_DEVICE __host__ __device__
#else
#define USEARCH_B200_HOST_DEVICE
#endif

namespace usearch_b200 {

/* the 64-bit finalizer both key tables hash with: key_map_t here and the table in HBM (device_keys.h) */
USEARCH_B200_HOST_DEVICE inline uint64_t key_hash(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return k;
}

/* key -> slot(s): open addressing over the host copy of the keys, built on first use. Plays the role of
 * index_dense_gt::slot_lookup_ (index_dense.hpp:462-500); a `multi` index keeps one entry per (key, slot). */
struct key_map_t {
    std::vector<uint32_t> cells; /* slot, or EMPTY_SLOT / TOMB */
    std::vector<uint64_t> const* keys = nullptr;
    size_t used = 0;
    bool built = false;
    static constexpr uint32_t TOMB = 0xFFFFFFFEu;
    static size_t hash(uint64_t k) { return (size_t)key_hash(k); }
    void clear() { cells.clear(); used = 0; built = false; }
    void rebuild(std::vector<uint64_t> const& host_keys, uint64_t free_key, size_t expect) {
        keys = &host_keys;
        size_t cap = 64;
        while (cap < 2 * std::max(expect, host_keys.size()) + 2) cap <<= 1;
        cells.assign(cap, EMPTY_SLOT);
        used = 0;
        built = true;
        for (size_t s = 0; s < host_keys.size(); ++s)
            if (host_keys[s] != free_key) insert(host_keys[s], (uint32_t)s);
    }
    void insert(uint64_t key, uint32_t slot) { /* keys->at(slot) == key must already hold */
        if ((used + 1) * 2 > cells.size()) { /* grow: re-insert the live cells */
            std::vector<uint32_t> old;
            old.swap(cells);
            cells.assign(old.size() * 2, EMPTY_SLOT);
            used = 0;
            for (uint32_t c : old)
                if (c != EMPTY_SLOT && c != TOMB) insert((*keys)[c], c);
        }
        size_t const mask = cells.size() - 1;
        size_t h = hash(key) & mask;
        while (cells[h] != EMPTY_SLOT && cells[h] != TOMB) h = (h + 1) & mask;
        cells[h] = slot;
        used += 1;
    }
    template <class F> void for_each(uint64_t key, F&& f) const { /* f(slot, cell index) -> bool keep going */
        if (cells.empty()) return;
        size_t const mask = cells.size() - 1;
        for (size_t h = hash(key) & mask; cells[h] != EMPTY_SLOT; h = (h + 1) & mask)
            if (cells[h] != TOMB && (*keys)[cells[h]] == key)
                if (!f(cells[h], h)) return;
    }
    bool contains(uint64_t key) const {
        bool hit = false;
        for_each(key, [&](uint32_t, size_t) { hit = true; return false; });
        return hit;
    }
    size_t count(uint64_t key) const {
        size_t n = 0;
        for_each(key, [&](uint32_t, size_t) { ++n; return true; });
        return n;
    }
    void erase_cell(size_t h) { cells[h] = TOMB; }
};

} // namespace usearch_b200
