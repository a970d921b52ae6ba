// Native unit test of the device key -> slot table (usearch_b200/csrc/device_keys.h) run on the host: the same insert and
// probe the CUDA kernels run, with the claim made by a plain compare-and-set. No CUDA, no GPU.
#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>

#include "device_keys.h"

using namespace usearch_b200;

#define EXPECT(cond)                                                               \
    do {                                                                           \
        if (!(cond)) {                                                             \
            std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            return 1;                                                              \
        }                                                                          \
    } while (0)

struct claim_t {
    bool operator()(uint32_t* word, uint32_t slot) const {
        if (*word != EMPTY_SLOT) return false;
        *word = slot;
        return true;
    }
};

/* the table the build kernel makes from slot -> key, inserting the slots in `order` */
static std::vector<key_cell_t> build(std::vector<uint64_t> const& keys, uint64_t free_key, std::vector<uint32_t> const& order,
                                     size_t live) {
    std::vector<key_cell_t> cells(key_table_cells(live));
    for (key_cell_t& c : cells) c.key = ~0ull, c.slot = EMPTY_SLOT, c.unused = ~0u;
    for (uint32_t s : order)
        if (keys[s] != free_key) key_table_insert(cells.data(), cells.size() - 1, keys[s], s, claim_t());
    return cells;
}

static std::vector<uint32_t> found(std::vector<key_cell_t> const& cells, uint64_t key) {
    std::vector<uint32_t> slots;
    key_table_for_each(cells.data(), cells.size() - 1, key, [&](uint32_t s) { slots.push_back(s); });
    std::sort(slots.begin(), slots.end());
    return slots;
}

int main() {
    EXPECT(sizeof(key_cell_t) == 16 && alignof(key_cell_t) == 16);
    EXPECT(key_table_cells(0) == 64 && key_table_cells(32) == 64 && key_table_cells(33) == 128);
    for (size_t live : {1ul, 31ul, 64ul, 1000ul, 4097ul, 10000000ul}) {
        size_t const cells = key_table_cells(live);
        EXPECT((cells & (cells - 1)) == 0 && cells >= 64 && cells >= 2 * live && (cells == 64 || cells < 4 * live));
    }

    // a multi index: one key with 1000 entries, keys with 1..5 entries, key 0, clustered hashes, removed slots
    uint64_t const free_key = ~0ull;
    std::mt19937_64 rng(11);
    std::vector<uint64_t> keys;
    for (uint32_t s = 0; s < 1000; ++s) keys.push_back(42);
    for (uint32_t k = 0; k < 3000; ++k)
        for (uint32_t r = 0; r <= k % 5; ++r) keys.push_back(k * 0x9E3779B97F4A7C15ull);
    std::shuffle(keys.begin(), keys.end(), rng);
    size_t live = 0;
    for (size_t s = 0; s < keys.size(); ++s) {
        if (s % 13 == 0) keys[s] = free_key;
        live += keys[s] != free_key;
    }

    // what the host map finds, per key
    key_map_t map;
    map.rebuild(keys, free_key, keys.size());
    auto want = [&](uint64_t key) {
        std::vector<uint32_t> slots;
        map.for_each(key, [&](uint32_t s, size_t) { slots.push_back(s); return true; });
        std::sort(slots.begin(), slots.end());
        return slots;
    };

    std::vector<uint32_t> order(keys.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = (uint32_t)i;
    for (int trial = 0; trial < 5; ++trial) {
        if (trial) std::shuffle(order.begin(), order.end(), rng);
        else std::reverse(order.begin(), order.end());
        std::vector<key_cell_t> const cells = build(keys, free_key, order, live);
        size_t used = 0;
        for (key_cell_t const& c : cells) used += c.slot != EMPTY_SLOT;
        EXPECT(used == live && 2 * used <= cells.size());
        EXPECT((ptrdiff_t)found(cells, 42).size() == std::count(keys.begin(), keys.end(), 42ull) && found(cells, 42).size() > 900);
        EXPECT(found(cells, 42) == want(42));
        for (uint32_t k = 0; k < 3000; ++k) EXPECT(found(cells, k * 0x9E3779B97F4A7C15ull) == want(k * 0x9E3779B97F4A7C15ull));
        EXPECT(found(cells, free_key).empty() && found(cells, 7).empty() && found(cells, 1ull << 40).empty());
    }
    std::printf("DEVICE_KEYS_OK\n");
    return 0;
}
