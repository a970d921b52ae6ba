/*
 *  device_keys.h — the key -> slot table that device lookups probe in HBM (plain C++11 when no CUDA compiler reads it,
 *  so tests/native/test_device_keys.cpp runs the same insert and probe on the host).
 *
 *  Open addressing with linear probing over a power-of-two number of 16-byte cells {key, slot, unused}: one probe is one
 *  aligned 16-byte load and needs no read of keys[slot]. A cell is empty while its slot is EMPTY_SLOT; an inserter claims
 *  it by compare-and-swap on the slot word and then writes the key, and every probe runs in a later launch than the
 *  inserts. A multi index holds one cell per (key, slot), so which cell an entry lands in depends on the order the
 *  inserts win their claims, but the set of slots found under each key does not.
 */
#pragma once
#include <cstddef>
#include <cstdint>

#include "key_map.h"

namespace usearch_b200 {

struct alignas(16) key_cell_t {
    uint64_t key;
    uint32_t slot; /* EMPTY_SLOT: the cell is free (all bytes 0xFF is an empty table) */
    uint32_t unused;
};

/* cells for `live` entries: a power of two, at least 64 and at least 2 x live, so the load factor stays <= 1/2 */
inline size_t key_table_cells(size_t live) {
    size_t cells = 64;
    while (cells < 2 * live) cells <<= 1;
    return cells;
}

/* (key, slot) into the first cell of key's probe sequence that `claim(&cell.slot, slot)` takes */
template <class claim_t>
USEARCH_B200_HOST_DEVICE inline void key_table_insert(key_cell_t* cells, uint64_t mask, uint64_t key, uint32_t slot, claim_t claim) {
    for (uint64_t h = key_hash(key) & mask;; h = (h + 1) & mask)
        if (cells[h].slot == EMPTY_SLOT && claim(&cells[h].slot, slot)) {
            cells[h].key = key;
            return;
        }
}

/* visit(slot) for every entry stored under `key`, in probe order */
template <class visit_t>
USEARCH_B200_HOST_DEVICE inline void key_table_for_each(key_cell_t const* cells, uint64_t mask, uint64_t key, visit_t visit) {
    for (uint64_t h = key_hash(key) & mask;; h = (h + 1) & mask) {
        key_cell_t const c = cells[h];
        if (c.slot == EMPTY_SLOT) return;
        if (c.key == key) visit(c.slot);
    }
}

} // namespace usearch_b200
