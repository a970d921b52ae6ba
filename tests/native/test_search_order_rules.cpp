/*
 *  The search's NaN rules (usearch_b200/csrc/search_order.h) against the reference's containers: random sequences of
 *  pushes, pops and bounded inserts over a pool of NaN (two payloads and both signs), +-inf, +-0, ties and finite values.
 *    - `next`: every pop is done twice, by max_heap_gt::shift_down restated (less = a.d > b.d on stored distances), and
 *      as pop_warp does it: every internal node's choice bit from heap_goes_right first, then the walk down those bits,
 *      stopping at the first level where heap_stops_above(last, child). The two heaps must be equal element for element.
 *    - `top`: every insert is placed by std::lower_bound (sorted_buffer_gt::insert) and by top_position under the
 *      kernel's flag, updated by top_may_hold_nan. The positions and the buffers must be equal.
 *  Build: g++ -std=c++17 -O2 -I usearch_b200/csrc; run: ./a.out [sequences]
 */
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "search_order.h"

using namespace usearch_b200;

struct cand_t {
    float d;
    uint32_t s;
};

static uint64_t failures = 0, heap_pops = 0, heap_nan_pops = 0, top_inserts = 0, top_probed = 0;

static bool same(cand_t a, cand_t b) {
    uint32_t x, y;
    std::memcpy(&x, &a.d, 4);
    std::memcpy(&y, &b.d, 4);
    return x == y && a.s == b.s;
}

static bool same(std::vector<cand_t> const& a, std::vector<cand_t> const& b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
        if (!same(a[i], b[i])) return false;
    return true;
}

static void fail(char const* what, std::vector<cand_t> const& before) {
    if (failures < 10) {
        std::printf("FAIL %s on [", what);
        for (cand_t c : before) std::printf(" %g", c.d);
        std::printf(" ]\n");
    }
    ++failures;
}

/* ---- max_heap_gt restated: 0-based, less(a, b) = a.d > b.d ----------------------------------------------------------- */

static bool less_heap(cand_t a, cand_t b) { return a.d > b.d; }

static void shift_up(std::vector<cand_t>& h, size_t i) {
    for (; i && less_heap(h[(i - 1) / 2], h[i]); i = (i - 1) / 2) std::swap(h[(i - 1) / 2], h[i]);
}

static void shift_down(std::vector<cand_t>& h, size_t i) {
    size_t max_idx = i;
    size_t const left = 2 * i + 1, right = 2 * i + 2;
    if (left < h.size() && less_heap(h[max_idx], h[left])) max_idx = left;
    if (right < h.size() && less_heap(h[max_idx], h[right])) max_idx = right;
    if (i != max_idx) {
        std::swap(h[i], h[max_idx]);
        shift_down(h, max_idx);
    }
}

static void pop_reference(std::vector<cand_t>& h) {
    std::swap(h[0], h.back());
    h.pop_back();
    shift_down(h, 0);
}

/* pop_warp's order, 1-based as the kernel stores the heap: choice bits of every internal node, the walk, the stop */
static void pop_warp_order(std::vector<cand_t>& h0) {
    size_t const size = h0.size(), n = size - 1;
    std::vector<cand_t> h(size + 2);
    for (size_t i = 0; i < size; ++i) h[i + 1] = h0[i];
    if (n > 0) {
        cand_t const last = h[size];
        std::vector<bool> right(n + 1, false);
        for (size_t p = 1; 2 * p + 1 <= n; ++p) right[p] = heap_goes_right(h[2 * p].d, h[2 * p + 1].d);
        std::vector<size_t> path; /* path[k] = node on level k + 1 */
        for (size_t p = 1; 2 * p <= n;) {
            p = 2 * p + (right[p] ? 1 : 0);
            path.push_back(p);
        }
        size_t moves = path.size();
        for (size_t k = 0; k < path.size(); ++k)
            if (heap_stops_above(last.d, h[path[k]].d)) { moves = k; break; }
        size_t parent = 1;
        for (size_t k = 0; k < moves; ++k) {
            h[parent] = h[path[k]];
            parent = path[k];
        }
        h[parent] = last;
    }
    h0.assign(h.begin() + 1, h.begin() + (long)size); /* elements 1..n */
}

/* ---- sorted_buffer_gt::insert(element, limit) and the kernel's placement ------------------------------------------- */

static void insert_at(std::vector<cand_t>& t, size_t slot, size_t limit, cand_t c) {
    if (t.size() == limit) t.pop_back();
    t.insert(t.begin() + (long)slot, c);
}

static float pool_value(std::mt19937_64& rng, int kind_count) {
    static uint32_t const nans[] = {0x7FC00000u, 0xFFC00000u, 0x7FFFFFFFu, 0x7FA00001u};
    uint32_t const kind = (uint32_t)(rng() % (uint64_t)kind_count);
    float f;
    switch (kind) {
    case 0: std::memcpy(&f, &nans[rng() % 4], 4); return f;
    case 1: return INFINITY;
    case 2: return -INFINITY;
    case 3: return 0.f;
    case 4: return -0.f;
    case 5: case 6: case 7: return (float)(1 + rng() % 3); /* ties */
    default: return std::ldexp((float)(rng() % 1000) - 500.f, (int)(rng() % 20) - 10);
    }
}

static void run_sequence(std::mt19937_64& rng) {
    int const kinds = 6 + (int)(rng() % 6); /* some sequences are all special values */
    uint32_t const limit = 1 + (uint32_t)(rng() % 40);
    uint32_t const steps = 20 + (uint32_t)(rng() % 200);
    std::vector<cand_t> heap, top;
    bool top_nan = false;
    uint32_t id = 0;
    for (uint32_t step = 0; step < steps; ++step) {
        uint64_t const op = rng() % 8;
        if (op < 3 && !heap.empty()) { /* pop */
            std::vector<cand_t> want = heap, got = heap;
            pop_reference(want);
            pop_warp_order(got);
            ++heap_pops;
            for (cand_t c : heap) heap_nan_pops += std::isnan(c.d) ? 1 : 0;
            if (!same(want, got)) fail("pop", heap);
            heap = want;
            continue;
        }
        cand_t const c{pool_value(rng, kinds), id++};
        if (op < 6) { /* push */
            heap.push_back(c);
            shift_up(heap, heap.size() - 1);
        } else { /* bounded insert into `top` */
            size_t const want = (size_t)(std::lower_bound(top.begin(), top.end(), c,
                                                          [](cand_t const& a, cand_t const& b) { return a.d < b.d; }) -
                                         top.begin());
            size_t const got = top_position([&](uint32_t i) { return top[i].d; }, (uint32_t)top.size(), c.d, top_nan);
            ++top_inserts;
            top_probed += top_nan ? 1 : 0;
            if (want != got) fail("top position", top);
            if (want == limit) continue;
            top_nan = top_may_hold_nan(top_nan, c.d);
            insert_at(top, want, limit, c);
        }
    }
}

int main(int argc, char** argv) {
    uint64_t const sequences = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 200000;
    std::mt19937_64 rng(20261018);
    for (uint64_t i = 0; i < sequences; ++i) run_sequence(rng);
    std::printf("pops: %llu (NaN entries seen %llu), top inserts: %llu (probed %llu), failures: %llu\n",
                (unsigned long long)heap_pops, (unsigned long long)heap_nan_pops, (unsigned long long)top_inserts,
                (unsigned long long)top_probed, (unsigned long long)failures);
    return failures ? 1 : 0;
}
