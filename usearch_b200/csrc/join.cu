/*
 *  join.cu — `join` (index.hpp:4345-4543, index_dense.hpp:1762-1786) and `pairwise_distance` by key
 *  (index_dense.hpp:808-862) on the GPU.
 *
 *  join: the reference pops a free man, runs `women.search(man, i)` for his i-th proposal (index_gt::search, no predicate:
 *  removed women can be proposed to) and proposes to the last result. index_gt::search runs with
 *  ef = max(expansion, count) and ends with sort + shrink(count) (index.hpp:3052-3073), so for every i <= expansion the
 *  result is the first i rows of one search with count min(P, expansion), counters included; exact search has the same
 *  prefix property (its order does not depend on count). So:
 *    1. ONE batched launch of the search kernel (or the exact kernel) answers proposals 1..min(P, expansion) of every man:
 *       the men's rows already in HBM are the queries, the women's handle runs with no deleted bits (no predicate) and
 *       with keys = slots, so the results are women slots;
 *    2. a proposal i > expansion (only when the caller asks for P > expansion) is a search of its own with count i, run
 *       for all men the first time the replay needs it;
 *    3. pair_distances_kernel gives, per proposal column, metric(woman, man): the husband's distance of the reference;
 *    4. join_resolve.h replays the one-thread FIFO on the host.
 */
#include <algorithm>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "cuda_check.h"
#include "frozen_index.h"
#include "join_resolve.h"

namespace usearch_b200 {

namespace {

/* adds the wall-clock milliseconds of its scope to `to` */
struct elapsed_into_t {
    double& to;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    ~elapsed_into_t() { to += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};

constexpr size_t JOIN_CHUNK = 1u << 18; /* men per search launch: bounds the result buffers */

struct join_scratch_t {
    device_buffer_t<uint64_t> iota, keys;
    device_buffer_t<float> dists, pair_out;
    device_buffer_t<uint32_t> counts, computed, visited, slot_a, slot_b;
};

/* the women's handle as index_gt::search sees it: every slot a candidate (no predicate), results reported as slots,
 * expansion_search = the join's expansion. Restored when the join ends. */
struct as_plain_graph_t {
    frozen_index_t& ix;
    device_index_t saved;
    size_t saved_expansion;
    as_plain_graph_t(frozen_index_t& w, uint64_t const* slot_keys, size_t expansion) : ix(w), saved(w.d), saved_expansion(w.expansion_search) {
        ix.d.keys = slot_keys;
        ix.d.deleted_bits = nullptr;
        ix.expansion_search = expansion;
    }
    ~as_plain_graph_t() {
        ix.d = saved;
        ix.expansion_search = saved_expansion;
    }
};

} // namespace

char const* frozen_index_t::join(frozen_index_t& other, size_t max_proposals, bool exact, std::vector<uint64_t>& a_keys,
                                 std::vector<uint64_t>& b_keys, size_t stats_out[4]) {
    a_keys.clear();
    b_keys.clear();
    for (int i = 0; i < 4; ++i) stats_out[i] = 0;
    for (int i = 0; i < 3; ++i) last_join_ms[i] = 0.f;
    if (this == &other) return "Can't join with itself, consider copying";
    /* both handles for the whole call, always in the same order so that two joins in opposite directions cannot deadlock */
    frozen_index_t* first = this < &other ? this : &other;
    frozen_index_t* second = this < &other ? &other : this;
    std::lock_guard<std::mutex> lock_first(first->mutex);
    std::lock_guard<std::mutex> lock_second(second->mutex);
    if (metric != other.metric || scalar != other.scalar || dimensions != other.dimensions)
        return "Can't join indexes of different metrics, scalar kinds or dimensions";
    if (stream.device != other.stream.device) return "Can't join indexes that live on different devices";
    if (shards || other.shards) return "Can't join a sharded handle: it holds one shard of its index";
    if (max_proposals > JOIN_MAX_PROPOSALS) return "max_proposals above 65535 would overflow the per-man proposal counter";

    /* index.hpp:4369-4380: the smaller side proposes; `size()` counts removed entries too */
    bool const swapped = other.size < size;
    frozen_index_t& men = swapped ? other : *this;
    frozen_index_t& women = swapped ? *this : other;
    size_t const nm = men.size, nw = women.size;
    if (!nm) return nullptr; /* the reference would take log(0) here */
    if (!men.loaded || !women.loaded || men.d.n < nm || women.d.n < nw) return "Index is not on the device";
    size_t const P = join_proposals(nm, max_proposals);
    size_t expansion = std::max(expansion_search, other.expansion_search); /* python/lib.cpp:790 */
    if (!expansion) expansion = 64;                                         /* index.hpp:3029-3030 */
    if (char const* e = women.ensure_context()) return e;
    cudaStream_t const s = women.stream;

    join_scratch_t js;
    if (char const* e = js.iota.reserve(nw)) return e;
    if (char const* e = iota_u64_device(js.iota.ptr, nw, s)) return e;
    as_plain_graph_t plain(women, js.iota.ptr, expansion);
    size_t const vs = men.d.vec_stride;
    size_t const chunk = std::min(nm, JOIN_CHUNK);

    /* one batched search with count k over every man: per man his k result slots / distances, count and counters */
    std::vector<uint32_t> h_slots, h_counts, h_computed, h_visited;
    std::vector<float> h_dists;
    std::vector<uint64_t> h_keys;
    double search_ms = 0, pairs_ms = 0;
    auto search_all = [&](size_t k) -> char const* {
        elapsed_into_t timer{search_ms};
        h_slots.resize(nm * k); h_dists.resize(nm * k); h_keys.resize(chunk * k);
        h_counts.resize(nm); h_computed.resize(nm); h_visited.resize(nm);
        if (char const* e = js.keys.reserve(chunk * k)) return e;
        if (char const* e = js.dists.reserve(chunk * k)) return e;
        if (char const* e = js.counts.reserve(chunk)) return e;
        if (char const* e = js.computed.reserve(chunk)) return e;
        if (char const* e = js.visited.reserve(chunk)) return e;
        for (size_t begin = 0; begin < nm; begin += chunk) {
            size_t const nq = std::min(chunk, nm - begin);
            void const* queries = men.d.vectors + begin * vs;
            if (exact) {
                if (char const* e = exact_search_device(women.d, women.stream.sm_count, queries, nq, vs, k, false, true, js.keys.ptr, js.dists.ptr,
                                                        js.counts.ptr, women.exact_scratch, s))
                    return e;
                women.kernel_launches += 2;
            } else if (char const* e = women.search_device(queries, nq, vs, k, js.keys.ptr, js.dists.ptr, js.counts.ptr, js.computed.ptr,
                                                           js.visited.ptr, s))
                return e;
            CU(cudaMemcpyAsync(h_keys.data(), js.keys.ptr, nq * k * 8, cudaMemcpyDeviceToHost, s));
            CU(cudaMemcpyAsync(h_dists.data() + begin * k, js.dists.ptr, nq * k * 4, cudaMemcpyDeviceToHost, s));
            CU(cudaMemcpyAsync(h_counts.data() + begin, js.counts.ptr, nq * 4, cudaMemcpyDeviceToHost, s));
            if (!exact) {
                CU(cudaMemcpyAsync(h_computed.data() + begin, js.computed.ptr, nq * 4, cudaMemcpyDeviceToHost, s));
                CU(cudaMemcpyAsync(h_visited.data() + begin, js.visited.ptr, nq * 4, cudaMemcpyDeviceToHost, s));
            }
            CU(cudaStreamSynchronize(s));
            for (size_t j = 0; j < nq * k; ++j) h_slots[begin * k + j] = (uint32_t)h_keys[j];
        }
        if (exact) /* search_exact_ (index.hpp:4252-4268) measures every slot and visits none */
            for (size_t m = 0; m < nm; ++m) { h_computed[m] = (uint32_t)nw; h_visited[m] = 0; }
        return nullptr;
    };

    /* metric(woman, man) for the woman each man proposes to in one column: one launch */
    std::vector<uint32_t> man_slots(nm);
    for (size_t m = 0; m < nm; ++m) man_slots[m] = (uint32_t)m;
    if (char const* e = js.slot_b.reserve(nm)) return e;
    if (char const* e = js.slot_a.reserve(nm)) return e;
    if (char const* e = js.pair_out.reserve(nm)) return e;
    CU(cudaMemcpyAsync(js.slot_b.ptr, man_slots.data(), nm * 4, cudaMemcpyHostToDevice, s));
    auto swapped_distances = [&](join_column_t& col) -> char const* {
        elapsed_into_t timer{pairs_ms};
        col.from_woman.resize(nm);
        CU(cudaMemcpyAsync(js.slot_a.ptr, col.woman.data(), nm * 4, cudaMemcpyHostToDevice, s));
        if (char const* e = pair_distances_device(women.d, men.d, js.slot_a.ptr, js.slot_b.ptr, nm, js.pair_out.ptr, s)) return e;
        women.kernel_launches += 1;
        CU(cudaMemcpyAsync(col.from_woman.data(), js.pair_out.ptr, nm * 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        return nullptr;
    };
    /* column i from row min(i, count) - 1 of a search with count k */
    auto take_column = [&](join_column_t& col, size_t i, size_t k) {
        col.woman.resize(nm); col.distance.resize(nm); col.computed.resize(nm); col.visited.resize(nm);
        for (size_t m = 0; m < nm; ++m) {
            size_t const found = h_counts[m];
            if (!found) { col.woman[m] = JOIN_MISSING; col.distance[m] = 0.f; }
            else {
                size_t const row = m * k + std::min(i, found) - 1;
                col.woman[m] = h_slots[row];
                col.distance[m] = h_dists[row];
            }
            col.computed[m] = h_computed[m];
            col.visited[m] = h_visited[m];
        }
    };

    /* columns 1..K from one search; K = min(P, expansion) (exact: every column) */
    size_t const K = exact ? P : std::min(P, expansion);
    if (char const* e = search_all(K)) return e;
    std::vector<join_column_t> columns(P + 1);
    std::vector<bool> ready(P + 1, false), taken(P + 1, false);
    for (size_t i = 1; i <= K; ++i) { take_column(columns[i], i, K); taken[i] = true; }
    auto column = [&](size_t i, join_column_t const*& out) -> char const* {
        if (!ready[i]) {
            if (!taken[i]) { /* a proposal beyond the expansion: its own search, count = ef = i */
                if (char const* e = search_all(i)) return e;
                take_column(columns[i], i, i);
                taken[i] = true;
            }
            for (size_t m = 0; m < nm; ++m)
                if (columns[i].woman[m] >= nw) return "A proposal search returned no candidates";
            if (char const* e = swapped_distances(columns[i])) return e;
            ready[i] = true;
        }
        out = &columns[i];
        return nullptr;
    };

    std::vector<uint32_t> man_to_woman;
    join_stats_t st;
    double replay_ms = 0;
    double const before = search_ms + pairs_ms;
    {
        elapsed_into_t timer{replay_ms};
        if (char const* e = join_replay(nm, nw, P, column, man_to_woman, st)) return e;
    }
    /* wall clock: proposal search (launches and copies back) | pair distances | the host replay without the columns it
     * waited for */
    last_join_ms[0] = (float)search_ms;
    last_join_ms[1] = (float)pairs_ms;
    last_join_ms[2] = (float)(replay_ms - (search_ms + pairs_ms - before));

    /* export (index.hpp:4522-4532): ascending men slots; removed entries carry the free key */
    a_keys.reserve(st.intersection_size);
    b_keys.reserve(st.intersection_size);
    for (size_t m = 0; m < nm; ++m) {
        uint32_t const w = man_to_woman[m];
        if (w == JOIN_MISSING) continue;
        uint64_t const man_key = men.host_keys[m], woman_key = women.host_keys[w];
        a_keys.push_back(swapped ? woman_key : man_key);
        b_keys.push_back(swapped ? man_key : woman_key);
    }
    stats_out[0] = st.intersection_size;
    stats_out[1] = st.engagements;
    stats_out[2] = st.visited_members;
    stats_out[3] = st.computed_distances;
    return nullptr;
}

char const* frozen_index_t::pairwise_distances(uint64_t const* left, uint64_t const* right, size_t n, float* out) {
    std::lock_guard<std::mutex> lock(mutex);
    float const infinite = FLT_MAX; /* aggregated_distances_t defaults (index_dense.hpp:752-757) */
    for (size_t i = 0; i < n; ++i) out[i] = infinite;
    if (!n || !size || !loaded) return nullptr;
    build_key_map();
    /* every (left slot, right slot) combination of every request, then the minimum per request on the host */
    std::vector<uint32_t> sa, sb;
    std::vector<size_t> owner;
    std::vector<uint32_t> ls, rs;
    for (size_t i = 0; i < n; ++i) {
        ls.clear(); rs.clear();
        key_map.for_each(left[i], [&](uint32_t slot, size_t) { ls.push_back(slot); return true; });
        key_map.for_each(right[i], [&](uint32_t slot, size_t) { rs.push_back(slot); return true; });
        for (uint32_t a : ls)
            for (uint32_t b : rs) { sa.push_back(a); sb.push_back(b); owner.push_back(i); }
    }
    if (sa.empty()) return nullptr;
    if (char const* e = ensure_context()) return e;
    size_t const pairs = sa.size();
    device_buffer_t<uint32_t> d_a, d_b;
    device_buffer_t<float> d_out;
    if (char const* e = d_a.reserve(pairs)) return e;
    if (char const* e = d_b.reserve(pairs)) return e;
    if (char const* e = d_out.reserve(pairs)) return e;
    CU(cudaMemcpyAsync(d_a.ptr, sa.data(), pairs * 4, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_b.ptr, sb.data(), pairs * 4, cudaMemcpyHostToDevice, stream));
    if (char const* e = pair_distances_device(d, d, d_a.ptr, d_b.ptr, pairs, d_out.ptr, stream)) return e;
    kernel_launches += 1;
    std::vector<float> h(pairs);
    CU(cudaMemcpyAsync(h.data(), d_out.ptr, pairs * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    /* one pair per request unless `multi`: the distance as it is (NaN included); a multi index folds with std::min as the
     * reference's loop does (index_dense.hpp:842-857) */
    for (size_t j = 0; j < pairs; ++j) out[owner[j]] = multi ? std::min(out[owner[j]], h[j]) : h[j];
    return nullptr;
}

} // namespace usearch_b200
