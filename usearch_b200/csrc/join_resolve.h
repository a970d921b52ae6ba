/*
 *  join_resolve.h — the host half of `join` (plain C++11, no CUDA): the reference's stable-marriage loop
 *  (index.hpp:4345-4543, `unum::usearch::join`) replayed decision for decision as its one-thread run makes them.
 *  Unit-tested natively against the reference's own proposals in tests/test_join_resolve.py.
 *
 *  The searches and distances it needs arrive as COLUMNS: column i holds, for every man, what proposal i of that man
 *  is — the woman he proposes to (`candidates.back()` of `women.search(man, i)`), the distance of that match
 *  (metric(man, woman)), the distance the other way round (metric(woman, man), what she measures when he is her husband
 *  and someone else proposes) and the two counters of that search. A provider builds a column the first time the
 *  replay asks for it; the device side (join.cu) answers columns 1..min(P, expansion) from one batched search.
 */
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <vector>

namespace usearch_b200 {

struct join_stats_t { /* join_result_t, index.hpp:1577-1590 */
    size_t intersection_size = 0, engagements = 0, visited_members = 0, computed_distances = 0;
};

struct join_column_t {
    std::vector<uint32_t> woman;     /* [men] slot of the woman proposal i goes to */
    std::vector<float> distance;     /* [men] metric(man, woman): `match.distance` */
    std::vector<float> from_woman;   /* [men] metric(woman, man): her distance to him once he is her husband */
    std::vector<uint64_t> computed;  /* [men] computed_distances of that search */
    std::vector<uint64_t> visited;   /* [men] visited_members of that search */
};

constexpr uint32_t JOIN_MISSING = 0xFFFFFFFFu;
constexpr size_t JOIN_MAX_PROPOSALS = 65535; /* the reference counts proposals in uint16_t */

/* `max_proposals == 0` (index.hpp:4378-4379): log(men) + threads, truncated, then clamped to the men. This library
 * replays the one-thread run, so `threads` is 1 unless a caller wants the value a wider executor would use. */
inline size_t join_proposals(size_t men, size_t max_proposals, size_t threads = 1) {
    if (max_proposals == 0) max_proposals = (size_t)(std::log((double)men) + (double)threads);
    return max_proposals < men ? max_proposals : men;
}

/*
 *  The replay. `men` / `women` are the sizes AFTER the role swap (men <= women), removed entries included.
 *  `column(i, out)` (i >= 1) sets `out` to column i and returns NULL, or returns an error message.
 *  On success `man_to_woman[m]` is the woman of man m or JOIN_MISSING; the pairs are exported in ascending man order.
 */
template <class column_at>
char const* join_replay(size_t men, size_t women, size_t max_proposals, column_at&& column, std::vector<uint32_t>& man_to_woman,
                        join_stats_t& stats) {
    stats = join_stats_t{};
    man_to_woman.assign(men, JOIN_MISSING);
    if (!men) return nullptr;
    std::vector<uint32_t> woman_to_man(women, JOIN_MISSING);
    std::vector<float> husband_distance(women, 0.f); /* metric(woman, husband), measured when he proposed */
    std::vector<uint16_t> proposals(men, 0);
    std::deque<uint32_t> free_men; /* ring_gt: push at one end, pop at the other, initially in slot order */
    for (size_t m = 0; m < men; ++m) free_men.push_back((uint32_t)m);
    while (!free_men.empty()) {
        uint32_t const m = free_men.front();
        free_men.pop_front();
        if (proposals[m] >= max_proposals) continue; /* out of proposals: dropped, stays single */
        size_t const i = ++proposals[m];
        join_column_t const* col = nullptr;
        if (char const* e = column(i, col)) return e;
        stats.visited_members += col->visited[m];
        stats.computed_distances += col->computed[m];
        uint32_t const w = col->woman[m];
        if (w >= women) return "A proposal search returned no candidates";
        uint32_t const husband = woman_to_man[w];
        if (husband == JOIN_MISSING) {
            man_to_woman[m] = w;
            woman_to_man[w] = m;
            husband_distance[w] = col->from_woman[m];
            stats.engagements += 1;
        } else if (husband_distance[w] > col->distance[m]) { /* strict: on a tie she keeps her husband */
            man_to_woman[husband] = JOIN_MISSING;
            man_to_woman[m] = w;
            woman_to_man[w] = m;
            husband_distance[w] = col->from_woman[m];
            stats.engagements += 1;
            free_men.push_back(husband);
        } else
            free_men.push_back(m);
    }
    for (size_t m = 0; m < men; ++m)
        if (man_to_woman[m] != JOIN_MISSING) stats.intersection_size += 1;
    return nullptr;
}

} // namespace usearch_b200
