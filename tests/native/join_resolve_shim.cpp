// C entry over usearch_b200/csrc/join_resolve.h for tests/test_join_resolve.py: the replay fed with precomputed columns.
// Columns are dense [columns x men] arrays; asking for a column past `columns` is an error.
#include <cstddef>
#include <cstdint>
#include <vector>

#include "join_resolve.h"

using namespace usearch_b200;

extern "C" char const* join_replay_columns(size_t men, size_t women, size_t max_proposals, size_t columns, uint32_t const* woman,
                                           float const* distance, float const* from_woman, uint64_t const* computed,
                                           uint64_t const* visited, uint32_t* man_to_woman_out, size_t* stats4_out, size_t* asked_out) {
    std::vector<join_column_t> cols(columns + 1);
    std::vector<bool> ready(columns + 1, false);
    size_t asked = 0;
    auto column = [&](size_t i, join_column_t const*& out) -> char const* {
        if (i == 0 || i > columns) return "column out of range";
        if (!ready[i]) {
            size_t const o = (i - 1) * men;
            join_column_t& c = cols[i];
            c.woman.assign(woman + o, woman + o + men);
            c.distance.assign(distance + o, distance + o + men);
            c.from_woman.assign(from_woman + o, from_woman + o + men);
            c.computed.assign(computed + o, computed + o + men);
            c.visited.assign(visited + o, visited + o + men);
            ready[i] = true;
            asked = i > asked ? i : asked;
        }
        out = &cols[i];
        return nullptr;
    };
    std::vector<uint32_t> m2w;
    join_stats_t st;
    if (char const* e = join_replay(men, women, join_proposals(men, max_proposals), column, m2w, st)) return e;
    for (size_t m = 0; m < men; ++m) man_to_woman_out[m] = m2w[m];
    stats4_out[0] = st.intersection_size;
    stats4_out[1] = st.engagements;
    stats4_out[2] = st.visited_members;
    stats4_out[3] = st.computed_distances;
    *asked_out = asked;
    return nullptr;
}
