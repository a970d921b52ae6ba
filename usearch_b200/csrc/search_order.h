/*
 *  search_order.h — where the search's `next` heap and `top` buffer put an element when a distance is NaN. Plain C++
 *  (host and device): search_kernel.cu and warp_primitives.cuh run these rules, tests/native/test_search_order_rules.cpp
 *  holds them to std::lower_bound and to a restatement of max_heap_gt::shift_down.
 *
 *  `next` (max_heap_gt, index.hpp:819-834, distances stored as +d with reversed compares): shift_down keeps `best` =
 *  last.d, moves it to le.d if last.d > le.d, then to re.d if best > re.d, and stops when neither moved. When le.d is a
 *  number, the element goes right iff re.d < min(last.d, le.d), i.e. iff re.d < le.d and last.d > re.d. When le.d is
 *  NaN, last.d > le.d is false, so best stays last.d and the element goes right iff last.d > re.d. So the child the walk
 *  can take is fixed without looking at `last`:
 *
 *    right  iff  re.d < le.d || le.d is NaN,   left otherwise,
 *
 *  and the element moves there iff last.d > child.d. That is the order pop_warp evaluates: choice bits first, the stop
 *  level after.
 *
 *  `top` (sorted_buffer_gt::insert, index.hpp:928-939) puts d at std::lower_bound(top, d). While `top` holds no NaN it is
 *  sorted under `<` (-0 and +0 compare equal), and lower_bound equals the number of stored distances below d, for a
 *  NaN d as well (nothing is below NaN: position 0). A NaN that enters `top` leaves it unsorted, and from then on only
 *  the probe sequence of libstdc++'s lower_bound gives the reference's position.
 */
#pragma once

#include <cstdint>

#if defined(__CUDACC__)
#define SO_HD __host__ __device__ __forceinline__
#else
#define SO_HD inline
#endif

namespace usearch_b200 {

/* shift_down's child: right iff re < le, or le is NaN (ties go left) */
SO_HD bool heap_goes_right(float le, float re) { return re < le || le != le; }

/* the sifted element stays above the chosen child */
SO_HD bool heap_stops_above(float last, float child) { return !(last > child); }

/* std::lower_bound over `len` elements read through `at(i)`, probed as libstdc++ probes (stl_algobase.h,
 * __lower_bound): halve the range, step past the middle iff *middle < d */
template <class At> SO_HD uint32_t probe_lower_bound(At const& at, uint32_t len, float d) {
    uint32_t first = 0;
    while (len > 0) {
        uint32_t const half = len >> 1;
        if (at(first + half) < d) {
            first += half + 1;
            len -= half + 1;
        } else
            len = half;
    }
    return first;
}

/* whether `top` may hold a NaN once d has entered it; the flag never clears (the probe is right either way) */
SO_HD bool top_may_hold_nan(bool has_nan, float d) { return has_nan || d != d; }

/* where `top` puts d: the count of smaller elements (the kernels count with ballots) while `top` holds no NaN, the
 * probe once it may */
template <class At> SO_HD uint32_t top_position(At const& at, uint32_t size, float d, bool has_nan) {
    if (has_nan) return probe_lower_bound(at, size, d);
    uint32_t below = 0;
    for (uint32_t i = 0; i < size; ++i) below += at(i) < d ? 1u : 0u;
    return below;
}

} // namespace usearch_b200
