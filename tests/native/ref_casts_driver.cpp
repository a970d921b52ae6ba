/*
 *  ref_casts_driver.cpp — TEST INFRASTRUCTURE: the reference's scalar casts, exported.
 *
 *  Compiled at test time by tests/cast_reference.py against the unmodified reference headers, with the defines of the
 *  oracle's parity build (USEARCH_USE_SIMSIMD=1, USEARCH_USE_FP16LIB=0), so that the casts are the ones the oracle's
 *  reference library runs. tests/test_scalar_casts.py and tests/native/test_scalar_casts.cpp hold
 *  usearch_b200/csrc/scalar_casts.h to it.
 */
#include <cstddef>
#include <cstring>

#include <usearch/index_dense.hpp>

using namespace unum::usearch;

extern "C" {

/* cast_gt<from, to> (index_plugins.hpp:1105-1224) over `rows` dense rows: casts_punned_t::make(to).from[from], what
 * index_dense_gt holds as `casts_` and runs in add_ / search_ (casts_.from) and, with the roles swapped, in get_
 * (casts_.to). Same kinds copy, as those callers do when the cast declines. A b1 target is OR-ed into the caller's bytes
 * past the last whole byte (cast_to_b1x8_gt clears dims / 8 bytes only). Returns 0 on success. */
int ref_cast(int from_char, int to_char, void const* src, std::size_t rows, std::size_t dimensions, void* dst) {
    scalar_kind_t const from = static_cast<scalar_kind_t>(from_char), to = static_cast<scalar_kind_t>(to_char);
    std::size_t const from_bytes = (dimensions * bits_per_scalar(from) + 7) / 8;
    std::size_t const to_bytes = (dimensions * bits_per_scalar(to) + 7) / 8;
    cast_punned_t cast = casts_punned_t::make(to).from[from];
    if (!cast || !from_bytes || !to_bytes) return -1;
    for (std::size_t r = 0; r != rows; ++r) {
        byte_t const* in = static_cast<byte_t const*>(src) + r * from_bytes;
        byte_t* out = static_cast<byte_t*>(dst) + r * to_bytes;
        if (!cast(in, dimensions, out)) std::memcpy(out, in, to_bytes);
    }
    return 0;
}

} // extern "C"
