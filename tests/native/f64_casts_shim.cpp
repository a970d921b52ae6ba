// The host casts of `get` out of an f64 index (usearch_b200/csrc/f64_casts.h), exported for tests/test_f64_oracle.py.
#include "f64_casts.h"

extern "C" {
void shim_f64_to_i8(double const* x, size_t dims, int8_t* out) { usearch_b200::cast_f64_to_i8(x, dims, out); }
void shim_f64_to_b1(double const* x, size_t dims, uint8_t* out) { usearch_b200::cast_f64_to_b1(x, dims, out); }
}
