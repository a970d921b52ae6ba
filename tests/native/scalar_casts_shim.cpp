// The host casts of usearch_b200/csrc/scalar_casts.h (`get`, and the element conversions the device casts share),
// exported for tests/test_scalar_casts.py.
#include "scalar_casts.h"

extern "C" {
int shim_cast_row(uint32_t from, uint32_t to, size_t dims, uint8_t const* src, uint8_t* dst) {
    return usearch_b200::cast_row_host(from, to, dims, src, dst) ? 1 : 0;
}
// element conversions on raw bits, so that a signalling NaN reaches them unquieted
uint16_t shim_f32_to_f16(uint32_t bits) { return usearch_b200::f32_to_f16_bits(usearch_b200::sc_bits_f32(bits)); }
uint16_t shim_f32_to_bf16(uint32_t bits) { return usearch_b200::f32_to_bf16_bits(usearch_b200::sc_bits_f32(bits)); }
uint32_t shim_f16_to_f32(uint16_t h) { return usearch_b200::sc_f32_bits(usearch_b200::f16_bits_to_f32(h)); }
}
