/*
 *  Every f32 bit pattern through f32 -> f16 and f32 -> bf16, and every f16 / bf16 pattern back to f32: the element
 *  conversions of usearch_b200/csrc/scalar_casts.h against the reference's own cast_gt (`ref_cast` of
 *  tests/native/ref_casts_driver.cpp, loaded from the library given as argv[1]). A mismatch prints the input bits and
 *  both outputs.
 *
 *  Build: g++ -O2 -std=c++17 -I usearch_b200/csrc test_scalar_casts.cpp -ldl
 *  Run:   ./a.out <ref_casts_driver library> [stride]   (stride 1, the default, is all 2^32 patterns)
 */
#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "scalar_casts.h"

using namespace usearch_b200;

using ref_cast_t = int (*)(int, int, void const*, size_t, size_t, void*);

static ref_cast_t ref_cast;
static unsigned long long failures = 0;

static void report(char const* what, uint32_t in, uint32_t want, uint32_t got) {
    if (++failures <= 20) std::printf("%s: input %08x reference %08x ours %08x\n", what, in, want, got);
}

/* f32 -> `to` for the patterns first, first + stride, ... below 2^32, in chunks */
static void sweep_from_f32(uint32_t to, char const* what, uint64_t stride) {
    size_t const chunk = 1u << 22;
    std::vector<uint32_t> in(chunk);
    std::vector<uint16_t> want(chunk);
    uint64_t next = 0, checked = 0;
    while (next < (1ull << 32)) {
        size_t n = 0;
        for (; n < chunk && next < (1ull << 32); ++n, next += stride) in[n] = (uint32_t)next;
        if (ref_cast(SCALAR_F32, to, in.data(), 1, n, want.data())) { std::printf("ref_cast failed\n"); std::exit(2); }
        for (size_t i = 0; i < n; ++i) {
            float f;
            std::memcpy(&f, &in[i], 4);
            uint16_t const got = to == SCALAR_F16 ? f32_to_f16_bits(f) : f32_to_bf16_bits(f);
            if (got != want[i]) report(what, in[i], want[i], got);
        }
        checked += n;
    }
    std::printf("%s: %llu patterns\n", what, (unsigned long long)checked);
}

/* every 16-bit pattern of `from` -> f32 */
static void sweep_to_f32(uint32_t from, char const* what) {
    std::vector<uint16_t> in(1u << 16);
    std::vector<uint32_t> want(1u << 16);
    for (uint32_t i = 0; i < (1u << 16); ++i) in[i] = (uint16_t)i;
    if (ref_cast(from, SCALAR_F32, in.data(), 1, in.size(), want.data())) { std::printf("ref_cast failed\n"); std::exit(2); }
    for (uint32_t i = 0; i < (1u << 16); ++i) {
        float const f = from == SCALAR_F16 ? f16_bits_to_f32(in[i]) : bf16_bits_to_f32(in[i]);
        uint32_t got;
        std::memcpy(&got, &f, 4);
        if (got != want[i]) report(what, in[i], want[i], got);
    }
    std::printf("%s: 65536 patterns\n", what);
}

int main(int argc, char** argv) {
    if (argc < 2) { std::printf("usage: %s <reference library> [stride]\n", argv[0]); return 2; }
    void* lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
    if (!lib) { std::printf("dlopen: %s\n", dlerror()); return 2; }
    ref_cast = reinterpret_cast<ref_cast_t>(dlsym(lib, "ref_cast"));
    if (!ref_cast) { std::printf("no ref_cast in %s\n", argv[1]); return 2; }
    uint64_t const stride = argc > 2 ? std::strtoull(argv[2], nullptr, 10) : 1;
    if (stride == 0) { std::printf("stride must be positive\n"); return 2; }
    sweep_to_f32(SCALAR_F16, "f16 -> f32");
    sweep_to_f32(SCALAR_BF16, "bf16 -> f32");
    sweep_from_f32(SCALAR_F16, "f32 -> f16", stride);
    sweep_from_f32(SCALAR_BF16, "f32 -> bf16", stride);
    std::printf("failures: %llu\n", failures);
    return failures ? 1 : 0;
}
