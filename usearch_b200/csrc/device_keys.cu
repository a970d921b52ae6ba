/*
 *  device_keys.cu — lookups by key for callers whose keys are already in HBM: count, get and filtered search. The first
 *  two probe the key -> slot table of device_keys.h, built from the device `keys` array on the first lookup after any
 *  change of the key -> slot relation (`keys_generation`); filtered search needs no table, it sorts the allowed keys on
 *  the device and builds a bitmap over slots from them, for device keys and for host keys uploaded first.
 */
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <climits>

#include "cuda_check.h"
#include "device_keys.h"
#include "frozen_index.h"

namespace usearch_b200 {

namespace {

/* output bytes of one chunk of get_many_device when the chunk-row knob is 0, as in get_many */
constexpr size_t GET_CHUNK_BYTES = 64ull << 20;

char const* const ERR_TOO_MANY_ALLOWED = "Too many allowed keys in one call";

struct claim_cas_t {
    __device__ bool operator()(uint32_t* word, uint32_t slot) const { return atomicCAS(word, EMPTY_SLOT, slot) == EMPTY_SLOT; }
};

__global__ void key_table_build_kernel(uint64_t const* keys, uint32_t n, uint64_t free_key, key_cell_t* cells, uint64_t mask) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        uint64_t const key = keys[s];
        if (key != free_key) key_table_insert(cells, mask, key, s, claim_cas_t{});
    }
}

__global__ void key_table_count_kernel(key_cell_t const* cells, uint64_t mask, uint64_t const* keys, size_t n, uint32_t* counts) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t c = 0;
        key_table_for_each(cells, mask, keys[i], [&](uint32_t) { ++c; });
        counts[i] = c;
    }
}

/* rows[i * per_key ...] <- the min(count, per_key) lowest slots under keys[i], ascending, then EMPTY_SLOT; counts[i] <- how
 * many. A bounded max-heap keeps the lowest ones while the probe walks the key's cells, and a heap sort orders them. */
__global__ void key_table_select_kernel(key_cell_t const* cells, uint64_t mask, uint64_t const* keys, size_t n, size_t per_key,
                                        uint32_t* rows, uint32_t* counts) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t* heap = rows + i * per_key;
        size_t held = 0;
        auto sift_down = [&](size_t at, size_t end) {
            for (;;) {
                size_t child = 2 * at + 1;
                if (child >= end) return;
                if (child + 1 < end && heap[child + 1] > heap[child]) ++child;
                if (heap[at] >= heap[child]) return;
                uint32_t const t = heap[at]; heap[at] = heap[child]; heap[child] = t;
                at = child;
            }
        };
        key_table_for_each(cells, mask, keys[i], [&](uint32_t slot) {
            if (held < per_key) {
                size_t at = held++;
                heap[at] = slot;
                while (at && heap[(at - 1) / 2] < heap[at]) {
                    size_t const up = (at - 1) / 2;
                    uint32_t const t = heap[at]; heap[at] = heap[up]; heap[up] = t;
                    at = up;
                }
            } else if (slot < heap[0]) {
                heap[0] = slot;
                sift_down(0, held);
            }
        });
        for (size_t end = held; end > 1; --end) {
            uint32_t const t = heap[0]; heap[0] = heap[end - 1]; heap[end - 1] = t;
            sift_down(0, end - 1);
        }
        for (size_t j = held; j < per_key; ++j) heap[j] = EMPTY_SLOT;
        counts[i] = (uint32_t)held;
    }
}

/* row i of `out` (`out_stride` bytes apart, `bpv` bytes written) <- row slots[i] of `vectors`, or zeros for EMPTY_SLOT.
 * gather_rows_kernel writes packed rows and has no empty row; this one also serves strided caller rows. */
__global__ void gather_rows_or_zero_kernel(uint4 const* vectors, uint32_t const* slots, size_t n, uint32_t chunks16, uint32_t bpv,
                                           uint8_t* out, size_t out_stride) {
    bool const whole = ((bpv | out_stride | (uintptr_t)out) & 15) == 0, words = ((bpv | out_stride | (uintptr_t)out) & 3) == 0;
    for (size_t i = blockIdx.x; i < n; i += gridDim.x) {
        uint32_t const slot = slots[i];
        uint4 const* src = vectors + (size_t)slot * chunks16;
        uint8_t* dst = out + i * out_stride;
        for (uint32_t j = threadIdx.x; j < chunks16; j += blockDim.x) {
            uint4 const v = slot == EMPTY_SLOT ? make_uint4(0, 0, 0, 0) : __ldg(src + j);
            uint32_t const at = j * 16;
            if (whole) {
                *reinterpret_cast<uint4*>(dst + at) = v;
                continue;
            }
            auto w = [&](uint32_t k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }; /* registers, not a local array */
            uint32_t const end = min(bpv - at, 16u);
            if (words)
                for (uint32_t b = 0; b < end; b += 4) *reinterpret_cast<uint32_t*>(dst + at + b) = w(b >> 2);
            else
                for (uint32_t b = 0; b < end; ++b) dst[at + b] = (uint8_t)(w(b >> 2) >> (8 * (b & 3)));
        }
    }
}

unsigned grid_for(size_t items, int sm_count) { return (unsigned)std::max<size_t>(1, std::min<size_t>((items + 255) / 256, (size_t)sm_count * 16)); }

} // namespace

char const* frozen_index_t::ensure_key_table(cudaStream_t s) {
    if (key_table.cells.ptr && key_table.generation == keys_generation) return nullptr;
    size_t const cells = key_table_cells(size - count_deleted);
    if (char const* e = key_table.cells.reserve(cells)) return e;
    CU(cudaMemsetAsync(key_table.cells.ptr, 0xFF, cells * sizeof(key_cell_t), s));
    key_table.mask = cells - 1;
    key_table_build_kernel<<<grid_for(size, stream.sm_count), 256, 0, s>>>(d.keys, (uint32_t)size, free_key, key_table.cells.ptr,
                                                                          key_table.mask);
    CU(cudaGetLastError());
    kernel_launches += 1;
    key_table.generation = keys_generation;
    return nullptr;
}

/* usearch_b200_count_many with device keys and counts */
char const* frozen_index_t::count_many_device(uint64_t const* keys, size_t n, uint32_t* counts_out, cudaStream_t s) {
    if (char const* e = ensure_context()) return e;
    if (!n) return nullptr;
    if (!loaded || !size) {
        CU(cudaMemsetAsync(counts_out, 0, n * 4, s));
    } else {
        if (char const* e = ensure_key_table(s)) return e;
        key_table_count_kernel<<<grid_for(n, stream.sm_count), 256, 0, s>>>(key_table.cells.ptr, key_table.mask, keys, n, counts_out);
        CU(cudaGetLastError());
        kernel_launches += 1;
    }
    CU(cudaStreamSynchronize(s));
    return nullptr;
}

/* usearch_b200_get_many with device keys and outputs, key i owning rows i * max_per_key ..: the slots of every row first
 * (one thread per key), then per chunk of rows one gather, straight into the caller's rows when no cast is needed, else
 * into scratch and cast from there. */
char const* frozen_index_t::get_many_device(uint64_t const* keys, size_t n, size_t max_per_key, void* out, size_t out_stride,
                                            uint32_t out_scalar, uint32_t* counts_out, cudaStream_t s) {
    if (char const* e = ensure_context()) return e;
    if (!bits_per_scalar(out_scalar)) return "Unknown scalar kind!";
    if (!n) return nullptr;
    size_t const out_bytes = (dimensions * bits_per_scalar(out_scalar) + 7) / 8, bpv = d.bytes_per_vector;
    if (out_stride == 0) out_stride = out_bytes;
    uint8_t* const out_rows = static_cast<uint8_t*>(out);
    if (!loaded || !size || !max_per_key) { /* no rows to read: the counts, and every row, are zero */
        CU(cudaMemsetAsync(counts_out, 0, n * 4, s));
        if (max_per_key && out_stride >= out_bytes) CU(cudaMemset2DAsync(out_rows, out_stride, 0, out_bytes, n * max_per_key, s));
        CU(cudaStreamSynchronize(s));
        return nullptr;
    }
    if (out_stride < out_bytes) return "Output stride is smaller than a vector";
    if (max_per_key > 0xFFFFFFFFull / n) return "Too many rows in one call";
    size_t const total = n * max_per_key;

    if (char const* e = ensure_key_table(s)) return e;
    if (char const* e = lookup_slots.reserve(total)) return e;
    key_table_select_kernel<<<grid_for(n, stream.sm_count), 256, 0, s>>>(key_table.cells.ptr, key_table.mask, keys, n, max_per_key,
                                                                        lookup_slots.ptr, counts_out);
    CU(cudaGetLastError());
    kernel_launches += 1;

    bool const cast = out_scalar != scalar;
    uint4 const* const rows = reinterpret_cast<uint4 const*>(d.vectors);
    if (!cast) {
        gather_rows_or_zero_kernel<<<(unsigned)std::min<size_t>(total, 65535), 128, 0, s>>>(rows, lookup_slots.ptr, total, d.chunks16,
                                                                                          (uint32_t)bpv, out_rows, out_stride);
        CU(cudaGetLastError());
        kernel_launches += 1;
        CU(cudaStreamSynchronize(s));
        return nullptr;
    }
    /* zero rows cast to zero rows in every kind; a packed output takes the cast directly, a strided one through scratch so
     * that the bytes between the caller's rows stay untouched */
    size_t chunk = tune.get_chunk_rows > 0 ? (size_t)tune.get_chunk_rows : std::max<size_t>(1, GET_CHUNK_BYTES / std::max(bpv, out_bytes));
    chunk = std::min(chunk, total);
    bool const packed = out_stride == out_bytes;
    if (char const* e = lookup_gathered.reserve(chunk * bpv)) return e;
    if (!packed)
        if (char const* e = lookup_casted.reserve(chunk * out_bytes)) return e;
    for (size_t lo = 0; lo < total; lo += chunk) {
        size_t const m = std::min(chunk, total - lo);
        gather_rows_or_zero_kernel<<<(unsigned)std::min<size_t>(m, 65535), 128, 0, s>>>(rows, lookup_slots.ptr + lo, m, d.chunks16,
                                                                                      (uint32_t)bpv, lookup_gathered.ptr, bpv);
        CU(cudaGetLastError());
        uint8_t* const dst = packed ? out_rows + lo * out_bytes : lookup_casted.ptr;
        if (char const* e = cast_rows_device(lookup_gathered.ptr, bpv, scalar, dst, out_bytes, out_scalar, dimensions, m, s)) return e;
        if (!packed)
            CU(cudaMemcpy2DAsync(out_rows + lo * out_stride, out_stride, lookup_casted.ptr, out_bytes, out_bytes, m,
                                 cudaMemcpyDeviceToDevice, s));
        kernel_launches += 2;
    }
    CU(cudaStreamSynchronize(s));
    return nullptr;
}

/* usearch_b200_filtered_search_many with device queries, allowed keys and outputs: the allowed keys sorted on the device
 * into `allowed_keys`, then the slot bitmap the search filters by */
char const* frozen_index_t::filtered_search_device(void const* d_queries, size_t nq, size_t stride, size_t k, uint64_t const* allowed,
                                                   size_t allowed_count, uint64_t* d_keys, float* d_dists, uint32_t* d_counts,
                                                   uint32_t* d_computed, uint32_t* d_visited, cudaStream_t s) {
    if (char const* e = ensure_context()) return e;
    if (nq == 0 || k == 0) return nullptr;
    if (allowed_count > (size_t)INT_MAX) return ERR_TOO_MANY_ALLOWED;
    search_filter_t filter;
    if (loaded && size) {
        int const m = (int)allowed_count;
        if (char const* e = allowed_keys.reserve(std::max<size_t>(allowed_count, 1))) return e;
        if (char const* e = allow_bits.reserve((size + 31) / 32)) return e;
        if (m) {
            size_t temp_bytes = 0;
            CU(cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, allowed, allowed_keys.ptr, m, 0, 64, s));
            if (char const* e = allowed_sort_temp.reserve(temp_bytes)) return e;
            CU(cub::DeviceRadixSort::SortKeys(allowed_sort_temp.ptr, temp_bytes, allowed, allowed_keys.ptr, m, 0, 64, s));
            kernel_launches += 1;
        }
        CU(search_build_allow_bits(d, allowed_keys.ptr, (uint32_t)m, allow_bits.ptr, s));
        filter.allow_bits = allow_bits.ptr;
    }
    return search_device(d_queries, nq, stride, k, d_keys, d_dists, d_counts, d_computed, d_visited, s, false, filter);
}

/* usearch_b200_filtered_search_many and usearch_filtered_search: the host keys staged on the device as given, then sorted
 * and applied by filtered_search_device (cub's sort must not write over its input) */
char const* frozen_index_t::filtered_search_host(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                                                 uint64_t const* allowed, size_t allowed_count, host_results_t const& out, size_t* total) {
    if (nq == 0 || k == 0) return nullptr;
    std::lock_guard<std::mutex> lock(mutex);
    if (!loaded || d.n == 0) return answer_empty(nq, k, out);
    if (allowed_count > (size_t)INT_MAX) return ERR_TOO_MANY_ALLOWED; /* refused before 16 GiB of keys are uploaded */
    return search_round_trip(q, nq, stride, query_scalar, k, out, total,
                             [&](void const* dq, size_t vs, device_results_t const& r) -> char const* {
        if (char const* e = stage_keys(allowed, allowed_count)) return e;
        return filtered_search_device(dq, nq, vs, k, key_stage.ptr, allowed_count, r.keys, r.dists, r.counts, r.computed, r.visited, stream);
    });
}

} // namespace usearch_b200
