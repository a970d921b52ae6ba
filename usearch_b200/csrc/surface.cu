/*
 *  surface.cu — reading an index back out: the vectors under many keys, the live keys, a full copy of a handle and the
 *  graph's statistics. These are the parts of index_dense_gt that the reference's Python `Index` uses besides search and
 *  mutation (python/lib.cpp:801-809, :924-1003, :1312-1341; index_dense.hpp:1595-1650; index.hpp:3133-3225).
 */
#include "cuda_check.h"
#include "frozen_index.h"
#include "prefilter_bound.h"

#include <algorithm>
#include <cstring>

namespace usearch_b200 {

namespace {

/* output bytes of one chunk of get_many when the chunk-row knob is 0: two chunks in flight keep the device and pinned
 * scratch near 4 x this */
constexpr size_t GET_CHUNK_BYTES = 64ull << 20;
constexpr uint32_t STATS_SMEM_LEVELS = 64;

/* row i of `out` (packed, `bpv` bytes a row) <- row slots[i] of `vectors`, read as whole 16-byte chunks: the inverse of
 * builder.cu's scatter_rows_kernel */
__global__ void gather_rows_kernel(uint4 const* vectors, uint32_t const* slots, uint32_t n, uint32_t chunks16, uint32_t bpv,
                                   uint8_t* out) {
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        uint4 const* src = vectors + (size_t)slots[i] * chunks16;
        uint8_t* dst = out + (size_t)i * bpv;
        for (uint32_t j = threadIdx.x; j < chunks16; j += blockDim.x) {
            uint4 const v = __ldg(src + j);
            uint32_t const at = j * 16;
            if ((bpv & 15u) == 0) {
                *reinterpret_cast<uint4*>(dst + at) = v;
                continue;
            }
            auto w = [&](uint32_t k) { return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w; }; /* registers, not a local array */
            uint32_t const end = min(bpv - at, 16u);
            if ((bpv & 3u) == 0)
                for (uint32_t b = 0; b < end; b += 4) *reinterpret_cast<uint32_t*>(dst + at + b) = w(b >> 2);
            else
                for (uint32_t b = 0; b < end; ++b) dst[at + b] = (uint8_t)(w(b >> 2) >> (8 * (b & 3)));
        }
    }
}

/* edges[l] += the entries != EMPTY_SLOT of every level-l list of slots [0, n). A warp per slot walks its layer-0 row and
 * then its rows on levels 1 .. levels[s], reduces each row in the warp and adds it to the block's per-level sums, which
 * go to `edges` once per block. */
__global__ void graph_stats_kernel(device_index_t const ix, int16_t const* levels, uint32_t n, uint32_t nlevels,
                                   unsigned long long* edges) {
    __shared__ unsigned long long block_edges[STATS_SMEM_LEVELS];
    for (uint32_t l = threadIdx.x; l < STATS_SMEM_LEVELS; l += blockDim.x) block_edges[l] = 0;
    __syncthreads();
    uint32_t const lane = threadIdx.x & 31;
    uint32_t const warps = gridDim.x * (blockDim.x >> 5);
    for (uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < n; s += warps) {
        int const top = levels[s];
        for (int l = 0; l <= top; ++l) {
            uint32_t const width = l ? ix.m : ix.m0;
            uint32_t const* row = l ? ix.upper + ((size_t)ix.upper_base[s] + (size_t)(l - 1)) * ix.m_stride
                                    : ix.nbr0 + (size_t)s * ix.m0_stride;
            uint32_t c = 0;
            for (uint32_t j = lane; j < width; j += 32) c += row[j] != EMPTY_SLOT ? 1u : 0u;
            c = __reduce_add_sync(0xffffffffu, c);
            if (lane == 0 && c) {
                if ((uint32_t)l < STATS_SMEM_LEVELS) atomicAdd(block_edges + l, (unsigned long long)c);
                else atomicAdd(edges + l, (unsigned long long)c);
            }
        }
    }
    __syncthreads();
    for (uint32_t l = threadIdx.x; l < min(nlevels, STATS_SMEM_LEVELS); l += blockDim.x)
        if (block_edges[l]) atomicAdd(edges + l, block_edges[l]);
}

} // namespace

/* index_dense_gt::get for many keys (python/lib.cpp:971-1003): the slots under each key, up to `max_per_key` of them in
 * ascending slot order (the selection get_vectors makes), then per chunk one gather, the cast to `out_scalar` when it
 * differs, and one D2H copy. Chunk c + 1 is gathered on the handle's stream while chunk c is copied on a second one, and
 * the host moves chunk c - 1 from pinned memory into `out` meanwhile. */
char const* frozen_index_t::get_many(uint64_t const* keys, size_t n, size_t max_per_key, void* out, size_t out_stride,
                                     uint32_t out_scalar, size_t* counts, size_t* rows) {
    *rows = 0;
    if (char const* e = ensure_context()) return e;
    if (!bits_per_scalar(out_scalar)) return "Unknown scalar kind!";
    std::fill(counts, counts + n, (size_t)0);
    if (!loaded || !size || !max_per_key || !n) return nullptr;
    size_t const out_bytes = (dimensions * bits_per_scalar(out_scalar) + 7) / 8, bpv = d.bytes_per_vector;
    if (out_stride == 0) out_stride = out_bytes;
    if (out_stride < out_bytes) return "Output stride is smaller than a vector";

    build_key_map();
    std::vector<uint32_t> slots;
    slots.reserve(n);
    for (size_t i = 0; i < n; ++i) {
        size_t const before = slots.size();
        key_map.for_each(keys[i], [&](uint32_t slot, size_t) { slots.push_back(slot); return slots.size() - before < max_per_key; });
        std::sort(slots.begin() + (ptrdiff_t)before, slots.end()); /* insertion order */
        counts[i] = slots.size() - before;
    }
    size_t const total = slots.size();
    if (!total) return nullptr;
    if (total > 0xFFFFFFFFull) return "Too many rows in one call";

    size_t chunk = tune.get_chunk_rows > 0 ? (size_t)tune.get_chunk_rows : std::max<size_t>(1, GET_CHUNK_BYTES / std::max(bpv, out_bytes));
    chunk = std::min(chunk, total);
    bool const cast = out_scalar != scalar;
    device_buffer_t<uint32_t> d_slots;
    device_buffer_t<uint8_t> gathered[2], casted[2];
    pinned_buffer_t<uint8_t> staged[2];
    if (char const* e = d_slots.reserve(total)) return e;
    for (int b = 0; b < 2 && b * chunk < total; ++b) {
        if (char const* e = gathered[b].reserve(chunk * bpv)) return e;
        if (cast)
            if (char const* e = casted[b].reserve(chunk * out_bytes)) return e;
        if (char const* e = staged[b].reserve(chunk * out_bytes)) return e;
    }
    cuda_stream_t copy_stream(stream.device);
    if (char const* e = copy_stream.open()) return e;
    cuda_event_t ready[2], copied[2];
    for (int b = 0; b < 2; ++b) {
        CU(ready[b].create());
        CU(copied[b].create());
    }
    CU(cudaMemcpyAsync(d_slots.ptr, slots.data(), total * 4, cudaMemcpyHostToDevice, stream));

    size_t const chunks = (total + chunk - 1) / chunk;
    auto drain = [&](size_t c) -> char const* { /* chunk c: pinned -> the caller's rows */
        int const b = (int)(c & 1);
        size_t const lo = c * chunk, m = std::min(chunk, total - lo);
        CU(cudaEventSynchronize(copied[b]));
        uint8_t* dst = static_cast<uint8_t*>(out) + lo * out_stride;
        if (out_stride == out_bytes) std::memcpy(dst, staged[b].ptr, m * out_bytes);
        else
            for (size_t r = 0; r < m; ++r) std::memcpy(dst + r * out_stride, staged[b].ptr + r * out_bytes, out_bytes);
        return nullptr;
    };
    for (size_t c = 0; c < chunks; ++c) {
        int const b = (int)(c & 1);
        if (c >= 2) /* frees both buffers of this parity */
            if (char const* e = drain(c - 2)) return e;
        size_t const lo = c * chunk, m = std::min(chunk, total - lo);
        gather_rows_kernel<<<(unsigned)std::min<size_t>(m, 65535), 128, 0, stream>>>(
            reinterpret_cast<uint4 const*>(d.vectors), d_slots.ptr + lo, (uint32_t)m, d.chunks16, (uint32_t)bpv, gathered[b].ptr);
        CU(cudaGetLastError());
        uint8_t const* src = gathered[b].ptr;
        if (cast) {
            if (char const* e = cast_rows_device(gathered[b].ptr, bpv, scalar, casted[b].ptr, out_bytes, out_scalar, dimensions, m, stream))
                return e;
            src = casted[b].ptr;
        }
        CU(cudaEventRecord(ready[b], stream));
        CU(cudaStreamWaitEvent(copy_stream, ready[b], 0));
        CU(cudaMemcpyAsync(staged[b].ptr, src, m * out_bytes, cudaMemcpyDeviceToHost, copy_stream));
        CU(cudaEventRecord(copied[b], copy_stream));
    }
    for (size_t c = chunks >= 2 ? chunks - 2 : 0; c < chunks; ++c)
        if (char const* e = drain(c)) return e;
    kernel_launches += chunks * (cast ? 2 : 1);
    *rows = total;
    return nullptr;
}

/* index_dense_gt::export_keys (index_dense.hpp:1595-1608) in slot order: the live keys from the `offset`-th on, at most
 * `limit` of them; returns how many were written */
size_t frozen_index_t::export_keys(size_t offset, size_t limit, uint64_t* out) const {
    size_t written = 0, seen = 0;
    for (size_t s = 0; s < host_keys.size() && written < limit; ++s) {
        if (host_keys[s] == free_key) continue;
        if (seen++ >= offset) out[written++] = host_keys[s];
    }
    return written;
}

/* out[i] = the offsets[i]-th live key in slot order, for offsets in any order: one walk over the keys */
char const* frozen_index_t::export_keys_at(size_t const* offsets, size_t n, uint64_t* out) const {
    size_t const live = size - count_deleted;
    std::vector<size_t> order(n);
    for (size_t i = 0; i < n; ++i) {
        if (offsets[i] >= live) return "Offset out of range";
        order[i] = i;
    }
    std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return offsets[a] < offsets[b]; });
    size_t next = 0, seen = 0;
    for (size_t s = 0; s < host_keys.size() && next < n; ++s) {
        if (host_keys[s] == free_key) continue;
        while (next < n && offsets[order[next]] == seen) out[order[next++]] = host_keys[s];
        ++seen;
    }
    return next == n ? nullptr : "Offset out of range";
}

/* index_dense_gt::copy (index_dense.hpp:1615-1650): a new handle on the same device with every HBM array copied at this
 * handle's capacity on this handle's stream, and every piece of host state copied, the free-slot queue in its order */
char const* frozen_index_t::copy_into(frozen_index_t& c) {
    if (char const* e = ensure_context()) return e;
    if (shards) return "Can't copy a sharded handle: it holds one shard of its index";
    c.stream.device = stream.device;
    if (char const* e = c.ensure_context()) return e;
    CU(cudaSetDevice(stream.device));
    auto clone = [&](auto const& from, auto& to) -> char const* {
        if (!from.ptr) return nullptr;
        if (char const* e = to.reserve(from.capacity)) return e;
        CU(cudaMemcpyAsync(to.ptr, from.ptr, from.capacity * sizeof(*from.ptr), cudaMemcpyDeviceToDevice, stream));
        return nullptr;
    };
    if (char const* e = clone(hbm.vectors, c.hbm.vectors)) return e;
    if (char const* e = clone(hbm.keys, c.hbm.keys)) return e;
    if (char const* e = clone(hbm.nbr0, c.hbm.nbr0)) return e;
    if (char const* e = clone(hbm.upper_base, c.hbm.upper_base)) return e;
    if (char const* e = clone(hbm.upper, c.hbm.upper)) return e;
    if (char const* e = clone(hbm.deleted_bits, c.hbm.deleted_bits)) return e;
    if (char const* e = clone(hbm.norms, c.hbm.norms)) return e;
    if (char const* e = clone(hbm.codes, c.hbm.codes)) return e;
    if (char const* e = clone(hbm.shadow, c.hbm.shadow)) return e;
    CU(cudaStreamSynchronize(stream));

    c.metric = metric; c.scalar = scalar;
    c.dimensions = dimensions; c.connectivity = connectivity; c.connectivity_base = connectivity_base;
    c.expansion_add = expansion_add; c.expansion_search = expansion_search;
    c.multi = multi; c.free_key = free_key;
    c.size = size; c.count_deleted = count_deleted;
    c.levels = levels;
    c.host_keys = host_keys;
    c.key_map = key_map;
    c.key_map.keys = &c.host_keys;
    c.free_slots = free_slots;
    c.reuse_removed = reuse_removed;
    c.capacity = capacity; c.upper_capacity = upper_capacity; c.upper_rows = upper_rows;
    c.level_seed = level_seed;
    c.tune = tune;
    c.d = d;
    /* the views move to the copy's arrays; an array this handle has not allocated stays absent (its view is NULL) */
    auto view = [](auto const* mine, auto const& copy) { return mine ? copy.ptr : nullptr; };
    c.d.vectors = view(d.vectors, c.hbm.vectors);
    c.d.keys = view(d.keys, c.hbm.keys);
    c.d.nbr0 = view(d.nbr0, c.hbm.nbr0);
    c.d.upper_base = view(d.upper_base, c.hbm.upper_base);
    c.d.upper = view(d.upper, c.hbm.upper);
    c.d.deleted_bits = view(d.deleted_bits, c.hbm.deleted_bits);
    c.d.norms = view(d.norms, c.hbm.norms);
    c.d.codes = view(d.codes, c.hbm.codes);
    c.d.shadow = view(d.shadow, c.hbm.shadow);
    c.hbm_bytes = hbm_bytes;
    c.loaded = loaded;
    return nullptr;
}

/* Entries per level (index_gt::stats, index.hpp:3133-3225): nodes[l] = members whose level is >= l, from the host
 * levels; edges[l] = the entries their level-l lists hold, from one launch over the lists. Removed members count, as
 * the reference loops over every slot below size(). An empty index gives empty vectors. */
char const* frozen_index_t::graph_levels(std::vector<uint64_t>& nodes, std::vector<uint64_t>& edges) {
    nodes.clear();
    edges.clear();
    if (char const* e = ensure_context()) return e;
    if (!loaded || !size) return nullptr;
    size_t const n = std::min<size_t>(size, d.n);
    int top = 0;
    for (size_t s = 0; s < n; ++s) top = std::max<int>(top, levels[s]);
    std::vector<uint64_t> at_level((size_t)top + 1, 0);
    for (size_t s = 0; s < n; ++s) at_level[(size_t)levels[s]] += 1;
    nodes.assign((size_t)top + 1, 0);
    uint64_t at_or_above = 0;
    for (int l = top; l >= 0; --l) nodes[(size_t)l] = at_or_above += at_level[(size_t)l];
    device_buffer_t<int16_t> d_levels;
    device_buffer_t<unsigned long long> d_edges;
    if (char const* e = d_levels.reserve(n)) return e;
    if (char const* e = d_edges.reserve((size_t)top + 1)) return e;
    CU(cudaMemcpyAsync(d_levels.ptr, levels.data(), n * 2, cudaMemcpyHostToDevice, stream));
    CU(cudaMemsetAsync(d_edges.ptr, 0, ((size_t)top + 1) * 8, stream));
    unsigned const blocks = (unsigned)std::min<size_t>((n + 7) / 8, (size_t)stream.sm_count * 8);
    graph_stats_kernel<<<blocks, 256, 0, stream>>>(d, d_levels.ptr, (uint32_t)n, (uint32_t)top + 1, d_edges.ptr);
    CU(cudaGetLastError());
    kernel_launches += 1;
    edges.assign((size_t)top + 1, 0);
    CU(cudaMemcpyAsync(edges.data(), d_edges.ptr, ((size_t)top + 1) * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    return nullptr;
}

} // namespace usearch_b200
