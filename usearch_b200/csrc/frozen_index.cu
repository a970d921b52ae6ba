/*
 *  frozen_index.cu — host side of the GPU search backend: parse the reference's v2 serialisation,
 *  lay the graph out as flat arrays in HBM, plan launches, run batches, retry scratch overflows.
 *
 *  Reference behaviour mirrored here (file:line under /root/reference/include/usearch):
 *    index_dense.hpp:1084-1188  load_from_stream: [u32 rows, u32 cols][matrix][64-byte head][graph]
 *    index_dense.hpp:42-79      index_dense_head_t field order
 *    index.hpp:3322-3382        graph: 40-byte header | int16 levels | node tapes
 *    index.hpp:2116-2195        node tape: key u64 | level i16 | {u32 n, slot[M0]} | level x {u32 n, slot[M]}
 *    index.hpp:3016-3075        expansion = max(config.expansion or 64, wanted)
 *    index_plugins.hpp:1105-1224 query casts
 */
#include "cuda_check.h"
#include "frozen_index.h"
#include "prefilter_bound.h"
#include "scalar_casts.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

namespace usearch_b200 {

namespace {

uint64_t rd_u64(uint8_t const* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
uint32_t rd_u32(uint8_t const* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
int16_t rd_i16(uint8_t const* p) { int16_t v; std::memcpy(&v, p, 2); return v; }
uint32_t ceil2(uint64_t v) { uint64_t r = 1; while (r < v) r <<= 1; return (uint32_t)std::min<uint64_t>(r, 1ull << 31); }
uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }


} // namespace

int default_device() {
    if (char const* dev = std::getenv("USEARCH_B200_DEVICE")) return std::atoi(dev);
    if (char const* rank = std::getenv("LOCAL_RANK")) return std::atoi(rank);
    return 0;
}

size_t bits_per_scalar(uint32_t s) { /* index_plugins.hpp:237-257 */
    switch (s) {
    case SCALAR_B1: return 1;
    case SCALAR_I8: return 8;
    case SCALAR_F16: case SCALAR_BF16: return 16;
    case SCALAR_F32: return 32;
    case SCALAR_F64: return 64;
    default: return 0;
    }
}

void frozen_index_t::release_device() {
    hbm = hbm_arrays_t{};
    d = device_index_t{};
    hbm_bytes = 0;
    loaded = false;
    size = 0;
    count_deleted = 0;
    free_slots.clear();
    capacity = 0;
    upper_capacity = 0;
    upper_rows = 0;
    visited_zeroed_words = 0;
    levels.clear();
    host_keys.clear();
    key_map.clear();
    key_table = key_table_t{};
    key_set_scratch = key_set_scratch_t{};
    keys_generation += 1;
}

char const* frozen_index_t::ensure_context() {
    if (char const* e = stream.open()) return e;
    if (!ev_end) {
        CU(ev_begin.create());
        CU(ev_end.create());
    }
    return nullptr;
}

char const* frozen_index_t::counts_reserve_all(size_t nq) {
    if (char const* e = counts.reserve(nq)) return e;
    if (char const* e = computed.reserve(nq)) return e;
    if (char const* e = cycles.reserve(nq)) return e;
    if (char const* e = h_counts.reserve(nq)) return e;
    if (char const* e = h_computed.reserve(nq)) return e;
    if (char const* e = h_cycles.reserve(nq)) return e;
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------- */
/*  v2 blob -> HBM                                                                                */
/* ---------------------------------------------------------------------------------------------- */

char const* frozen_index_t::load_blob(uint8_t const* blob, size_t length) {
    if (char const* e = ensure_context()) return e;
    release_device();

    uint8_t const* p = blob;
    uint8_t const* const end = blob + length;
    if (length < 8 + 64 + 40) return "File is corrupted and lacks matrix dimensions";
    uint64_t const rows = rd_u32(p), cols = rd_u32(p + 4);
    p += 8;
    if ((uint64_t)(end - p) < rows * cols + 64 + 40) return "File is corrupted and lacks a header";
    uint8_t const* const matrix = p;
    p += rows * cols;
    if (std::memcmp(p, "usearch", 7) != 0) return "Magic header mismatch - the file isn't an index";
    uint16_t version_major;
    std::memcpy(&version_major, p + 7, 2);
    if (version_major != 2) return "File format may be different, please rebuild";
    uint32_t const head_metric = p[13], head_scalar = p[14], head_key = p[15], head_slot = p[16];
    if (head_key != 14 /* u64_k */) return "Key type doesn't match, consider rebuilding";
    if (head_slot != 15 /* u32_k */) return "Slot type doesn't match, consider rebuilding";
    uint64_t const count_present = rd_u64(p + 17), deleted = rd_u64(p + 25), dims = rd_u64(p + 33);
    bool const head_multi = p[41] != 0;
    p += 64;
    (void)count_present;
    if (!search_supported(head_metric, head_scalar))
        return "This metric / scalar kind has no sm_90a kernel and the backend has no CPU fallback";
    size_t const bpv = (dims * bits_per_scalar(head_scalar) + 7) / 8;
    if (rows && cols != bpv) return "Matrix columns do not match bytes per vector";

    uint64_t const n = rd_u64(p), m = rd_u64(p + 8), m0 = rd_u64(p + 16), max_level = rd_u64(p + 24), entry = rd_u64(p + 32);
    p += 40;
    if (n != rows) return "Index size and the number of vectors doesn't match";
    if (n >= 0xFFFFFFFFull) return "Too many entries for 32-bit slots";
    if (n && (m < 2 || m0 < 2)) return "Connectivity is too low";
    if ((uint64_t)(end - p) < n * 2) return "File is corrupted and can't fit all the levels";
    uint8_t const* const levels_bytes = p;
    p += n * 2;

    /* host fields are committed only when the whole file has been accepted (see `commit` below) */
    auto commit = [&](device_index_t const& accepted, size_t rows_in_upper) {
        metric = head_metric;
        scalar = head_scalar;
        dimensions = dims;
        connectivity = m;
        connectivity_base = m0;
        multi = head_multi;
        size = n;
        count_deleted = deleted;
        capacity = n;
        upper_rows = rows_in_upper;
        upper_capacity = std::max<size_t>(rows_in_upper, 1);
        d = accepted;
        loaded = true;
    };
    if (n && max_level > 0x7FFF) return "File is corrupted: level out of range";

    device_index_t ix;
    ix.n = (uint32_t)n;
    ix.m = (uint32_t)m;
    ix.m0 = (uint32_t)m0;
    ix.m_stride = round_up((uint32_t)m, 4);
    ix.m0_stride = round_up((uint32_t)m0, 4);
    ix.entry_slot = (uint32_t)entry;
    ix.max_level = (int32_t)max_level;
    ix.dims = (uint32_t)dims;
    ix.bytes_per_vector = (uint32_t)bpv;
    ix.vec_stride = round_up((uint32_t)bpv, 16);
    ix.chunks16 = (uint32_t)(ix.vec_stride / 16);
    ix.metric = head_metric;
    ix.scalar = head_scalar;
    if (search_needs_shadow(ix)) ix.code_stride = search_code_stride(ix);
    if (n == 0) {
        commit(ix, 0);
        upper_capacity = 0;
        return nullptr;
    }
    if (entry >= n) return "File is corrupted: entry slot out of range";

    /* pass 1: levels, upper row offsets, tape offsets */
    levels.resize(n);
    host_keys.resize(n);
    struct drop_host_state_t { /* a rejected file leaves no trace in the handle */
        frozen_index_t* self;
        bool armed = true;
        ~drop_host_state_t() { if (armed) { self->levels.clear(); self->host_keys.clear(); self->release_device(); } }
    } drop_host_state{this};
    std::vector<uint32_t> upper_base(n);
    uint64_t upper_rows = 0;
    size_t const nb = m * 4 + 4, nb0 = m0 * 4 + 4;
    {
        uint8_t const* q = p;
        for (uint64_t i = 0; i < n; ++i) {
            int16_t level = rd_i16(levels_bytes + 2 * i);
            if (level < 0) return "File is corrupted: negative level";
            levels[i] = level;
            upper_base[i] = level ? (uint32_t)upper_rows : EMPTY_SLOT;
            upper_rows += (uint64_t)level;
            size_t node_bytes = 10 + nb0 + nb * (size_t)level;
            if ((size_t)(end - q) < node_bytes) return "File is corrupted and can't fit all the nodes";
            q += node_bytes;
        }
        if (upper_rows >= 0xFFFFFFFFull) return "Too many upper-level rows";
        /* the descent starts on `max_level` at the entry point (index.hpp:3963-3975): it must own that many rows */
        if ((uint64_t)levels[entry] != max_level) return "File is corrupted: entry point and top level disagree";
    }

    /* device allocations */
    size_t const bytes_vectors = (size_t)n * ix.vec_stride, bytes_keys = (size_t)n * 8,
                 bytes_nbr0 = (size_t)n * ix.m0_stride * 4, bytes_ub = (size_t)n * 4,
                 bytes_upper = std::max<size_t>(upper_rows, 1) * ix.m_stride * 4, bytes_deleted = ((size_t)n + 31) / 32 * 4;
    if (char const* e = hbm.vectors.reserve(bytes_vectors)) return e;
    if (char const* e = hbm.keys.reserve(n)) return e;
    if (char const* e = hbm.nbr0.reserve((size_t)n * ix.m0_stride)) return e;
    if (char const* e = hbm.upper_base.reserve(n)) return e;
    if (char const* e = hbm.upper.reserve(std::max<size_t>(upper_rows, 1) * ix.m_stride)) return e;
    hbm_bytes = bytes_vectors + bytes_keys + bytes_nbr0 + bytes_ub + bytes_upper;

    /* vectors: slot-major matrix, rows padded to 16 bytes */
    if (ix.vec_stride == bpv) {
        CU(cudaMemcpy(hbm.vectors.ptr, matrix, bytes_vectors, cudaMemcpyHostToDevice));
    } else {
        CU(cudaMemset(hbm.vectors.ptr, 0, bytes_vectors));
        CU(cudaMemcpy2D(hbm.vectors.ptr, ix.vec_stride, matrix, bpv, bpv, n, cudaMemcpyHostToDevice));
    }

    /* pass 2: node tapes -> keys, nbr0 rows, upper rows; converted and uploaded in chunks */
    size_t const chunk_nodes = 1u << 18;
    std::vector<uint64_t> h_keys(std::min<size_t>(n, chunk_nodes));
    std::vector<uint32_t> h_nbr0(std::min<size_t>(n, chunk_nodes) * ix.m0_stride);
    std::vector<uint32_t> h_upper;
    std::vector<uint32_t> h_deleted(((size_t)n + 31) / 32, 0u);
    bool any_deleted = false;
    uint8_t const* q = p;
    for (uint64_t begin = 0; begin < n; begin += chunk_nodes) {
        uint64_t const stop = std::min<uint64_t>(n, begin + chunk_nodes);
        uint64_t const first_upper_row = [&] { for (uint64_t i = begin; i < stop; ++i) if (levels[i]) return (uint64_t)upper_base[i]; return upper_rows; }();
        uint64_t chunk_upper_rows = 0;
        for (uint64_t i = begin; i < stop; ++i) chunk_upper_rows += (uint64_t)levels[i];
        h_upper.assign(chunk_upper_rows * ix.m_stride, EMPTY_SLOT);
        std::fill(h_nbr0.begin(), h_nbr0.begin() + (stop - begin) * ix.m0_stride, EMPTY_SLOT);
        uint64_t row = 0;
        for (uint64_t i = begin; i < stop; ++i) {
            uint64_t key = rd_u64(q);
            h_keys[i - begin] = key;
            host_keys[i] = key;
            if (key == free_key) { h_deleted[i >> 5] |= 1u << (i & 31); any_deleted = true; }
            uint8_t const* list = q + 10;
            uint32_t c0 = std::min<uint32_t>(rd_u32(list), (uint32_t)m0);
            uint32_t* dst0 = h_nbr0.data() + (i - begin) * ix.m0_stride;
            /* A self-link or a repeated slot in a layer-0 list can never pass `visits.set()` in
             * search_to_find_in_base_ (index.hpp:4221): the expanded node and the first occurrence are
             * already marked. Dropping them here changes nothing observable and lets the kernel issue
             * every visited test of a row at once. */
            uint32_t kept = 0;
            for (uint32_t j = 0; j < c0; ++j) {
                uint32_t s = rd_u32(list + 4 + 4 * j);
                if (s >= n) return "File is corrupted: neighbour slot out of range";
                bool drop = s == (uint32_t)i;
                for (uint32_t t = 0; t < kept && !drop; ++t) drop = dst0[t] == s;
                if (!drop) dst0[kept++] = s;
            }
            list += nb0;
            for (int16_t l = 0; l < levels[i]; ++l, ++row, list += nb) {
                uint32_t c = std::min<uint32_t>(rd_u32(list), (uint32_t)m);
                uint32_t* dst = h_upper.data() + row * ix.m_stride;
                for (uint32_t j = 0; j < c; ++j) {
                    uint32_t s = rd_u32(list + 4 + 4 * j);
                    if (s >= n) return "File is corrupted: neighbour slot out of range";
                    /* a search on level l+1 reads row l+1 of every member it reaches: the member must have it */
                    if (levels[s] < l + 1) return "File is corrupted: link to a member that is absent from that level";
                    dst[j] = s;
                }
            }
            q = list;
        }
        CU(cudaMemcpy(hbm.keys.ptr + begin, h_keys.data(), (stop - begin) * 8, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(hbm.nbr0.ptr + begin * ix.m0_stride, h_nbr0.data(), (stop - begin) * ix.m0_stride * 4, cudaMemcpyHostToDevice));
        if (chunk_upper_rows)
            CU(cudaMemcpy(hbm.upper.ptr + first_upper_row * ix.m_stride, h_upper.data(), chunk_upper_rows * ix.m_stride * 4,
                          cudaMemcpyHostToDevice));
    }
    CU(cudaMemcpy(hbm.upper_base.ptr, upper_base.data(), bytes_ub, cudaMemcpyHostToDevice));
    if (any_deleted) {
        if (char const* e = hbm.deleted_bits.reserve(bytes_deleted / 4)) return e;
        CU(cudaMemcpy(hbm.deleted_bits.ptr, h_deleted.data(), bytes_deleted, cudaMemcpyHostToDevice));
        hbm_bytes += bytes_deleted;
    }
    ix.vectors = hbm.vectors.ptr;
    ix.keys = hbm.keys.ptr;
    ix.nbr0 = hbm.nbr0.ptr;
    ix.upper_base = hbm.upper_base.ptr;
    ix.upper = hbm.upper.ptr;
    ix.deleted_bits = hbm.deleted_bits.ptr;
    if (search_needs_norms(head_metric, head_scalar)) {
        if (char const* e = hbm.norms.reserve(n)) return e;
        hbm_bytes += (size_t)n * 4;
        CU(search_compute_norms(ix, hbm.norms.ptr, stream));
        CU(cudaStreamSynchronize(stream));
        ix.norms = hbm.norms.ptr;
    }
    if (ix.code_stride) {
        if (char const* e = hbm.codes.reserve((size_t)n * ix.code_stride)) return e;
        if (char const* e = hbm.shadow.reserve(n)) return e;
        hbm_bytes += (size_t)n * (ix.code_stride + sizeof(pf_record_t));
        CU(search_compute_shadow(ix, ix.norms, hbm.codes.ptr, hbm.shadow.ptr, stream));
        CU(cudaStreamSynchronize(stream));
        ix.codes = hbm.codes.ptr;
        ix.shadow = hbm.shadow.ptr;
    }
    drop_host_state.armed = false;
    commit(ix, upper_rows);
    /* reindex_keys_ (index_dense.hpp:2160-2188): removed slots queue up for reuse in ascending order */
    for (uint64_t i = 0; i < n; ++i)
        if (host_keys[i] == free_key) free_slots.push_back((uint32_t)i);
    return nullptr;
}

size_t frozen_index_t::serialized_length() const {
    size_t const nb = connectivity * 4 + 4, nb0 = connectivity_base * 4 + 4;
    size_t total = 8 + size * d.bytes_per_vector + 64 + 40 + size * 2;
    for (size_t i = 0; i < size; ++i) total += 10 + nb0 + nb * (size_t)levels[i];
    return total;
}

/* Re-serialise the frozen index into the reference's v2 format (index_dense.hpp:994-1062,
 * index.hpp:3276-3317) by downloading the SoA arrays. */
char const* frozen_index_t::save_blob(uint8_t* out, size_t length) const {
    if (length < serialized_length()) return "Failed to serialize into stream";
    CU(cudaSetDevice(stream.device));
    size_t const n = size, bpv = d.bytes_per_vector;
    uint8_t* p = out;
    uint32_t dims32[2] = {(uint32_t)n, (uint32_t)bpv};
    std::memcpy(p, dims32, 8);
    p += 8;
    if (n) {
        if (d.vec_stride == bpv) CU(cudaMemcpy(p, d.vectors, n * bpv, cudaMemcpyDeviceToHost));
        else CU(cudaMemcpy2D(p, bpv, d.vectors, d.vec_stride, bpv, n, cudaMemcpyDeviceToHost));
    }
    p += n * bpv;
    std::memset(p, 0, 64);
    std::memcpy(p, "usearch", 7);
    uint16_t version[3] = {2, 21, 0};
    std::memcpy(p + 7, version, 6);
    p[13] = (uint8_t)metric;
    p[14] = (uint8_t)scalar;
    p[15] = 14; /* u64 keys */
    p[16] = 15; /* u32 slots */
    uint64_t present = n - count_deleted, deleted = count_deleted, dims = dimensions;
    std::memcpy(p + 17, &present, 8);
    std::memcpy(p + 25, &deleted, 8);
    std::memcpy(p + 33, &dims, 8);
    p[41] = multi ? 1 : 0;
    p += 64;
    uint64_t header[5] = {n, connectivity, connectivity_base, (uint64_t)d.max_level, d.entry_slot};
    std::memcpy(p, header, 40);
    p += 40;
    if (!n) return nullptr;
    std::memcpy(p, levels.data(), n * 2);
    p += n * 2;
    std::vector<uint64_t> h_keys(n);
    std::vector<uint32_t> h_nbr0((size_t)n * d.m0_stride), h_ub(n);
    size_t upper_rows = 0;
    for (size_t i = 0; i < n; ++i) upper_rows += (size_t)levels[i];
    std::vector<uint32_t> h_upper(std::max<size_t>(upper_rows, 1) * d.m_stride);
    CU(cudaMemcpy(h_keys.data(), d.keys, n * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(h_nbr0.data(), d.nbr0, h_nbr0.size() * 4, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(h_ub.data(), d.upper_base, n * 4, cudaMemcpyDeviceToHost));
    if (upper_rows) CU(cudaMemcpy(h_upper.data(), d.upper, upper_rows * d.m_stride * 4, cudaMemcpyDeviceToHost));
    size_t const nb = connectivity * 4 + 4, nb0 = connectivity_base * 4 + 4;
    auto write_list = [&](uint32_t const* row, uint32_t cap, size_t bytes) {
        std::memset(p, 0, bytes);
        uint32_t c = 0;
        while (c < cap && row[c] != EMPTY_SLOT) ++c;
        std::memcpy(p, &c, 4);
        std::memcpy(p + 4, row, (size_t)c * 4);
        p += bytes;
    };
    for (size_t i = 0; i < n; ++i) {
        std::memcpy(p, &h_keys[i], 8);
        std::memcpy(p + 8, &levels[i], 2);
        p += 10;
        write_list(h_nbr0.data() + i * d.m0_stride, d.m0, nb0);
        for (int16_t l = 0; l < levels[i]; ++l) write_list(h_upper.data() + ((size_t)h_ub[i] + l) * d.m_stride, d.m, nb);
    }
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------- */
/*  launch planning                                                                               */
/* ---------------------------------------------------------------------------------------------- */

char const* frozen_index_t::plan(uint32_t k, uint32_t visited_cap_override, launch_plan_t& pl, uint32_t ef_override,
                                 bool grouped) const {
    uint32_t ef = (uint32_t)(expansion_search ? expansion_search : 64); /* index.hpp:3029-3030 */
    ef = std::max(ef, k);                                               /* index.hpp:3052 */
    if (ef_override) ef = ef_override; /* the builder searches with expansion_add (index.hpp:2854) */
    pl.ef = ef;
    /* `visits` covers every slot the arrays have room for, so that its size does not change while members are added */
    uint64_t const visit_slots = std::max<uint64_t>(capacity, d.n);
    uint32_t const list_cap = round_up(std::max(d.m0, d.m), 32);
    /* an SM has 228 KB of shared memory and charges 1 KB per resident CTA on top of its request */
    size_t const smem_sm = 228 * 1024, cta_tax = 1024, smem_cta_max = 227 * 1024;
    uint32_t const min_heap = 128 * 8;
    /* The prefilter's s32 dot products are exact while dims 127^2 < 2^31: above that it is off. Only a plain search can
     * run it (the builder's INSERT kernel never does), and its shared memory is reserved only then. Where that layout
     * does not fit, the search goes without the prefilter rather than fail. */
    bool const s32_exact = (uint64_t)d.dims * 127u * 127u < (1ull << 31);
    uint32_t fixed = 0;
    for (bool pf = d.codes && tune.prefilter && s32_exact && !ef_override;; pf = false) {
        /* per-warp (= per-CTA) shared memory: query | top | candidates | mbarriers | TMA slots | heap head */
        uint32_t off = 0;
        off += d.chunks16 * 16;          /* query */
        uint32_t const top_smem = ef > 256 ? round_up(ef * 4, 16) : 0; /* ef <= 256: `top` lives in registers */
        pl.off_top_d = off; off += top_smem;
        pl.off_top_s = off; off += top_smem;
        pl.off_cand_s = off; off += list_cap * 4;
        pl.off_cand_d = off; off += list_cap * 4;
        /* prefilter: the tensor-core k-steps read 32 code bytes at a time, so the query split is zero-padded to that */
        pl.qsplit_len = pf ? round_up(d.code_stride, 32) : 0;
        pl.off_surv_b2 = pl.off_qsplit = 0;
        if (pf) { /* prefilter: the survivors' stored squared norms, and the query split q1 | q2 */
            pl.off_surv_b2 = off; off += list_cap * 4;
            pl.off_qsplit = off; off += 2 * pl.qsplit_len;
        }
        pl.off_bars = off; off += 256; /* 32 mbarriers */
        off = round_up(off, 128);
        pl.off_stage = off;
        int const slots = search_stage_slots(d); /* slots of one set: 32 / LPV */
        int const forced_sets = tune.stage_sets;
        pl.stage_sets = 1;
        pl.stage_stride = 0;
        if (slots) {
            /* slot stride = 16*LPV mod 128 bytes: the lanes of a quarter-warp then read disjoint banks */
            pl.stage_stride = round_up(d.chunks16 * 16, 128) + search_stage_pad(d);
            /* double-buffer the slots when at least 4 warps per SM still fit */
            size_t const two = off + 2 * (size_t)slots * pl.stage_stride + min_heap + cta_tax;
            pl.stage_sets = smem_sm / two >= 4 ? 2u : 1u;
            /* short vectors of the 16-warp kernels: resident warps beat double buffering (search_kernel.cu, dispatch) */
            if (search_single_stage_set(d)) pl.stage_sets = 1;
            /* prefilter on: a hop reads few rows, so resident warps beat double buffering (C2 on one H100 SXM at 700 W: 14.9 ms
             * per 4096-query launch with one set and 7 warps per SM, 18.2 ms with two sets and 4) */
            if (d.codes && tune.prefilter) pl.stage_sets = 1;
            if (forced_sets == 1 || forced_sets == 2) pl.stage_sets = (uint32_t)forced_sets;
        }
        uint32_t const stage_bytes = (uint32_t)slots * pl.stage_sets * pl.stage_stride;
        off += stage_bytes;
        pl.off_heap = off;
        /* prefilter: the int8 codes of a pass fill the stage area in whole m16n8k32 tiles of 16 rows (<= 64). A row stride
         * that is an odd multiple of 16 bytes puts the 8 rows of every ldmatrix matrix in distinct bank groups. */
        pl.code_smem_stride = pf ? pl.qsplit_len + 16 : 0;
        pl.code_pass = pf ? std::min<uint32_t>(64, stage_bytes / pl.code_smem_stride) & ~15u : 0;
        pl.prefilter = pl.code_pass >= 16;
        fixed = off;
        if (!pf || fixed + min_heap <= smem_cta_max) break;
    }
    if (fixed + min_heap > smem_cta_max) return "Expansion or dimensionality too large for on-chip state";
    int const forced_warps = tune.warps_per_sm;
    uint32_t warps_sm = (uint32_t)std::min<size_t>(smem_sm / (fixed + min_heap + cta_tax), (size_t)search_max_warps_per_sm(d));
    if (forced_warps > 0) warps_sm = std::min<uint32_t>(warps_sm, (uint32_t)forced_warps);
    warps_sm = std::max(warps_sm, 1u);
    auto head_bytes = [&](uint32_t warps) { /* the shared memory left to the heap head at `warps` per SM */
        uint32_t const budget = std::min<uint32_t>((uint32_t)(smem_sm / warps - cta_tax), (uint32_t)smem_cta_max);
        return std::min<uint32_t>((budget - fixed) & ~15u, 4096 * 8);
    };
    /* Prefilter on: a hop is short, and a pop that leaves the warp-wide `pop_warp` (a head below the heap, which sends the
     * pops to lane 0's serial walk and the HBM tail) is expensive. So plan for one warp per SM fewer when that lifts a head
     * below PF_MIN_HEAP_HEAD entries. At 768-d (M=32, ef=128) a 7-warp budget leaves a 200-entry head, below the average
     * per-query heap maximum of 353, and the 128-byte granularity of shared-memory allocation lets only 6 of those warps
     * be resident anyway (792 blocks on 132 SMs); a 6-warp budget gives the same 6 warps an 896-entry head. 10M x 768 f32
     * cosine on one H100 SXM at 400 W: 13.61 -> 12.77 ms per 4096-query launch (medians of three), heap_pop 0.63 M ->
     * 0.31 M cycles per query (DESIGN §8). */
    constexpr uint32_t PF_MIN_HEAP_HEAD = 512;
    if (pl.prefilter && forced_warps <= 0 && tune.heap_head <= 0 && warps_sm > 2 && head_bytes(warps_sm) / 8 < PF_MIN_HEAP_HEAD)
        warps_sm -= 1;
    uint32_t heap_bytes = head_bytes(warps_sm);
    /* the heap_head knob: a smaller head sends more of the heap to its HBM tail; the root stays in shared memory */
    if (tune.heap_head > 0) heap_bytes = std::min<uint32_t>(heap_bytes, (uint32_t)std::max(tune.heap_head / 2, 1) * 16);
    pl.heap_smem_cap = heap_bytes / 8; /* even: heap_bytes is a multiple of 16 */
    pl.smem_per_warp = fixed + pl.heap_smem_cap * 8;
    pl.smem_per_block = pl.smem_per_warp;
    pl.warps_per_sm_target = warps_sm;

    /* scratch per warp. `scale` (1, 8, 64, ...) grows it for the retry of overflowed queries. */
    uint64_t const scale = visited_cap_override ? visited_cap_override : 1;
    uint64_t const enough = (uint64_t)2 * (visit_slots + d.m0 + 1); /* a hash table this large can never overflow */
    static int const forced = [] { /* test hook: USEARCH_B200_VISITED=hash|bitmap|bitmap_log */
        char const* v = std::getenv("USEARCH_B200_VISITED");
        return !v ? 0 : (std::strcmp(v, "hash") == 0 ? 1 : (std::strcmp(v, "bitmap") == 0 ? 2 : (std::strcmp(v, "bitmap_log") == 0 ? 3 : 0)));
    }();
    static uint64_t const shrink = [] { /* test hook: start with undersized scratch to exercise the retry path */
        char const* v = std::getenv("USEARCH_B200_SCRATCH_SHRINK");
        return v && std::atoi(v) > 0 ? (uint64_t)std::atoi(v) : (uint64_t)1;
    }();
    uint64_t const bitmap_words = round_up((uint32_t)((visit_slots + 31) / 32), 4);
    uint64_t const max_warps_guess = (uint64_t)stream.sm_count * 32;
    bool const bitmaps_fit = bitmap_words * 4 * std::min<uint64_t>(max_warps_guess, (uint64_t)stream.sm_count * pl.warps_per_sm_target) <= BITMAP_SCRATCH_BUDGET;
    if (forced == 2 || forced == 3 || (forced == 0 && bitmaps_fit)) {
        /* BITMAP visits: one bit per slot, exact, never overflows */
        pl.visited_bitmap_words = (uint32_t)bitmap_words;
        pl.visited_cap = 0;
        pl.visit_log_cap = (forced == 3 || (forced == 0 && visit_slots > BITMAP_WIPE_MAX_SLOTS))
                               ? (uint32_t)std::max<uint64_t>(32768 / shrink, 64) : 0u;
        uint64_t spill = std::max<uint64_t>(1024, (uint64_t)8 * ef) * scale / shrink;
        spill = std::max<uint64_t>(spill, 16);
        pl.heap_spill_cap = (uint32_t)std::min<uint64_t>(spill, visit_slots + 1);
        pl.maxed = pl.heap_spill_cap >= visit_slots;
    } else {
        pl.visited_bitmap_words = 0;
        pl.visit_log_cap = 0;
        uint64_t want = std::max<uint64_t>((uint64_t)2 * ef * d.m0 * scale, 2048) / shrink;
        pl.visited_cap = std::max<uint32_t>(ceil2(std::min<uint64_t>(want, enough)), 64);
        /* pushes <= visited entries <= cap/2, so this spill can not overflow before `visits` does */
        pl.heap_spill_cap = pl.visited_cap / 2;
        pl.maxed = pl.visited_cap >= enough;
    }

    int per_sm = 0;
    CU(search_occupancy(d, &per_sm, pl.smem_per_block, grouped));
    if (per_sm < 1) return "Kernel does not fit on an SM";
    per_sm = std::min<int>(per_sm, (int)pl.warps_per_sm_target);
    pl.blocks = per_sm * stream.sm_count;
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------- */
/*  batched search on device buffers                                                              */
/* ---------------------------------------------------------------------------------------------- */

/* scratch for `warps` resident warps under plan `pl`, and the launch arguments that describe it */
char const* frozen_index_t::prepare_launch(launch_plan_t const& pl, size_t warps, search_args_t& a, cudaStream_t s) {
    if (char const* e = work_counter.reserve(2)) return e;
    size_t const words = warps * pl.visited_words_per_warp();
    bool const grown = words > visited.capacity;
    if (char const* e = visited.reserve(words)) return e;
    if (grown) visited_zeroed_words = 0;
    if (pl.visit_log_cap) { /* logged bitmaps rely on an all-zero slab between queries */
        if (char const* e = visit_log.reserve(warps * pl.visit_log_cap)) return e;
        if (visited_zeroed_words < words) {
            if (cudaMemsetAsync(visited.ptr, 0, words * 4, s) != cudaSuccess) return "CUDA failure: memset";
            visited_zeroed_words = words;
        }
    } else
        visited_zeroed_words = 0; /* wiped per query with other contents in between */
    if (char const* e = heap_spill.reserve(warps * pl.heap_spill_cap)) return e;
    a = search_args_t{};
    a.ef = pl.ef;
    a.work_counter = work_counter.ptr;
    a.visited = visited.ptr;
    a.visited_cap = pl.visited_cap;
    a.visited_bitmap_words = pl.visited_bitmap_words;
    a.visit_log = pl.visit_log_cap ? visit_log.ptr : nullptr;
    a.visit_log_cap = pl.visit_log_cap;
    a.heap_spill = heap_spill.ptr;
    a.heap_spill_cap = pl.heap_spill_cap;
    a.heap_smem_cap = pl.heap_smem_cap;
    a.smem_per_warp = pl.smem_per_warp;
    a.off_top_d = pl.off_top_d; a.off_top_s = pl.off_top_s; a.off_cand_s = pl.off_cand_s;
    a.off_cand_d = pl.off_cand_d; a.off_heap = pl.off_heap;
    a.off_bars = pl.off_bars; a.off_stage = pl.off_stage; a.stage_stride = pl.stage_stride;
    a.stage_sets = pl.stage_sets;
    a.prefilter = pl.prefilter ? 1u : 0u;
    a.code_pass = pl.code_pass;
    a.code_smem_stride = pl.code_smem_stride;
    a.off_surv_b2 = pl.off_surv_b2;
    a.off_qsplit = pl.off_qsplit; a.qsplit_len = pl.qsplit_len;
    return nullptr;
}

char const* frozen_index_t::search_device(void const* d_queries, size_t nq, size_t stride, size_t k, uint64_t* d_keys,
                                          float* d_dists, uint32_t* d_counts, uint32_t* d_computed, uint32_t* d_cycles,
                                          cudaStream_t s, bool defer, search_filter_t const& filter) {
    if (nq == 0 || k == 0) return nullptr;
    if (nq > 0x7FFFFFFFull) return "Too many queries in one batch";
    if (char const* e = ensure_context()) return e;
    if (!loaded || d.n == 0) { /* no matches, no error (index.hpp:3036-3037) */
        CU(search_fill_empty(d_keys, d_dists, d_counts, d_computed, d_cycles, nq, k, s));
        return nullptr;
    }
    launch_plan_t pl;
    if (char const* e = plan((uint32_t)k, 0, pl)) return e;
    /* a small batch does not need the whole grid */
    int const wpb = search_warps_per_block();
    int blocks = (int)std::min<size_t>((size_t)pl.blocks, (nq + wpb - 1) / wpb);
    size_t warps = (size_t)blocks * wpb;

    if (char const* e = h_status.reserve(nq)) return e;
    uint32_t* status_ptr = nullptr;
    if (defer) { /* every batch in flight owns its status words until search_finish has looked at them */
        if (pending_status.size() == pending.size()) pending_status.emplace_back();
        device_buffer_t<uint32_t>& buf = pending_status[pending.size()];
        if (char const* e = buf.reserve(nq)) return e;
        pending.push_back(pending_search_t{buf.ptr, search_args_t{}, pl.maxed, s});
        status_ptr = buf.ptr;
    } else {
        if (char const* e = status.reserve(nq)) return e;
        status_ptr = status.ptr;
    }
    search_args_t a;
    if (char const* e = prepare_launch(pl, warps, a, s)) return e;
    a.queries = static_cast<uint8_t const*>(d_queries);
    a.query_stride = stride;
    a.nq = (uint32_t)nq;
    a.k = (uint32_t)k;
    a.out_keys = d_keys;
    a.out_dists = d_dists;
    a.out_counts = d_counts;
    a.out_computed = d_computed;
    a.out_visited = d_cycles;
    a.status = status_ptr;
    a.allow_bits = filter.allow_bits;
    a.cluster_end_level = filter.cluster_end_level;

    if (profile_phases) {
        if (char const* e = phase_cycles.reserve(PHASE_COUNTERS)) return e;
        a.phase_cycles = phase_cycles.ptr;
    }
    CU(cudaMemsetAsync(work_counter.ptr, 0, 8, s));
    CU(cudaEventRecord(ev_begin, s));
    CU(search_launch(d, a, blocks, pl.smem_per_block, s));
    CU(cudaEventRecord(ev_end, s));
    kernel_launches += 1;
    if (defer) { /* enqueue only: search_finish synchronises, looks at the status words and retries what overflowed */
        pending.back().args = a;
        return nullptr;
    }
    CU(cudaMemcpyAsync(h_status.ptr, status.ptr, nq * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaEventElapsedTime(&last_kernel_ms, ev_begin, ev_end));
    return retry_overflowed(a, pl.maxed, s);
}

/* every deferred batch: wait, then give the queries whose scratch overflowed their retry */
char const* frozen_index_t::search_finish() {
    char const* first_error = nullptr;
    for (pending_search_t& p : pending) {
        char const* e = cuda_error(cudaStreamSynchronize(p.stream));
        if (!e) e = h_status.reserve(p.args.nq);
        if (!e) e = cuda_error(cudaMemcpy(h_status.ptr, p.status, (size_t)p.args.nq * 4, cudaMemcpyDeviceToHost));
        if (!e) e = retry_overflowed(p.args, p.maxed, p.stream);
        if (e && !first_error) first_error = e;
    }
    pending.clear();
    if (ev_begin && ev_end && !first_error) cudaEventElapsedTime(&last_kernel_ms, ev_begin, ev_end);
    return first_error;
}

/* scratch overflow (h_status holds the status words of the launch described by `a`): rerun just those queries with 8x
 * larger tables until they fit. The scan covers query ids 0 .. a.nq-1: a caller that launched through `query_list` passes
 * `a.nq` as the id range, with every word outside the launch already STATUS_OK. */
char const* frozen_index_t::retry_overflowed(search_args_t const& a, bool maxed, cudaStream_t s) {
    size_t const nq = a.nq, k = a.k;
    int const wpb = search_warps_per_block();
    std::vector<uint32_t> failed;
    for (size_t i = 0; i < nq; ++i)
        if (h_status.ptr[i] != STATUS_OK) failed.push_back((uint32_t)i);
    uint64_t scale = 1;
    while (!failed.empty()) {
        if (maxed) return "Search scratch overflow that full-size scratch could not fix";
        scale *= 8;
        launch_plan_t rp;
        if (char const* e = plan((uint32_t)k, (uint32_t)std::min<uint64_t>(scale, 1u << 30), rp, 0, a.allow_groups != nullptr)) return e;
        maxed = rp.maxed;
        size_t const bytes_per_warp = (size_t)rp.visited_words_per_warp() * 4 + (size_t)rp.heap_spill_cap * 8;
        size_t max_warps = std::max<size_t>(wpb, ((size_t)2 << 30) / bytes_per_warp / wpb * wpb);
        int rblocks = (int)std::min<size_t>({(size_t)rp.blocks, (failed.size() + wpb - 1) / wpb, max_warps / wpb});
        rblocks = std::max(rblocks, 1);
        size_t rwarps = (size_t)rblocks * wpb;
        if (char const* e = retry_list.reserve(failed.size())) return e;
        CU(cudaMemcpyAsync(retry_list.ptr, failed.data(), failed.size() * 4, cudaMemcpyHostToDevice, s));
        search_args_t r;
        if (char const* e = prepare_launch(rp, rwarps, r, s)) return e;
        r.queries = a.queries; r.query_stride = a.query_stride; r.k = a.k;
        r.out_keys = a.out_keys; r.out_dists = a.out_dists; r.out_counts = a.out_counts;
        r.out_computed = a.out_computed; r.out_visited = a.out_visited; r.status = a.status;
        r.allow_bits = a.allow_bits; r.cluster_end_level = a.cluster_end_level; r.phase_cycles = a.phase_cycles;
        r.allow_groups = a.allow_groups; r.allow_group_base = a.allow_group_base; r.allow_words = a.allow_words;
        r.nq = (uint32_t)failed.size();
        r.query_list = retry_list.ptr;
        CU(cudaMemsetAsync(work_counter.ptr, 0, 8, s));
        CU(search_launch(d, r, rblocks, rp.smem_per_block, s));
        kernel_launches += 1;
        CU(cudaMemcpyAsync(h_status.ptr, a.status, nq * 4, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        std::vector<uint32_t> still;
        for (uint32_t qi : failed)
            if (h_status.ptr[qi] != STATUS_OK) still.push_back(qi);
        failed.swap(still);
    }
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------- */
/*  batched search on host buffers: H2D + kernel + D2H inside the call                            */
/* ---------------------------------------------------------------------------------------------- */

/* host rows of `query_scalar` -> `queries` on the device in the index's scalar kind, rows zero-padded to vec_stride. The cast
 * (index_dense_gt::search_ casts every query with casts_.from_*, index_dense.hpp:2060-2066) runs on the device. */
char const* frozen_index_t::upload_queries(void const* q, size_t nq, size_t stride, uint32_t query_scalar) {
    size_t const vs = d.vec_stride ? d.vec_stride : 16, bpv = d.bytes_per_vector;
    size_t const src_bytes = (dimensions * bits_per_scalar(query_scalar) + 7) / 8;
    if (!src_bytes) return "Unknown scalar kind!";
    if (stride < src_bytes) { /* single-query callers pass 0; rows can not overlap */
        if (nq != 1 && stride != 0) return "Query stride is smaller than a vector";
        stride = src_bytes;
    }
    if (query_scalar == scalar) {
        if (vs != bpv) CU(cudaMemsetAsync(queries.ptr, 0, nq * vs, stream));
        CU(cudaMemcpy2DAsync(queries.ptr, vs, q, stride, bpv, nq, cudaMemcpyHostToDevice, stream));
        return nullptr;
    }
    if (char const* e = cast_stage.reserve(nq * src_bytes)) return e;
    CU(cudaMemcpy2DAsync(cast_stage.ptr, src_bytes, q, stride, src_bytes, nq, cudaMemcpyHostToDevice, stream));
    return cast_rows_device(cast_stage.ptr, src_bytes, query_scalar, queries.ptr, vs, scalar, dimensions, nq, stream);
}

char const* frozen_index_t::stage_keys(uint64_t const* keys, size_t n) {
    if (char const* e = key_stage.reserve(std::max<size_t>(n, 1))) return e;
    if (n) CU(cudaMemcpyAsync(key_stage.ptr, keys, n * 8, cudaMemcpyHostToDevice, stream));
    return nullptr;
}

char const* answer_empty(size_t nq, size_t k, host_results_t const& out) {
    for (size_t i = 0; i < nq; ++i) {
        uint64_t* krow = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(out.keys) + i * out.keys_stride);
        uint32_t* drow = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(out.dists) + i * out.dists_stride);
        for (size_t j = 0; j < k; ++j) { krow[j] = 0; drow[j] = SNAN_BITS; }
        if (out.counts) out.counts[i] = 0;
        if (out.computed) out.computed[i] = 0;
        if (out.visited) out.visited[i] = 0;
    }
    return nullptr;
}

char const* frozen_index_t::search_round_trip(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                                              host_results_t const& out, size_t* total, device_search_t const& search) {
    if (char const* e = ensure_context()) return e;
    size_t const vs = d.vec_stride ? d.vec_stride : 16;
    if (char const* e = queries.reserve(nq * vs)) return e;
    if (char const* e = out_keys.reserve(nq * k)) return e;
    if (char const* e = out_dists.reserve(nq * k)) return e;
    if (char const* e = counts_reserve_all(nq)) return e;
    if (char const* e = upload_queries(q, nq, stride, query_scalar)) return e;
    if (char const* e = search(queries.ptr, vs, device_results_t{out_keys.ptr, out_dists.ptr, counts.ptr, out.computed ? computed.ptr : nullptr,
                                                                 out.visited ? cycles.ptr : nullptr}))
        return e;

    if (out.keys_stride == k * 8 && out.dists_stride == k * 4) {
        CU(cudaMemcpyAsync(out.keys, out_keys.ptr, nq * k * 8, cudaMemcpyDeviceToHost, stream));
        CU(cudaMemcpyAsync(out.dists, out_dists.ptr, nq * k * 4, cudaMemcpyDeviceToHost, stream));
    } else {
        CU(cudaMemcpy2DAsync(out.keys, out.keys_stride, out_keys.ptr, k * 8, k * 8, nq, cudaMemcpyDeviceToHost, stream));
        CU(cudaMemcpy2DAsync(out.dists, out.dists_stride, out_dists.ptr, k * 4, k * 4, nq, cudaMemcpyDeviceToHost, stream));
    }
    CU(cudaMemcpyAsync(h_counts.ptr, counts.ptr, nq * 4, cudaMemcpyDeviceToHost, stream));
    if (out.computed) CU(cudaMemcpyAsync(h_computed.ptr, computed.ptr, nq * 4, cudaMemcpyDeviceToHost, stream));
    if (out.visited) CU(cudaMemcpyAsync(h_cycles.ptr, cycles.ptr, nq * 4, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    size_t sum = 0;
    for (size_t i = 0; i < nq; ++i) {
        sum += h_counts.ptr[i];
        if (out.counts) out.counts[i] = h_counts.ptr[i];
        if (out.computed) out.computed[i] = h_computed.ptr[i];
        if (out.visited) out.visited[i] = h_cycles.ptr[i];
    }
    *total = sum;
    return nullptr;
}

char const* frozen_index_t::search_host(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                                        host_results_t const& out, size_t* total) {
    if (nq == 0 || k == 0) return nullptr;
    std::lock_guard<std::mutex> lock(mutex);
    if (!loaded || d.n == 0) return answer_empty(nq, k, out);
    return search_round_trip(q, nq, stride, query_scalar, k, out, total, [&](void const* dq, size_t vs, device_results_t const& r) {
        return search_device(dq, nq, vs, k, r.keys, r.dists, r.counts, r.computed, r.visited, stream);
    });
}

/* index_gt::cluster (index.hpp:3115-3116): the greedy descent over levels max..`level`, with level 0 treated as level 1 */
char const* frozen_index_t::cluster_host(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t level, uint64_t* keys,
                                         float* dists, uint64_t* computed_out, uint64_t* visited_out) {
    if (nq == 0) return nullptr;
    std::lock_guard<std::mutex> lock(mutex);
    if (!loaded || d.n == 0) return "No clusters to identify";
    search_filter_t filter;
    filter.cluster_end_level = level <= 1 ? 0 : (int)std::min<size_t>(level, 0x7FFF) - 1;
    size_t total = 0;
    host_results_t const out{keys, 8, dists, 4, nullptr, computed_out, visited_out};
    return search_round_trip(q, nq, stride, query_scalar, 1, out, &total, [&](void const* dq, size_t vs, device_results_t const& r) {
        return search_device(dq, nq, vs, 1, r.keys, r.dists, r.counts, r.computed, r.visited, stream, false, filter);
    });
}

/* One query per call, many calling threads: gather what is waiting into one batch. The first caller to find no leader
 * becomes it, takes every queued request of the same (scalar kind, count) as its own, runs them through search_host as one
 * batch, hands the rows back and repeats until the queue is empty. */
char const* frozen_index_t::search_single(void const* query, uint32_t query_scalar, size_t count, uint64_t* keys, float* dists,
                                          size_t* found) {
    single_request_t mine{query, query_scalar, count, keys, dists, 0, nullptr, false};
    std::unique_lock<std::mutex> lock(gather_mutex);
    gather_queue.push_back(&mine);
    while (!mine.done && gather_leader) gather_cv.wait(lock);
    if (mine.done) { *found = mine.found; return mine.error; }
    gather_leader = true;
    while (!gather_queue.empty()) {
        /* the batch: every waiting request that matches the head's shape */
        std::vector<single_request_t*> batch, rest;
        for (single_request_t* r : gather_queue)
            (r->scalar == gather_queue[0]->scalar && r->count == gather_queue[0]->count ? batch : rest).push_back(r);
        gather_queue.swap(rest);
        lock.unlock();
        size_t const nq = batch.size(), k = batch[0]->count;
        size_t const qbytes = (dimensions * bits_per_scalar(batch[0]->scalar) + 7) / 8;
        char const* e = nullptr;
        if (nq == 1) {
            size_t total = 0;
            e = search_host(batch[0]->query, 1, 0, batch[0]->scalar, k, host_results_t{batch[0]->keys, k * 8, batch[0]->dists, k * 4}, &total);
            batch[0]->found = total;
        } else {
            std::vector<uint8_t> q(nq * qbytes);
            std::vector<uint64_t> out_k(nq * k);
            std::vector<float> out_d(nq * k);
            std::vector<size_t> cnt(nq);
            for (size_t i = 0; i < nq; ++i) std::memcpy(q.data() + i * qbytes, batch[i]->query, qbytes);
            size_t total = 0;
            e = search_host(q.data(), nq, qbytes, batch[0]->scalar, k, host_results_t{out_k.data(), k * 8, out_d.data(), k * 4, cnt.data()},
                            &total);
            for (size_t i = 0; i < nq && !e; ++i) {
                std::memcpy(batch[i]->keys, out_k.data() + i * k, k * 8);
                std::memcpy(batch[i]->dists, out_d.data() + i * k, k * 4);
                batch[i]->found = cnt[i];
            }
        }
        lock.lock();
        gathered_batches += 1;
        gathered_queries += nq;
        for (single_request_t* r : batch) { r->error = e; r->done = true; }
        gather_cv.notify_all();
    }
    gather_leader = false;
    gather_cv.notify_all(); /* a request that slipped in while the leader was leaving elects a new one */
    *found = mine.found;
    return mine.error;
}

/* ---------------------------------------------------------------------------------------------- */
/*  exact (brute-force) search: host wrappers around exact_kernel.cu                              */
/* ---------------------------------------------------------------------------------------------- */

/* index_gt::search(exact = true) (index.hpp:3047-3051 -> search_exact_ :4251-4268) for a batch of host queries */
char const* frozen_index_t::exact_host(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k, host_results_t const& out,
                                       size_t* total) {
    if (nq == 0 || k == 0) return nullptr;
    std::lock_guard<std::mutex> lock(mutex);
    if (!loaded || d.n == 0) return answer_empty(nq, k, out);
    return search_round_trip(q, nq, stride, query_scalar, k, out, total,
                             [&](void const* dq, size_t vs, device_results_t const& r) -> char const* {
        if (char const* e = exact_search_device(d, stream.sm_count, dq, nq, vs, k, false, false, r.keys, r.dists, r.counts, exact_scratch, stream))
            return e;
        kernel_launches += 2;
        return nullptr;
    });
}

/* usearch_distance: both vectors to the device, one warp, the metric struct of the search kernels */
char const* pair_distance_host(void const* a, void const* b, uint32_t scalar, size_t dimensions, uint32_t metric, float* result) {
    cuda_stream_t s(default_device());
    if (char const* e = s.open()) return e;
    size_t const bpv = (dimensions * bits_per_scalar(scalar) + 7) / 8, vs = (bpv + 15) / 16 * 16;
    if (vs > 48 * 1024) return "Vector too long for a single-pair distance";
    device_index_t ix;
    ix.dims = (uint32_t)dimensions;
    ix.bytes_per_vector = (uint32_t)bpv;
    ix.vec_stride = vs;
    ix.chunks16 = (uint32_t)(vs / 16);
    ix.metric = metric;
    ix.scalar = scalar;
    device_buffer_t<uint8_t> pair;
    device_buffer_t<float> out;
    if (char const* e = pair.reserve(2 * vs)) return e;
    if (char const* e = out.reserve(1)) return e;
    CU(cudaMemsetAsync(pair.ptr, 0, 2 * vs, s));
    CU(cudaMemcpyAsync(pair.ptr, a, bpv, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(pair.ptr + vs, b, bpv, cudaMemcpyHostToDevice, s));
    if (char const* e = pair_distance_device(ix, pair.ptr, pair.ptr + vs, out.ptr, s)) return e;
    CU(cudaMemcpyAsync(result, out.ptr, 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return nullptr;
}

/* ---------------------------------------------------------------------------------------------- */
/*  lookups and edits by key                                                                      */
/* ---------------------------------------------------------------------------------------------- */

/* index_dense_gt::rename (index_dense.hpp:1554-1580): every entry under `from` gets the key `to` */
char const* frozen_index_t::rename_key(uint64_t from, uint64_t to, size_t* renamed) {
    *renamed = 0;
    if (!loaded || !size) return nullptr;
    keys_generation += 1;
    if (char const* e = ensure_context()) return e;
    if (to == free_key) return "Key is reserved for removed entries";
    build_key_map();
    if (!multi && key_map.contains(to)) return "Renaming impossible, the key is already in use";
    std::vector<uint32_t> slots;
    key_map.for_each(from, [&](uint32_t slot, size_t cell) { slots.push_back(slot); key_map.erase_cell(cell); return true; });
    for (uint32_t slot : slots) {
        host_keys[slot] = to;
        key_map.insert(to, slot);
        CU(cudaMemcpy(const_cast<uint64_t*>(d.keys) + slot, &to, 8, cudaMemcpyHostToDevice));
    }
    *renamed = slots.size();
    return nullptr;
}

/* index_dense_gt::get (index_dense.hpp:781-786 -> get_ :2121-2150): up to `max_count` vectors stored under `key` */
char const* frozen_index_t::get_vectors(uint64_t key, size_t max_count, void* out, uint32_t out_scalar, size_t* found) {
    *found = 0;
    if (!loaded || !size || !max_count) return nullptr;
    if (char const* e = ensure_context()) return e;
    size_t const out_bytes = (dimensions * bits_per_scalar(out_scalar) + 7) / 8;
    if (!out_bytes) return "Unknown scalar kind!";
    build_key_map();
    std::vector<uint32_t> slots;
    key_map.for_each(key, [&](uint32_t slot, size_t) { slots.push_back(slot); return slots.size() < max_count; });
    std::sort(slots.begin(), slots.end()); /* insertion order */
    std::vector<uint8_t> row(d.vec_stride);
    for (size_t i = 0; i < slots.size(); ++i) {
        CU(cudaMemcpy(row.data(), d.vectors + (size_t)slots[i] * d.vec_stride, d.bytes_per_vector, cudaMemcpyDeviceToHost));
        /* index_dense_gt::get_ casts with casts_.to_* (index_dense.hpp:2121-2150) */
        if (char const* e = cast_row_host(scalar, out_scalar, dimensions, row.data(), static_cast<uint8_t*>(out) + i * out_bytes)) return e;
    }
    *found = slots.size();
    return nullptr;
}

} // namespace usearch_b200
