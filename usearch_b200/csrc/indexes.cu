/*
 *  indexes.cu — several indexes searched as one on a single GPU: the reference's `Indexes` (python/lib.cpp:74-107,
 *  :321-402), with its one-thread results.
 *
 *  The reference searches every shard for every query and folds each shard's result into the query's row with
 *  search_result_t::merge_into (index.hpp:2650-2670). Run on one thread, shards are folded in merge order, each result in
 *  its stored order, into rows that start empty. Here one search call
 *      1. uploads the queries once and casts them on the device to each shard's scalar kind,
 *      2. runs every shard's own batched search (or exact search) on the group's stream, each writing its slice of
 *         packed per-shard rows [S][nq][count],
 *      3. folds those rows with merge_into_kernel: a warp per query, the row in shared memory, every fold replaying
 *         merge_into exactly (libstdc++'s lower_bound probe, then the shift),
 *      4. copies the merged rows and counters back once.
 *  The NCCL sharded search (shards.cu) orders ties by (distance, shard, position) instead; the two merges share nothing.
 */
#include <algorithm>
#include <cstring>
#include <mutex>

#include "cuda_check.h"
#include "frozen_index.h"

namespace usearch_b200 {

namespace {

/* Shared memory of one warp's row: `k` keys then `k` distances. Warps per block shrink as `k` grows. */
constexpr size_t MERGE_MAX_SMEM = 227u << 10;

/* merge_into (index.hpp:2650-2670) of shard 0's row, then shard 1's, ... into an empty row of `k`, for query q:
 *     offset = std::lower_bound(row, row + merged, d)        libstdc++'s probe: halve len, test *mid < d
 *     skip if offset == k
 *     shift merged - offset - (merged == k) entries right, write the candidate, merged += merged != k
 * Distances compare as floats (-0.0 ties +0.0; any comparison with NaN is false). Inputs: keys / dists [S][nq][k],
 * counts [S][nq] (clamped to k); computed / visited [S][nq] or null. Outputs [nq][k] padded with key 0 and SNAN_BITS. */
__global__ void merge_into_kernel(uint64_t const* __restrict__ keys, float const* __restrict__ dists, uint32_t const* __restrict__ counts,
                                  uint32_t const* __restrict__ computed, uint32_t const* __restrict__ visited, uint32_t shards,
                                  uint32_t nq, uint32_t k, uint64_t* __restrict__ out_keys, float* __restrict__ out_dists,
                                  uint32_t* __restrict__ out_counts, uint64_t* __restrict__ out_computed,
                                  uint64_t* __restrict__ out_visited) {
    extern __shared__ __align__(16) unsigned char smem[];
    uint32_t const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t const warps = blockDim.x >> 5;
    uint32_t const q = blockIdx.x * warps + warp;
    if (q >= nq) return; /* whole warps leave together */
    uint64_t* row_k = reinterpret_cast<uint64_t*>(smem) + (size_t)warp * k;
    float* row_d = reinterpret_cast<float*>(smem + (size_t)warps * k * 8) + (size_t)warp * k;

    uint32_t merged = 0;
    for (uint32_t s = 0; s < shards; ++s) {
        size_t const slice = (size_t)s * nq + q;
        uint32_t const found = min(counts[slice], k);
        uint64_t const* in_k = keys + slice * k;
        float const* in_d = dists + slice * k;
        for (uint32_t c0 = 0; c0 < found; c0 += 32) {
            uint32_t const m = min(32u, found - c0);
            uint64_t my_k = 0;
            float my_d = 0.f;
            if (lane < m) { my_k = in_k[c0 + lane]; my_d = in_d[c0 + lane]; }
            for (uint32_t j = 0; j < m; ++j) {
                uint64_t const key = __shfl_sync(0xffffffffu, my_k, j);
                float const d = __shfl_sync(0xffffffffu, my_d, j);
                /* std::lower_bound, every lane on the same (broadcast) shared-memory probes */
                uint32_t first = 0, len = merged;
                while (len > 0) {
                    uint32_t const half = len >> 1, mid = first + half;
                    if (row_d[mid] < d) { first = mid + 1; len -= half + 1; }
                    else len = half;
                }
                if (first == k) continue;
                uint32_t const worse = merged - first - (merged == k ? 1u : 0u);
                /* move [first, first + worse) one place right, 32 entries at a time from the top down */
                for (uint32_t hi = first + worse; hi > first;) {
                    uint32_t const lo = hi - first > 32 ? hi - 32 : first;
                    uint32_t const i = lo + lane;
                    uint64_t vk = 0;
                    float vd = 0.f;
                    if (i < hi) { vk = row_k[i]; vd = row_d[i]; }
                    __syncwarp();
                    if (i < hi) { row_k[i + 1] = vk; row_d[i + 1] = vd; }
                    __syncwarp();
                    hi = lo;
                }
                if (lane == 0) { row_k[first] = key; row_d[first] = d; }
                __syncwarp();
                merged += merged != k ? 1u : 0u;
            }
        }
    }
    for (uint32_t i = lane; i < k; i += 32) { /* dump_to padding (index.hpp:2715-2720) */
        out_keys[(size_t)q * k + i] = i < merged ? row_k[i] : 0;
        out_dists[(size_t)q * k + i] = i < merged ? row_d[i] : __uint_as_float(SNAN_BITS);
    }
    if (computed || visited) {
        unsigned long long c = 0, v = 0;
        for (uint32_t s = lane; s < shards; s += 32) {
            if (computed) c += computed[(size_t)s * nq + q];
            if (visited) v += visited[(size_t)s * nq + q];
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            c += __shfl_xor_sync(0xffffffffu, c, o);
            v += __shfl_xor_sync(0xffffffffu, v, o);
        }
        if (lane == 0) { out_computed[q] = c; out_visited[q] = v; }
    }
    if (lane == 0) out_counts[q] = merged;
}

char const* merge_into_launch(uint64_t const* keys, float const* dists, uint32_t const* counts, uint32_t const* computed,
                              uint32_t const* visited, size_t shards, size_t nq, size_t k, uint64_t* out_keys, float* out_dists,
                              uint32_t* out_counts, uint64_t* out_computed, uint64_t* out_visited, cudaStream_t s) {
    if (!nq || !k) return nullptr;
    if (nq > 0x7FFFFFFFull || shards > 0xFFFFFFFFull) return "Too many queries or shards in one merge";
    size_t const per_warp = k * 12;
    if (per_warp > MERGE_MAX_SMEM) return "count too large for the merge: one row must fit in shared memory";
    size_t const warps = std::max<size_t>(1, std::min<size_t>(4, MERGE_MAX_SMEM / per_warp));
    size_t const smem = warps * per_warp;
    if (smem > (48u << 10))
        CU(cudaFuncSetAttribute(merge_into_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    unsigned const blocks = (unsigned)((nq + warps - 1) / warps);
    merge_into_kernel<<<blocks, (unsigned)(warps * 32), smem, s>>>(keys, dists, counts, computed, visited, (uint32_t)shards,
                                                                    (uint32_t)nq, (uint32_t)k, out_keys, out_dists, out_counts,
                                                                    out_computed, out_visited);
    return cuda_error(cudaGetLastError());
}

/* queries of one scalar kind and row stride, shared by every shard that takes them */
struct query_rows_t {
    uint32_t scalar = 0;
    size_t stride = 0;
    bool ready = false; /* holds this call's queries */
    device_buffer_t<uint8_t> rows;
};

} // namespace

struct index_group_t {
    std::vector<frozen_index_t*> members; /* borrowed, in merge order; the same handle may appear more than once */
    std::mutex mutex;                     /* one search (or merge) of the group at a time */
    cuda_stream_t stream;
    cuda_event_t ev_begin, ev_merge, ev_end;
    float last_ms[2] = {0.f, 0.f}; /* searches | merge kernel, of the last search */
    device_buffer_t<uint8_t> raw_queries;
    std::vector<query_rows_t> casts;
    device_buffer_t<uint64_t> keys;
    device_buffer_t<float> dists;
    device_buffer_t<uint32_t> counts, computed, visited;
    device_buffer_t<uint8_t> merged; /* keys u64[nq*k] | computed u64[nq] | visited u64[nq] | distances f32[nq*k] | counts u32[nq] */
    pinned_buffer_t<uint8_t> h_merged;

    char const* ensure_stream(int on_device) {
        if (stream && stream.device == on_device) return nullptr;
        /* the device scratch of the previous device cannot serve this one */
        raw_queries.release();
        casts.clear();
        keys.release(); dists.release(); counts.release(); computed.release(); visited.release(); merged.release();
        h_merged.release();
        stream = cuda_stream_t(on_device);
        if (char const* e = stream.open()) return e;
        CU(ev_begin.create());
        CU(ev_merge.create());
        CU(ev_end.create());
        return nullptr;
    }
    /* the raw queries in `scalar` with rows `stride` bytes apart (zero-padded), cast on the device once per kind */
    char const* rows_for(uint32_t scalar, size_t stride, uint32_t query_scalar, size_t src_bytes, size_t nq, size_t dims,
                         uint8_t const*& out) {
        query_rows_t* c = nullptr;
        for (query_rows_t& r : casts)
            if (r.scalar == scalar && r.stride == stride) c = &r;
        if (!c) {
            casts.emplace_back();
            c = &casts.back();
            c->scalar = scalar;
            c->stride = stride;
        }
        out = c->rows.ptr;
        if (c->ready) return nullptr;
        if (char const* e = c->rows.reserve(nq * stride)) return e;
        if (char const* e = cast_rows_device(raw_queries.ptr, src_bytes, query_scalar, c->rows.ptr, stride, scalar, dims, nq, stream))
            return e;
        c->ready = true;
        out = c->rows.ptr;
        return nullptr;
    }
    char const* search(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k, bool exact, uint64_t* keys_out,
                       float* dists_out, size_t* counts_out, uint64_t* computed_out, uint64_t* visited_out, size_t* total);
};

index_group_t* index_group_create() { return new index_group_t(); }
void index_group_free(index_group_t* g) { delete g; }

void index_group_merge(index_group_t& g, frozen_index_t* member) {
    std::lock_guard<std::mutex> lock(g.mutex);
    g.members.push_back(member);
}

size_t index_group_size(index_group_t& g) {
    std::lock_guard<std::mutex> lock(g.mutex);
    size_t total = 0;
    for (frozen_index_t* m : g.members) total += m->size - m->count_deleted;
    return total;
}

float const* index_group_last_ms(index_group_t& g) { return g.last_ms; }

char const* index_group_search(index_group_t& g, void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k, bool exact,
                               uint64_t* keys, float* dists, size_t* counts, uint64_t* computed, uint64_t* visited, size_t* total) {
    std::lock_guard<std::mutex> lock(g.mutex);
    return g.search(q, nq, stride, query_scalar, k, exact, keys, dists, counts, computed, visited, total);
}

char const* index_group_t::search(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k, bool exact,
                                  uint64_t* keys_out, float* dists_out, size_t* counts_out, uint64_t* computed_out,
                                  uint64_t* visited_out, size_t* total) {
    if (total) *total = 0;
    if (nq == 0 || k == 0) return nullptr;
    if (nq > 0x7FFFFFFFull) return "Too many queries in one batch";
    size_t const S = members.size();
    if (!S) { /* no shards: no matches, no error, as an empty index answers */
        for (size_t i = 0; i < nq * k; ++i) { keys_out[i] = 0; std::memcpy(dists_out + i, &SNAN_BITS, 4); }
        for (size_t i = 0; i < nq; ++i) {
            if (counts_out) counts_out[i] = 0;
            if (computed_out) computed_out[i] = 0;
            if (visited_out) visited_out[i] = 0;
        }
        return nullptr;
    }
    size_t const dims = members[0]->dimensions;
    for (frozen_index_t* m : members) {
        if (m->dimensions != dims) return "Can't search indexes of different dimensions together";
        if (m->stream.device != members[0]->stream.device) return "Can't search indexes that live on different devices together";
        if (m->shards) return "Can't search a sharded handle in Indexes: it holds one shard of its index";
    }
    /* every distinct handle for the whole call, in ascending address order, as join does: no two calls can deadlock */
    std::vector<frozen_index_t*> distinct(members);
    std::sort(distinct.begin(), distinct.end());
    distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
    std::vector<std::unique_lock<std::mutex>> locks;
    locks.reserve(distinct.size());
    for (frozen_index_t* m : distinct) locks.emplace_back(m->mutex);

    if (char const* e = ensure_stream(members[0]->stream.device)) return e;
    cudaStream_t const s = stream;
    size_t const src_bytes = (dims * bits_per_scalar(query_scalar) + 7) / 8;
    if (!src_bytes) return "Unknown scalar kind!";
    if (stride < src_bytes) {
        if (nq != 1 && stride != 0) return "Query stride is smaller than a vector";
        stride = src_bytes;
    }
    if (char const* e = raw_queries.reserve(nq * src_bytes)) return e;
    if (char const* e = keys.reserve(S * nq * k)) return e;
    if (char const* e = dists.reserve(S * nq * k)) return e;
    if (char const* e = counts.reserve(S * nq)) return e;
    if (char const* e = computed.reserve(S * nq)) return e;
    if (char const* e = visited.reserve(S * nq)) return e;
    size_t const merged_bytes = nq * k * 12 + nq * 20;
    if (char const* e = merged.reserve(merged_bytes)) return e;
    if (char const* e = h_merged.reserve(merged_bytes)) return e;
    for (query_rows_t& c : casts) c.ready = false;

    CU(cudaEventRecord(ev_begin, s));
    CU(cudaMemcpy2DAsync(raw_queries.ptr, src_bytes, q, stride, src_bytes, nq, cudaMemcpyHostToDevice, s));
    size_t exact_computed = 0; /* search_exact_ (index.hpp:4251-4268) measures every live member and visits none */
    auto run_shard = [&](size_t i) -> char const* {
        frozen_index_t& m = *members[i];
        uint64_t* sk = keys.ptr + i * nq * k;
        float* sd = dists.ptr + i * nq * k;
        uint32_t* sc = counts.ptr + i * nq;
        uint32_t* scomp = computed.ptr + i * nq;
        uint32_t* svis = visited.ptr + i * nq;
        if (char const* e = m.ensure_context()) return e;
        if (!m.loaded || m.d.n == 0) { /* no matches, no error (index.hpp:3036-3037) */
            CU(search_fill_empty(sk, sd, sc, scomp, svis, nq, k, s));
            return nullptr;
        }
        uint8_t const* rows = nullptr;
        if (char const* e = rows_for(m.scalar, m.d.vec_stride, query_scalar, src_bytes, nq, dims, rows)) return e;
        if (exact) {
            if (char const* e = exact_search_device(m.d, m.stream.sm_count, rows, nq, m.d.vec_stride, k, false, false, sk, sd, sc,
                                                    m.exact_scratch, s))
                return e;
            m.kernel_launches += 2;
            CU(cudaMemsetAsync(scomp, 0, nq * 4, s));
            CU(cudaMemsetAsync(svis, 0, nq * 4, s));
            exact_computed += m.size - m.count_deleted;
            return nullptr;
        }
        return m.search_device(rows, nq, m.d.vec_stride, k, sk, sd, sc, scomp, svis, s, true);
    };
    char const* error = nullptr;
    for (size_t i = 0; i < S && !error; ++i) error = run_shard(i);
    /* the deferred searches, also after a failed launch: wait, then retry the queries whose scratch overflowed, as a
     * single search does */
    for (frozen_index_t* m : distinct)
        if (!m->pending.empty()) /* exact searches and empty shards defer nothing */
            if (char const* e = m->search_finish()) error = error ? error : e;
    if (error) return error;

    uint8_t* p = merged.ptr;
    uint64_t* mk = reinterpret_cast<uint64_t*>(p);
    uint64_t* mcomp = mk + nq * k;
    uint64_t* mvis = mcomp + nq;
    float* md = reinterpret_cast<float*>(mvis + nq);
    uint32_t* mc = reinterpret_cast<uint32_t*>(md + nq * k);
    CU(cudaEventRecord(ev_merge, s));
    if (char const* e = merge_into_launch(keys.ptr, dists.ptr, counts.ptr, computed.ptr, visited.ptr, S, nq, k, mk, md, mc, mcomp, mvis, s))
        return e;
    CU(cudaEventRecord(ev_end, s));
    CU(cudaMemcpyAsync(h_merged.ptr, p, merged_bytes, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaEventElapsedTime(&last_ms[0], ev_begin, ev_merge));
    CU(cudaEventElapsedTime(&last_ms[1], ev_merge, ev_end));

    uint8_t const* h = h_merged.ptr;
    std::memcpy(keys_out, h, nq * k * 8);
    std::memcpy(dists_out, h + nq * k * 8 + nq * 16, nq * k * 4);
    uint64_t const* hcomp = reinterpret_cast<uint64_t const*>(h + nq * k * 8);
    uint64_t const* hvis = hcomp + nq;
    uint32_t const* hc = reinterpret_cast<uint32_t const*>(h + nq * k * 12 + nq * 16);
    size_t sum = 0;
    for (size_t i = 0; i < nq; ++i) {
        sum += hc[i];
        if (counts_out) counts_out[i] = hc[i];
        if (computed_out) computed_out[i] = hcomp[i] + exact_computed;
        if (visited_out) visited_out[i] = hvis[i];
    }
    if (total) *total = sum;
    return nullptr;
}

/* the merge kernel on host rows: keys / distances [shards][nq][k], counts [shards][nq] -> merged [nq][k], counts [nq] */
char const* indexes_merge_host(uint64_t const* keys, float const* dists, uint32_t const* counts, size_t shards, size_t nq, size_t k,
                               uint64_t* out_keys, float* out_dists, uint32_t* out_counts) {
    if (!nq || !k) return nullptr;
    cuda_stream_t s(default_device());
    if (char const* e = s.open()) return e;
    size_t const rows = std::max<size_t>(shards, 1) * nq;
    device_buffer_t<uint64_t> dk, ok;
    device_buffer_t<float> dd, od;
    device_buffer_t<uint32_t> dc, oc;
    if (char const* e = dk.reserve(rows * k)) return e;
    if (char const* e = dd.reserve(rows * k)) return e;
    if (char const* e = dc.reserve(rows)) return e;
    if (char const* e = ok.reserve(nq * k)) return e;
    if (char const* e = od.reserve(nq * k)) return e;
    if (char const* e = oc.reserve(nq)) return e;
    if (shards) {
        CU(cudaMemcpyAsync(dk.ptr, keys, shards * nq * k * 8, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(dd.ptr, dists, shards * nq * k * 4, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(dc.ptr, counts, shards * nq * 4, cudaMemcpyHostToDevice, s));
    }
    if (char const* e = merge_into_launch(dk.ptr, dd.ptr, dc.ptr, nullptr, nullptr, shards, nq, k, ok.ptr, od.ptr, oc.ptr, nullptr,
                                          nullptr, s))
        return e;
    CU(cudaMemcpyAsync(out_keys, ok.ptr, nq * k * 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(out_dists, od.ptr, nq * k * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(out_counts, oc.ptr, nq * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return nullptr;
}

} // namespace usearch_b200
