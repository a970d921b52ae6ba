/*
 *  shards.cu — the sharded search behind the C ABI (SURVEY.md §8 row a16 / §8e).
 *
 *  The reference shards on the CPU (`Indexes`, python/lib.cpp:74-107): every query is searched in every shard and the
 *  per-shard results are merged by distance (`search_typed(dense_indexes_py_t&)`, python/lib.cpp:321-402 ->
 *  search_result_t::merge_into, index.hpp:2650-2670). Here one process per GPU holds one shard; a sharded search is
 *      1. the batched search of this shard, its kernel writing keys | distances | counts straight into ONE packed payload,
 *      2. ONE ncclAllGather of that payload (NVLink / NVSwitch) on the same stream,
 *      3. merge_topk_kernel: a warp per query, a lane per shard holding the head of that shard's ascending list; k rounds of
 *         a warp arg-min ordered by (distance, shard, position) — deterministic, where the reference's tie order depends
 *         on which thread reaches the per-query lock first (SURVEY.md §3.3).
 *  NCCL is bound at run time (dlopen of libnccl.so.2: the copy torch ships when the host process is a torch process, the
 *  system library for a plain C client), so the library has no link-time dependency on it and single-GPU users never load it.
 *  The 128-byte ncclUniqueId travels over whatever control plane the host side has (torch.distributed, MPI, a file).
 */
#include <dlfcn.h>

#include <cstring>

#include "cuda_check.h"
#include "frozen_index.h"

namespace usearch_b200 {

namespace {


/* ---- the five NCCL entry points this file needs, resolved at run time (nccl.h: ncclResult_t == int, 0 = success) ---- */

struct nccl_unique_id_t { char internal[128]; };
typedef void* nccl_comm_t;
enum { NCCL_UINT8 = 1 }; /* ncclDataType_t: ncclInt8 0, ncclUint8 1, ... */

struct nccl_api_t {
    void* lib = nullptr;
    int (*get_unique_id)(nccl_unique_id_t*) = nullptr;
    int (*comm_init_rank)(nccl_comm_t*, int, nccl_unique_id_t, int) = nullptr;
    int (*all_gather)(void const*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*comm_destroy)(nccl_comm_t) = nullptr;
    char const* (*get_error_string)(int) = nullptr;
    char const* load() {
        if (lib) return nullptr;
        char const* names[] = {"libnccl.so.2", "libnccl.so"};
        for (char const* name : names)
            if ((lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL))) break;
        if (!lib) return "NCCL is not available: libnccl.so.2 could not be loaded";
        get_unique_id = reinterpret_cast<decltype(get_unique_id)>(dlsym(lib, "ncclGetUniqueId"));
        comm_init_rank = reinterpret_cast<decltype(comm_init_rank)>(dlsym(lib, "ncclCommInitRank"));
        all_gather = reinterpret_cast<decltype(all_gather)>(dlsym(lib, "ncclAllGather"));
        comm_destroy = reinterpret_cast<decltype(comm_destroy)>(dlsym(lib, "ncclCommDestroy"));
        get_error_string = reinterpret_cast<decltype(get_error_string)>(dlsym(lib, "ncclGetErrorString"));
        if (!get_unique_id || !comm_init_rank || !all_gather || !comm_destroy) return "NCCL is not available: symbols missing";
        return nullptr;
    }
    char const* check(int rc) const {
        if (rc == 0) return nullptr;
        static thread_local char message[200];
        std::snprintf(message, sizeof(message), "NCCL failure: %s", get_error_string ? get_error_string(rc) : "unknown");
        return message;
    }
};

nccl_api_t& nccl() {
    static nccl_api_t api;
    return api;
}

/* ---- the merge ------------------------------------------------------------------------------------------------------- */

/* payload of one shard for nq queries and k results each: keys u64[nq*k] | distances f32[nq*k] | counts u32[nq], padded to 16 B */
__host__ __device__ inline size_t payload_bytes(size_t nq, size_t k) { return (nq * (12 * k + 4) + 15) / 16 * 16; }

__global__ void merge_topk_kernel(uint8_t const* gathered, size_t stride, int world, uint32_t nq, uint32_t k, uint64_t* out_keys,
                                  uint32_t* out_dist_bits, uint32_t* out_counts) {
    uint32_t const q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int const lane = threadIdx.x & 31;
    if (q >= nq) return; /* whole warps leave together */
    /* lane r walks shard r's ascending list */
    uint8_t const* mine = gathered + (size_t)lane * stride;
    uint64_t const* keys = reinterpret_cast<uint64_t const*>(mine) + (size_t)q * k;
    float const* dists = reinterpret_cast<float const*>(mine + (size_t)nq * k * 8) + (size_t)q * k;
    uint32_t count = 0;
    if (lane < world) count = min(reinterpret_cast<uint32_t const*>(mine + (size_t)nq * k * 12)[q], k);
    uint32_t head = 0;
    float head_d = 0.f;
    if (head < count) head_d = dists[head];
    uint32_t total = 0;
    for (uint32_t i = 0; i < k; ++i) {
        /* arg-min over the lanes that still hold an entry: (is-NaN, distance, shard) ascending */
        bool const have = head < count;
        bool best_nan = !have || head_d != head_d;
        float best = have && !best_nan ? head_d : 0.f;
        int who = have ? lane : 64;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            bool const o_nan = __shfl_xor_sync(0xffffffffu, (int)best_nan, o) != 0;
            float const o_d = __shfl_xor_sync(0xffffffffu, best, o);
            int const o_who = __shfl_xor_sync(0xffffffffu, who, o);
            bool take;
            if (o_who == 64) take = false;
            else if (who == 64) take = true;
            else if (o_nan != best_nan) take = best_nan; /* numbers before NaNs */
            else if (!o_nan && o_d != best) take = o_d < best;
            else take = o_who < who;
            if (take) { best_nan = o_nan; best = o_d; who = o_who; }
        }
        if (who == 64) break; /* uniform: every list is exhausted */
        if (lane == who) {
            out_keys[(size_t)q * k + i] = keys[head];
            out_dist_bits[(size_t)q * k + i] = __float_as_uint(head_d);
            head += 1;
            if (head < count) head_d = dists[head];
        }
        total += 1;
    }
    for (uint32_t i = total + lane; i < k; i += 32) { /* dump_to padding (index.hpp:2715-2720) */
        out_keys[(size_t)q * k + i] = 0;
        out_dist_bits[(size_t)q * k + i] = SNAN_BITS;
    }
    if (lane == 0) out_counts[q] = total;
}

} // namespace

struct shard_group_t {
    int rank = 0, world = 1;
    nccl_comm_t comm = nullptr;
    device_buffer_t<uint8_t> send, recv;
    ~shard_group_t() {
        if (comm) nccl().comm_destroy(comm);
    }
};

size_t shards_payload_bytes(size_t nq, size_t k) { return payload_bytes(nq, k); }

cudaError_t shards_merge_launch(uint8_t const* gathered, size_t stride, int world, size_t nq, size_t k, uint64_t* keys, float* dists,
                                uint32_t* counts, cudaStream_t s) {
    unsigned const threads = 128, blocks = (unsigned)((nq * 32 + threads - 1) / threads);
    merge_topk_kernel<<<blocks, threads, 0, s>>>(gathered, stride, world, (uint32_t)nq, (uint32_t)k, keys,
                                                 reinterpret_cast<uint32_t*>(dists), counts);
    return cudaGetLastError();
}

char const* shards_unique_id(void* out128) {
    if (char const* e = nccl().load()) return e;
    nccl_unique_id_t id;
    if (char const* e = nccl().check(nccl().get_unique_id(&id))) return e;
    std::memcpy(out128, &id, 128);
    return nullptr;
}

void frozen_index_t::leave_shards() {
    delete shards;
    shards = nullptr;
}

/* collective: every rank of the group calls it with the same id */
char const* frozen_index_t::join_shards(int rank, int world, void const* unique_id128) {
    if (world < 1 || world > 32 || rank < 0 || rank >= world) return "Shard rank / world size out of range (1..32 shards)";
    if (char const* e = ensure_context()) return e;
    leave_shards();
    shards = new shard_group_t();
    shards->rank = rank;
    shards->world = world;
    if (world == 1) return nullptr;
    if (char const* e = nccl().load()) return e;
    nccl_unique_id_t id;
    std::memcpy(&id, unique_id128, 128);
    return nccl().check(nccl().comm_init_rank(&shards->comm, world, id, rank));
}

/* this shard's search + all-gather + merge; queries and outputs in device memory; every rank receives the merged rows */
char const* frozen_index_t::sharded_search_device(void const* d_queries, size_t nq, size_t stride, size_t k, uint64_t* d_keys,
                                                  float* d_dists, uint32_t* d_counts, uint32_t* d_computed, uint32_t* d_cycles,
                                                  cudaStream_t s) {
    if (!shards || shards->world == 1) return search_device(d_queries, nq, stride, k, d_keys, d_dists, d_counts, d_computed, d_cycles, s);
    if (nq == 0 || k == 0) return nullptr;
    size_t const bytes = payload_bytes(nq, k);
    if (char const* e = shards->send.reserve(bytes)) return e;
    if (char const* e = shards->recv.reserve(bytes * (size_t)shards->world)) return e;
    uint8_t* p = shards->send.ptr;
    if (char const* e = search_device(d_queries, nq, stride, k, reinterpret_cast<uint64_t*>(p), reinterpret_cast<float*>(p + nq * k * 8),
                                      reinterpret_cast<uint32_t*>(p + nq * k * 12), d_computed, d_cycles, s))
        return e;
    if (char const* e = nccl().check(nccl().all_gather(shards->send.ptr, shards->recv.ptr, bytes, NCCL_UINT8, shards->comm, s))) return e;
    CU(shards_merge_launch(shards->recv.ptr, bytes, shards->world, nq, k, d_keys, d_dists, d_counts, s));
    kernel_launches += 1;
    return nullptr;
}

/* the same on host buffers: H2D of the queries and D2H of the merged rows inside the call */
char const* frozen_index_t::sharded_search_host(void const* q, size_t nq, size_t stride, uint32_t query_scalar, size_t k,
                                                host_results_t const& out, size_t* total) {
    if (nq == 0 || k == 0) return nullptr;
    std::lock_guard<std::mutex> lock(mutex);
    if (char const* e = ensure_context()) return e;
    if (!configured()) return "Index is not initialized";
    if (!loaded) /* an empty shard still takes part in the exchange */
        if (char const* e = reserve_slots(0)) return e;
    return search_round_trip(q, nq, stride, query_scalar, k, out, total, [&](void const* dq, size_t vs, device_results_t const& r) {
        return sharded_search_device(dq, nq, vs, k, r.keys, r.dists, r.counts, r.computed, r.visited, stream);
    });
}

/* `world` payloads (host memory, back to back, each shards_payload_bytes(nq, k) long) -> merged rows (host memory): the
 * merge kernel on its own, for single-process multi-shard callers and for the parity tests */
char const* shards_merge_host(void const* payloads, int world, size_t nq, size_t k, uint64_t* keys, float* dists, uint32_t* counts) {
    if (world < 1 || world > 32) return "Shard rank / world size out of range (1..32 shards)";
    if (!nq || !k) return nullptr;
    cuda_stream_t s(default_device());
    if (char const* e = s.open()) return e;
    size_t const bytes = payload_bytes(nq, k);
    device_buffer_t<uint8_t> in;
    device_buffer_t<uint64_t> dk;
    device_buffer_t<float> dd;
    device_buffer_t<uint32_t> dc;
    if (char const* e = in.reserve(bytes * (size_t)world)) return e;
    if (char const* e = dk.reserve(nq * k)) return e;
    if (char const* e = dd.reserve(nq * k)) return e;
    if (char const* e = dc.reserve(nq)) return e;
    CU(cudaMemcpyAsync(in.ptr, payloads, bytes * (size_t)world, cudaMemcpyHostToDevice, s));
    CU(shards_merge_launch(in.ptr, bytes, world, nq, k, dk.ptr, dd.ptr, dc.ptr, s));
    CU(cudaMemcpyAsync(keys, dk.ptr, nq * k * 8, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(dists, dd.ptr, nq * k * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(counts, dc.ptr, nq * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return nullptr;
}

} // namespace usearch_b200
