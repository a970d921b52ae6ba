/*
 *  exact_free.cu — usearch_exact_search (c/lib.cpp:468-501) and its device twin: brute force over a caller's raw matrix,
 *  keys are dataset row numbers.
 *
 *  The dataset is scanned in chunks of rows. A chunk is a device_index_t over rows laid out like an index's (vec_stride
 *  apart, zero tails); the exact kernels scan it (exact_kernel.cu), and the merge folds its lists into the top-k of the
 *  chunks before, carried in the output rows, as one more segment. The order is total, so every cut of the dataset gives
 *  the one-chunk result bit for bit. The plan (chunk_rows):
 *    - rows per chunk from free HBM, after the queries, the outputs and the scan's scratch, over two chunk buffers, so
 *      that chunk c + 1 loads while chunk c is scanned; a dataset larger than HBM simply takes more chunks;
 *    - a host dataset that fits is still cut into up to 8 chunks of at least 256 MB, so that its upload hides under the
 *      scans: only the first upload and the last scan are exposed;
 *    - device rows that already have the layout are scanned in place, as one chunk;
 *    - USEARCH_B200_EXACT_CHUNK_ROWS forces the rows per chunk (tests cross many boundaries on small data).
 *  Host rows are pageable memory, which an asynchronous copy cannot overlap. The host copies them (with a few threads,
 *  honouring the caller's stride, tails zeroed) into a ring of pinned slots, and each slot is uploaded on a copy stream:
 *  the host fills one slot while the one before uploads and the previous chunk is scanned. The host waits only to reuse
 *  a slot whose upload has not finished.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "cuda_check.h"
#include "frozen_index.h"

namespace usearch_b200 {
namespace {

constexpr size_t CHUNK_MIN_BYTES = 256ull << 20; /* a host dataset up to this size is one chunk */
constexpr size_t CHUNKS_FOR_OVERLAP = 8;          /* a fitting host dataset: the first upload and the last scan are 1/8 each */
constexpr size_t SLOT_BYTES = 64ull << 20;        /* one pinned staging slot */
constexpr unsigned SLOTS = 4;
constexpr size_t HBM_MARGIN = 512ull << 20;       /* left free: the context and the allocator's rounding */
constexpr size_t FILL_SPLIT_BYTES = 4ull << 20;   /* a slot fill smaller than this runs on the calling thread */

char const* const NO_DEVICE = "No CUDA device: the GPU search backend has no CPU fallback";

size_t forced_chunk_rows() { /* test hook: USEARCH_B200_EXACT_CHUNK_ROWS=<rows per chunk> */
    static size_t const rows = [] {
        char const* v = std::getenv("USEARCH_B200_EXACT_CHUNK_ROWS");
        return v && std::atoll(v) > 0 ? (size_t)std::atoll(v) : (size_t)0;
    }();
    return rows;
}

/* the row layout, metric and scalar kind of a free search: rows padded to whole 16-byte chunks */
device_index_t free_shape(uint32_t scalar, size_t dimensions, uint32_t metric) {
    size_t const bpv = (dimensions * bits_per_scalar(scalar) + 7) / 8, vs = (bpv + 15) / 16 * 16;
    device_index_t ix;
    ix.n = 1;
    ix.dims = (uint32_t)dimensions;
    ix.bytes_per_vector = (uint32_t)bpv;
    ix.vec_stride = vs;
    ix.chunks16 = (uint32_t)(vs / 16);
    ix.metric = metric;
    ix.scalar = scalar;
    return ix;
}

/* the refusals both entries share, in the order the free search has always checked them */
char const* check_counts(size_t n, size_t nq, size_t k) {
    if (!nq || !k) return nullptr;
    if (k > n) return "More neighbours requested than the dataset holds";
    if (n >= 0xFFFFFFFFull) return "Too many entries for 32-bit slots";
    return nullptr;
}

/* device memory the scan needs besides the chunk buffers: queries, dense outputs, and a bound on exact_run's scratch
 * (partial lists capped near 1 GB unless one segment's lists exceed it, their counts, the merged lists of count > 256) */
size_t fixed_bytes(size_t nq, size_t vs, size_t k) {
    size_t const lists = std::max<size_t>((size_t)1 << 30, nq * k * 8);
    return nq * vs + nq * k * 16 + lists + lists / 2 + nq * k * 8 + nq * 8;
}

/* where the rows of a chunk come from: rows [first, first + count) into `dst`, rows vec_stride apart with zero tails,
 * enqueued on the copy stream */
struct chunk_source_t {
    virtual ~chunk_source_t() = default;
    virtual char const* load(size_t first, size_t count, uint8_t* dst) = 0;
};

/* rows of a host matrix through the ring of pinned slots */
struct host_source_t final : chunk_source_t {
    uint8_t const* rows;
    size_t stride, bpv, vs, n;
    unsigned threads;
    cudaStream_t copy;
    size_t slot_rows = 0;
    pinned_buffer_t<uint8_t> ring;
    cuda_event_t uploaded[SLOTS];
    bool pending[SLOTS] = {};
    unsigned next = 0;

    host_source_t(void const* data, size_t stride_, size_t bpv_, size_t vs_, size_t n_, unsigned threads_, cudaStream_t copy_)
        : rows(static_cast<uint8_t const*>(data)), stride(stride_), bpv(bpv_), vs(vs_), n(n_), threads(threads_), copy(copy_) {}

    /* rows [first, first + count) of the matrix into `slot`, each padded to vs with zeros */
    void fill_rows(uint8_t* slot, size_t first, size_t lo, size_t hi) const {
        if (stride == vs && bpv == vs) {
            std::memcpy(slot + lo * vs, rows + (first + lo) * stride, (hi - lo) * vs);
            return;
        }
        for (size_t i = lo; i < hi; ++i) {
            std::memcpy(slot + i * vs, rows + (first + i) * stride, bpv);
            if (vs != bpv) std::memset(slot + i * vs + bpv, 0, vs - bpv);
        }
    }
    void fill(uint8_t* slot, size_t first, size_t count) const {
        unsigned const t = count * bpv >= FILL_SPLIT_BYTES ? std::max(1u, threads) : 1u;
        std::vector<std::thread> pool;
        unsigned started = 1;
        for (; started < t; ++started) {
            try {
                pool.emplace_back([=] { fill_rows(slot, first, count * started / t, count * (started + 1) / t); });
            } catch (...) {
                break; /* no thread to spare: the calling thread copies the rest */
            }
        }
        fill_rows(slot, first, 0, count / t);
        if (started < t) fill_rows(slot, first, count * started / t, count);
        for (std::thread& th : pool) th.join();
    }

    char const* load(size_t first, size_t count, uint8_t* dst) override {
        if (!ring.ptr) {
            slot_rows = std::max<size_t>(1, std::min(SLOT_BYTES / vs, n));
            if (char const* e = ring.reserve(SLOTS * slot_rows * vs)) return e;
            for (cuda_event_t& ev : uploaded) CU(ev.create(cudaEventDisableTiming));
        }
        for (size_t done = 0; done < count;) {
            size_t const r = std::min(slot_rows, count - done);
            unsigned const s = next;
            next = (next + 1) % SLOTS;
            if (pending[s]) CU(cudaEventSynchronize(uploaded[s])); /* the slot's last upload has read it */
            uint8_t* const slot = ring.ptr + (size_t)s * slot_rows * vs;
            fill(slot, first + done, r);
            CU(cudaMemcpyAsync(dst + done * vs, slot, r * vs, cudaMemcpyHostToDevice, copy));
            CU(cudaEventRecord(uploaded[s], copy));
            pending[s] = true;
            done += r;
        }
        return nullptr;
    }
};

/* rows of a device matrix whose layout the kernels cannot read in place: repacked by a 2D copy */
struct device_source_t final : chunk_source_t {
    uint8_t const* rows;
    size_t stride, bpv, vs;
    cudaStream_t copy;
    device_source_t(void const* data, size_t stride_, size_t bpv_, size_t vs_, cudaStream_t copy_)
        : rows(static_cast<uint8_t const*>(data)), stride(stride_), bpv(bpv_), vs(vs_), copy(copy_) {}
    char const* load(size_t first, size_t count, uint8_t* dst) override {
        CU(cudaMemcpy2DAsync(dst, vs, rows + first * stride, stride, bpv, count, cudaMemcpyDeviceToDevice, copy));
        return nullptr;
    }
};

/* rows per chunk. `buffers` chunk buffers (0: the rows are scanned in place) share free HBM after `fixed` bytes. */
char const* chunk_rows(size_t n, size_t vs, size_t per_row_extra, size_t fixed, unsigned buffers, bool overlap, size_t* rows) {
    size_t r = n;
    if (buffers) {
        size_t free_bytes = 0, total_bytes = 0;
        CU(cudaMemGetInfo(&free_bytes, &total_bytes));
        size_t const per_row = buffers * vs + per_row_extra;
        if (free_bytes < fixed + HBM_MARGIN + per_row) return "Out of GPU memory!";
        r = std::min(n, (free_bytes - fixed - HBM_MARGIN) / per_row);
        if (overlap) {
            size_t const chunks = std::max<size_t>(1, std::min(CHUNKS_FOR_OVERLAP, n * vs / CHUNK_MIN_BYTES));
            r = std::min(r, (n + chunks - 1) / chunks);
        }
    }
    if (size_t const forced = forced_chunk_rows()) r = std::min(n, forced);
    *rows = r;
    return nullptr;
}

/* one free search, chunk by chunk */
struct free_run_t {
    device_index_t shape;              /* metric, scalar kind and row layout */
    size_t n = 0;                      /* dataset rows */
    uint8_t const* in_place = nullptr; /* rows already laid out (vec_stride apart, zero tails), or null: `source` loads them */
    chunk_source_t* source = nullptr;
    cudaStream_t stream = nullptr;     /* scans, merges and every buffer's allocation */
    cudaStream_t copy = nullptr;       /* loads; the same stream, or a second one that overlaps them with the scans */
    bool overlap = false;              /* cut a fitting dataset for overlap */
    int sm_count = 0;
};

/* before the buffers of run_chunks go back to the pool (in `stream` order), `stream` waits for what `copy` still does */
struct join_copy_t {
    cudaStream_t stream, copy;
    ~join_copy_t() {
        if (copy == stream) return;
        cuda_event_t copied;
        if (copied.create(cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(copied, copy) != cudaSuccess ||
            cudaStreamWaitEvent(stream, copied, 0) != cudaSuccess) {
            cudaGetLastError();
            cudaStreamSynchronize(copy); /* no event: wait here instead */
        }
    }
};

char const* run_chunks(free_run_t const& r, uint8_t const* d_queries, size_t nq, size_t query_stride, size_t k, uint64_t* d_keys,
                       float* d_dists, uint32_t* d_counts) {
    size_t const vs = r.shape.vec_stride, bpv = r.shape.bytes_per_vector;
    bool const norms = search_needs_norms(r.shape.metric, r.shape.scalar);
    unsigned const buffers = r.in_place ? 0u : (r.copy == r.stream ? 1u : 2u);
    size_t const extra = (norms ? 4 : 0) + (r.shape.scalar == SCALAR_I8 ? 4 : 0); /* norms, i8 self dots */
    size_t rows = 0;
    if (char const* e = chunk_rows(r.n, vs, extra, fixed_bytes(nq, vs, k), buffers, r.overlap, &rows)) return e;
    size_t const chunks = (r.n + rows - 1) / rows;

    stream_buffer_t<uint8_t> buf0(r.stream), buf1(r.stream), scratch(r.stream);
    stream_buffer_t<uint8_t>* const buf[2] = {&buf0, &buf1};
    stream_buffer_t<float> row_norms(r.stream);
    for (unsigned b = 0; b < buffers; ++b) {
        if (char const* e = buf[b]->reserve(rows * vs)) return e;
        if (vs != bpv) CU(cudaMemsetAsync(buf[b]->ptr, 0, rows * vs, r.stream)); /* the loads write bpv bytes of each row */
    }
    if (norms)
        if (char const* e = row_norms.reserve(rows)) return e;
    join_copy_t const join{r.stream, r.copy};
    cuda_event_t ready[2], done[2];
    if (buffers == 2) {
        cuda_event_t allocated;
        for (unsigned b = 0; b < 2; ++b) {
            CU(ready[b].create(cudaEventDisableTiming));
            CU(done[b].create(cudaEventDisableTiming));
        }
        CU(allocated.create(cudaEventDisableTiming));
        CU(cudaEventRecord(allocated, r.stream));
        CU(cudaStreamWaitEvent(r.copy, allocated, 0)); /* the buffers exist in stream order */
    }

    for (size_t c = 0; c < chunks; ++c) {
        size_t const first = c * rows, count = std::min(rows, r.n - first);
        unsigned const b = (unsigned)(c & 1u) % std::max(1u, buffers);
        device_index_t ix = r.shape;
        ix.n = (uint32_t)count;
        if (r.in_place) {
            ix.vectors = r.in_place + first * vs;
        } else {
            if (buffers == 2 && c >= 2) CU(cudaStreamWaitEvent(r.copy, done[b], 0)); /* chunk c - 2 is scanned */
            if (char const* e = r.source->load(first, count, buf[b]->ptr)) return e;
            if (buffers == 2) {
                CU(cudaEventRecord(ready[b], r.copy));
                CU(cudaStreamWaitEvent(r.stream, ready[b], 0));
            }
            ix.vectors = buf[b]->ptr;
        }
        if (norms) {
            CU(search_compute_norms(ix, row_norms.ptr, r.stream));
            ix.norms = row_norms.ptr;
        }
        if (char const* e = exact_search_chunk_device(ix, r.sm_count, d_queries, nq, query_stride, k, (uint32_t)first, c > 0, d_keys,
                                                      d_dists, d_counts, scratch, r.stream))
            return e;
        if (buffers == 2) CU(cudaEventRecord(done[b], r.stream));
    }
    return nullptr;
}

/* the device a caller's array lives on, or -1 when it is not device memory */
int device_of(void const* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged ? at.device : -1;
}

struct restore_device_t {
    int device = -1;
    ~restore_device_t() {
        if (device >= 0) cudaSetDevice(device);
    }
};

} // namespace

/* usearch_exact_search (c/lib.cpp:468-501): many-to-many over host matrices; keys are dataset row numbers */
char const* exact_search_free(void const* dataset, size_t n, size_t dataset_stride, void const* queries_h, size_t nq, size_t queries_stride,
                              uint32_t scalar, size_t dimensions, uint32_t metric, size_t k, size_t threads, uint64_t* keys,
                              size_t keys_stride, float* distances, size_t distances_stride) {
    if (!search_supported(metric, scalar)) return "This metric / scalar kind has no sm_90a kernel and the backend has no CPU fallback";
    if (!nq || !k) return nullptr;
    if (char const* e = check_counts(n, nq, k)) return e;
    cuda_stream_t s(default_device()), copy(default_device());
    if (char const* e = s.open()) return e;
    if (char const* e = copy.open()) return e;
    device_index_t const shape = free_shape(scalar, dimensions, metric);
    if (char const* e = exact_search_check(shape, k)) return e;
    size_t const bpv = shape.bytes_per_vector, vs = shape.vec_stride;
    unsigned const fill_threads = threads ? (unsigned)std::min<size_t>(threads, 64)
                                          : std::max(1u, std::min(8u, std::thread::hardware_concurrency()));
    host_source_t source(dataset, dataset_stride, bpv, vs, n, fill_threads, copy);
    char const* e = [&]() -> char const* {
        stream_buffer_t<uint8_t> d_queries(s);
        stream_buffer_t<uint64_t> d_keys(s);
        stream_buffer_t<float> d_dists(s);
        stream_buffer_t<uint32_t> d_counts(s);
        if (char const* e = d_queries.reserve(nq * vs)) return e;
        if (char const* e = d_keys.reserve(nq * k)) return e;
        if (char const* e = d_dists.reserve(nq * k)) return e;
        if (char const* e = d_counts.reserve(nq)) return e;
        if (vs != bpv) CU(cudaMemsetAsync(d_queries.ptr, 0, nq * vs, s));
        CU(cudaMemcpy2DAsync(d_queries.ptr, vs, queries_h, queries_stride, bpv, nq, cudaMemcpyHostToDevice, s));
        free_run_t r;
        r.shape = shape;
        r.n = n;
        r.source = &source;
        r.stream = s;
        r.copy = copy;
        r.overlap = true;
        r.sm_count = s.sm_count;
        if (char const* e = run_chunks(r, d_queries.ptr, nq, vs, k, d_keys.ptr, d_dists.ptr, d_counts.ptr)) return e;
        CU(cudaMemcpy2DAsync(keys, keys_stride, d_keys.ptr, k * 8, k * 8, nq, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpy2DAsync(distances, distances_stride, d_dists.ptr, k * 4, k * 4, nq, cudaMemcpyDeviceToHost, s));
        return nullptr;
    }();
    /* the pinned ring and the caller's rows outlive every copy that reads them */
    char const* const e_copy = cuda_error(cudaStreamSynchronize(copy));
    char const* const e_scan = cuda_error(cudaStreamSynchronize(s));
    return e ? e : (e_copy ? e_copy : e_scan);
}

/* the same over device matrices, in the caller's stream, without waiting for it */
char const* exact_search_free_device(void const* dataset, size_t n, size_t dataset_stride, void const* queries, size_t nq,
                                     size_t queries_stride, uint32_t scalar, size_t dimensions, uint32_t metric, size_t k, uint64_t* keys,
                                     size_t keys_stride, float* distances, size_t distances_stride, cudaStream_t stream) {
    if (!search_supported(metric, scalar)) return "This metric / scalar kind has no sm_90a kernel and the backend has no CPU fallback";
    if (!nq || !k) return nullptr;
    if (char const* e = check_counts(n, nq, k)) return e;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
        cudaGetLastError();
        return NO_DEVICE;
    }
    if (!dataset || !queries || !keys || !distances) return "The dataset, queries and outputs must be device arrays";
    int const device = device_of(dataset);
    if (device < 0 || device_of(queries) != device || device_of(keys) != device || device_of(distances) != device)
        return "The dataset, queries and outputs must be device arrays on one device";
    device_index_t const shape = free_shape(scalar, dimensions, metric);
    size_t const bpv = shape.bytes_per_vector, vs = shape.vec_stride;
    if (!keys_stride) keys_stride = k * 8;
    if (!distances_stride) distances_stride = k * 4;
    if (dataset_stride < bpv || queries_stride < bpv || keys_stride < k * 8 || distances_stride < k * 4)
        return "A row stride is shorter than its row";
    if (char const* e = exact_search_check(shape, k)) return e;
    restore_device_t restore;
    CU(cudaGetDevice(&restore.device));
    CU(cudaSetDevice(device));
    int sm_count = 0;
    CU(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));

    /* the kernels read vec_stride bytes per row, vec_stride apart: in place only when that is the caller's layout */
    auto aligned = [](void const* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    bool const rows_in_place = aligned(dataset) && dataset_stride == vs && bpv == vs;
    bool const queries_in_place = aligned(queries) && queries_stride % 16 == 0 && bpv == vs;
    stream_buffer_t<uint8_t> d_queries(stream);
    stream_buffer_t<uint64_t> d_keys(stream);
    stream_buffer_t<float> d_dists(stream);
    stream_buffer_t<uint32_t> d_counts(stream);
    if (char const* e = d_keys.reserve(nq * k)) return e;
    if (char const* e = d_dists.reserve(nq * k)) return e;
    if (char const* e = d_counts.reserve(nq)) return e;
    uint8_t const* q = static_cast<uint8_t const*>(queries);
    size_t q_stride = queries_stride;
    if (!queries_in_place) {
        if (char const* e = d_queries.reserve(nq * vs)) return e;
        if (vs != bpv) CU(cudaMemsetAsync(d_queries.ptr, 0, nq * vs, stream));
        CU(cudaMemcpy2DAsync(d_queries.ptr, vs, queries, queries_stride, bpv, nq, cudaMemcpyDeviceToDevice, stream));
        q = d_queries.ptr;
        q_stride = vs;
    }
    device_source_t source(dataset, dataset_stride, bpv, vs, stream);
    free_run_t r;
    r.shape = shape;
    r.n = n;
    r.in_place = rows_in_place ? static_cast<uint8_t const*>(dataset) : nullptr;
    r.source = &source;
    r.stream = stream;
    r.copy = stream;
    r.sm_count = sm_count;
    if (char const* e = run_chunks(r, q, nq, q_stride, k, d_keys.ptr, d_dists.ptr, d_counts.ptr)) return e;
    CU(cudaMemcpy2DAsync(keys, keys_stride, d_keys.ptr, k * 8, k * 8, nq, cudaMemcpyDeviceToDevice, stream));
    CU(cudaMemcpy2DAsync(distances, distances_stride, d_dists.ptr, k * 4, k * 4, nq, cudaMemcpyDeviceToDevice, stream));
    return nullptr;
}

} // namespace usearch_b200
