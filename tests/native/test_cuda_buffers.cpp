// Native unit test of the CUDA resource owners (usearch_b200/csrc/cuda_buffers.h): no GPU. The runtime calls the header
// makes are answered by the stand-ins below, which count what is live, refuse to free what they never handed out, and can
// be told to fail the next allocation.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <utility>
#include <vector>

#include "cuda_buffers.h"

using namespace usearch_b200;

namespace {

std::set<void*> live_device, live_pinned, live_streams, live_events;
int allocations = 0;     // every successful cudaMalloc / cudaHostAlloc
int bad_frees = 0;       // frees of a pointer that is not live: a double free or a stray pointer
bool fail_next = false;  // the next allocation or creation fails
int device_count = 1;
size_t last_bytes = 0;   // the size of the last allocation asked for

cudaError_t take(std::set<void*>& live, void** out, size_t bytes) {
    last_bytes = bytes;
    if (fail_next) {
        fail_next = false;
        return cudaErrorMemoryAllocation;
    }
    void* p = std::malloc(bytes ? bytes : 1);
    live.insert(p);
    *out = p;
    return cudaSuccess;
}

cudaError_t give_back(std::set<void*>& live, void* p) {
    if (!live.erase(p)) {
        ++bad_frees;
        return cudaErrorInvalidValue;
    }
    std::free(p);
    return cudaSuccess;
}

size_t live_total() { return live_device.size() + live_pinned.size() + live_streams.size() + live_events.size(); }

} // namespace

extern "C" {
cudaError_t cudaMalloc(void** p, size_t bytes) {
    cudaError_t e = take(live_device, p, bytes);
    allocations += e == cudaSuccess;
    return e;
}
cudaError_t cudaFree(void* p) { return give_back(live_device, p); }
cudaError_t cudaHostAlloc(void** p, size_t bytes, unsigned int) {
    cudaError_t e = take(live_pinned, p, bytes);
    allocations += e == cudaSuccess;
    return e;
}
cudaError_t cudaFreeHost(void* p) { return give_back(live_pinned, p); }
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
char const* cudaGetErrorString(cudaError_t) { return "stand-in error"; }
cudaError_t cudaGetDeviceCount(int* count) {
    *count = device_count;
    return cudaSuccess;
}
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaDeviceGetAttribute(int* value, cudaDeviceAttr, int) {
    *value = 132;
    return cudaSuccess;
}
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned int) {
    void* p = nullptr;
    cudaError_t e = take(live_streams, &p, 1);
    if (e == cudaSuccess) *s = static_cast<cudaStream_t>(p);
    return e;
}
cudaError_t cudaStreamDestroy(cudaStream_t s) { return give_back(live_streams, s); }
cudaError_t cudaEventCreate(cudaEvent_t* ev) {
    void* p = nullptr;
    cudaError_t e = take(live_events, &p, 1);
    if (e == cudaSuccess) *ev = static_cast<cudaEvent_t>(p);
    return e;
}
cudaError_t cudaEventDestroy(cudaEvent_t ev) { return give_back(live_events, ev); }
}

#define EXPECT(cond)                                                                 \
    do {                                                                             \
        if (!(cond)) {                                                               \
            std::fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);   \
            return 1;                                                                \
        }                                                                            \
    } while (0)

// reserve, grow-only reuse, failure, moves and scope exit of one buffer type
template <typename Buffer> int check_buffer(std::set<void*> const& live, char const* out_of_memory) {
    {
        Buffer a;
        EXPECT(a.ptr == nullptr && a.capacity == 0);
        EXPECT(a.reserve(100) == nullptr && a.ptr && a.capacity == 100 && live.size() == 1);
        int const before = allocations;
        EXPECT(a.reserve(100) == nullptr && a.reserve(7) == nullptr && a.reserve(0) == nullptr);
        EXPECT(allocations == before && a.capacity == 100); // no allocation while it fits
        EXPECT(a.reserve(101) == nullptr && a.capacity == 101 && live.size() == 1 && allocations == before + 1);

        fail_next = true; // a failed growth leaves the owner empty, with the old allocation freed
        char const* e = a.reserve(1000);
        EXPECT(e && std::strcmp(e, out_of_memory) == 0);
        EXPECT(a.ptr == nullptr && a.capacity == 0 && live.empty());
        EXPECT(a.reserve(5) == nullptr && live.size() == 1);

        Buffer b(std::move(a)); // move construction: the allocation changes hands
        EXPECT(a.ptr == nullptr && a.capacity == 0 && b.ptr && b.capacity == 5 && live.size() == 1);
        Buffer c;
        EXPECT(c.reserve(9) == nullptr && live.size() == 2);
        void* const moved = b.ptr;
        c = std::move(b); // move assignment frees the target's own allocation
        EXPECT(c.ptr == moved && c.capacity == 5 && b.ptr == nullptr && b.capacity == 0 && live.size() == 1);
        Buffer& same = c;
        c = std::move(same); // self-assignment keeps it
        EXPECT(c.ptr == moved && live.size() == 1);
        c.release(); // early release, and a destructor after it frees nothing twice
        EXPECT(c.ptr == nullptr && c.capacity == 0 && live.empty());
        EXPECT(b.reserve(3) == nullptr && live.size() == 1);
    }
    EXPECT(live.empty() && bad_frees == 0);

    // a growing vector of structs that each hold a buffer (the group's per-kind query rows): every reallocation moves the
    // buffers, and none may be freed twice or lost
    struct rows_t {
        int kind = 0;
        Buffer rows;
    };
    {
        std::vector<rows_t> casts;
        for (int i = 0; i < 300; ++i) {
            casts.emplace_back();
            casts.back().kind = i;
            EXPECT(casts.back().rows.reserve((size_t)i + 1) == nullptr);
            EXPECT(live.size() == (size_t)i + 1);
        }
        for (int i = 0; i < 300; ++i) EXPECT(casts[i].kind == i && casts[i].rows.capacity == (size_t)i + 1 && live.count(casts[i].rows.ptr));
        casts.erase(casts.begin(), casts.begin() + 100);
        EXPECT(live.size() == 200);
    }
    EXPECT(live.empty() && bad_frees == 0);
    return 0;
}

int main() {
    if (check_buffer<device_buffer_t<float>>(live_device, "Out of GPU memory!")) return 1;
    if (check_buffer<pinned_buffer_t<uint64_t>>(live_pinned, "Out of pinned host memory!")) return 1;
    {
        device_buffer_t<uint64_t> a; // capacity counts elements
        EXPECT(a.reserve(3) == nullptr && last_bytes == 24);
    }

    // streams: nothing is created before open(); open() creates once and reads the SM count
    {
        cuda_stream_t s(3);
        EXPECT(!s && s.device == 3 && live_streams.empty());
        EXPECT(s.open() == nullptr && s && s.sm_count == 132 && live_streams.size() == 1);
        cudaStream_t const first = s;
        EXPECT(s.open() == nullptr && s.handle == first && live_streams.size() == 1);

        cuda_stream_t t(std::move(s));
        EXPECT(!s && t.handle == first && t.device == 3 && t.sm_count == 132 && live_streams.size() == 1);
        cuda_stream_t u(1);
        EXPECT(u.open() == nullptr && live_streams.size() == 2);
        u = std::move(t); // the target's own stream is destroyed
        EXPECT(u.handle == first && u.device == 3 && !t && live_streams.size() == 1);
        u = cuda_stream_t(5); // how a device change replaces a stream
        EXPECT(!u && u.device == 5 && live_streams.empty());

        fail_next = true;
        char const* e = u.open();
        EXPECT(e && std::strcmp(e, "Out of GPU memory!") == 0 && !u && live_streams.empty());
        device_count = 0;
        e = u.open();
        EXPECT(e && std::strcmp(e, "No CUDA device: the GPU search backend has no CPU fallback") == 0 && live_streams.empty());
        device_count = 1;

        std::vector<cuda_stream_t> many;
        for (int i = 0; i < 300; ++i) {
            many.emplace_back(i);
            EXPECT(many.back().open() == nullptr && live_streams.size() == (size_t)i + 1);
        }
        for (int i = 0; i < 300; ++i) EXPECT(many[i].device == i && live_streams.count(many[i].handle));
    }
    EXPECT(live_streams.empty() && bad_frees == 0);

    // events: create() replaces the event held
    {
        cuda_event_t a;
        EXPECT(!a && live_events.empty());
        EXPECT(a.create() == cudaSuccess && a && live_events.size() == 1);
        EXPECT(a.create() == cudaSuccess && a && live_events.size() == 1);
        cuda_event_t b(std::move(a));
        EXPECT(!a && b && live_events.size() == 1);
        cuda_event_t c;
        EXPECT(c.create() == cudaSuccess && live_events.size() == 2);
        c = std::move(b);
        EXPECT(c && !b && live_events.size() == 1);
        fail_next = true;
        EXPECT(c.create() == cudaErrorMemoryAllocation && !c && live_events.empty());

        std::vector<cuda_event_t> many;
        for (int i = 0; i < 300; ++i) {
            many.emplace_back();
            EXPECT(many.back().create() == cudaSuccess && live_events.size() == (size_t)i + 1);
        }
    }
    EXPECT(live_events.empty() && bad_frees == 0);
    EXPECT(live_total() == 0);
    std::printf("CUDA_BUFFERS_OK\n");
    return 0;
}
