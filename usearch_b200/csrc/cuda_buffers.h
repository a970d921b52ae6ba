/*
 *  cuda_buffers.h — owners of the CUDA resources the host side holds: device and pinned host buffers, device buffers
 *  taken and given back in stream order, a stream with its device, and events. Each frees what it holds when it is destroyed or assigned over, and can be moved but not
 *  copied, so no code keeps a list of what to free. Plain C++ against the runtime API: tests/native/test_cuda_buffers.cpp
 *  compiles it with g++ and a counting stand-in for the runtime.
 */
#pragma once
#include <cuda_runtime_api.h>

#include <cstddef>
#include <utility>

#include "cuda_check.h"

namespace usearch_b200 {

/* `capacity` elements of T in device memory (Pinned = false) or page-locked host memory (Pinned = true) */
template <typename T, bool Pinned> struct cuda_buffer_t {
    T* ptr = nullptr;
    size_t capacity = 0; /* elements */

    cuda_buffer_t() = default;
    cuda_buffer_t(cuda_buffer_t&& other) noexcept
        : ptr(std::exchange(other.ptr, nullptr)), capacity(std::exchange(other.capacity, 0)) {}
    cuda_buffer_t& operator=(cuda_buffer_t&& other) noexcept {
        if (this != &other) {
            release();
            ptr = std::exchange(other.ptr, nullptr);
            capacity = std::exchange(other.capacity, 0);
        }
        return *this;
    }
    cuda_buffer_t(cuda_buffer_t const&) = delete;
    cuda_buffer_t& operator=(cuda_buffer_t const&) = delete;
    ~cuda_buffer_t() { release(); }

    /* room for at least `n` elements; growing does not keep the contents. On failure the buffer is empty. */
    char const* reserve(size_t n) {
        if (n <= capacity) return nullptr;
        release();
        void* p = nullptr;
        if ((Pinned ? cudaHostAlloc(&p, n * sizeof(T), cudaHostAllocDefault) : cudaMalloc(&p, n * sizeof(T))) != cudaSuccess) {
            cudaGetLastError();
            return Pinned ? "Out of pinned host memory!" : "Out of GPU memory!";
        }
        ptr = static_cast<T*>(p);
        capacity = n;
        return nullptr;
    }
    void release() {
        if (ptr) {
            if (Pinned) cudaFreeHost(ptr);
            else cudaFree(ptr);
        }
        ptr = nullptr;
        capacity = 0;
    }
};

template <typename T> using device_buffer_t = cuda_buffer_t<T, false>;
template <typename T> using pinned_buffer_t = cuda_buffer_t<T, true>;

/* `capacity` elements of T in device memory taken and given back in the order of `stream` (cudaMallocAsync /
 * cudaFreeAsync), for a call that owns scratch but must not wait for its stream: the memory returns to the pool only
 * after the work enqueued on `stream` before the release. */
template <typename T> struct stream_buffer_t {
    T* ptr = nullptr;
    size_t capacity = 0; /* elements */
    cudaStream_t stream = nullptr;

    explicit stream_buffer_t(cudaStream_t s) : stream(s) {}
    stream_buffer_t(stream_buffer_t const&) = delete;
    stream_buffer_t& operator=(stream_buffer_t const&) = delete;
    ~stream_buffer_t() { release(); }

    /* room for at least `n` elements; growing does not keep the contents. On failure the buffer is empty. */
    char const* reserve(size_t n) {
        if (n <= capacity) return nullptr;
        release();
        void* p = nullptr;
        if (cudaMallocAsync(&p, n * sizeof(T), stream) != cudaSuccess) {
            cudaGetLastError();
            return "Out of GPU memory!";
        }
        ptr = static_cast<T*>(p);
        capacity = n;
        return nullptr;
    }
    void release() {
        if (ptr) cudaFreeAsync(ptr, stream);
        ptr = nullptr;
        capacity = 0;
    }
};

/* one runtime handle, destroyed with `destroy` */
template <typename H, cudaError_t (*destroy)(H)> struct cuda_handle_t {
    H handle = nullptr;

    cuda_handle_t() = default;
    cuda_handle_t(cuda_handle_t&& other) noexcept : handle(std::exchange(other.handle, nullptr)) {}
    cuda_handle_t& operator=(cuda_handle_t&& other) noexcept {
        if (this != &other) {
            release();
            handle = std::exchange(other.handle, nullptr);
        }
        return *this;
    }
    cuda_handle_t(cuda_handle_t const&) = delete;
    cuda_handle_t& operator=(cuda_handle_t const&) = delete;
    ~cuda_handle_t() { release(); }
    operator H() const { return handle; }

    void release() {
        if (handle) destroy(handle);
        handle = nullptr;
    }
};

struct cuda_event_t : cuda_handle_t<cudaEvent_t, cudaEventDestroy> {
    /* a new event on the current device in place of the one held */
    cudaError_t create() {
        release();
        return cudaEventCreate(&handle);
    }
    /* the same with cudaEventCreateWithFlags (cudaEventDisableTiming for events that only order streams) */
    cudaError_t create(unsigned int flags) {
        release();
        return cudaEventCreateWithFlags(&handle, flags);
    }
};

/* a non-blocking stream on `device` and that device's SM count, created by the first open() */
struct cuda_stream_t : cuda_handle_t<cudaStream_t, cudaStreamDestroy> {
    int device = 0;
    int sm_count = 0;

    cuda_stream_t() = default;
    explicit cuda_stream_t(int on_device) : device(on_device) {}

    /* makes `device` current on the calling thread, and creates the stream if there is none yet */
    char const* open() {
        int count = 0;
        if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
            cudaGetLastError();
            return "No CUDA device: the GPU search backend has no CPU fallback";
        }
        CU(cudaSetDevice(device));
        if (!handle) {
            CU(cudaStreamCreateWithFlags(&handle, cudaStreamNonBlocking));
            CU(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
        }
        return nullptr;
    }
};

} // namespace usearch_b200
