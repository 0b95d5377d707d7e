/*
 * cuda_buffers.hpp -- how a batch owns host and device memory (host code only).
 *
 * The POA batch (b200poa.cu) and the aligner batch (b200aln.cu) allocate through these types and nothing else: a member's
 * destructor frees what it holds, so a batch is released by deleting it.  The owner must synchronise every stream that
 * may still use a buffer before the buffer is destroyed.  All types are move-only.  DeviceGuard is how the batches and
 * the racon shim (host/) switch devices.
 */
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <utility>

namespace b200buf {

/* Grow-only device buffer: need() re-allocates, contents lost, when the bytes asked for exceed the capacity. */
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    DevBuf& operator=(DevBuf&& o) noexcept {
        std::swap(p, o.p);
        std::swap(cap, o.cap);
        return *this;
    }
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    cudaError_t need(size_t bytes, bool slack = true) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        const size_t want = bytes + (slack ? bytes / 4 : 0) + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
};

/* Grow-only page-locked host buffer, contents preserved: reserve() keeps the first `used` bytes. */
struct PinnedBuf {
    uint8_t* p = nullptr;
    size_t cap = 0, used = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    PinnedBuf(PinnedBuf&& o) noexcept
        : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)), used(std::exchange(o.used, 0)) {}
    PinnedBuf& operator=(PinnedBuf&& o) noexcept {
        std::swap(p, o.p);
        std::swap(cap, o.cap);
        std::swap(used, o.used);
        return *this;
    }
    ~PinnedBuf() {
        if (p) cudaFreeHost(p);
    }
    bool reserve(size_t bytes) {
        if (bytes <= cap) return true;
        size_t want = std::max<size_t>(bytes, cap * 2);
        want = std::max<size_t>(want, (size_t)1 << 20);
        uint8_t* q = nullptr;
        if (cudaHostAlloc(reinterpret_cast<void**>(&q), want, cudaHostAllocDefault) != cudaSuccess) return false;
        if (used) std::memcpy(q, p, used);
        if (p) cudaFreeHost(p);
        p = q;
        cap = want;
        return true;
    }
};

/* A table of `count` elements in page-locked host memory and the same count on the device, allocated once; upload and
 * download copy the first n elements asynchronously on the given stream. */
template <class T>
class Mirror {
  public:
    Mirror() = default;
    Mirror(const Mirror&) = delete;
    Mirror& operator=(const Mirror&) = delete;
    Mirror(Mirror&& o) noexcept : h_(std::exchange(o.h_, nullptr)), d_(std::exchange(o.d_, nullptr)) {}
    Mirror& operator=(Mirror&& o) noexcept {
        std::swap(h_, o.h_);
        std::swap(d_, o.d_);
        return *this;
    }
    ~Mirror() {
        if (h_) cudaFreeHost(h_);
        if (d_) cudaFree(d_);
    }
    cudaError_t alloc(size_t count) {
        cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&d_), count * sizeof(T));
        if (e != cudaSuccess) {
            d_ = nullptr;
            return e;
        }
        e = cudaHostAlloc(reinterpret_cast<void**>(&h_), count * sizeof(T), cudaHostAllocDefault);
        if (e != cudaSuccess) h_ = nullptr;
        return e;
    }
    T* h() const { return h_; }
    T* d() const { return d_; }
    cudaError_t upload(size_t n, cudaStream_t s) const {
        return cudaMemcpyAsync(d_, h_, n * sizeof(T), cudaMemcpyHostToDevice, s);
    }
    cudaError_t download(size_t n, cudaStream_t s) const {
        return cudaMemcpyAsync(h_, d_, n * sizeof(T), cudaMemcpyDeviceToHost, s);
    }

  private:
    T* h_ = nullptr;
    T* d_ = nullptr;
};

/* Makes `dev` the current device for a scope and restores the previous one (GenomeWorks' scoped_device_switch). */
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

} // namespace b200buf
