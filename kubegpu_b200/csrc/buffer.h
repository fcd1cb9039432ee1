// buffer.h -- the owning buffer type of the libkgpu handle (host code).
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <utility>

namespace kgpu {

// T[capacity()] in device memory (Pinned = false) or pinned host memory (Pinned = true), freed by its destructor
// on the device it was allocated on.  Move-only; reads as a T * in kernel arguments and copies.
template <typename T, bool Pinned = false>
class Buffer {
  public:
    Buffer() = default;
    Buffer(const Buffer &) = delete;
    Buffer &operator=(const Buffer &) = delete;
    Buffer(Buffer &&o) noexcept : p_(std::exchange(o.p_, nullptr)), cap_(std::exchange(o.cap_, 0)), dev_(o.dev_) {}
    Buffer &operator=(Buffer &&o) noexcept {
        if (this != &o) {
            reset();
            p_ = std::exchange(o.p_, nullptr);
            cap_ = std::exchange(o.cap_, 0);
            dev_ = o.dev_;
        }
        return *this;
    }
    ~Buffer() { reset(); }

    // Room for at least n elements on the current device.  Grows only: when it must, it discards the contents and
    // allocates max(n, grow_to) elements, so that callers can leave headroom for a slowly growing size.  A failed
    // allocation leaves the buffer empty (null, capacity 0).
    cudaError_t reserve(int64_t n, int64_t grow_to = 0) {
        if (n <= cap_) return cudaSuccess;
        reset();
        const int64_t cap = std::max(n, grow_to);
        void *p = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&p, (size_t)cap * sizeof(T)) : cudaMalloc(&p, (size_t)cap * sizeof(T));
        if (e != cudaSuccess) return e;
        cudaGetDevice(&dev_);
        p_ = static_cast<T *>(p);
        cap_ = cap;
        return cudaSuccess;
    }

    // Frees the buffer on the device it was allocated on; the current device stays as it was.
    void reset() {
        if (!p_) return;
        int cur = dev_;
        cudaGetDevice(&cur);
        if (cur != dev_) cudaSetDevice(dev_);
        if (Pinned) cudaFreeHost(p_); else cudaFree(p_);
        if (cur != dev_) cudaSetDevice(cur);
        p_ = nullptr;
        cap_ = 0;
    }

    T *get() const { return p_; }
    operator T *() const { return p_; }
    int64_t capacity() const { return cap_; }

  private:
    T *p_ = nullptr;
    int64_t cap_ = 0;
    int dev_ = 0;
};

template <typename T>
using DeviceBuffer = Buffer<T, false>;
template <typename T>
using PinnedBuffer = Buffer<T, true>;

}  // namespace kgpu
