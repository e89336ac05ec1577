// devbuf.cuh -- DevBuf<T>, the single owner of one cudaMalloc allocation, and the process-wide count of the bytes all
// DevBufs hold (gpb200_device_bytes).  Private to the engine's translation units.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstddef>
#include <cstdint>

namespace engine __attribute__((visibility("hidden"))) {
inline std::atomic<int64_t> g_device_bytes{0};
}  // namespace engine

// Move-only.  A failed allocation leaves the buffer empty (null, size 0) and returns the runtime's error, so no stale
// pointer survives it.  It converts to T* so that the schedules read a buffer as the pointer it holds.
template <class T>
class DevBuf {
public:
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            reset();
            p_ = o.p_; n_ = o.n_;
            o.p_ = nullptr; o.n_ = 0;
        }
        return *this;
    }
    ~DevBuf() { reset(); }

    T* data() const { return p_; }
    operator T*() const { return p_; }
    size_t size() const { return n_; }
    size_t bytes() const { return n_ * sizeof(T); }

    // frees, then allocates n elements (the old and the new allocation never coexist)
    cudaError_t alloc(size_t n) {
        reset();
        void* p = nullptr;
        const cudaError_t e = cudaMalloc(&p, n * sizeof(T));
        if (e != cudaSuccess) return e;
        p_ = static_cast<T*>(p); n_ = n;
        engine::g_device_bytes += (int64_t)bytes();
        return cudaSuccess;
    }
    // grow-only: reallocates (contents lost) only when n exceeds the capacity
    cudaError_t ensure(size_t n) { return n <= n_ ? cudaSuccess : alloc(n); }
    void reset() {
        if (p_) {
            cudaFree(p_);
            engine::g_device_bytes -= (int64_t)bytes();
        }
        p_ = nullptr; n_ = 0;
    }

private:
    T* p_ = nullptr;
    size_t n_ = 0;
};
