// cuda_util.h — the host runtime's CUDA error macro and owners of device memory, pinned host memory, streams and events.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <string>
#include <utility>

#include "../../include/b200post.h"

namespace b200post {

void set_error(const std::string &msg);

// On failure: error text "<expr>: <CUDA message>", the non-sticky error cleared, and OUT_OF_MEMORY or CUDA returned.
#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t e__ = (expr);                                                                        \
        if (e__ != cudaSuccess) {                                                                        \
            ::b200post::set_error(std::string(#expr) + ": " + cudaGetErrorString(e__));                  \
            cudaGetLastError();                                                                          \
            return e__ == cudaErrorMemoryAllocation ? B200POST_ERR_OUT_OF_MEMORY : B200POST_ERR_CUDA;    \
        }                                                                                                \
    } while (0)

// n elements of T in device memory (cudaMalloc) or pinned host memory (cudaMallocHost); freed on destruction
template <class T, bool Pinned>
class CudaBuffer {
public:
    CudaBuffer() = default;
    CudaBuffer(CudaBuffer &&o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    CudaBuffer &operator=(CudaBuffer &&o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
    ~CudaBuffer() { reset(); }
    T *get() const { return p_; }
    size_t size() const { return n_; }
    // frees the old allocation first, then allocates n elements (contents undefined)
    cudaError_t resize(size_t n) {
        reset();
        void *p = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
        if (e == cudaSuccess) { p_ = static_cast<T *>(p); n_ = n; }
        return e;
    }
    cudaError_t grow(size_t n) { return n <= n_ ? cudaSuccess : resize(n); }
    void reset() {
        if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr; n_ = 0;
    }

private:
    T *p_ = nullptr;
    size_t n_ = 0;
};
template <class T> using DeviceBuffer = CudaBuffer<T, false>;
template <class T> using PinnedBuffer = CudaBuffer<T, true>;

// a cudaStream_t or cudaEvent_t, destroyed with its owner
template <class H, cudaError_t (*Create)(H *, unsigned int), cudaError_t (*Destroy)(H)>
class CudaHandle {
public:
    CudaHandle() = default;
    CudaHandle(CudaHandle &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    CudaHandle &operator=(CudaHandle &&o) noexcept { std::swap(h_, o.h_); return *this; }
    ~CudaHandle() { reset(); }
    H get() const { return h_; }
    // destroys the old handle, then creates a new one with `flags`
    cudaError_t create(unsigned int flags) {
        reset();
        const cudaError_t e = Create(&h_, flags);
        if (e != cudaSuccess) h_ = nullptr;
        return e;
    }
    void reset() { if (h_) Destroy(h_); h_ = nullptr; }

private:
    H h_ = nullptr;
};
using Stream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;
using Event = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;

}  // namespace b200post
