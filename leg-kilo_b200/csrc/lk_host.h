// lk_host.h — host-side owners of device and page-locked memory, and the one CUDA error path of the host code.
// Every cudaMalloc / cudaFree of the library is here: a buffer is freed by its destructor, so no error return leaks.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <utility>

#include "../../include/legkilo_b200.h"

// Evaluate a CUDA runtime call; on failure clear the sticky error, describe the call in `err` and return
// LK_ERR_OUT_OF_MEMORY (allocation failed) or LK_ERR_CUDA from the enclosing function.
#define LK_CUDA(err, expr)                                                                        \
    do {                                                                                          \
        cudaError_t e__ = (expr);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            cudaGetLastError();                                                                   \
            (err) = std::string(#expr) + ": " + cudaGetErrorString(e__);                          \
            return e__ == cudaErrorMemoryAllocation ? LK_ERR_OUT_OF_MEMORY : LK_ERR_CUDA;         \
        }                                                                                         \
    } while (0)

namespace lk {

// One device allocation, freed with its owner. Move-only.
class DevBuf {
   public:
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }  // o frees the old one
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { reset(); }

    // Exactly `bytes`, the old contents freed first. Zero bytes still gives a pointer: CUB reads a null
    // temporary-storage pointer as a size query.
    cudaError_t alloc(size_t bytes) {
        reset();
        const size_t want = bytes ? bytes : 16;
        const cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { p = nullptr; return e; }
        cap = want;
        return cudaSuccess;
    }
    // At least `bytes`, with 1/8 slack so that a slowly growing size does not reallocate every call. The contents are
    // not kept across a growth.
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        reset();
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            e = cudaMalloc(&p, bytes);
            if (e != cudaSuccess) { p = nullptr; return e; }
            want = bytes;
        }
        cap = want;
        return cudaSuccess;
    }
    void reset() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <class T>
    T* as() const { return reinterpret_cast<T*>(p); }

    void* p = nullptr;
    size_t cap = 0;  // bytes
};

// Page-locked host memory (staging of the packed small inputs / outputs), freed with its owner. Move-only.
class PinnedBuf {
   public:
    PinnedBuf() = default;
    PinnedBuf(PinnedBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    PinnedBuf& operator=(PinnedBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }  // o frees the old one
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { reset(); }
    // At least `bytes` with 1/4 slack; the contents are not kept across a growth.
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        reset();
        const cudaError_t e = cudaHostAlloc(&p, bytes + bytes / 4 + 4096, cudaHostAllocDefault);
        if (e != cudaSuccess) { p = nullptr; return e; }
        cap = bytes + bytes / 4 + 4096;
        return cudaSuccess;
    }
    void reset() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
    }

    void* p = nullptr;
    size_t cap = 0;
};

}  // namespace lk
