// lk_host.h — host-side owners of device and page-locked memory, the one CUDA error path of the host code, and the host
// entry points of the units without a launcher in lk_kernels.h.
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

// Offsets inside the packed staging blocks are 256-byte aligned.
constexpr size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

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

// Host entry points of the decode / preprocessing (lk_preprocess.cu) and leg-kinematics (lk_kinematics.cu) units, called
// behind lk_api.cu's argument checks; each states its preconditions where it is defined. Declared here, which both units
// include, rather than in lk_kernels.h, whose device headers would give their modules a watchdog note (lk_async.cuh).
int decode_pointcloud2s_device(uint32_t n_msgs, const uint8_t* const* h_data, const uint32_t* h_n, const double* h_stamps,
                               const lk_pc2_layout& L, float blind, int filter_num, double time_scale, float* h_pts_out,
                               float* h_intensity_out, uint32_t* h_out_offs, double* h_begin, double* h_end, DevBuf& scratch,
                               cudaStream_t s, std::string& err);
int preprocess_scans_device(uint32_t n_scans, const float* h_pts_in, const uint32_t* h_offs, float leaf, const double* h_begin,
                            float* h_pts_out, uint32_t* h_scan_off, uint32_t* h_scan_bptr, uint32_t* h_boff, float* h_bcurv,
                            double* h_btimes, DevBuf& scratch, cudaStream_t s, std::string& err);
size_t leg_kinematics_scratch_bytes(uint32_t n);
int leg_kinematics_device(const lk_leg_cfg& cfg, const lk_leg_state* h_in, uint32_t n, int redundancy,
                          lk_leg_track* track, lk_kinimu_meas* h_out, uint32_t* n_out, void* scratch, cudaStream_t s,
                          std::string& err);

}  // namespace lk
