// lk_async.cuh — mbarrier and 1-D TMA bulk-copy primitives (PTX) for sm_90a.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lk {

// Watchdog notes of this translation unit's kernels: a wait that never completes is bounded, leaves a code here and
// lets the kernel finish (with garbage), so that a broken invariant shows up as an error instead of a hung device.
//   [0] first code (1 mbarrier wait, 2 root-slot publication, 3 octree descent, 4 root-table probe) [1] block [2] thread [3] detail
static __device__ uint32_t lk_stall_note[8];
__device__ __forceinline__ void stall_note(uint32_t code, uint32_t detail) {
    if (atomicCAS(&lk_stall_note[0], 0u, code) == 0u) {
        lk_stall_note[1] = blockIdx.x; lk_stall_note[2] = threadIdx.x; lk_stall_note[3] = detail;
        __threadfence();
    }
}

// the global nanosecond timer, for the kernels' optional trace stamps
__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// ---- mbarrier / bulk-copy primitives (PTX) ----------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    for (uint32_t spins = 0;; ++spins) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
        if (ok) return;
        if (spins > (1u << 24)) {  // seconds: a bulk copy that never arrives (see lk_stall_note)
            stall_note(1u, parity);
            return;
        }
    }
}
// 1-D TMA bulk copy global -> shared::cta; size multiple of 16, both addresses 16-B aligned.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the same between this thread's view of global memory and the bulk copies it issues next
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

__device__ __forceinline__ void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async();
}

}  // namespace lk

namespace lk {
// Ampere-style asynchronous 16-byte copy global -> shared (LDGSTS in SASS); completes per thread.
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
}  // namespace lk

namespace lk {
// plain arrival (release at CTA scope)
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrival that fires when all cp.async issued so far by this thread have landed; does not add to the
// pending count, so the barrier's init count must include it
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
template <int ID, int NTHREADS>
__device__ __forceinline__ void named_barrier_sync() {
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(NTHREADS) : "memory");
}
template <int REGS>
__device__ __forceinline__ void warpgroup_reg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS));
}
template <int REGS>
__device__ __forceinline__ void warpgroup_reg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS));
}
}  // namespace lk

namespace lk {
// the same primitives on 32-bit shared-window addresses (no generic->shared conversion per call)
__device__ __forceinline__ void cp_async16_s(uint32_t dst_smem, const void* src_gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void mbar_arrive_s(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive_noinc_s(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait_s(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
}  // namespace lk
