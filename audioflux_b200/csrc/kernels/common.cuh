// common.cuh -- small device/host helpers shared by the kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../af_internal.h"

#define AF_LAUNCH_CHECK(what)                                                        \
    do {                                                                             \
        af_count_launch(1);                                                          \
        cudaError_t e__ = cudaGetLastError();                                        \
        if (e__ != cudaSuccess) return af_fail(AF_ERR_CUDA, "%s launch: %s", what, cudaGetErrorString(e__)); \
    } while (0)

// dynamic shared memory above the default 48 KB needs the kernel's opt-in before its launch
template <typename K>
static inline int af_smem_optin(K kernel, size_t bytes, const char *name) {
    if (bytes <= 48 * 1024) return AF_OK;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    return e == cudaSuccess ? AF_OK : af_fail(AF_ERR_CUDA, "cudaFuncSetAttribute(%s): %s", name, cudaGetErrorString(e));
}

// CTA size: `want` threads, clamped to [lo, hi]
static inline int af_cta_threads(int want, int hi, int lo = 32) { return want < lo ? lo : want > hi ? hi : want; }

__device__ __forceinline__ uint32_t af_smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier + 1-D TMA bulk copy (cp.async.bulk) ------------------------------------------
__device__ __forceinline__ void af_mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(af_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void af_fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void af_mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(af_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void af_mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(af_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool af_mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(af_smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait: a protocol bug must trap, never hang the GPU
__device__ __forceinline__ void af_mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!af_mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();
    }
}
// same wait for helper warps that idle most of the time: suspend-time hint (ns) keeps them asleep in hardware
// instead of spinning through issue slots the compute warps need; an arrival still wakes them at once
__device__ __forceinline__ void af_mbar_wait_sleepy(uint64_t *bar, uint32_t parity) {
    uint32_t spins = 0, ok = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(af_smem_u32(bar)), "r"(parity), "r"(2000u) : "memory");
        if (ok) break;
        if (++spins > (1u << 22)) __trap();
    }
}
// global -> shared bulk async copy; bytes, src and dst must be multiples of 16
__device__ __forceinline__ void af_tma_load_1d(void *dstSmem, const void *srcGmem, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(af_smem_u32(dstSmem)), "l"(srcGmem), "r"(bytes), "r"(af_smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float2 af_cmul(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
