// mfcc_common.cuh -- what the fused MFCC kernels (mfcc_fused.cu = v1, mfcc_fused2.cu = v2) share: the DCT epilogue's
// 3xTF32 mma.sync, the TMA bulk stores, the rectify, the host side of a launch, and the four host functions each kernel
// file exports (declared at the end; mfcc_plan.cu wraps them into the one plan type of af_internal.h).
#pragma once
#include <math.h>
#include <stdlib.h>
#include "common.cuh"

constexpr int kMfccMaxNum = 128;    // filters (padded)
constexpr int kMfccMaxPeers = 15;   // extra destinations of the output tile (P2P stores to peer GPUs)

// ---- device -------------------------------------------------------------------------------------------------------
// ACC[0..3] += A . B, mma.sync m16n8k8 TF32 (A: 4 registers, B: 2).  A macro: as an inline function taking the
// accumulator array by reference it changes the register allocation of k_mfcc_fused2<2>.
#define AF_MMA_TF32(ACC, A0, A1, A2, A3, B0, B1)                                                              \
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" \
        : "+f"(ACC[0]), "+f"(ACC[1]), "+f"(ACC[2]), "+f"(ACC[3])                                              \
        : "r"(A0), "r"(A1), "r"(A2), "r"(A3), "r"(B0), "r"(B1))
// TF32 split by truncation: hi = top 19 bits, lo = (x - hi) (exact), again cut to 19 bits
__device__ __forceinline__ void af_tf32_split(float x, uint32_t &hi, uint32_t &lo) {
    hi = __float_as_uint(x) & 0xffffe000u;
    lo = __float_as_uint(x - __uint_as_float(hi)) & 0xffffe000u;
}

__device__ __forceinline__ void af_fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void af_bulk_store(void *dstGmem, const void *srcSmem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(dstGmem), "r"(af_smem_u32(srcSmem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void af_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void af_bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void af_bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ float af_mfcc_rectify(float v, int rectify) {
    if (rectify == CepstralRectify_CubicRoot) return powf(v, 1.0f / 3.0f);
    return __log2f(v < 1e-8f ? 1e-8f : v) * 0.30102999566398120f;      // log10 via MUFU.LG2
}

// ---- host ---------------------------------------------------------------------------------------------------------
// n-blocks of 8 coefficients the DCT epilogue computes (the kernels' template argument CT)
inline int af_mfcc_ct(int ccNum) { return ccNum <= 16 ? 2 : ccNum <= 24 ? 3 : ccNum <= 40 ? 5 : 8; }
// row pitch of the DCT B operand: pitch % 32 == 8 makes the (k0 + t, n0 + g) fragment reads hit 32 different banks
__host__ __device__ constexpr int af_mfcc_dct_pitch(int ct) { return ct <= 5 ? 40 : 72; }

// DCT table as the mma B operand: D^T[m][c] with row pitch af_mfcc_dct_pitch(ct); rows m >= num and columns
// c >= ccNum are zero.  dct: ccNum x num.
inline int af_mfcc_dct_upload(float **dDct, const float *dct, int num, int ccNum, int ct) {
    const int pitch = af_mfcc_dct_pitch(ct);
    float *dt = static_cast<float *>(calloc((size_t)kMfccMaxNum * pitch, sizeof(float)));
    if (!dt) return AF_ERR_NOMEM;
    for (int m = 0; m < num; m++)
        for (int c = 0; c < ccNum; c++) dt[(size_t)m * pitch + c] = dct[(size_t)c * num + m];
    const int rc = af_dev_upload(reinterpret_cast<void **>(dDct), dt, sizeof(float) * (size_t)kMfccMaxNum * pitch);
    free(dt);
    return rc;
}

// one bulk store per destination needs 16-byte aligned tiles: rows of a multiple of 4 floats and aligned bases
inline int af_mfcc_bulk_store_ok(int rowFloats, const float *out, int nPeer, float *const *peerOut) {
    int bulk = rowFloats % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    for (int d = 0; d < nPeer; d++) if (reinterpret_cast<uintptr_t>(peerOut[d]) & 15) bulk = 0;
    return bulk;
}

// launch kernels[i] (the instantiations CT = 2, 3, 5, 8) for ct with `smem` bytes of dynamic shared memory, one
// persistent CTA per SM (fewer for fewer tiles)
template <typename P>
inline int af_mfcc_launch_ct(void (*const kernels[4])(P), const char *name, int ct, long long tiles, int threads,
                             int smem, void *stream, const P &p) {
    int sms = af_sm_count();
    if (sms <= 0) sms = 132;
    const long long grid = tiles < (long long)sms ? tiles : (long long)sms;
    void (*k)(P) = kernels[ct == 2 ? 0 : ct == 3 ? 1 : ct == 5 ? 2 : 3];
    const int rc = af_smem_optin(k, smem, name);
    if (rc) return rc;
    k<<<(unsigned)grid, threads, smem, (cudaStream_t)stream>>>(p);
    AF_LAUNCH_CHECK(name);
    return AF_OK;
}

// the four host functions of each kernel file (mfcc_fused.cu: af_mfcc1_*, mfcc_fused2.cu: af_mfcc2_*).  build: the
// kernel's device tables for a bank [num][1025] and a DCT [ccNum][num]; launch (arguments checked by af_launch_mfcc):
// rawMel = 1 stops after the bank (out: batch x T x num), else the first ccNum cepstral coefficients (out: batch x T x
// ccNum, and the same offset of every peerOut).
int af_mfcc1_supported(int fftLength, int num, int ccNum, const AfBands *bands);
int af_mfcc1_plan_build(void **plan, int fftLength, int num, int ccNum, const float *window, const float *bank,
                        const AfBands *bands, const float *dct, int dataType);
int af_mfcc1_launch(void *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                    int rectifyType, float *out, int nPeer, float *const *peerOut, int rawMel, void *stream);
void af_mfcc1_plan_free(void *plan);
int af_mfcc2_supported(int fftLength, int num, int ccNum, const float *bank);
int af_mfcc2_plan_build(void **plan, int fftLength, int num, int ccNum, const float *window, const float *bank,
                        const float *dct, int dataType);
int af_mfcc2_launch(void *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                    int rectifyType, float *out, int nPeer, float *const *peerOut, int rawMel, void *stream);
void af_mfcc2_plan_free(void *plan);
