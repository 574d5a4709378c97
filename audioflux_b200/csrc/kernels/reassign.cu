// reassign.cu -- time-frequency reassignment: coordinates, indices and the scatter of the STFT cells.
//
// Replaces steps 3-5 of reassignObj_reassign (src/reassign_algorithm.c:200-217): `_reassignObj_reassignTimeFre`
// (:612-703, complex divides S_dh / S_h and S_th / S_h -> reassigned frequency / time), `_reassignObj_filterTimeFre`
// (:709-822, threshold on |S_h|^2, clip to the axes) and `_reassignObj_rearrage` (:224-414, roundf to cell indices,
// order-1 further look-ups along the row, scatter-add of the sign-alternated S_h).  The three STFTs (windows h, dh,
// t.h) are kernels/stft_generic.cu.
//   * k_reassign_index: one thread per (clip, frame, bin), float32 operation by operation in the reference's order
//     (explicit _rn intrinsics: no FMA contraction, the roundf outcome is an integer);
//   * k_reassign_order: the row-local index iteration of order > 1, one CTA per (clip, frame); the row's scratch lives in
//     global memory (the accumulator planes, not yet in use), so any row length works;
//   * scatter: the reference adds the cells in (frame, bin) order into float planes; on the GPU the additions are made
//     order-independent instead: every cell is scaled by a per-clip power of two (max |S_h| -> [2^35, 2^36)) and added
//     as a 64-bit integer (atomicAdd on unsigned long long is associative), so the result is bit-stable for any
//     schedule and carries 36 bits below the clip's maximum -- finer than the reference's own float32 running sum.
#include <math.h>
#include "common.cuh"

namespace {

__device__ __forceinline__ int c_float_to_int(float v) {          // `int i = v;` on the reference's x86 build
    if (!(fabsf(v) < 2147483648.0f)) return (int)0x80000000;       // NaN, +-inf, out of range -> INT_MIN (cvttss2si)
    return (int)v;
}

struct ReParams {
    int T, W, batch, reType, order, resultType;
    float thresh2;                 // thresh * thresh (float product, as the reference writes it)
    float freStep, fmax;           // __vlinspace(0, samplate / 2, W): fre[j] = 0 + j * step
    float hop, sr;                 // timeArr[i] = (i * hop) / sr
    float tmax;
    float cFre, cTime;             // (float)(-0.5 samplate / pi), (float)(1 / samplate)
    float halfN;                   // (float)(fftLength / 2)
};

__device__ __forceinline__ float fre_of(const ReParams &p, int j) { return __fadd_rn(0.0f, __fmul_rn((float)j, p.freStep)); }
__device__ __forceinline__ float time_of(const ReParams &p, int i) { return __fdiv_rn(__fmul_rn((float)i, p.hop), p.sr); }

__global__ void __launch_bounds__(256) k_reassign_index(const float *__restrict__ r1, const float *__restrict__ i1,
                                                        const float *__restrict__ r2, const float *__restrict__ i2,
                                                        const float *__restrict__ r3, const float *__restrict__ i3,
                                                        ReParams p, int *__restrict__ tIdx, int *__restrict__ fIdx) {
    const long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)p.batch * p.T * p.W;
    if (cell >= total) return;
    const int j = (int)(cell % p.W);
    const int i = (int)((cell / p.W) % p.T);
    const float c = r1[cell], d = i1[cell];
    const float den = __fadd_rn(__fmul_rn(c, c), __fmul_rn(d, d));           // |S_h|^2 (also __complexDiv's divisor)
    const bool keep = den >= p.thresh2;
    const float fj = fre_of(p, j), ti = time_of(p, i);
    float vf = fj, vt = ti;
    if (p.reType == 0 || p.reType == 1) {                                      // Reassign_All / Reassign_Fre
        const float a = r2[cell], b = i2[cell];
        const float im = __fdiv_rn(__fsub_rn(__fmul_rn(b, c), __fmul_rn(a, d)), den);
        float v = __fadd_rn(__fmul_rn(im, p.cFre), fj);
        if (!keep) v = fj;
        if (v < 0.0f) v = 0.0f;
        if (v > p.fmax) v = p.fmax;
        vf = v;
    }
    if (p.reType == 0 || p.reType == 2) {                                      // Reassign_All / Reassign_Time
        const float a = r3[cell], b = i3[cell];
        const float re = __fdiv_rn(__fadd_rn(__fmul_rn(a, c), __fmul_rn(b, d)), den);
        float v = __fadd_rn(__fmul_rn(re, p.cTime), ti);
        if (!keep) v = ti;
        if (v < 0.0f) v = 0.0f;
        if (v > p.tmax) v = p.tmax;
        vt = v;
    }
    // roundf((t - tmin) (T - 1) / (tmax - tmin)), roundf((f - fmin) (N / 2) / (fmax - fmin)); tmin = fmin = 0
    int it = 0;
    if (p.T > 1) it = c_float_to_int(roundf(__fdiv_rn(__fmul_rn(__fsub_rn(vt, 0.0f), (float)(p.T - 1)), __fsub_rn(p.tmax, 0.0f))));
    tIdx[cell] = it;
    fIdx[cell] = c_float_to_int(roundf(__fdiv_rn(__fmul_rn(__fsub_rn(vf, 0.0f), p.halfN), __fsub_rn(p.fmax, 0.0f))));
}

// order > 1: tmp[j] = fIdx[fIdx[j]] where the index stays in the row; tmp keeps its previous value elsewhere (it starts
// at zero and is NOT cleared between iterations, reassign_algorithm.c:325-343)
__global__ void __launch_bounds__(256) k_reassign_order(int *fIdx, int *scratch, int W, int order) {
    int *cur = fIdx + (size_t)blockIdx.x * W, *tmp = scratch + (size_t)blockIdx.x * W;
    for (int j = threadIdx.x; j < W; j += blockDim.x) tmp[j] = 0;
    __syncthreads();
    for (int k = 0; k < order - 1; k++) {
        for (int j = threadIdx.x; j < W; j += blockDim.x) {
            const int v = cur[j];
            if (v >= 0 && v < W) tmp[j] = cur[v];
        }
        __syncthreads();
        for (int j = threadIdx.x; j < W; j += blockDim.x) cur[j] = tmp[j];
        __syncthreads();
    }
}

// per-clip maximum of |re|, |im| of S_h as float bits (non-negative floats order like unsigned integers)
__global__ void __launch_bounds__(256) k_reassign_absmax(const float *__restrict__ r1, const float *__restrict__ i1, long long perClip,
                                                         unsigned *__restrict__ maxBits) {
    const int clip = blockIdx.y;
    const float *a = r1 + (size_t)clip * perClip, *b = i1 + (size_t)clip * perClip;
    unsigned m = 0;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < perClip; k += (long long)gridDim.x * blockDim.x) {
        const float x = fabsf(a[k]), y = fabsf(b[k]);
        if (x < INFINITY) m = max(m, __float_as_uint(x));
        if (y < INFINITY) m = max(m, __float_as_uint(y));
    }
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&maxBits[clip], m);
}

// power-of-two scale that brings a clip's largest component into [2^35, 2^36) (amplitudes: < 2^36.5)
__device__ __forceinline__ float clip_scale(unsigned maxBits) {
    int e = (int)(maxBits >> 23) - 127;                // max in [2^e, 2^(e+1))
    int s = 35 - e;
    s = s > 126 ? 126 : (s < -126 ? -126 : s);
    return __uint_as_float((unsigned)(s + 127) << 23);
}

__global__ void __launch_bounds__(256) k_reassign_scatter(const float *__restrict__ r1, const float *__restrict__ i1,
                                                          const int *__restrict__ tIdx, const int *__restrict__ fIdx, ReParams p,
                                                          const unsigned *__restrict__ maxBits,
                                                          unsigned long long *__restrict__ accRe, unsigned long long *__restrict__ accIm) {
    const long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long perClip = (long long)p.T * p.W;
    if (cell >= (long long)p.batch * perClip) return;
    const int clip = (int)(cell / perClip);
    const int j = (int)(cell % p.W);
    const int it = tIdx[cell], jf = fIdx[cell];
    if (it < 0 || it >= p.T || jf < 0 || jf >= p.W) return;
    float v1 = r1[cell], v2 = i1[cell];
    if (j & 1) { v1 = -v1; v2 = -v2; }
    const float s = clip_scale(maxBits[clip]);
    const long long dst = (long long)clip * perClip + (long long)it * p.W + jf;
    if (p.resultType == 0) {
        const long long a = __float2ll_rn(v1 * s), b = __float2ll_rn(v2 * s);
        if (a) atomicAdd(&accRe[dst], (unsigned long long)a);
        if (b) atomicAdd(&accIm[dst], (unsigned long long)b);
    } else {
        const float amp = sqrtf(__fadd_rn(__fmul_rn(v1, v1), __fmul_rn(v2, v2)));
        const long long a = __float2ll_rn(amp * s);
        if (a) atomicAdd(&accRe[dst], (unsigned long long)a);
    }
}

// out += acc / scale (the reference ADDS into the caller's planes)
__global__ void __launch_bounds__(256) k_reassign_finish(const unsigned long long *__restrict__ accRe, const unsigned long long *__restrict__ accIm,
                                                         const unsigned *__restrict__ maxBits, long long perClip, int batch, int resultType,
                                                         float *__restrict__ outRe, float *__restrict__ outIm) {
    const long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= (long long)batch * perClip) return;
    const double inv = 1.0 / (double)clip_scale(maxBits[cell / perClip]);
    outRe[cell] = __fadd_rn(outRe[cell], (float)((double)(long long)accRe[cell] * inv));
    if (resultType == 0) outIm[cell] = __fadd_rn(outIm[cell], (float)((double)(long long)accIm[cell] * inv));
}

}  // namespace

extern "C" int af_launch_reassign(const AfReassignArgs *a, const float *r1, const float *i1, const float *r2, const float *i2,
                                  const float *r3, const float *i3, int *tIdx, int *fIdx, unsigned *maxBits,
                                  unsigned long long *accRe, unsigned long long *accIm, float *outRe, float *outIm, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const int W = a->fftLength / 2 + 1;
    const long long perClip = (long long)a->timeLength * W, total = perClip * a->batch;
    if (total <= 0) return AF_OK;
    ReParams p;
    p.T = a->timeLength; p.W = W; p.batch = a->batch; p.reType = a->reType; p.order = a->order; p.resultType = a->resultType;
    p.thresh2 = a->thresh * a->thresh;
    const float start = 0.0f, stop = (float)(a->samplate / 2.0);
    p.freStep = (stop - start) / (float)(W - 1 > 0 ? W - 1 : 1);
    p.fmax = start + (float)(W - 1) * p.freStep;
    p.hop = (float)a->slideLength; p.sr = (float)a->samplate;
    p.tmax = ((float)(a->timeLength - 1) * p.hop) / p.sr;
    p.cFre = (float)(-0.5 * a->samplate / M_PI);
    p.cTime = (float)(1.0 / a->samplate);
    p.halfN = (float)(a->fftLength / 2);
    const unsigned blocks = (unsigned)((total + 255) / 256);
    k_reassign_index<<<blocks, 256, 0, st>>>(r1, i1, r2, i2, r3, i3, p, tIdx, fIdx);
    AF_LAUNCH_CHECK("k_reassign_index");
    if (a->order > 1) {
        k_reassign_order<<<(unsigned)((long long)a->batch * a->timeLength), 256, 0, st>>>(fIdx, (int *)accRe, W, a->order);
        AF_LAUNCH_CHECK("k_reassign_order");
    }
    cudaError_t e = cudaMemsetAsync(maxBits, 0, sizeof(unsigned) * (size_t)a->batch, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(accRe, 0, sizeof(unsigned long long) * (size_t)total, st);
    if (e == cudaSuccess && a->resultType == 0) e = cudaMemsetAsync(accIm, 0, sizeof(unsigned long long) * (size_t)total, st);
    if (e != cudaSuccess) return af_fail(AF_ERR_CUDA, "reassign memset: %s", cudaGetErrorString(e));
    const unsigned gx = (unsigned)((perClip + 256 * 8 - 1) / (256 * 8));
    k_reassign_absmax<<<dim3(gx > 0 ? gx : 1, (unsigned)a->batch), 256, 0, st>>>(r1, i1, perClip, maxBits);
    AF_LAUNCH_CHECK("k_reassign_absmax");
    k_reassign_scatter<<<blocks, 256, 0, st>>>(r1, i1, tIdx, fIdx, p, maxBits, accRe, accIm);
    AF_LAUNCH_CHECK("k_reassign_scatter");
    k_reassign_finish<<<blocks, 256, 0, st>>>(accRe, accIm, maxBits, perClip, a->batch, a->resultType, outRe, outIm);
    AF_LAUNCH_CHECK("k_reassign_finish");
    return AF_OK;
}
