// wavelet.cu -- the discrete wavelet transforms (sm_90a): DWTObj, WPTObj and SWTObj (src/dwt_algorithm.c,
// src/wpt_algorithm.c, src/swt_algorithm.c), which pad, convolve and decimate level by level on one core.
//
// The reference materialises the periodic padding (__periodPadding) and takes a valid (DWT / WPT) or full (SWT)
// convolution of the padded signal.  Both branches of that padding put x[(m - half) mod L] at padded index m (half =
// filter length / 2), so every kernel here reads the unpadded signal with modulo indexing instead:
//   DWT / WPT: a[i] = conv_valid(pad(x), loD)[2i+1] = sum_j loD[j] x[(2i + dec - half - j) mod L];
//   SWT level with dilation s: keep = conv_full(pad(x), dilated loD)[up + t] = sum_j loD[j] x[(t + up/2 - j s) mod n],
//   up = dec * s.
// tests/test_wavelet_cpu.py checks the identity against the literal padding for every (length, filter length) pair
// the three objects produce.
//
// k_wavelet_level: one thread per (clip, node, output pair), all nodes of a level in one launch; the filters (at most
// 80 taps) in shared memory.  k_wavelet_expand: one thread per four output columns of mDataArr, which looks up the
// coefficients that feed them (coalesced 16-byte stores where mDataArr is 16-byte aligned, else 4-byte stores; the
// coefficient reads hit L1/L2).  k_swt_level: one thread
// per output sample of one level, both filters.
#include <stdint.h>
#include <cuda_runtime.h>
#include "../af_internal.h"
#include "common.cuh"

#define AF_WAVELET_MAX_DEC 80

__global__ void __launch_bounds__(256) k_wavelet_level(AfWaveletLevel p) {
    __shared__ float sLo[AF_WAVELET_MAX_DEC], sHi[AF_WAVELET_MAX_DEC];
    for (int j = threadIdx.x; j < p.dec; j += blockDim.x) { sLo[j] = p.loD[j]; sHi[j] = p.hiD[j]; }
    __syncthreads();
    const int half = p.L >> 1;
    const long long perClip = (long long)p.nodes * half;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= perClip * p.batch) return;
    const int b = (int)(idx / perClip);
    const int r = (int)(idx - (long long)b * perClip);
    const int k = r / half, i = r - k * half;
    const float *x = p.in + b * p.inStride + (long long)k * p.L;
    const int mask = p.L - 1;
    const int m0 = 2 * i + p.dec - p.dec / 2;
    float a = 0.f, d = 0.f;
    for (int j = 0; j < p.dec; j++) {
        const float v = __ldg(x + ((m0 - j) & mask));
        a = fmaf(sLo[j], v, a);
        d = fmaf(sHi[j], v, d);
    }
    const int g = p.nodeBase + k;
    const int swap = p.wpt && g && !(g & 1);
    p.lo[b * p.loStride + (long long)k * p.L + (swap ? half : 0) + i] = a;
    p.hi[b * p.hiStride + (long long)k * p.L + (swap ? 0 : half) + i] = d;
}

// four consecutive columns of one row per thread: one 16-byte store when `out` is 16-byte aligned (vec), else four
// 4-byte stores (a caller's device pointer need only be float-aligned)
__global__ void __launch_bounds__(256) k_wavelet_expand(const float *__restrict__ coef, int log2n, int rows, int wpt,
                                                        int vec, long long total4, float *__restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total4) return;
    const unsigned plane = (unsigned)(idx >> (log2n - 2));
    const int j = (int)(idx & ((1 << (log2n - 2)) - 1)) * 4;
    const unsigned r = plane % (unsigned)rows;
    const long long b = plane / (unsigned)rows;
    int base, shift;
    if (wpt) {
        shift = 31 - __clz(rows);
        base = r << (log2n - shift);
    } else {
        base = 2 << r;
        shift = log2n - r - 1;
    }
    const float *c = coef + (b << log2n) + base;
    const float4 v = make_float4(__ldg(c + (j >> shift)), __ldg(c + ((j + 1) >> shift)), __ldg(c + ((j + 2) >> shift)),
                                 __ldg(c + ((j + 3) >> shift)));
    float *o = out + idx * 4;
    if (vec) {
        *reinterpret_cast<float4 *>(o) = v;
    } else {
        o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
    }
}

__global__ void __launch_bounds__(256) k_swt_level(const float *__restrict__ in, long long inStride,
                                                   const float *__restrict__ loD, const float *__restrict__ hiD, int dec,
                                                   int n, int s, int batch, float *__restrict__ lo,
                                                   float *__restrict__ hi, long long outStride) {
    __shared__ float sLo[AF_WAVELET_MAX_DEC], sHi[AF_WAVELET_MAX_DEC];
    for (int j = threadIdx.x; j < dec; j += blockDim.x) { sLo[j] = loD[j]; sHi[j] = hiD[j]; }
    __syncthreads();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * batch) return;
    const int b = (int)(idx / n);
    const int t = (int)(idx - (long long)b * n);
    const float *x = in + b * inStride;
    const long long up = (long long)dec * s;
    const int step = (int)(s % n);
    int m = (int)((t + up / 2) % n);
    float a = 0.f, d = 0.f;
    for (int j = 0; j < dec; j++) {
        const float v = __ldg(x + m);
        a = fmaf(sLo[j], v, a);
        d = fmaf(sHi[j], v, d);
        m -= step;
        if (m < 0) m += n;
    }
    lo[b * outStride + t] = a;
    hi[b * outStride + t] = d;
}

static unsigned blocks_for(long long work) { return (unsigned)((work + 255) / 256); }

extern "C" int af_launch_wavelet_level(const AfWaveletLevel *a, void *stream) {
    const long long work = (long long)a->batch * a->nodes * (a->L / 2);
    if (work <= 0) return AF_OK;
    if (a->dec < 1 || a->dec > AF_WAVELET_MAX_DEC) return af_fail(AF_ERR_ARG, "af_launch_wavelet_level: dec=%d", a->dec);
    k_wavelet_level<<<blocks_for(work), 256, 0, (cudaStream_t)stream>>>(*a);
    AF_LAUNCH_CHECK("k_wavelet_level");
    return AF_OK;
}

extern "C" int af_launch_wavelet_expand(const float *coef, int log2n, int rows, int wpt, int batch, float *out,
                                        void *stream) {
    const long long planes = (long long)batch * rows;
    if (planes <= 0) return AF_OK;
    if (log2n < 2 || planes > 0xffffffffLL)
        return af_fail(AF_ERR_ARG, "af_launch_wavelet_expand: log2n=%d, %lld rows", log2n, planes);
    const long long total4 = planes << (log2n - 2);
    const int vec = ((uintptr_t)out & 15) == 0;
    k_wavelet_expand<<<blocks_for(total4), 256, 0, (cudaStream_t)stream>>>(coef, log2n, rows, wpt, vec, total4, out);
    AF_LAUNCH_CHECK("k_wavelet_expand");
    return AF_OK;
}

extern "C" int af_launch_swt_level(const float *in, long long inStride, const float *loD, const float *hiD, int dec,
                                   int n, int s, int batch, float *lo, float *hi, long long outStride, void *stream) {
    const long long work = (long long)n * batch;
    if (work <= 0) return AF_OK;
    if (dec < 1 || dec > AF_WAVELET_MAX_DEC) return af_fail(AF_ERR_ARG, "af_launch_swt_level: dec=%d", dec);
    k_swt_level<<<blocks_for(work), 256, 0, (cudaStream_t)stream>>>(in, inStride, loD, hiD, dec, n, s, batch, lo, hi,
                                                                     outStride);
    AF_LAUNCH_CHECK("k_swt_level");
    return AF_OK;
}
