// deconv.cu -- cepstral deconvolution of constant-Q spectra: cqtObj_cqhc / cqtObj_deconv (src/cqt_algorithm.c:662-781).
// Per frame (row of `num` magnitudes / powers, zero-padded to L = ceilPow2(2 num)):
//     X = FFT_L(row), m = |X|;   timbre = Re IFFT_L(m);   pitch = Re IFFT_L(X / max(m, 1e-16))
// cqhc keeps timbre[round(binPerOctave log2(j + 1))], j < hcNum; deconv the first num samples of both sequences.
// One CTA per frame, shared-memory Stockham transforms (stockham.cuh; IFFT = conj . FFT . conj / L as fftObj_ifft,
// src/dsp/fft_algorithm.c:559-623).
#include <math.h>
#include "common.cuh"
#include "stockham.cuh"

namespace {

__global__ void __launch_bounds__(128) k_cq_deconv(const float *__restrict__ in, int num, int L, int log2L, int mode, int hcNum,
                                                   int bpo, float *__restrict__ out0, float *__restrict__ out1) {
    extern __shared__ float2 sm[];
    float2 *a = sm, *b = sm + L, *X = sm + 2 * L;
    float *mag = reinterpret_cast<float *>(sm + 3 * L);
    const long long row = blockIdx.x;
    const float *src = in + row * num;
    for (int k = threadIdx.x; k < L; k += blockDim.x) a[k] = make_float2(k < num ? src[k] : 0.0f, 0.0f);
    __syncthreads();
    float2 *r = af_stockham(a, b, L, log2L);
    for (int k = threadIdx.x; k < L; k += blockDim.x) {
        const float2 v = r[k];
        X[k] = v;
        mag[k] = sqrtf(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)));
    }
    __syncthreads();
    const float inv = 1.0f / (float)L;
    for (int k = threadIdx.x; k < L; k += blockDim.x) a[k] = make_float2(mag[k], 0.0f);     // conj of a real sequence
    __syncthreads();
    r = af_stockham(a, b, L, log2L);
    if (mode == 0) {
        for (int j = threadIdx.x; j < hcNum; j += blockDim.x) {
            const int idx = (int)roundf((float)bpo * log2f((float)(j + 1)));
            out0[row * hcNum + j] = idx < L ? r[idx].x * inv : 0.0f;
        }
        return;
    }
    for (int j = threadIdx.x; j < num; j += blockDim.x) out0[row * num + j] = r[j].x * inv;
    __syncthreads();
    for (int k = threadIdx.x; k < L; k += blockDim.x) {
        float m = mag[k];
        if (m < 1e-16f) m = 1e-16f;
        a[k] = make_float2(X[k].x / m, -(X[k].y / m));
    }
    __syncthreads();
    r = af_stockham(a, b, L, log2L);
    for (int j = threadIdx.x; j < num; j += blockDim.x) out1[row * num + j] = r[j].x * inv;
}

}  // namespace

// mode 0: out0 [rows][hcNum] (cqhc); mode 1: out0 = timbre, out1 = pitch, each [rows][num] (deconv)
extern "C" int af_launch_cq_deconv(const float *in, int rows, int num, int mode, int hcNum, int bpo, float *out0, float *out1,
                                   void *stream) {
    if (rows <= 0) return AF_OK;
    int L = 1, lg = 0;
    while (L < 2 * num) { L <<= 1; lg++; }                 /* util_ceilPowerTwo(2 * num) */
    const size_t smem = sizeof(float2) * 3 * (size_t)L + sizeof(float) * (size_t)L;
    if (smem > 200 * 1024) return af_fail(AF_ERR_UNSUPPORTED, "cqhc / deconv: num=%d too large", num);
    const int rc = af_smem_optin(k_cq_deconv, smem, "k_cq_deconv");
    if (rc) return rc;
    k_cq_deconv<<<(unsigned)rows, 128, smem, (cudaStream_t)stream>>>(in, num, L, lg, mode, hcNum, bpo, out0, out1);
    AF_LAUNCH_CHECK("k_cq_deconv");
    return AF_OK;
}
