// stft_generic.cu -- framed real FFT for any power-of-two fftLength in [2, 2^20].
//
// Replaces the reference's per-frame loop `__vmul(window) ; fftObj_fft` (src/stft_algorithm.c:696-715,
// 790-801), the Hermitian mirror of `_fftObj_fft` (src/dsp/fft_algorithm.c:309-317) and the
// T x n -> T x (n/2+1) compaction `__mccut` (src/reassign_algorithm.c:600-604), plus the |S|^2 /
// |S| / S^2 passes of bftObj_bft (src/bft_algorithm.c:458-504) as store modes.
//
// One CTA per frame.  The n real samples are packed as n/2 complex points, transformed by a
// shared-memory Stockham radix-4 (+ one radix-2 when log2(n/2) is odd) autosort FFT and unpacked
// with the real-FFT post-pass.  This is the general path; the MFCC configuration has its own
// fused kernel (mfcc_fused.cu).  Frames longer than 16384 points (the reference accepts radix2Exp up to 30,
// src/stft_algorithm.c:114-117) do not fit a CTA: they are gathered (window, padding) into a workspace, transformed by the
// four-step forward legs of the CWT path (af_launch_fft_rows, kernels/cwt.cu) and written out by a mode-specific pass.
#include <math.h>
#include "common.cuh"
#include "stockham.cuh"

namespace {

struct StftParams {
    const float *data;
    const float *window;
    float *outRe, *outIm;
    long long dataStride;   // floats between clips
    int n, nc, log2nc;
    int hop, timeLength, padLeft, validLength;
    int padMode;            // PaddingMode_Constant | Reflect | Wrap for samples outside [0, validLength)
    float padValue1, padValue2;   // constant mode: value left / right of the data
    int mode;
    float normValue;
    const float2 *tw;       // twiddle tables of af_twiddle_table(log2nc), or null
};


// sample s of the logical (padded) signal of one clip: x[0:valid] with, outside, a constant (left / right value),
// the mirror image without repeating the edge sample (period 2(valid-1), == __vpad_center2 of the reference,
// src/vector/flux_vectorOp.c:654-723) or the periodic extension (__vpad_center3, :736-770).  Reflect / wrap of fewer
// than two samples pad nothing (zeros), as in the reference.
__device__ __forceinline__ float padded_sample(const StftParams &p, const float *x, int s) {
    const int v = p.validLength;
    if (s >= 0 && s < v) return x[s];
    if (p.padMode == PaddingMode_Constant) return s < 0 ? p.padValue1 : p.padValue2;
    if (v < 2) return 0.0f;
    if (p.padMode == PaddingMode_Wrap) { int j = s % v; if (j < 0) j += v; return x[j]; }
    const int period = 2 * (v - 1);
    int j = s % period; if (j < 0) j += period;
    return x[j < v ? j : period - j];
}

__global__ void k_stft_generic(StftParams p) {
    extern __shared__ float2 smem[];
    float2 *a = smem, *b = smem + p.nc;
    const int frame = blockIdx.x % p.timeLength;
    const int clip = blockIdx.x / p.timeLength;
    const float *x = p.data + (long long)clip * p.dataStride;
    const int nc = p.nc, n = p.n;

    // load + window, 2 real samples -> 1 complex point; logical signal = pad(padLeft) ++ x[0:valid] ++ pad
    const int base = frame * p.hop - p.padLeft;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) {
        int s0 = base + 2 * i, s1 = s0 + 1;
        float v0 = padded_sample(p, x, s0);
        float v1 = padded_sample(p, x, s1);
        if (p.window) { v0 *= p.window[2 * i]; v1 *= p.window[2 * i + 1]; }
        a[i] = make_float2(v0, v1);
    }
    __syncthreads();

    a = af_stockham(a, b, nc, p.log2nc, p.tw);      // forward complex FFT of the nc packed points (stockham.cuh)

    // real-FFT post-pass: X[k] = E[k] + W_n^k O[k], k = 0..nc
    const int width = nc + 1;
    const long long row = (long long)clip * p.timeLength + frame;
    for (int k = threadIdx.x; k <= nc; k += blockDim.x) {
        // (written out rather than through af_real_bin: with FMA contraction on, the helper's inlined form rounds the
        // imaginary part differently here, and the STFT planes must not change)
        float2 zk = a[k == nc ? 0 : k], zp = a[k == 0 ? 0 : nc - k];
        float er = 0.5f * (zk.x + zp.x), ei = 0.5f * (zk.y - zp.y);
        float orr = 0.5f * (zk.y + zp.y), oi = -0.5f * (zk.x - zp.x);
        float2 w = p.tw ? __ldg(p.tw + nc + k) : af_twiddle(k, n);     // exp(-2 pi i k / n), second half of the table
        float xr = er + (w.x * orr - w.y * oi), xi = ei + (w.x * oi + w.y * orr);
        if (k == 0 || k == nc) xi = 0.0f;
        switch (p.mode) {
        case AF_STFT_FULL: {
            float *re = p.outRe + row * n, *im = p.outIm + row * n;
            re[k] = xr; im[k] = xi;
            if (k > 0 && k < nc) { re[n - k] = xr; im[n - k] = -xi; }
        } break;
        case AF_STFT_HALF:
            p.outRe[row * width + k] = xr; p.outIm[row * width + k] = xi;
            break;
        case AF_STFT_SQUARE:
            p.outRe[row * width + k] = xr * xr - xi * xi; p.outIm[row * width + k] = 2.0f * xr * xi;
            break;
        case AF_STFT_POWER: {
            float v = xr * xr + xi * xi;
            if (p.normValue != 1.0f) v = powf(v, p.normValue);
            p.outRe[row * width + k] = v;
        } break;
        default:
            p.outRe[row * width + k] = sqrtf(xr * xr + xi * xi);
        }
    }
}

// fftLength 2: X0 = x0 + x1, X1 = x0 - x1 (kept for API completeness: radix2Exp = 1 is legal)
__global__ void k_stft_n2(StftParams p, long long frames) {
    long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= frames) return;
    const int frame = (int)(f % p.timeLength);
    const int clip = (int)(f / p.timeLength);
    const float *x = p.data + (long long)clip * p.dataStride;
    int s0 = frame * p.hop - p.padLeft;
    float v0 = padded_sample(p, x, s0);
    float v1 = padded_sample(p, x, s0 + 1);
    if (p.window) { v0 *= p.window[0]; v1 *= p.window[1]; }
    float X[2] = {v0 + v1, v0 - v1};
    for (int k = 0; k < 2; k++) {
        float xr = X[k];
        long long o = f * 2 + k;
        switch (p.mode) {
        case AF_STFT_FULL: case AF_STFT_HALF: p.outRe[o] = xr; p.outIm[o] = 0.0f; break;
        case AF_STFT_SQUARE: p.outRe[o] = xr * xr; p.outIm[o] = 0.0f; break;
        case AF_STFT_POWER: p.outRe[o] = p.normValue != 1.0f ? powf(xr * xr, p.normValue) : xr * xr; break;
        default: p.outRe[o] = fabsf(xr);
        }
    }
}


// ---- long frames (n > 16384): gather -> four-step forward FFT (cwt.cu) -> mode-specific write-out ----
__global__ void __launch_bounds__(256) k_frames_gather(StftParams p, long long frame0, int nf, float *__restrict__ frames) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)nf * p.n) return;
    const long long f = frame0 + i / p.n;
    const int j = (int)(i % p.n);
    const int frame = (int)(f % p.timeLength), clip = (int)(f / p.timeLength);
    float v = padded_sample(p, p.data + (long long)clip * p.dataStride, frame * p.hop - p.padLeft + j);
    if (p.window) v *= p.window[j];
    frames[i] = v;
}

__global__ void __launch_bounds__(256) k_long_post(StftParams p, long long frame0, int nf, const float2 *__restrict__ spec) {
    const int nc = p.n / 2, width = nc + 1;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)nf * width) return;
    const long long f = i / width, row = frame0 + f;
    const int k = (int)(i % width);
    const float2 X = spec[f * p.n + k];
    const float xr = X.x, xi = (k == 0 || k == nc) ? 0.0f : X.y;
    const int n = p.n;
    switch (p.mode) {
    case AF_STFT_FULL: {
        float *re = p.outRe + row * n, *im = p.outIm + row * n;
        re[k] = xr; im[k] = xi;
        if (k > 0 && k < nc) { re[n - k] = xr; im[n - k] = -xi; }
    } break;
    case AF_STFT_HALF: p.outRe[row * width + k] = xr; p.outIm[row * width + k] = xi; break;
    case AF_STFT_SQUARE: p.outRe[row * width + k] = xr * xr - xi * xi; p.outIm[row * width + k] = 2.0f * xr * xi; break;
    case AF_STFT_POWER: {
        float v = xr * xr + xi * xi;
        if (p.normValue != 1.0f) v = powf(v, p.normValue);
        p.outRe[row * width + k] = v;
    } break;
    default: p.outRe[row * width + k] = sqrtf(xr * xr + xi * xi);
    }
}

}  // namespace

static int launch_stft_long(StftParams p, long long frames, cudaStream_t st);

extern "C" int af_launch_stft(const AfFrameSrc *src, int mode, float normValue, float *outRe, float *outIm, void *stream) {
    const int n = src->fftLength;
    if (n < 2 || (n & (n - 1))) return af_fail(AF_ERR_ARG, "fftLength %d is not a power of two", n);
    if (n > (1 << 20)) return af_fail(AF_ERR_UNSUPPORTED, "STFT fftLength %d > 2^20 is not supported", n);
    const long long frames = (long long)src->batch * src->timeLength;
    if (frames <= 0) return AF_OK;
    if (frames > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "too many frames in one launch");
    StftParams p;
    p.data = src->data; p.window = src->window; p.outRe = outRe; p.outIm = outIm;
    p.dataStride = src->dataLength; p.n = n; p.nc = n / 2;
    p.log2nc = 0; while ((1 << p.log2nc) < p.nc) p.log2nc++;
    p.hop = src->slideLength; p.timeLength = src->timeLength; p.padLeft = src->padLeft;
    p.validLength = src->validLength; p.mode = mode; p.normValue = normValue;
    p.padMode = src->padMode; p.padValue1 = src->padValue1; p.padValue2 = src->padValue2;
    cudaStream_t st = (cudaStream_t)stream;
    if (n > 16384) return launch_stft_long(p, frames, st);
    p.tw = n >= 4 ? af_twiddle_table(p.log2nc) : nullptr;
    if (n == 2) {
        k_stft_n2<<<(unsigned)((frames + 255) / 256), 256, 0, st>>>(p, frames);
        AF_LAUNCH_CHECK("k_stft_n2");
        return AF_OK;
    }
    const size_t smem = sizeof(float2) * 2 * (size_t)p.nc;
    const int rc = af_smem_optin(k_stft_generic, smem, "k_stft_generic");
    if (rc) return rc;
    k_stft_generic<<<(unsigned)frames, af_cta_threads(p.nc / 4, 1024), smem, st>>>(p);
    AF_LAUNCH_CHECK("k_stft_generic");
    return AF_OK;
}

// frames of more than 16384 points: chunks of frames (af_fft_rows_chunk) through a stream-ordered workspace
static int launch_stft_long(StftParams p, long long frames, cudaStream_t st) {
    const int n = p.n;
    int log2n = 0;
    while ((1 << log2n) < n) log2n++;
    const long long chunk = af_fft_rows_chunk(log2n, frames);
    const size_t specBytes = af_fft_rows_workspace_bytes(log2n, (int)chunk);
    void *ws = nullptr;
    cudaError_t e = cudaMallocAsync(&ws, specBytes + sizeof(float) * (size_t)n * chunk, st);
    if (e != cudaSuccess) return af_cuda_check(e, "cudaMallocAsync(long-frame STFT workspace)");
    float2 *spec = static_cast<float2 *>(ws);
    float *dFrames = reinterpret_cast<float *>(static_cast<char *>(ws) + specBytes);
    int rc = AF_OK;
    for (long long f0 = 0; f0 < frames && rc == AF_OK; f0 += chunk) {
        const int nf = (int)(frames - f0 < chunk ? frames - f0 : chunk);
        const long long cells = (long long)nf * n;
        k_frames_gather<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(p, f0, nf, dFrames);
        af_count_launch(1);
        if ((rc = af_launch_fft_rows(dFrames, log2n, nf, spec, st))) break;
        const long long outCells = (long long)nf * (n / 2 + 1);
        k_long_post<<<(unsigned)((outCells + 255) / 256), 256, 0, st>>>(p, f0, nf, spec);
        af_count_launch(1);
        if ((e = cudaGetLastError()) != cudaSuccess) rc = af_cuda_check(e, "long-frame STFT launch");
    }
    cudaFreeAsync(ws, st);
    return rc;
}
