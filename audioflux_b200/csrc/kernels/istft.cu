// istft.cu -- inverse STFT: per-frame complex inverse FFT, synthesis window, overlap-add, window-sum normalisation.
//
// Replaces stftObj_istft (src/stft_algorithm.c:304-409): for every frame  y_t = Re(IFFT_n(X_t))  (fftObj_ifft:
// conj -> forward FFT -> conj, divided by n, src/dsp/fft_algorithm.c:559-623), then
//     data[j] <- ( data[j] + sum_t y_t[j - t hop] w^e[j - t hop] ) / max-guarded( sum_t w^(e+1)[j - t hop] )
// with e = 1 ('weight', methodType 0) or e = 0 ('overlap-add'); a window sum below 1e-6 is replaced by 1.
// Two kernels: frames (one CTA per frame, shared-memory Stockham FFT) and a gather over the <= n/hop frames that
// cover an output sample, summed in ascending frame order like the reference's loop (bit-stable, no atomics).
// Frames of 2^15 .. 2^20 points (the reference accepts radix2Exp up to 30, src/stft_algorithm.c:114-117) do not fit a
// CTA: Re(IFFT_n(X)) is taken from ONE real-input forward transform of the four-step legs (af_launch_fft_rows,
// kernels/cwt.cu) by the Hartley identity -- with H = the Hermitian part of X (the only part Re(IFFT) sees) and the real sequence
// c[k] = Re H[k] + Im H[k],  C = FFT_n(c):   Re(IFFT_n(X))[j] = (Re C[j] + Im C[j]) / n.
#include <math.h>
#include "common.cuh"
#include "stockham.cuh"

namespace {

// spec planes [rows][width] with width = n (full spectrum) or n/2+1 (half: the rest is the Hermitian mirror)
__global__ void k_istft_frames(const float *__restrict__ re, const float *__restrict__ im, int width, int n, int log2n,
                               const float *__restrict__ window, int weightMode, float *__restrict__ frames,
                               const float2 *__restrict__ tw) {
    extern __shared__ float2 smem[];
    float2 *a = smem, *b = smem + n;
    const long long row = blockIdx.x;
    const float *r = re + row * width, *q = im + row * width;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        float xr, xi;
        if (k < width) { xr = r[k]; xi = q[k]; }
        else { xr = r[n - k]; xi = -q[n - k]; }
        a[k] = make_float2(xr, -xi);                 // conj in; the conj out only flips the unused imaginary part
    }
    __syncthreads();
    a = af_stockham(a, b, n, log2n, tw);
    const float inv = 1.0f / (float)n;
    float *f = frames + row * n;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        float v = a[j].x * inv;
        if (weightMode && window) v *= window[j];
        f[j] = v;
    }
}

// same transform for frames whose ping-pong buffers do not fit shared memory (fftLength 16384: 2 x 128 KB): the in-place
// passes of af_fft_inplace_dif over ONE buffer, result in bit-reversed order, undone while the frame is written out.
// Only this size takes the path; the Stockham kernel above is 2-3x faster where it fits.
__global__ void k_istft_frames_inplace(const float *__restrict__ re, const float *__restrict__ im, int width, int n, int log2n,
                                       const float *__restrict__ window, int weightMode, float *__restrict__ frames,
                                       const float2 *__restrict__ tw) {
    extern __shared__ float2 smem[];
    float2 *a = smem;
    const long long row = blockIdx.x;
    const float *r = re + row * width, *q = im + row * width;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        float xr, xi;
        if (k < width) { xr = r[k]; xi = q[k]; }
        else { xr = r[n - k]; xi = -q[n - k]; }
        a[k] = make_float2(xr, -xi);
    }
    __syncthreads();
    af_fft_inplace_dif(a, n, tw);
    const float inv = 1.0f / (float)n;
    float *f = frames + row * n;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        float v = a[af_brev(j, log2n)].x * inv;
        if (weightMode && window) v *= window[j];
        f[j] = v;
    }
}

__global__ void k_istft_ola(const float *__restrict__ frames, int n, int hop, int timeLength, int dataLength,
                            const float *__restrict__ window, int weightMode, float *__restrict__ data, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const long long clip = i / dataLength;
    const int j = (int)(i - clip * dataLength);
    int t0 = j - n + 1;
    t0 = t0 <= 0 ? 0 : (t0 + hop - 1) / hop;
    int t1 = j / hop;
    if (t1 > timeLength - 1) t1 = timeLength - 1;
    float acc = data[i], norm = 0.0f;
    const float *f = frames + clip * (long long)timeLength * n;
    for (int t = t0; t <= t1; t++) {
        const int k = j - t * hop;
        acc = acc + f[(long long)t * n + k];
        const float w = window ? window[k] : 1.0f;
        norm = norm + (weightMode ? w * w : w);      // w^(e+1)
    }
    if (norm < 1e-6f) norm = 1.0f;
    data[i] = acc / norm;
}

// ---- long frames: c = Re H + Im H of the (mirrored) planes -> four-step forward FFT -> (Re C + Im C) / n ----
__global__ void __launch_bounds__(256) k_istft_long_pre(const float *__restrict__ re, const float *__restrict__ im, int width, int n,
                                                        long long row0, int nf, float *__restrict__ c) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)nf * n) return;
    const long long f = i / n;
    const int k = (int)(i - f * n), km = k ? n - k : 0;
    const float *r = re + (row0 + f) * width, *q = im + (row0 + f) * width;
    // X[k] as k_istft_frames reads it: the planes below `width`, the Hermitian mirror above
    const float xr = k < width ? r[k] : r[n - k], xi = k < width ? q[k] : -q[n - k];
    const float yr = km < width ? r[km] : r[n - km], yi = km < width ? q[km] : -q[n - km];
    c[i] = 0.5f * (xr + yr) + 0.5f * (xi - yi);
}

__global__ void __launch_bounds__(256) k_istft_long_post(const float2 *__restrict__ spec, int n, long long row0, int nf,
                                                         const float *__restrict__ window, int weightMode, float *__restrict__ frames) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)nf * n) return;
    const int j = (int)(i % n);
    const float2 C = spec[i];
    float v = (C.x + C.y) * (1.0f / (float)n);
    if (weightMode && window) v *= window[j];
    frames[row0 * n + i] = v;
}

}  // namespace

// frames of more than 16384 points: chunks of frames (af_fft_rows_chunk) through a stream-ordered workspace, as the
// forward side does (stft_generic.cu)
static int launch_istft_frames_long(const float *re, const float *im, int width, int n, int log2n, long long rows,
                                    const float *window, int weightMode, float *frames, cudaStream_t st) {
    const long long chunk = af_fft_rows_chunk(log2n, rows);
    const size_t specBytes = af_fft_rows_workspace_bytes(log2n, (int)chunk);
    void *ws = nullptr;
    cudaError_t e = cudaMallocAsync(&ws, specBytes + sizeof(float) * (size_t)n * chunk, st);
    if (e != cudaSuccess) return af_cuda_check(e, "cudaMallocAsync(long-frame ISTFT workspace)");
    float2 *spec = static_cast<float2 *>(ws);
    float *c = reinterpret_cast<float *>(static_cast<char *>(ws) + specBytes);
    int rc = AF_OK;
    for (long long r0 = 0; r0 < rows && rc == AF_OK; r0 += chunk) {
        const int nf = (int)(rows - r0 < chunk ? rows - r0 : chunk);
        const long long cells = (long long)nf * n;
        k_istft_long_pre<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(re, im, width, n, r0, nf, c);
        af_count_launch(1);
        if ((rc = af_launch_fft_rows(c, log2n, nf, spec, st))) break;
        k_istft_long_post<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(spec, n, r0, nf, window, weightMode, frames);
        af_count_launch(1);
        if ((e = cudaGetLastError()) != cudaSuccess) rc = af_cuda_check(e, "long-frame ISTFT launch");
    }
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int af_launch_istft(const float *re, const float *im, int width, int fftLength, int slideLength, int timeLength,
                               int batch, const float *window, int methodType, float *frames, float *data, void *stream) {
    if (timeLength <= 0 || batch <= 0) return AF_OK;
    int log2n = 0;
    while ((1 << log2n) < fftLength) log2n++;
    if (fftLength > (1 << 20)) return af_fail(AF_ERR_UNSUPPORTED, "istft: fftLength %d > 2^20 is not supported", fftLength);
    const int weightMode = methodType == 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int dataLength = (timeLength - 1) * slideLength + fftLength;
    const long long total = (long long)batch * dataLength;
    if (fftLength > 16384) {
        int rc = launch_istft_frames_long(re, im, width, fftLength, log2n, (long long)batch * timeLength, window, weightMode, frames, st);
        if (rc) return rc;
        k_istft_ola<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(frames, fftLength, slideLength, timeLength, dataLength, window,
                                                                    weightMode, data, total);
        AF_LAUNCH_CHECK("k_istft_ola");
        return AF_OK;
    }
    const bool inplace = af_fft_inplace(fftLength);
    const size_t smem = sizeof(float2) * (inplace ? 1 : 2) * (size_t)fftLength;
    const int rc = inplace ? af_smem_optin(k_istft_frames_inplace, smem, "k_istft_frames_inplace")
                           : af_smem_optin(k_istft_frames, smem, "k_istft_frames");
    if (rc) return rc;
    const int threads = af_cta_threads(fftLength / 4, 1024);
    if (inplace)
        k_istft_frames_inplace<<<(unsigned)((long long)batch * timeLength), threads, smem, st>>>(re, im, width, fftLength, log2n, window,
                                                                                                weightMode, frames, af_twiddle_table(log2n));
    else
        k_istft_frames<<<(unsigned)((long long)batch * timeLength), threads, smem, st>>>(re, im, width, fftLength, log2n, window,
                                                                                        weightMode, frames, af_twiddle_table(log2n));
    AF_LAUNCH_CHECK("k_istft_frames");
    k_istft_ola<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(frames, fftLength, slideLength, timeLength, dataLength, window,
                                                                weightMode, data, total);
    AF_LAUNCH_CHECK("k_istft_ola");
    return AF_OK;
}
