// cepstrogram.cu -- the cepstrogram (sm_90a), replacing the pass chain of __cepstrogramObj_spectrogram
// (src/cepstrogram_algorithm.c:127-298): STFT, power, log, inverse FFT, lifter and two forward FFTs, each over T x N
// float planes.
//
// k_cepstrogram: one CTA per frame (for N <= 256 a group of frames, one after the other).  Every N-point transform is a
// real-input FFT: the N reals packed as N/2 complex points, a Stockham transform in shared memory (stockham.cuh,
// twiddles from af_twiddle_table) and the real-FFT post-pass.  The post-pass of each transform writes the next
// transform's input straight into the free Stockham buffer, so per frame:
//   1. the windowed frame is read coalesced from the clip (frames overlap: re-reads hit L1 / L2), or the frame's STFT row
//      from the caller's planes (kPlanes; the transform of step 2 is skipped);
//   2. forward FFT; L[k] = logf(max(re^2 + im^2, 1e-16)) (:219-229), written as the real even sequence L[k] = L[N-k];
//   3. y = FFT_N(L) / N, which equals Re IFFT_N(L) for a real even L (:232-234); cep = y[0 .. N/2] (:236-239); the
//      envelope's input, y on {0 .. c} mirrored to {N-c .. N-1} (:257-262), is written as step 2 wrote L;
//   4. env = Re FFT_N(that) (:264-265);
//   5. det = Re FFT_N(y on {c+1 .. N-c}) (:283-287), from y[0 .. N/2] kept in shared memory.  Its own transform keeps
//      its error relative to its own size: the closed form L - env + y[c] cos(2 pi c k / N) would subtract two numbers
//      the size of L to get one that can be 35x smaller.  At c = N/2 the set is empty and the transform gives exact 0.
// No spectrum, log spectrum or cepstrum plane goes through HBM.  Requested outputs only: steps 4 and 5 run only for
// env and det.
#include "common.cuh"
#include "stockham.cuh"

namespace {

struct CepsParams {
    const float *data, *window, *specRe, *specIm;
    float *cep, *env, *det;
    const float2 *tw;              // af_twiddle_table(log2nc), null for N = 2
    long long frames;
    int n, nc, log2nc, cepNum, framesPerCta;
    int dataLength, hop, timeLength, specWidth;
};

__device__ __forceinline__ float log_power(float re, float im) { return logf(fmaxf(re * re + im * im, 1e-16f)); }

template <bool kPlanes>
__global__ void __launch_bounds__(1024) k_cepstrogram(CepsParams p) {
    extern __shared__ float2 smem[];
    const int n = p.n, nc = p.nc, c = p.cepNum, width = nc + 1;
    float2 *const A = smem, *const B = smem + nc;
    float *const ys = reinterpret_cast<float *>(smem + 2 * nc);        // y[0 .. N/2], when det is requested
    const float inv = 1.0f / (float)n;
    const long long f0 = (long long)blockIdx.x * p.framesPerCta;
    const long long f1 = min(p.frames, f0 + p.framesPerCta);
    for (long long f = f0; f < f1; f++) {
        const size_t row = (size_t)f * width;
        float2 *L;                                                     // the even log spectrum, packed
        if (kPlanes) {
            const float *re = p.specRe + (size_t)f * p.specWidth, *im = p.specIm + (size_t)f * p.specWidth;
            L = A;
            for (int k = threadIdx.x; k <= nc; k += blockDim.x) {
                float v = log_power(__ldg(re + k), __ldg(im + k));
                if (p.specWidth == n && k > 0 && k < nc) v = 0.5f * (v + log_power(__ldg(re + n - k), __ldg(im + n - k)));
                af_put_even(reinterpret_cast<float *>(L), n, k, v);
            }
        } else {
            const long long clip = f / p.timeLength, t = f % p.timeLength;
            const float *x = p.data + clip * p.dataLength + t * p.hop;
            float *a = reinterpret_cast<float *>(A);
            if (p.window)
                for (int j = threadIdx.x; j < n; j += blockDim.x) a[j] = __ldg(x + j) * __ldg(p.window + j);
            else
                for (int j = threadIdx.x; j < n; j += blockDim.x) a[j] = __ldg(x + j);
            __syncthreads();
            const float2 *X = af_stockham(A, B, nc, p.log2nc, p.tw);
            L = X == A ? B : A;
            for (int k = threadIdx.x; k <= nc; k += blockDim.x) {
                const float2 z = af_real_bin(X, af_real_tw(p.tw, nc, k), k, nc);
                af_put_even(reinterpret_cast<float *>(L), n, k, log_power(z.x, z.y));
            }
        }
        __syncthreads();

        const float2 *Y = af_stockham(L, L == A ? B : A, nc, p.log2nc, p.tw);
        float2 *F = Y == A ? B : A;                                    // free: the envelope's input, packed
        for (int k = threadIdx.x; k <= nc; k += blockDim.x) {
            const float y = af_real_bin(Y, af_real_tw(p.tw, nc, k), k, nc).x * inv;
            if (p.cep) p.cep[row + k] = y;
            if (p.env) af_put_even(reinterpret_cast<float *>(F), n, k, k <= c ? y : 0.0f);
            if (p.det) ys[k] = y;
        }
        __syncthreads();

        if (p.env) {
            const float2 *V = af_stockham(F, F == A ? B : A, nc, p.log2nc, p.tw);
            for (int k = threadIdx.x; k <= nc; k += blockDim.x) p.env[row + k] = af_real_bin(V, af_real_tw(p.tw, nc, k), k, nc).x;
            F = V == A ? B : A;
        }
        if (p.det) {                                                   // y on {c+1 .. N-c}, y[m] = y[N-m] above N/2
            float *d = reinterpret_cast<float *>(F);
            for (int m = threadIdx.x; m < n; m += blockDim.x) d[m] = m > c && m <= n - c ? ys[m <= nc ? m : n - m] : 0.0f;
            __syncthreads();
            const float2 *W = af_stockham(F, F == A ? B : A, nc, p.log2nc, p.tw);
            for (int k = threadIdx.x; k <= nc; k += blockDim.x) p.det[row + k] = af_real_bin(W, af_real_tw(p.tw, nc, k), k, nc).x;
        }
        __syncthreads();                                               // the buffers are free for the next frame
    }
}

template <bool kPlanes>
int launch(const CepsParams &p, unsigned grid, int threads, size_t smem, cudaStream_t st) {
    const int rc = af_smem_optin(k_cepstrogram<kPlanes>, smem, "k_cepstrogram");
    if (rc) return rc;
    k_cepstrogram<kPlanes><<<grid, threads, smem, st>>>(p);
    AF_LAUNCH_CHECK("k_cepstrogram");
    return AF_OK;
}

}  // namespace

extern "C" int af_launch_cepstrogram(const AfCepsArgs *a, void *stream) {
    const int n = 1 << a->log2n, nc = n / 2;
    if (a->log2n < 1 || n > AF_CEPS_MAX_N)
        return af_fail(AF_ERR_UNSUPPORTED, "cepstrogram: %d points; 2 .. %d are supported", n, AF_CEPS_MAX_N);
    if (a->cepNum < 1 || a->cepNum > nc) return af_fail(AF_ERR_ARG, "cepstrogram: cepNum=%d; 1 .. %d", a->cepNum, nc);
    const bool planes = a->data == nullptr;
    CepsParams p;
    p.data = a->data; p.window = a->window; p.specRe = a->specRe; p.specIm = a->specIm;
    p.cep = a->cep; p.env = a->env; p.det = a->det;
    p.frames = planes ? (long long)a->rows : (long long)a->batch * a->timeLength;
    if (p.frames <= 0 || (!p.cep && !p.env && !p.det)) return AF_OK;
    if (planes && a->specWidth != n && a->specWidth != nc + 1)
        return af_fail(AF_ERR_ARG, "cepstrogram: specWidth=%d must be %d or %d", a->specWidth, n, nc + 1);
    p.n = n; p.nc = nc; p.log2nc = a->log2n - 1; p.cepNum = a->cepNum;
    p.dataLength = a->dataLength; p.hop = a->hop; p.timeLength = a->timeLength; p.specWidth = a->specWidth;
    p.tw = p.log2nc >= 1 ? af_twiddle_table(p.log2nc) : nullptr;
    p.framesPerCta = n <= 256 ? 2048 / n : 1;
    const long long grid = (p.frames + p.framesPerCta - 1) / p.framesPerCta;
    if (grid > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "cepstrogram: too many frames in one launch");
    const int threads = af_cta_threads(nc / 4, 1024);
    const size_t smem = sizeof(float2) * 2 * (size_t)nc + (p.det ? sizeof(float) * (size_t)(nc + 1) : 0);
    cudaStream_t st = (cudaStream_t)stream;
    return planes ? launch<true>(p, (unsigned)grid, threads, smem, st) : launch<false>(p, (unsigned)grid, threads, smem, st);
}
