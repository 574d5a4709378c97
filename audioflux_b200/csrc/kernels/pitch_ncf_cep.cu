// pitch_ncf_cep.cu -- pitch by the normalised correlation (sm_90a), replacing the frame loops of pitchNCFObj_pitch
// (src/mir/_pitch_ncf.c:380-494), and by the cepstrum, replacing those of pitchCEPObj_pitch (src/mir/_pitch_cep.c:381-474).
// The reference runs a 2n-point FFT and a 2n-point inverse per frame on one core and keeps a timeLength x 2n matrix.
//
// k_pitch_ncf and k_pitch_cep: one CTA per frame, everything in shared memory, one body (n = 2^log2n):
//   1. the windowed frame is read coalesced into the first half of a 2n-point real input packed as n complex points
//      (the second half is the zero padding) and transformed in place (af_fft_inplace_dif: bit-reversed order);
//   2. af_real_inverse turns the per-bin step of X, read by af_real_bin_brev, into n c, c the 2n-point inverse (1/2n
//      included): NCF |X_k|^2 = re*re + im*im, CEP logf of it (full-precision logf, as the reference's __vlog);
//   3. only the needed lags are read back (af_real_at).  NCF: slot j = minIndex .. maxIndex-1 holds
//      ((c[j+1] / n) * s) * (1 / rms), s = (float)(1/sqrtf(2n)) and rms = sqrtf((c[0] / n) * s), the reference's two
//      float scale factors in its order (/ n is exact); slot maxIndex is the reference's 0 that is never written.
//      CEP: slot k = minIndex .. maxIndex holds n c[k]; a power-of-two scale changes no comparison;
//   4. __vmax's first arg-max over the slots (vmax_take, block_argmax, vmax_first: a NaN first slot, as in silence
//      (0 * inf, or -inf - -inf) or a frame holding a NaN, stays the maximum), fre = samplate / (index + 1) in double.
// Only the clips are read from HBM and one float per frame is written.
//
// Shared memory: 8n bytes for the packed transform (and 256 bytes for the reductions): 32 KB at the defaults
// (n = 2^12) and 128 KB at n = 2^14, within the 227 KB a CTA may hold; n = 2^15 would need 256 KB, hence
// AFB200_PITCH_NCF_MAX_EXP = AFB200_PITCH_CEP_MAX_EXP = 14.
//
// The file is compiled with -fmad=false (Makefile): |X|^2, the real-FFT passes and the scale factors are rounded on
// their own, as in the reference.
#include "block_reduce.cuh"
#include "stockham.cuh"

namespace {

constexpr int kMaxThreads = 1024;
// 32 registers: 2048 threads per SM (65 536 registers / 32), the most an SM runs; the launcher sizes the CTAs so that
// the CTAs that fit in shared memory fill them
constexpr int kMinBlocks = 2;

struct LagParams {
    const float *data, *window;
    float *fre;
    const float2 *tw;              // af_twiddle_table(log2n): n-point butterflies and the 2n-point real-FFT passes
    int n, log2n, minIndex, maxIndex, samplate, dataLength, hop, T;
    float scale;                   // NCF: (float)(1.0 / sqrtf(2n))
};

template <int kMode>
__device__ __forceinline__ void pitch_lag(const LagParams &p) {
    extern __shared__ float2 smem[];
    __shared__ float redv[32];
    __shared__ int redi[32];
    const int n = p.n, tid = threadIdx.x, bd = blockDim.x;
    float2 *X = smem;                                                  // n complex points: the 2n-point real input
    const long long f = blockIdx.x, clip = f / p.T, t = f - clip * p.T;
    const float *x = p.data + clip * p.dataLength + t * p.hop;

    float *a = reinterpret_cast<float *>(X);
    for (int j = tid; j < 2 * n; j += bd) a[j] = j < n ? __ldg(x + j) * __ldg(p.window + j) : 0.0f;
    __syncthreads();
    af_fft_inplace_dif(X, n, p.tw);
    af_real_inverse(X, n, p.log2n, p.tw, [&](int k) {
        const float2 z = af_real_bin_brev(X, p.tw, k, n, p.log2n);
        const float pw = z.x * z.x + z.y * z.y;
        return make_float2(kMode == AF_PITCH_NCF ? pw : logf(pw), 0.0f);
    });

    const int lo = p.minIndex, hi = p.maxIndex;
    float bv = 0.0f;
    int bi = -1;
    float v0;
    if (kMode == AF_PITCH_NCF) {
        const float inv = 1.0f / (float)n;                             // exact
        const float rms = sqrtf(af_real_at(X, 0) * inv * p.scale);
        const float norm = (float)(1.0 / (double)rms);                 // :460-465
        for (int j = lo + tid; j <= hi; j += bd)
            vmax_take(j < hi ? af_real_at(X, j + 1) * inv * p.scale * norm : 0.0f, j, bv, bi);
        v0 = lo < hi ? af_real_at(X, lo + 1) * inv * p.scale * norm : 0.0f;
    } else {
        for (int k = lo + tid; k <= hi; k += bd) vmax_take(af_real_at(X, k), k, bv, bi);
        v0 = af_real_at(X, lo);
    }
    bi = block_argmax(bv, bi, redv, redi);
    if (tid == 0) p.fre[f] = (float)((double)p.samplate / (vmax_first(bi, v0, lo) + 1));
}

__global__ void __launch_bounds__(kMaxThreads, kMinBlocks) k_pitch_ncf(LagParams p) { pitch_lag<AF_PITCH_NCF>(p); }
__global__ void __launch_bounds__(kMaxThreads, kMinBlocks) k_pitch_cep(LagParams p) { pitch_lag<AF_PITCH_CEP>(p); }

}  // namespace

extern "C" int af_launch_pitch_ncf_cep(const AfPitchLagArgs *a, void *stream) {
    const bool ncf = a->mode == AF_PITCH_NCF;
    if (a->mode != AF_PITCH_NCF && a->mode != AF_PITCH_CEP) return af_fail(AF_ERR_ARG, "pitch NCF/CEP: mode %d", a->mode);
    const char *name = ncf ? "k_pitch_ncf" : "k_pitch_cep";
    if (a->log2n < 1 || a->log2n > AFB200_PITCH_NCF_MAX_EXP)
        return af_fail(AF_ERR_UNSUPPORTED, "%s: frame 2^%d; frames 2^1 .. 2^%d", name, a->log2n, AFB200_PITCH_NCF_MAX_EXP);
    const int n = 1 << a->log2n;
    if (a->minIndex < (ncf ? 1 : 0) || a->maxIndex < a->minIndex || a->maxIndex >= (ncf ? n : 2 * n))
        return af_fail(AF_ERR_ARG, "%s: lags %d .. %d", name, a->minIndex, a->maxIndex);
    const long long frames = (long long)a->batch * a->timeLength;
    if (frames <= 0) return AF_OK;
    if (frames > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "%s: too many frames in one launch", name);
    LagParams p;
    p.data = a->data; p.window = a->window; p.fre = a->fre;
    p.n = n; p.log2n = a->log2n; p.minIndex = a->minIndex; p.maxIndex = a->maxIndex; p.samplate = a->samplate;
    p.dataLength = a->dataLength; p.hop = a->hop; p.T = a->timeLength;
    p.scale = (float)(1.0 / sqrtf((float)(2 * n)));                   // :454, 1.0/sqrtf(corrFFTLength) as a float
    p.tw = af_twiddle_table(a->log2n);
    if (!p.tw) return af_fail(AF_ERR_CUDA, "%s: twiddle table 2^%d", name, a->log2n);
    const size_t smem = sizeof(float2) * (size_t)n;
    // as many threads as the CTAs that fit an SM's 228 KB of shared memory (1 KB each reserved) leave of the 2048 its
    // registers hold at the kernels' 32-register budget, and no more than one per butterfly
    const int fit = (int)((228u * 1024u) / (smem + 1024u)), want = (2048 / (fit > 1 ? fit : 1)) & ~31;
    const int threads = af_cta_threads(want, af_cta_threads(n / 2, kMaxThreads));
    int rc;
    if (ncf) {
        if ((rc = af_smem_optin(k_pitch_ncf, smem, name))) return rc;
        k_pitch_ncf<<<(unsigned)frames, threads, smem, (cudaStream_t)stream>>>(p);
    } else {
        if ((rc = af_smem_optin(k_pitch_cep, smem, name))) return rc;
        k_pitch_cep<<<(unsigned)frames, threads, smem, (cudaStream_t)stream>>>(p);
    }
    AF_LAUNCH_CHECK(name);
    return AF_OK;
}
