// pitch_pef.cu -- pitch by the pitch estimation filter (sm_90a), replacing the frame loops of pitchPEFObj_pitch
// (src/mir/_pitch_pef.c:258-426), which run a 2n-point FFT and an 8n-point correlation (forward and inverse) per frame on
// one core.
//
// k_pitch_pef: one CTA per frame, everything in shared memory (n = 2^log2n, P the filter's zero padding):
//   1. the windowed frame is read coalesced into the first half of a 2n-point real input packed as n complex points (the
//      second half is the zero padding); Stockham transform (stockham.cuh, twiddles from af_twiddle_table) and the
//      real-FFT post-pass give power[k] = re^2 + im^2, k = 0 .. n, kept in its own buffer;
//   2. s[P + i] = (y1 + (log[i] - x1)(y2 - y1)/(x2 - x1)) * bandWidth[i], i < 2n: __vinterp_linear's step with its
//      segment index from the object's table, the grids read from the device tables; s is zero elsewhere up to L;
//   3. s, packed as L/2 complex points, is transformed in place (af_fft_inplace_dif: bit-reversed order);
//      af_real_inverse turns S conj(F), S read by af_real_bin_brev and F the filter's spectrum, into (L/2) c, c the
//      correlation c[k] = sum_j filter[j] s[j + k mod L], read by af_real_at.  The scale is left in: a power-of-two
//      scale changes no comparison;
//   4. the first arg-max of c over the lags minIndex .. maxIndex (__vmax: vmax_take, block_argmax, vmax_first), and
//      fre = log[that lag].
// Only the clips are read from HBM and one float per frame is written.
//
// The transform length.  The reference correlates at 8n (P > 0) or 4n (P = 0).  Any L >= P + 2n (s fits) and
// L >= n + maxIndex + 1 gives the same lags 0 .. maxIndex up to rounding, because with j < n and k <= maxIndex no product
// filter[j] s[j + k] wraps.  P < n and maxIndex < 2n, so the host picks the smallest such power of two, at most 4n: the
// L/2 complex points (L <= 4n floats) reuse the two n-point Stockham buffers of step 1.  With the n + 1 power values that
// is 40 KB of shared memory per CTA at n = 2^11, 80 KB at 2^12 (two CTAs per SM) and 160 KB at 2^13; n = 2^14 would
// need 320 KB, above the 227 KB a CTA may hold, hence
// AFB200_PITCH_PEF_MAX_EXP = 13.
//
// The file is compiled with -fmad=false (Makefile): the power, each step of the interpolation and the weighting are
// rounded on their own, as in the reference.
#include "block_reduce.cuh"
#include "stockham.cuh"

namespace {

constexpr int kMaxThreads = 1024;

struct PefParams {
    const float *data, *window, *lin, *logf, *bw;
    const int *idx;
    const float2 *spec;            // filter spectrum, bins 0 .. L/2
    float *fre;
    const float2 *tw1;             // af_twiddle_table(log2n): n-point butterflies and the 2n-point post-pass
    const float2 *tw2;             // af_twiddle_table(log2L - 1): L/2-point butterflies and the L-point post-pass
    int n, log2n, nc, log2nc, pad, minIndex, maxIndex, dataLength, hop, T;
};

__device__ __forceinline__ float2 times_conj_filter(const PefParams &p, const float2 *z, int k) {
    const float2 x = af_real_bin_brev(z, p.tw2, k, p.nc, p.log2nc), f = __ldg(p.spec + k);
    return make_float2(x.x * f.x + x.y * f.y, x.y * f.x - x.x * f.y);
}

__global__ void __launch_bounds__(kMaxThreads) k_pitch_pef(PefParams p) {
    extern __shared__ float2 smem[];
    __shared__ float redv[32];
    __shared__ int redi[32];
    const int n = p.n, nc = p.nc, tid = threadIdx.x, bd = blockDim.x;
    float2 *S = smem;                                                  // 2n complex points (nc <= 2n)
    float *pw = reinterpret_cast<float *>(smem + 2 * n);               // n + 1 power values
    const long long f = blockIdx.x, clip = f / p.T, t = f - clip * p.T;
    const float *x = p.data + clip * p.dataLength + t * p.hop;

    float *a = reinterpret_cast<float *>(S);
    for (int j = tid; j < 2 * n; j += bd) a[j] = j < n ? __ldg(x + j) * __ldg(p.window + j) : 0.0f;
    __syncthreads();
    const float2 *X = af_stockham(S, S + n, n, p.log2n, p.tw1);
    for (int k = tid; k <= n; k += bd) {
        const float2 z = af_real_bin(X, __ldg(p.tw1 + n + k), k, n);   // exp(-2 pi i k / 2n)
        pw[k] = z.x * z.x + z.y * z.y;
    }
    __syncthreads();

    float *s = reinterpret_cast<float *>(S);                           // L = 2 nc real values
    const int L = 2 * nc, P = p.pad;
    for (int i = tid; i < L; i += bd) {
        float v = 0.0f;
        const int m = i - P;
        if (m >= 0 && m < 2 * n) {
            const int j = __ldg(p.idx + m);
            if (j < n) {
                const float x1 = __ldg(p.lin + j), x2 = __ldg(p.lin + j + 1), y1 = pw[j], y2 = pw[j + 1];
                v = y1 + (__ldg(p.logf + m) - x1) * (y2 - y1) / (x2 - x1);
            } else {
                v = pw[n];
            }
            v = v * __ldg(p.bw + m);
        }
        s[i] = v;
    }
    __syncthreads();

    af_fft_inplace_dif(S, nc, p.tw2);
    af_real_inverse(S, nc, p.log2nc, p.tw2, [&](int k) { return times_conj_filter(p, S, k); });

    const int lo = p.minIndex, hi = p.maxIndex;
    float bv = 0.0f;
    int bi = -1;
    for (int k = lo + tid; k <= hi; k += bd) vmax_take(af_real_at(S, k), k, bv, bi);
    bi = block_argmax(bv, bi, redv, redi);
    if (tid == 0) p.fre[f] = __ldg(p.logf + vmax_first(bi, af_real_at(S, lo), lo));
}

}  // namespace

extern "C" int af_launch_pitch_pef(const AfPitchPefArgs *a, void *stream) {
    if (a->log2n < 1 || a->log2n > AFB200_PITCH_PEF_MAX_EXP || a->log2L < a->log2n + 1 || a->log2L > a->log2n + 2)
        return af_fail(AF_ERR_UNSUPPORTED, "pitch PEF: frame 2^%d, transform 2^%d; frames 2^1 .. 2^%d, transforms 2n or 4n",
                       a->log2n, a->log2L, AFB200_PITCH_PEF_MAX_EXP);
    const int n = 1 << a->log2n;
    if (a->minIndex < 0 || a->maxIndex <= a->minIndex || a->maxIndex >= 2 * n)
        return af_fail(AF_ERR_ARG, "pitch PEF: lags %d .. %d", a->minIndex, a->maxIndex);
    PefParams p;
    const long long frames = (long long)a->batch * a->timeLength;
    if (frames <= 0) return AF_OK;
    if (frames > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "pitch PEF: too many frames in one launch");
    p.data = a->data; p.fre = a->fre;
    p.window = a->tables; p.lin = a->tables + AF_PEF_LIN(n); p.logf = a->tables + AF_PEF_LOG(n);
    p.bw = a->tables + AF_PEF_BW(n);
    p.idx = reinterpret_cast<const int *>(a->tables + AF_PEF_IDX(n));
    p.spec = reinterpret_cast<const float2 *>(a->tables + AF_PEF_SPEC(n));
    p.n = n; p.log2n = a->log2n; p.nc = 1 << (a->log2L - 1); p.log2nc = a->log2L - 1; p.pad = a->padNum;
    p.minIndex = a->minIndex; p.maxIndex = a->maxIndex;
    p.dataLength = a->dataLength; p.hop = a->hop; p.T = a->timeLength;
    p.tw1 = af_twiddle_table(a->log2n);
    p.tw2 = af_twiddle_table(p.log2nc);
    if (!p.tw1 || !p.tw2) return af_fail(AF_ERR_CUDA, "pitch PEF: twiddle tables 2^%d, 2^%d", a->log2n, p.log2nc);
    const int threads = af_cta_threads(p.nc / 2, kMaxThreads);
    const size_t smem = sizeof(float2) * 2 * (size_t)n + sizeof(float) * (size_t)(n + 1);
    const int rc = af_smem_optin(k_pitch_pef, smem, "k_pitch_pef");
    if (rc) return rc;
    k_pitch_pef<<<(unsigned)frames, threads, smem, (cudaStream_t)stream>>>(p);
    AF_LAUNCH_CHECK("k_pitch_pef");
    return AF_OK;
}
