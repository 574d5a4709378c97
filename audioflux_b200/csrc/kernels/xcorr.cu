// xcorr.cu -- cross-correlation and autocorrelation (sm_90a), replacing _xcorrObj_fft and the Coeff / __vmax passes of
// xcorrObj_xcorr (src/dsp/xcorr_algorithm.c:49-115, 182-243), which run two forward and one inverse M-point FFT per call
// on one core.
//
// k_xcorr (M <= 2^14): one CTA per pair, everything in one buffer per signal.
//   1. each signal, zero-padded to M, is packed as M/2 complex points (x[2j] + i x[2j+1]) and transformed in place
//      (af_fft_inplace_dif: bit-reversed order).  The two signals keep separate transforms: packing a and b into one
//      complex transform would let the louder leak into the quieter one;
//   2. af_real_inverse turns P = A conj(B) (|A|^2 for the autocorrelation), A and B read by af_real_bin_brev, into
//      nc r, r = IFFT_M(P) with the reference's 1/M and nc = M/2; af_real_at times 1/nc gives r;
//   3. the 2n-1 lags in the reference's order, divided by the Coeff scale, and __vmax's first arg-max.
// Longer rows (M = 2^15 .. 2^20): the zero-padded signals go through the CWT path's four-step forward legs
// (af_launch_fft_rows); k_xcorr_cross forms the Hermitian P and writes its Hartley sequence c = Re P + Im P; a second
// forward pass gives C, and Re C[j] + Im C[j] = M r[j].  k_xcorr_finish writes the lags and per-segment arg-max
// candidates, k_xcorr_argmax reduces them in a fixed order (no atomics).  The workspace belongs to the object and is kept
// between calls.
//
// Sums of squares are float products summed in double in a fixed order, like __vsum's double accumulator.  The file is
// compiled with -fmad=false (Makefile): the scale and the post-passes are rounded step by step.
#include "block_reduce.cuh"
#include "stockham.cuh"

namespace {

constexpr int kMaxThreads = 1024;
constexpr int kPadSegs = 32;            // long path: segments of a padded row (partial sums of squares per segment)
constexpr int kFinishSegs = 128;        // long path: segments of an output row (arg-max candidates per segment)
constexpr int kLongThreads = 256;

struct XcParams {
    const float *a, *b;
    float *out, *maxValue;
    int *maxIndex;
    const float2 *tw;                   // af_twiddle_table(log2nc): nc-point butterflies, then W_M^k for k <= nc
    int n, M, nc, log2nc, coeff;
};

// xcorrObj_xcorr's Coeff scale (:85-103): sqrtf of the product of the two float sums
__device__ __forceinline__ float coeff_scale(double s1, double s2) {
    const float f1 = (float)s1, f2 = (float)s2;
    return sqrtf(f1 * f2);
}

__device__ __forceinline__ float2 cross(const XcParams &p, const float2 *A, const float2 *B, int k) {
    const float2 x = af_real_bin_brev(A, p.tw, k, p.nc, p.log2nc);
    if (!p.b) return make_float2(x.x * x.x + x.y * x.y, 0.0f);
    const float2 y = af_real_bin_brev(B, p.tw, k, p.nc, p.log2nc);
    return make_float2(x.x * y.x + x.y * y.y, x.y * y.x - x.x * y.y);   // x conj(y)
}

__global__ void __launch_bounds__(kMaxThreads) k_xcorr(XcParams p) {
    extern __shared__ float2 smem[];
    __shared__ double redd[32];
    __shared__ float redv[32];
    __shared__ int redi[32];
    float2 *A = smem, *B = smem + p.nc;
    const int n = p.n, nc = p.nc, tid = threadIdx.x, bd = blockDim.x;
    const long long row = blockIdx.x;
    const float *x = p.a + row * n, *y = p.b ? p.b + row * n : nullptr;
    double s1 = 0.0, s2 = 0.0;
    for (int j = tid; j < nc; j += bd) {
        const int i0 = 2 * j, i1 = i0 + 1;
        const float x0 = i0 < n ? __ldg(x + i0) : 0.0f, x1 = i1 < n ? __ldg(x + i1) : 0.0f;
        A[j] = make_float2(x0, x1);
        s1 += (double)(x0 * x0) + (double)(x1 * x1);
        if (y) {
            const float y0 = i0 < n ? __ldg(y + i0) : 0.0f, y1 = i1 < n ? __ldg(y + i1) : 0.0f;
            B[j] = make_float2(y0, y1);
            s2 += (double)(y0 * y0) + (double)(y1 * y1);
        }
    }
    __syncthreads();
    af_fft_inplace_dif(A, nc, p.tw);
    if (y) af_fft_inplace_dif(B, nc, p.tw);
    af_real_inverse(A, nc, p.log2nc, p.tw, [&](int k) { return cross(p, A, B, k); });

    float scale = 1.0f;
    if (p.coeff) {
        s1 = block_sum(s1, redd);
        s2 = y ? block_sum(s2, redd) : s1;
        scale = coeff_scale(s1, s2);
    }
    const int L = 2 * n - 1, M = p.M;
    const float inv = 1.0f / (float)nc;
    auto at = [&](int j) {
        const int lag = j - (n - 1);
        const float v = af_real_at(A, lag < 0 ? lag + M : lag) * inv;
        return p.coeff ? v / scale : v;
    };
    float *o = p.out + row * L;
    float bv = 0.0f;
    int bi = -1;
    for (int j = tid; j < L; j += bd) {
        const float v = at(j);
        o[j] = v;
        vmax_take(v, j, bv, bi);
    }
    bi = block_argmax(bv, bi, redv, redi);
    if (tid == 0) {
        bi = vmax_first(bi, at(0), 0);
        if (p.maxValue) p.maxValue[row] = at(bi);
        if (p.maxIndex) p.maxIndex[row] = bi;
    }
}

// ---- long path ----

// rows [rows][M]: a's rows, then b's; partial sums of the float squares per segment -> sums[row][kPadSegs]
__global__ void __launch_bounds__(kLongThreads) k_xcorr_pad(const float *__restrict__ a, const float *__restrict__ b, int n,
                                                            int M, int nb, float *__restrict__ rows, double *__restrict__ sums) {
    __shared__ double redd[32];
    const int r = blockIdx.y, seg = M / kPadSegs;
    const float *x = r < nb ? a + (size_t)r * n : b + (size_t)(r - nb) * n;
    float *dst = rows + (size_t)r * M;
    double s = 0.0;
    for (int j = blockIdx.x * seg + threadIdx.x; j < (blockIdx.x + 1) * seg; j += blockDim.x) {
        const float v = j < n ? __ldg(x + j) : 0.0f;
        dst[j] = v;
        s += (double)(v * v);
    }
    s = block_sum(s, redd);
    if (threadIdx.x == 0) sums[(size_t)r * kPadSegs + blockIdx.x] = s;
}

// c[pair][k] = Re P + Im P, P = A conj(B) (|A|^2 without b): the Hartley sequence of the Hermitian P
__global__ void __launch_bounds__(kLongThreads) k_xcorr_cross(const float2 *__restrict__ spec, int M, int nb, int autoc,
                                                              float *__restrict__ c) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x, pair = blockIdx.y;
    if (k >= M) return;
    const float2 x = spec[(size_t)pair * M + k];
    float pr, pi;
    if (autoc) { pr = x.x * x.x + x.y * x.y; pi = 0.0f; }
    else {
        const float2 y = spec[(size_t)(nb + pair) * M + k];
        pr = x.x * y.x + x.y * y.y; pi = x.y * y.x - x.x * y.y;
    }
    c[(size_t)pair * M + k] = pr + pi;
}

__device__ __forceinline__ float long_scale(const double *sums, int pair, int nb, int autoc) {
    double s1 = 0.0, s2 = 0.0;
    for (int s = 0; s < kPadSegs; s++) s1 += sums[(size_t)pair * kPadSegs + s];
    if (autoc) s2 = s1;
    else for (int s = 0; s < kPadSegs; s++) s2 += sums[(size_t)(nb + pair) * kPadSegs + s];
    return coeff_scale(s1, s2);
}

// the lags of each pair from C = FFT_M(c): r[m] = (Re C[m] + Im C[m]) / M; one arg-max candidate per segment
__global__ void __launch_bounds__(kLongThreads) k_xcorr_finish(const float2 *__restrict__ spec, const double *__restrict__ sums,
                                                               int n, int M, int nb, int autoc, int coeff, float *__restrict__ out,
                                                               float *__restrict__ candV, int *__restrict__ candI) {
    __shared__ float redv[32];
    __shared__ int redi[32];
    const int pair = blockIdx.y, L = 2 * n - 1, seg = (L + kFinishSegs - 1) / kFinishSegs;
    const float scale = coeff ? long_scale(sums, pair, nb, autoc) : 1.0f;
    const float inv = 1.0f / (float)M;
    const float2 *C = spec + (size_t)pair * M;
    float *o = out + (size_t)pair * L;
    float bv = 0.0f;
    int bi = -1;
    const int j1 = min(L, (int)(blockIdx.x + 1) * seg);
    for (int j = blockIdx.x * seg + threadIdx.x; j < j1; j += blockDim.x) {
        const int lag = j - (n - 1);
        const float2 v2 = C[lag < 0 ? lag + M : lag];
        float v = (v2.x + v2.y) * inv;
        if (coeff) v = v / scale;
        o[j] = v;
        vmax_take(v, j, bv, bi);
    }
    bi = block_argmax(bv, bi, redv, redi);
    if (threadIdx.x == 0) {
        candV[(size_t)pair * kFinishSegs + blockIdx.x] = bi >= 0 ? o[bi] : 0.0f;
        candI[(size_t)pair * kFinishSegs + blockIdx.x] = bi;
    }
}

__global__ void __launch_bounds__(kFinishSegs) k_xcorr_argmax(const float *__restrict__ out, int n, const float *__restrict__ candV,
                                                              const int *__restrict__ candI, float *__restrict__ maxValue,
                                                              int *__restrict__ maxIndex) {
    __shared__ float redv[32];
    __shared__ int redi[32];
    const int pair = blockIdx.x, L = 2 * n - 1;
    const int t = threadIdx.x;
    int bi = block_argmax(candV[(size_t)pair * kFinishSegs + t], candI[(size_t)pair * kFinishSegs + t], redv, redi);
    if (t == 0) {
        const float *o = out + (size_t)pair * L;
        bi = vmax_first(bi, o[0], 0);
        if (maxValue) maxValue[pair] = o[bi];
        if (maxIndex) maxIndex[pair] = bi;
    }
}

int launch_long(const AfXcorrArgs *a, int M, int log2M, cudaStream_t st) {
    const int autoc = a->b == nullptr, per = autoc ? 1 : 2;
    // per pair: padded rows (per x M floats), the long FFT's workspace (per x M spectra + inter-leg slots), candidates and sums
    const size_t perPair = (size_t)per * M * sizeof(float) + af_fft_rows_workspace_bytes(log2M, per) +
                           (size_t)kFinishSegs * (sizeof(float) + sizeof(int)) + (size_t)per * kPadSegs * sizeof(double);
    int chunk = (int)(((size_t)512 << 20) / perPair);
    if (chunk < 1) chunk = 1;
    if (chunk > a->batch) chunk = a->batch;
    const size_t wsBytes = af_fft_rows_workspace_bytes(log2M, per * chunk);
    const size_t rowsBytes = (size_t)per * chunk * M * sizeof(float);
    const size_t candBytes = (size_t)chunk * kFinishSegs * (sizeof(float) + sizeof(int));
    const size_t sumBytes = (size_t)per * chunk * kPadSegs * sizeof(double);
    const size_t total = sumBytes + wsBytes + rowsBytes + candBytes;
    int rc;
    // a larger workspace replaces the old one only after every launch that used it has finished
    if (a->work->bytes < total && ((rc = af_fence_wait(*a->fence)) || (rc = af_devbuf_reserve(a->work, total)))) return rc;
    if ((rc = af_fence_order(*a->fence, st))) return rc;
    char *mem = static_cast<char *>(a->work->ptr);
    double *sums = reinterpret_cast<double *>(mem);
    float2 *ws = reinterpret_cast<float2 *>(mem + sumBytes);
    float *rows = reinterpret_cast<float *>(mem + sumBytes + wsBytes);
    float *candV = rows + (size_t)per * chunk * M;
    int *candI = reinterpret_cast<int *>(candV + (size_t)chunk * kFinishSegs);
    const int n = a->n, L = 2 * n - 1;
    cudaError_t e;
    for (int p0 = 0; p0 < a->batch && rc == AF_OK; p0 += chunk) {
        const int nb = a->batch - p0 < chunk ? a->batch - p0 : chunk;
        const float *pa = a->a + (size_t)p0 * n, *pb = autoc ? nullptr : a->b + (size_t)p0 * n;
        k_xcorr_pad<<<dim3(kPadSegs, per * nb), kLongThreads, 0, st>>>(pa, pb, n, M, nb, rows, sums);
        af_count_launch(1);
        if ((rc = af_launch_fft_rows(rows, log2M, per * nb, ws, st))) break;
        k_xcorr_cross<<<dim3((unsigned)((M + kLongThreads - 1) / kLongThreads), nb), kLongThreads, 0, st>>>(ws, M, nb, autoc, rows);
        af_count_launch(1);
        if ((rc = af_launch_fft_rows(rows, log2M, nb, ws, st))) break;
        float *out = a->out + (size_t)p0 * L;
        k_xcorr_finish<<<dim3(kFinishSegs, nb), kLongThreads, 0, st>>>(ws, sums, n, M, nb, autoc, a->coeff, out, candV, candI);
        af_count_launch(1);
        k_xcorr_argmax<<<nb, kFinishSegs, 0, st>>>(out, n, candV, candI, a->maxValue ? a->maxValue + p0 : nullptr,
                                                   a->maxIndex ? a->maxIndex + p0 : nullptr);
        af_count_launch(1);
        if ((e = cudaGetLastError()) != cudaSuccess) rc = af_cuda_check(e, "long xcorr launch");
    }
    const int rf = af_fence_record(a->fence, st);
    return rc ? rc : rf;
}

}  // namespace

extern "C" int af_launch_xcorr(const AfXcorrArgs *a, void *stream) {
    if (a->n < 1 || a->n > AFB200_XCORR_MAX_LENGTH)
        return af_fail(AF_ERR_UNSUPPORTED, "xcorr: length %d; 1 .. %d are supported", a->n, AFB200_XCORR_MAX_LENGTH);
    if (a->batch <= 0) return AF_OK;
    int log2M = 0;
    while ((1 << log2M) < 2 * a->n) log2M++;
    const int M = 1 << log2M;
    cudaStream_t st = (cudaStream_t)stream;
    if (M > AF_XCORR_SHORT_MAX) return launch_long(a, M, log2M, st);
    XcParams p;
    p.a = a->a; p.b = a->b; p.out = a->out; p.maxValue = a->maxValue; p.maxIndex = a->maxIndex;
    p.n = a->n; p.M = M; p.nc = M / 2; p.log2nc = log2M - 1; p.coeff = a->coeff;
    p.tw = p.log2nc >= 1 ? af_twiddle_table(p.log2nc) : nullptr;
    if (p.log2nc >= 1 && !p.tw) return af_fail(AF_ERR_CUDA, "xcorr: twiddle table 2^%d", p.log2nc);
    const size_t smem = sizeof(float2) * 2 * (size_t)p.nc;
    const int rc = af_smem_optin(k_xcorr, smem, "k_xcorr");
    if (rc) return rc;
    k_xcorr<<<(unsigned)a->batch, af_cta_threads(p.nc / 2, kMaxThreads), smem, st>>>(p);
    AF_LAUNCH_CHECK("k_xcorr");
    return AF_OK;
}
