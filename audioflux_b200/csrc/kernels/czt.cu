// czt.cu -- chirp z-transform (sm_90a), replacing _cztObj_czt (src/dsp/czt_algorithm.c:163-257), which runs three
// M-point FFTs per call on one core (the filter's included).
//
// k_czt: one CTA per row, one buffer of M = 2N complex points in shared memory.
//   1. g[n] = x[n] * pre[n] for n < N (the reference's A^-n W^(n^2/2) product, then the input, multiplied as :209-237
//      multiplies them), 0 above;
//   2. af_fft_inplace_dif (bit-reversed order), times H = FFT_M(h), which the object stores in the same order, and
//      conjugated;
//   3. af_fft_inplace_dit (natural order): y = conj(result) / M is the reference's IFFT_M(G H);
//   4. the head y[N-1+k] * post[k] and the tail y[N+k] as they are, k < N (:253-255).
// k_czt_filter: one CTA turns the chirp filter h into H in place, once per table change of the object.
//
// The file is compiled with -fmad=false (Makefile): the complex products are rounded step by step, as in the reference.
#include "common.cuh"
#include "stockham.cuh"

namespace {

constexpr int kMaxThreads = 1024;

struct CztParams {
    const float *re, *im;
    float *re3, *im3;
    const float2 *pre, *post, *H;
    const float2 *tw;                  // af_twiddle_table(log2m)
    int N, M, log2m;
};

__device__ __forceinline__ float2 cmul_ref(float2 a, float2 b) {   // __complexMul (src/vector/flux_complex.c:763-769)
    return make_float2(a.x * b.x - a.y * b.y, a.y * b.x + a.x * b.y);
}

__global__ void __launch_bounds__(kMaxThreads) k_czt(CztParams p) {
    extern __shared__ float2 a[];
    const int N = p.N, M = p.M, tid = threadIdx.x, bd = blockDim.x;
    const long long row = blockIdx.x;
    const float *re = p.re ? p.re + row * N : nullptr, *im = p.im ? p.im + row * N : nullptr;
    for (int j = tid; j < M; j += bd) {
        float2 g = make_float2(0.0f, 0.0f);
        if (j < N) {
            const float2 c = __ldg(p.pre + j);
            if (re && im) g = cmul_ref(c, make_float2(__ldg(re + j), __ldg(im + j)));
            else if (re) { const float v = __ldg(re + j); g = make_float2(c.x * v, c.y * v); }
            else { const float v = __ldg(im + j); g = make_float2(-c.y * v, c.x * v); }
        }
        a[j] = g;
    }
    __syncthreads();
    af_fft_inplace_dif(a, M, p.tw);
    for (int j = tid; j < M; j += bd) {
        const float2 v = cmul_ref(a[j], __ldg(p.H + j));
        a[j] = make_float2(v.x, -v.y);
    }
    __syncthreads();
    af_fft_inplace_dit(a, M, p.log2m, p.tw);
    const float inv = 1.0f / (float)M;
    float *o = p.re3 + row * M, *q = p.im3 + row * M;
    for (int k = tid; k < N; k += bd) {
        const float2 y = a[N - 1 + k];
        const float2 h = cmul_ref(make_float2(y.x * inv, -y.y * inv), __ldg(p.post + k));
        o[k] = h.x; q[k] = h.y;
        const float2 t = a[N + k];
        o[N + k] = t.x * inv; q[N + k] = -t.y * inv;
    }
}

__global__ void __launch_bounds__(kMaxThreads) k_czt_filter(float2 *H, int M, const float2 *tw) {
    extern __shared__ float2 a[];
    for (int j = threadIdx.x; j < M; j += blockDim.x) a[j] = H[j];
    __syncthreads();
    af_fft_inplace_dif(a, M, tw);
    for (int j = threadIdx.x; j < M; j += blockDim.x) H[j] = a[j];
}

}  // namespace

extern "C" int af_launch_czt_filter(float *H, int log2m, void *stream) {
    if (log2m < 1 || log2m > AFB200_CZT_MAX_EXP + 1) return af_fail(AF_ERR_UNSUPPORTED, "czt: 2^%d-point transforms", log2m);
    const int M = 1 << log2m;
    const float2 *tw = af_twiddle_table(log2m);
    if (!tw) return af_fail(AF_ERR_CUDA, "czt: twiddle table 2^%d", log2m);
    const size_t smem = sizeof(float2) * (size_t)M;
    const int rc = af_smem_optin(k_czt_filter, smem, "k_czt_filter");
    if (rc) return rc;
    k_czt_filter<<<1, af_cta_threads(M / 2, kMaxThreads), smem, (cudaStream_t)stream>>>(reinterpret_cast<float2 *>(H), M, tw);
    AF_LAUNCH_CHECK("k_czt_filter");
    return AF_OK;
}

extern "C" int af_launch_czt(const AfCztArgs *a, void *stream) {
    if (a->log2n < 0 || a->log2n > AFB200_CZT_MAX_EXP) return af_fail(AF_ERR_UNSUPPORTED, "czt: 2^%d points", a->log2n);
    if (!a->re && !a->im) return af_fail(AF_ERR_ARG, "czt: no input plane");
    if (a->batch <= 0) return AF_OK;
    CztParams p;
    p.N = 1 << a->log2n; p.M = 2 * p.N; p.log2m = a->log2n + 1;
    p.re = a->re; p.im = a->im; p.re3 = a->re3; p.im3 = a->im3;
    const float2 *t = reinterpret_cast<const float2 *>(a->tables);
    p.pre = t; p.post = t + p.N; p.H = t + 2 * p.N;
    p.tw = af_twiddle_table(p.log2m);
    if (!p.tw) return af_fail(AF_ERR_CUDA, "czt: twiddle table 2^%d", p.log2m);
    const size_t smem = sizeof(float2) * (size_t)p.M;
    const int rc = af_smem_optin(k_czt, smem, "k_czt");
    if (rc) return rc;
    k_czt<<<(unsigned)a->batch, af_cta_threads(p.M / 2, kMaxThreads), smem, (cudaStream_t)stream>>>(p);
    AF_LAUNCH_CHECK("k_czt");
    return AF_OK;
}
