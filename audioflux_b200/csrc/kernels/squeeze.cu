// squeeze.cu -- synchrosqueezing kernels: instantaneous-frequency row index and the row scatter.
//
// Replaces the tail of wsstObj_wsst (src/wsst_algorithm.c:246-341: complex divide W'/W, / 2 pi, frequency -> row index,
// scatter-add of W into the indexed rows) and of synsqObj_synsq (src/synsq_algorithm.c:147-300: atan2f phase, unwrap
// along time, first difference, / 2 pi, the same index and scatter).  The transforms themselves are kernels/cwt.cu.
//   * index: one thread per (row, time) cell, float32 operation by operation as the reference evaluates it (explicit
//     _rn intrinsics: nvcc would otherwise contract c*c + d*d, b*c - a*d and the |W|^2 threshold test into FMAs, and
//     an FMA can move a cell to another row or across the threshold); log2f and atan2f are the CUDA Math API's, so
//     the Octave / Log index and the synsq phase may differ from glibc's where those round differently.  The index
//     and scatter are checked cell by cell on the GPU's own planes by tests/test_gpu_scatter_cells.py;
//   * unwrap (synsq): the reference's sequential rule adds a multiple of 2 pi chosen from the distance to the previous
//     UNWRAPPED sample; with wrapped phases in (-pi, pi] that is a running count K_i of +-1 jumps (jump when the raw
//     difference leaves [-pi, pi]) and u_i = fl(p_i + 2 pi K_i) -- a prefix sum, done per row by one CTA;
//   * scatter: one thread per time column walks the rows in ascending order (the reference's order of the float
//     additions into a cell), so no atomics and bit-stable results.
#include <math.h>
#include "common.cuh"

namespace {

__device__ __forceinline__ int c_float_to_int(float v) {          // what `int i = v;` gives on the reference's x86 build
    if (!(fabsf(v) < 2147483648.0f)) return (int)0x80000000;       // NaN, +-inf, out of range -> INT_MIN (cvttss2si)
    return (int)v;
}

struct IndexParams {
    int num, n, scaleType;
    float fmin, fmax;              // freArr[0] / samplate, freArr[num-1] / samplate
    float l2min, l2den;            // log2f(fmin), log2f(fmax) - log2f(fmin)
    const float *norm;             // [num] freArr / samplate (mel / bark / erb: nearest band)
};

__device__ __forceinline__ int fre_index(const IndexParams &p, float f) {
    if (p.scaleType == SpectralFilterBankScale_Octave || p.scaleType == SpectralFilterBankScale_Log)
        return c_float_to_int(roundf(__fdiv_rn(__fmul_rn(__fsub_rn(log2f(fabsf(f)), p.l2min), (float)p.num), p.l2den)));
    if (p.scaleType == SpectralFilterBankScale_Linear || p.scaleType == SpectralFilterBankScale_Linspace)
        return c_float_to_int(roundf(__fdiv_rn(__fmul_rn(fabsf(__fsub_rn(f, p.fmin)), (float)p.num), __fsub_rn(p.fmax, p.fmin))));
    // mel / bark / erb: __arr_roundIndex -- the band whose normalised frequency is nearest, -1 outside [arr[0], arr[num-1])
    const float a = fabsf(f);
    if (!(a >= p.norm[0]) || !(a < p.norm[p.num - 1])) return -1;
    int lo = 0, hi = p.num - 1;                                      // arr[lo] <= a < arr[hi]
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (a >= p.norm[mid]) lo = mid; else hi = mid; }
    return (a - p.norm[lo]) < (p.norm[lo + 1] - a) ? lo : lo + 1;
}

// wsst: idx = index(Im(W' / W) / 2 pi)
__global__ void k_wsst_index(const float *wr, const float *wi, const float *dr, const float *di, IndexParams p, int *idx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)p.num * p.n) return;
    const float a = dr[i], b = di[i], c = wr[i], d = wi[i];
    // __complexDiv (src/vector/flux_complex.c): (a + ib) / (c + id), imaginary part (b c - a d) / (c^2 + d^2)
    const float den = __fadd_rn(__fmul_rn(c, c), __fmul_rn(d, d));
    const float im = __fdiv_rn(__fsub_rn(__fmul_rn(b, c), __fmul_rn(a, d)), den);
    idx[i] = fre_index(p, __fdiv_rn(im, 6.283185307179586f));
}

// u = fl(p + 2 pi K): the correction K * 2 pi rounded to double, then the sum (the reference's C expression; no DFMA)
__device__ __forceinline__ float unwrapped(float ph, int K) {
    return (float)__dadd_rn((double)ph, __dmul_rn(6.283185307179586, (double)K));
}

// synsq step 1-3: phase = atan2f(re, im) (the reference's argument order), unwrap along the row, first difference
// (d[0] = 0, last column repeats its neighbour), / 2 pi -> index.  One CTA per row.
constexpr int kUwThreads = 1024;
__global__ void __launch_bounds__(kUwThreads) k_synsq_index(const float *re, const float *im, IndexParams p, int *idx) {
    __shared__ int warpSum[32];
    const int row = blockIdx.x, n = p.n;
    const float *r = re + (size_t)row * n, *q = im + (size_t)row * n;
    int *out = idx + (size_t)row * n;
    const int per = (n + kUwThreads - 1) / kUwThreads;             // consecutive samples per thread
    const int i0 = threadIdx.x * per, i1 = min(n, i0 + per);
    // pass 1: jumps inside the thread's run (relative to its first sample's predecessor)
    int local = 0;
    float prev = i0 > 0 && i0 < n ? atan2f(r[i0 - 1], q[i0 - 1]) : 0.0f;
    for (int i = i0; i < i1; i++) {
        const float ph = atan2f(r[i], q[i]);
        if (i > 0) { const float dlt = __fsub_rn(ph, prev); if (dlt > 3.14159265358979f) local--; else if (dlt < -3.14159265358979f) local++; }
        prev = ph;
    }
    // block-wide exclusive scan of the per-thread jump counts
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    if (lane == 31) warpSum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = warpSum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += v; }
        warpSum[lane] = w;
    }
    __syncthreads();
    int K = inc - local + (warp > 0 ? warpSum[warp - 1] : 0);       // jumps before this thread's run

    // pass 2: unwrapped phase u = fl(p + 2 pi K), difference, index
    float uprev = 0.0f;
    if (i0 > 0 && i0 < n) uprev = unwrapped(atan2f(r[i0 - 1], q[i0 - 1]), K);
    prev = i0 > 0 && i0 < n ? atan2f(r[i0 - 1], q[i0 - 1]) : 0.0f;
    for (int i = i0; i < i1; i++) {
        const float ph = atan2f(r[i], q[i]);
        if (i > 0) { const float dlt = __fsub_rn(ph, prev); if (dlt > 3.14159265358979f) K--; else if (dlt < -3.14159265358979f) K++; }
        const float u = unwrapped(ph, K);
        const float f = __fdiv_rn(i > 0 ? __fsub_rn(u, uprev) : 0.0f, 6.283185307179586f);
        if (i < n - 1 || n == 1) out[i] = fre_index(p, f);
        if (i == n - 2) out[n - 1] = fre_index(p, f);      // last column repeats column n - 2
        prev = ph; uprev = u;
    }
}

// out[idx[i][j]][j] += W[i][j] for rows i ascending, where 0 <= idx < num and |W|^2 > thresh^2
__global__ void k_squeeze_scatter(const float *re, const float *im, const int *idx, int num, int n, float thresh2,
                                  float *outRe, float *outIm) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    for (int i = 0; i < num; i++) {
        const size_t k = (size_t)i * n + j;
        const int t = idx[k];
        const float v1 = re[k], v2 = im[k];
        if (t >= 0 && t < num && __fadd_rn(__fmul_rn(v1, v1), __fmul_rn(v2, v2)) > thresh2) {
            outRe[(size_t)t * n + j] += v1;
            outIm[(size_t)t * n + j] += v2;
        }
    }
}

IndexParams make_index_params(int num, int n, int scaleType, float fre0, float freLast, int samplate, const float *dNorm) {
    IndexParams p;
    p.num = num; p.n = n; p.scaleType = scaleType;
    p.fmin = fre0 / (float)samplate; p.fmax = freLast / (float)samplate;
    p.l2min = log2f(p.fmin); p.l2den = log2f(p.fmax) - log2f(p.fmin);
    p.norm = dNorm;
    return p;
}

}  // namespace

extern "C" int af_launch_wsst_index(const float *wr, const float *wi, const float *dr, const float *di, int num, int n,
                                    int scaleType, float fre0, float freLast, int samplate, const float *dNorm, int *idx,
                                    void *stream) {
    const long long total = (long long)num * n;
    if (total <= 0) return AF_OK;
    k_wsst_index<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        wr, wi, dr, di, make_index_params(num, n, scaleType, fre0, freLast, samplate, dNorm), idx);
    AF_LAUNCH_CHECK("k_wsst_index");
    return AF_OK;
}

extern "C" int af_launch_synsq_index(const float *re, const float *im, int num, int n, int scaleType, float fre0,
                                     float freLast, int samplate, const float *dNorm, int *idx, void *stream) {
    if (num <= 0 || n <= 0) return AF_OK;
    k_synsq_index<<<(unsigned)num, kUwThreads, 0, (cudaStream_t)stream>>>(
        re, im, make_index_params(num, n, scaleType, fre0, freLast, samplate, dNorm), idx);
    AF_LAUNCH_CHECK("k_synsq_index");
    return AF_OK;
}

extern "C" int af_launch_squeeze_scatter(const float *re, const float *im, const int *idx, int num, int n, float thresh,
                                         float *outRe, float *outIm, void *stream) {
    if (num <= 0 || n <= 0) return AF_OK;
    k_squeeze_scatter<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(re, im, idx, num, n, thresh * thresh, outRe, outIm);
    AF_LAUNCH_CHECK("k_squeeze_scatter");
    return AF_OK;
}
