// harmonic_ratio.cu -- the harmonic ratio (sm_90a), replacing the frame loop of harmonicRatioObj_harmonicRatio
// (src/mir/harmonicRatio_algorithm.c:172-287), which runs two 2W-point FFTs and five passes per frame on one core.
//
// k_harmonic_ratio: one CTA per frame.  With W the window and N = 2W:
//   1. the windowed frame is read coalesced into the first half of an N-point real input packed as W complex points
//      (the second half is the zero padding), Stockham transform in shared memory (stockham.cuh, twiddles from
//      af_twiddle_table) and the real-FFT post-pass;
//   2. P[k] = re^2 + im^2, written as the real even sequence P[k] = P[N-k] into the free buffer; r = FFT_N(P) / N is
//      Re IFFT_N(P), the reference's autocorrelation with its 1/N (:242-246).  r[0 .. maxLength] is kept;
//   3. the prefix sums of x^2 (a block scan; the reference sums sequentially, :249-256);
//   4. the crossing: the first j in 2 .. maxLength where r[j], r[j-1] change sign, zeros included (a block minimum);
//      minIndex = j - 1 (:259-266);
//   5. g[k] = r[j] / sqrtf(r[0] E[j] + 1e-16) with the sum in double (:270-273), its first arg-max (__vmax: vmax_take,
//      block_argmax, vmax_first) and the parabolic refinement in double (util_qaudInterp, :277-285).
// The minIndex of a frame without a crossing is the last one an earlier frame of the same call found (it lives outside
// the reference's frame loop).  That is the only coupling between frames, and it stays out of this pass: every frame
// stores its crossing (-1 for none) in minIdx, and only frames with one store their value.
//
// k_harmonic_ratio_carry: a grid-stride pass over the frames without a crossing.  Each takes the index of the last
// earlier frame of its clip that has one (0 when none; the reference starts every call at 0) and computes steps 1-5 with
// it.  No CTA waits on another: the indices come from the previous launch.
//
// The file is compiled with -fmad=false (Makefile): every float step is rounded on its own, as in the reference.
#include <climits>

#include "block_reduce.cuh"
#include "stockham.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kMaxThreads = 1024;

struct HrParams {
    const float *data, *window;
    float *value;
    int *minIdx;
    const float2 *tw;              // af_twiddle_table(log2w): W-point butterflies and the 2W-point post-pass
    long long frames;
    int w, log2w, maxLength, dataLength, hop, T;
};

// in-place inclusive prefix sum of s[0 .. n): each thread sums a run of consecutive values, then the runs are offset
__device__ void block_scan(float *s, int n, float *redv) {
    const int bd = blockDim.x, c = (n + bd - 1) / bd, lo = min(n, (int)threadIdx.x * c), hi = min(n, lo + c);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = bd >> 5;
    float run = 0.f;
    for (int i = lo; i < hi; i++) run += s[i];
    float incl = run;
    for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += u;
    }
    if (lane == 31) redv[warp] = incl;
    __syncthreads();
    float acc = incl - run;                                            // exclusive within the warp
    float before = 0.f;
    for (int k = 0; k < warp && k < nw; k++) before += redv[k];
    acc += before;
    for (int i = lo; i < hi; i++) { acc += s[i]; s[i] = acc; }
    __syncthreads();
}

// util_qaudInterp (src/util/flux_util.c): its 1e-16 and 0.25 make the arithmetic double
__device__ __forceinline__ float qaud_interp(float v1, float v2, float v3) {
    const float pp = (float)((double)(v3 - v1) / ((double)(2.0f * (2.0f * v2 - v3 - v1)) + 1e-16));
    return (float)((double)v2 - 0.25 * (double)(v1 - v3) * (double)pp);
}

// the value of frame f with minIndex m (m < 0: the frame's own crossing, stored in minIdx[f]; no value without one).
// A and B: W float2 each.  Every thread of the block calls it.
__device__ void hr_frame(const HrParams &p, long long f, int m, float2 *A, float2 *B, float *redv, int *redi) {
    const int W = p.w, n = 2 * W, L = p.maxLength, tid = threadIdx.x, bd = blockDim.x;
    const long long clip = f / p.T, t = f - clip * p.T;
    const float *x = p.data + clip * p.dataLength + t * p.hop;
    float *a = reinterpret_cast<float *>(A);
    for (int j = tid; j < n; j += bd) a[j] = j < W ? __ldg(x + j) * __ldg(p.window + j) : 0.0f;
    __syncthreads();
    const float2 *X = af_stockham(A, B, W, p.log2w, p.tw);
    float2 *P = X == A ? B : A;
    for (int k = tid; k <= W; k += bd) {
        const float2 z = af_real_bin(X, __ldg(p.tw + W + k), k, W);          // exp(-2 pi i k / 2W)
        af_put_even(reinterpret_cast<float *>(P), n, k, z.x * z.x + z.y * z.y);
    }
    __syncthreads();
    const float2 *Y = af_stockham(P, P == A ? B : A, W, p.log2w, p.tw);
    float *const r = reinterpret_cast<float *>(Y == A ? B : A);       // r[0 .. L]; the prefix sums E behind it
    float *const E = r + W;
    const float inv = 1.0f / (float)n;
    for (int k = tid; k <= L; k += bd) r[k] = af_real_bin(Y, __ldg(p.tw + W + k), k, W).x * inv;
    for (int j = tid; j < W; j += bd) {
        const float v = __ldg(x + j) * __ldg(p.window + j);
        E[j] = v * v;
    }
    __syncthreads();
    block_scan(E, W, redv);

    if (m < 0) {                                                       // the frame's own crossing
        int jm = INT_MAX;
        for (int j = 2 + tid; j <= L; j += bd) {
            const float r1 = r[j], r0 = r[j - 1];
            if ((r1 >= 0.f && r0 <= 0.f) || (r1 <= 0.f && r0 >= 0.f)) { jm = j; break; }
        }
        jm = block_reduce_int(jm, false, redi);
        m = jm == INT_MAX ? -1 : jm - 1;
        if (tid == 0) p.minIdx[f] = m;
        if (m < 0) return;                                             // block-uniform: the carry pass computes it
    }

    const float r0 = r[0];
    auto gamma = [&](int j) { return r[j] / sqrtf((float)((double)(r0 * E[W - 2 - j]) + 1e-16)); };
    const int len = L - m - 1;                                         // g[k] = gamma(m + 1 + k), k < len
    float bv = 0.f;
    int bi = -1;
    for (int k = tid; k < len; k += bd) vmax_take(gamma(m + 1 + k), k, bv, bi);
    bi = block_argmax(bv, bi, redv, redi);
    if (tid == 0) {
        float v = 0.0f;                                                // len 0: __vmax leaves the value at 0
        if (len > 0) {
            const int k = vmax_first(bi, gamma(m + 1), 0);
            const float g = gamma(m + 1 + k);
            v = k == 0 || k == len - 1 ? g : qaud_interp(gamma(m + k), g, gamma(m + 2 + k));
        }
        p.value[f] = v;
    }
}

__global__ void __launch_bounds__(kMaxThreads) k_harmonic_ratio(HrParams p) {
    extern __shared__ float2 smem[];
    __shared__ float redv[32];
    __shared__ int redi[32];
    hr_frame(p, blockIdx.x, -1, smem, smem + p.w, redv, redi);
}

__global__ void __launch_bounds__(kMaxThreads) k_harmonic_ratio_carry(HrParams p) {
    extern __shared__ float2 smem[];
    __shared__ float redv[32];
    __shared__ int redi[32];
    __shared__ int list[kMaxThreads];
    __shared__ int count;
    const int tid = threadIdx.x, bd = blockDim.x;
    const long long G = gridDim.x;
    for (long long k0 = 0; blockIdx.x + k0 * G < p.frames; k0 += bd) {
        // this CTA's frames blockIdx.x + k G, k0 <= k < k0 + bd: those without a crossing, listed in any order
        if (tid == 0) count = 0;
        __syncthreads();
        const long long f = blockIdx.x + (k0 + tid) * G;
        if (f < p.frames && __ldg(p.minIdx + f) < 0) list[atomicAdd(&count, 1)] = tid;
        __syncthreads();
        const int nl = count;
        for (int q = 0; q < nl; q++) {
            const long long g = blockIdx.x + (k0 + list[q]) * G;
            const long long clip = g / p.T;
            const int t = (int)(g - clip * p.T);
            const int *row = p.minIdx + clip * p.T;
            int m = 0;
            for (int t0 = t - 1; t0 >= 0; t0 -= bd) {                  // the last earlier frame with a crossing
                const int u = t0 - tid;
                const int hit = block_reduce_int(u >= 0 && __ldg(row + u) >= 0 ? u : -1, true, redi);
                if (hit >= 0) { m = __ldg(row + hit); break; }
            }
            hr_frame(p, g, m, smem, smem + p.w, redv, redi);
            __syncthreads();                                           // the buffers are free for the next frame
        }
        __syncthreads();                                               // count and list are rewritten next
    }
}

}  // namespace

extern "C" int af_launch_harmonic_ratio(const AfHarmonicRatioArgs *a, void *stream) {
    if (a->log2w < 1 || a->log2w > AFB200_HARMONIC_RATIO_MAX_EXP)
        return af_fail(AF_ERR_UNSUPPORTED, "harmonic ratio: window 2^%d; 2^1 .. 2^%d are supported", a->log2w,
                       AFB200_HARMONIC_RATIO_MAX_EXP);
    const int W = 1 << a->log2w;
    if (a->maxLength < 1 || a->maxLength > W - 1)
        return af_fail(AF_ERR_ARG, "harmonic ratio: maxLength=%d; 1 .. %d", a->maxLength, W - 1);
    HrParams p;
    p.data = a->data; p.window = a->window; p.value = a->value; p.minIdx = a->minIdx;
    p.frames = (long long)a->batch * a->timeLength;
    if (p.frames <= 0) return AF_OK;
    if (p.frames > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "harmonic ratio: too many frames in one launch");
    p.tw = af_twiddle_table(a->log2w);
    if (!p.tw) return af_fail(AF_ERR_CUDA, "harmonic ratio: twiddle table 2^%d", a->log2w);
    p.w = W; p.log2w = a->log2w; p.maxLength = a->maxLength;
    p.dataLength = a->dataLength; p.hop = a->hop; p.T = a->timeLength;
    const int threads = af_cta_threads(W / 4, kMaxThreads);
    const size_t smem = sizeof(float2) * 2 * (size_t)W;
    int rc;
    if ((rc = af_smem_optin(k_harmonic_ratio, smem, "k_harmonic_ratio")) ||
        (rc = af_smem_optin(k_harmonic_ratio_carry, smem, "k_harmonic_ratio_carry")))
        return rc;
    cudaStream_t st = (cudaStream_t)stream;
    k_harmonic_ratio<<<(unsigned)p.frames, threads, smem, st>>>(p);
    AF_LAUNCH_CHECK("k_harmonic_ratio");
    int perSm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, k_harmonic_ratio_carry, threads, smem);
    if (e != cudaSuccess) return af_cuda_check(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor(k_harmonic_ratio_carry)");
    long long grid = (long long)af_sm_count() * (perSm > 0 ? perSm : 1);
    if (grid < 1) grid = 1;
    if (grid > p.frames) grid = p.frames;
    k_harmonic_ratio_carry<<<(unsigned)grid, threads, smem, st>>>(p);
    AF_LAUNCH_CHECK("k_harmonic_ratio_carry");
    return AF_OK;
}
