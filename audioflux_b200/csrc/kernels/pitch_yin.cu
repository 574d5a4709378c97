// pitch_yin.cu -- pitch by YIN (sm_90a), replacing the frame loops of pitchYINObj_pitch (src/mir/_pitch_yin.c:350-625),
// which run three n-point FFTs per frame on one core and materialise every intermediate plane.
//
// k_pitch_yin: one CTA per frame, everything in shared memory (n = 2^log2n, nc = n/2, A = autoLength, M = maxIndex):
//   1. the frame x and y[j] = x[A - j] (j <= A, 0 beyond) are read into two n-point real inputs packed as nc complex
//      points each; one thread forms E, the running sum of x^2 over 0 .. A + M, in the reference's sequential float32
//      order;
//   2. both are transformed in place (af_fft_inplace_dif: bit-reversed order); af_real_inverse turns X Y, X and Y read
//      by af_real_bin_brev, into (n/2) c, c = IFFT_n(X Y), written over the packed x; r[k] = c[A + k] for k <= M (no
//      product x[m] x[m + k] wraps there), read by af_real_at and scaled by 2/n exactly;
//   3. e2, d and their 1e-6 clamps (in double, as fabs() compares), then one thread forms the running sum of
//      d[1 .. M] in the reference's order, and yin[k] = d[minIndex + k] / (mean + 1e-16) in double, as C promotes it;
//      e2 and the running sums are where the reference's float32 cancellation lies, so the correlation's rounding is
//      the only difference left;
//   4. the trough flags and the row minimum over contiguous runs of the yin row per thread: the first trough by a
//      block minimum, __vmin's first minimum by __vmax's steps (vmax_take, block_argmax, vmax_first) on -yin, and,
//      when the trough rows are requested, their positions by a block prefix count.  The parabolic offset of a trough
//      is done in double, as C promotes it.
// Only the clips are read from HBM.
//
// Shared memory: 8n bytes for the two packed transforms (later d and the running sums) and 4 (A + M + 1) bytes for E
// (later the yin row), at most 8n + 4n: 96 KB at n = 2^13 and 192 KB at n = 2^14, within the 227 KB a CTA may hold,
// hence AFB200_PITCH_YIN_MAX_EXP = 14.  At the defaults (n = 2^12, A = 2048, M = 1186) it is 45 KB: four CTAs of 384
// threads per SM.
//
// The file is compiled with -fmad=false (Makefile): x^2 and every step of e2, d, the mean and the offsets are rounded
// on their own, as in the reference.
#include <climits>

#include "block_reduce.cuh"
#include "stockham.cuh"

namespace {

constexpr int kMaxThreads = 1024;

struct YinParams {
    const float *data;
    float *fre, *value1, *value2, *mFre, *mTrough;
    int *lens;
    const float2 *tw;              // af_twiddle_table(log2n - 1), or null at n = 2
    int nc, log2nc, A, minIndex, M, Y, mLen, samplate, dataLength, hop, T;
    float thresh;
};

// the reference's clamp: fabs(v) >= 1e-6, a double comparison
__device__ __forceinline__ float clamp_small(float v) { return fabs((double)v) >= 1e-6 ? v : 0.0f; }

// :546-572
__device__ __forceinline__ bool is_trough(const float *y, int k, int Y, float th) {
    if (k >= Y - 1) return false;
    if (k == 0) return y[0] < y[1] && y[0] < th;
    return y[k] <= y[k + 1] && y[k] < y[k - 1] && y[k] < th;
}

// samplate / (minIndex + k + offset[k]), offset of __pitchYINObj_calInterp (:485-501)
__device__ __forceinline__ float trough_fre(const YinParams &p, const float *y, int k) {
    float off = 0.0f;
    if (k >= 1 && k <= p.Y - 2) {
        const float v1 = y[k - 1], v2 = y[k], v3 = y[k + 1];
        const float num = (v3 - v1) / 2.0f, den = (v1 + v3 - 2.0f * v2) / 2.0f;
        const float o = (float)((double)(-num) / ((double)(2.0f * den) + 1e-16));
        off = fabsf(o) <= 1.0f ? o : 0.0f;
    }
    return (float)p.samplate / ((float)(p.minIndex + k) + off);
}

// out[j] = in[0] + .. + in[j] (of in[i]^2 when squares), j < len, one float32 add after another as in the reference.
// One thread.  The loads of each run of kRun values are issued before its adds and stores: the compiler cannot move a
// shared-memory load above a store it may alias, so a plain loop would wait out the load latency at every step.
constexpr int kRun = 12;
__device__ __forceinline__ void running_sum(const float *in, int len, float *out, bool squares) {
    float s = 0.0f;
    for (int j0 = 0; j0 < len; j0 += kRun) {
        float v[kRun];
#pragma unroll
        for (int i = 0; i < kRun; i++) v[i] = in[min(j0 + i, len - 1)];
#pragma unroll
        for (int i = 0; i < kRun; i++) {
            if (j0 + i >= len) break;
            s = j0 + i ? s + (squares ? v[i] * v[i] : v[i]) : (squares ? v[i] * v[i] : v[i]);
            out[j0 + i] = s;
        }
    }
}

// exclusive prefix sum of v over the block in thread order, and the total.  red: 32 ints
__device__ int block_excl_scan(int v, int *red, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    __syncthreads();
    if (lane == 31) red[warp] = incl;
    __syncthreads();
    int base = 0, sum = 0;
    for (int w = 0; w < nw; w++) {
        if (w < warp) base += red[w];
        sum += red[w];
    }
    *total = sum;
    return base + incl - v;
}

__global__ void __launch_bounds__(kMaxThreads) k_pitch_yin(YinParams p) {
    extern __shared__ float2 smem[];
    __shared__ float redv[32];
    __shared__ int redi[32];
    const int nc = p.nc, n = 2 * nc, tid = threadIdx.x, bd = blockDim.x, A = p.A, M = p.M, Y = p.Y;
    float2 *X = smem, *Yc = smem + nc;                                 // packed x and packed y
    float *xs = reinterpret_cast<float *>(X), *ys = reinterpret_cast<float *>(Yc);
    float *E = reinterpret_cast<float *>(smem + n);                    // A + M + 1 energies, then the yin row
    const long long f = blockIdx.x, clip = f / p.T, t = f - clip * p.T;
    const float *x = p.data + clip * p.dataLength + t * p.hop;

    for (int j = tid; j < n; j += bd) {
        const float v = __ldg(x + j);
        xs[j] = v;
        if (j <= A) ys[A - j] = v;
        else ys[j] = 0.0f;
    }
    __syncthreads();
    if (tid == 0) running_sum(xs, A + M + 1, E, true);               // :388-398
    __syncthreads();

    af_fft_inplace_dif(X, nc, p.tw);
    af_fft_inplace_dif(Yc, nc, p.tw);
    af_real_inverse(X, nc, p.log2nc, p.tw, [&](int k) {
        return af_cmul(af_real_bin_brev(X, p.tw, k, nc, p.log2nc), af_real_bin_brev(Yc, p.tw, k, nc, p.log2nc));
    });

    const float inv = 1.0f / (float)nc;                               // the unscaled chain gives nc c; exact
    const float e0 = clamp_small(E[A] - E[0]);
    for (int j = tid; j <= M; j += bd)                                 // :375-415
        ys[j] = e0 + clamp_small(E[A + j] - E[j]) - 2.0f * clamp_small(af_real_at(X, A + j) * inv);
    __syncthreads();
    if (tid == 0) running_sum(ys + 1, M, xs, false);                  // :426-436, the sums of d[1 .. k+1]
    __syncthreads();
    float *yin = E;
    for (int k = tid; k < Y; k += bd) {                                // :438-453
        const float mean = xs[p.minIndex - 1 + k] / (float)(p.minIndex + k);
        yin[k] = (float)((double)ys[p.minIndex + k] / ((double)mean + 1e-16));
    }
    __syncthreads();

    // contiguous runs of the row per thread, so that a thread meets its indices in order
    const int per = (Y + bd - 1) / bd, k0 = min(Y, tid * per), k1 = min(Y, k0 + per);
    const float th = p.thresh;
    int first = INT_MAX, count = 0;
    float bv = 0.0f;
    int bi = -1;
    for (int k = k0; k < k1; k++) {
        if (is_trough(yin, k, Y, th)) {
            if (first == INT_MAX) first = k;
            count++;
        }
        vmax_take(-yin[k], k, bv, bi);
    }
    first = block_reduce_int(first, false, redi);
    if (p.value2) bi = block_argmax(bv, bi, redv, redi);
    if (tid == 0) {
        if (first < Y) {
            p.fre[f] = trough_fre(p, yin, first);
            if (p.value1) p.value1[f] = yin[first];
        }
        if (p.value2) p.value2[f] = yin[vmax_first(bi, yin[0], 0)];                    // __vmin
    }
    if (p.mFre || p.mTrough || p.lens) {                               // :585-625
        int total;
        int pos = block_excl_scan(count, redi, &total);
        const size_t row = (size_t)f * p.mLen;
        for (int k = k0; k < k1 && count; k++) {
            if (!is_trough(yin, k, Y, th)) continue;
            if (p.mTrough) p.mTrough[row + pos] = yin[k];
            if (p.mFre) p.mFre[row + pos] = trough_fre(p, yin, k);
            pos++;
        }
        for (int i = total + tid; i < p.mLen; i += bd) {
            if (p.mTrough) p.mTrough[row + i] = 0.0f;
            if (p.mFre) p.mFre[row + i] = 0.0f;
        }
        if (p.lens && tid == 0) p.lens[f] = total;
    }
}

}  // namespace

extern "C" int af_launch_pitch_yin(const AfPitchYinArgs *a, void *stream) {
    if (a->log2n < 1 || a->log2n > AFB200_PITCH_YIN_MAX_EXP)
        return af_fail(AF_ERR_UNSUPPORTED, "pitch YIN: frame 2^%d; frames 2^1 .. 2^%d", a->log2n, AFB200_PITCH_YIN_MAX_EXP);
    const int n = 1 << a->log2n;
    if (a->autoLength < 0 || a->minIndex < 1 || a->maxIndex < a->minIndex || a->maxIndex > n - 1 - a->autoLength)
        return af_fail(AF_ERR_ARG, "pitch YIN: autoLength %d, lags %d .. %d", a->autoLength, a->minIndex, a->maxIndex);
    if (!a->fre) return af_fail(AF_ERR_ARG, "pitch YIN: no frequency output");
    const long long frames = (long long)a->batch * a->timeLength;
    if (frames <= 0) return AF_OK;
    if (frames > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "pitch YIN: too many frames in one launch");
    YinParams p;
    p.data = a->data; p.fre = a->fre; p.value1 = a->value1; p.value2 = a->value2; p.mFre = a->mFre;
    p.mTrough = a->mTrough; p.lens = a->lens;
    p.nc = n / 2; p.log2nc = a->log2n - 1; p.A = a->autoLength; p.minIndex = a->minIndex; p.M = a->maxIndex;
    p.Y = a->maxIndex - a->minIndex + 1; p.mLen = p.Y / 2 + 1; p.samplate = a->samplate;
    p.dataLength = a->dataLength; p.hop = a->hop; p.T = a->timeLength; p.thresh = a->thresh;
    p.tw = p.log2nc ? af_twiddle_table(p.log2nc) : nullptr;
    if (p.log2nc && !p.tw) return af_fail(AF_ERR_CUDA, "pitch YIN: twiddle table 2^%d", p.log2nc);
    const size_t smem = sizeof(float2) * (size_t)n + sizeof(float) * (size_t)(a->autoLength + a->maxIndex + 1);
    // as many threads as the CTAs that fit an SM's 228 KB of shared memory (1 KB each reserved) leave of the 1536 its
    // registers hold at the kernel's 40-register budget, and no more than one per butterfly: the two sequential scans
    // of a CTA then overlap the other CTAs' transforms
    const int fit = (int)((228u * 1024u) / (smem + 1024u)), want = (1536 / (fit > 1 ? fit : 1)) & ~31;
    const int threads = af_cta_threads(want, af_cta_threads(p.nc / 2, kMaxThreads));
    const int rc = af_smem_optin(k_pitch_yin, smem, "k_pitch_yin");
    if (rc) return rc;
    k_pitch_yin<<<(unsigned)frames, threads, smem, (cudaStream_t)stream>>>(p);
    AF_LAUNCH_CHECK("k_pitch_yin");
    return AF_OK;
}
