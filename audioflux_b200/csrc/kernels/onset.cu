// onset.cu -- the two onset-specific steps of onsetObj_onset (src/mir/onset_algorithm.c) around the novelty function,
// which k_spectral (spectral.cu) computes.
//
// k_onset_maxfilter: the sliding max over bins of every frame (__mmaxfilter along axis 1, src/vector/flux_vector.c),
// one thread per output, window [k - order/2, k - 1 + order - order/2] clipped to the frame, folded left to right with
// the reference's `max < v` rule.  Max is exact, so the result is bit-identical.
//
// k_onset_pick: one CTA per clip, any number of frames (the clip stays in global memory, where the CTA's own writes
// are visible to it after a barrier):
//   1. min over the clip, then evn -= min and the max of the result, then evn /= max when max > 0 (a true division).
//      The block reductions give the sequential scan's result: a NaN first value is kept, later NaNs are passed over;
//   2. per tile of kThreads frames, each thread tests its frame: evn[i] equal to the max of [i - preMax, i - 1 +
//      postMax] and evn[i] >= mean([i - preAvg, i - 1 + postAvg]) + delta, the mean summed in float from the window's
//      left end and divided by its length, as __vmean does.  Given the same evn the decisions are bit-identical;
//   3. the candidates of the tile, one ballot word per warp, are walked in frame order by thread 0, which applies the
//      greedy `wait` suppression and writes the points;
//   4. the rest of the clip's points row is zeroed and its count stored.
// No product is formed anywhere in the file (sums, differences, one division), so nothing can be contracted into an FMA.
#include "block_reduce.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr unsigned FULL = 0xffffffffu;

__global__ void __launch_bounds__(256) k_onset_maxfilter(const float *__restrict__ in, long long n, int num, int left,
                                                         int right, float *__restrict__ out) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const long long r = e / num;
        const int k = (int)(e - r * num);
        const float *row = in + r * num;
        const int s = k - left >= 0 ? k - left : 0;
        const int t = k - 1 + right <= num - 1 ? k - 1 + right : num - 1;
        float m = __ldg(row + s);
        for (int j = s + 1; j <= t; j++) {
            const float v = __ldg(row + j);
            if (m < v) m = v;
        }
        out[e] = m;
    }
}

__global__ void __launch_bounds__(kThreads) k_onset_pick(const AfOnsetPickArgs a) {
    __shared__ float red[kWarps];
    __shared__ unsigned cand[kWarps];
    __shared__ int sCount;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, T = a.T;
    float *e = a.evn + (size_t)blockIdx.x * T;
    int *pts = a.points + (size_t)blockIdx.x * T;

    // 1. normalisation
    float mn = __int_as_float(0x7f800000);
    for (int i = tid; i < T; i += kThreads) mn = fminf(mn, e[i]);
    mn = block_reduce_float<kWarps>(mn, 0, red);
    const float e0 = e[0];
    if (e0 != e0) mn = e0;
    __syncthreads();                       // every thread has read e[0] before it changes
    float mx = -__int_as_float(0x7f800000);
    for (int i = tid; i < T; i += kThreads) {
        const float v = e[i] - mn;
        e[i] = v;
        mx = fmaxf(mx, v);
    }
    mx = block_reduce_float<kWarps>(mx, 1, red);       // its barriers publish the differences
    const float d0 = e[0];
    if (d0 != d0) mx = d0;
    __syncthreads();                       // every thread has read e[0] before it is divided
    if (mx > 0.f)
        for (int i = tid; i < T; i += kThreads) e[i] = e[i] / mx;
    __syncthreads();

    // 2-3. candidates per tile, then the suppression in frame order
    int pre = -a.wait - 1, count = 0;      // thread 0's
    for (int t0 = 0; t0 < T; t0 += kThreads) {
        const int i = t0 + tid;
        bool c = false;
        if (i < T) {
            const float v = e[i];
            const int s1 = i - a.preMax >= 0 ? i - a.preMax : 0;
            const int t1 = i + a.postMax < T ? i - 1 + a.postMax : T - 1;
            float m = e[s1];
            for (int j = s1 + 1; j <= t1; j++) {
                const float w = e[j];
                if (m < w) m = w;
            }
            if (v == m) {
                const int s2 = i - a.preAvg >= 0 ? i - a.preAvg : 0;
                const int t2 = i + a.postAvg < T ? i - 1 + a.postAvg : T - 1;
                float sum = 0.f;
                for (int j = s2; j <= t2; j++) sum += e[j];
                const float mean = sum / (float)(t2 - s2 + 1);
                c = v >= mean + a.delta;
            }
        }
        const unsigned bal = __ballot_sync(FULL, c);
        if (lane == 0) cand[warp] = bal;
        __syncthreads();
        if (tid == 0) {
            for (int w = 0; w < kWarps; w++) {
                for (unsigned bits = cand[w]; bits; bits &= bits - 1) {
                    const int f = t0 + 32 * w + __ffs(bits) - 1;
                    if (f - pre > a.wait) {
                        pts[count++] = f;
                        pre = f;
                    }
                }
            }
        }
        __syncthreads();                   // cand[] is rewritten by the next tile
    }

    // 4. zeros after the points, and the count
    if (tid == 0) {
        sCount = count;
        a.counts[blockIdx.x] = count;
    }
    __syncthreads();
    for (int i = sCount + tid; i < T; i += kThreads) pts[i] = 0;
}

}  // namespace

extern "C" int af_launch_onset_maxfilter(const float *in, long long rows, int num, int order, float *out, void *stream) {
    if (rows <= 0 || num <= 0) return AF_OK;
    if (order < 1) return af_fail(AF_ERR_ARG, "onset max filter: order %d", order);
    const long long n = rows * num;
    long long blocks = (n + 255) / 256;
    const long long cap = (long long)af_sm_count() * 16;     // grid-stride beyond a few waves
    if (cap > 0 && blocks > cap) blocks = cap;
    k_onset_maxfilter<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(in, n, num, order / 2, order - order / 2, out);
    AF_LAUNCH_CHECK("k_onset_maxfilter");
    return AF_OK;
}

extern "C" int af_launch_onset_pick(const AfOnsetPickArgs *a, void *stream) {
    if (a->clips <= 0 || a->T <= 0) return AF_OK;
    if (a->postMax < 1 || a->postAvg < 1 || a->preMax < 0 || a->preAvg < 0 || a->wait < 0)
        return af_fail(AF_ERR_ARG, "onset peak picking: windows %d/%d, %d/%d, wait %d", a->preMax, a->postMax, a->preAvg,
                       a->postAvg, a->wait);
    k_onset_pick<<<(unsigned)a->clips, kThreads, 0, (cudaStream_t)stream>>>(*a);
    AF_LAUNCH_CHECK("k_onset_pick");
    return AF_OK;
}
