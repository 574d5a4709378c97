// resample.cu -- the resampler (sm_90a), replacing the per-output loop of _resampleObj_resample
// (src/dsp/resample_algorithm.c:430-521) for a batch of clips in one launch.
//
// k_resample: one CTA per tile of consecutive outputs of one clip (grid = tiles x clips, flattened).  Per output i the
// index arithmetic is the reference's, in its types and rounding: t = (float)((double)i / ratio), n = floorf(t), the
// left phase scale * (t - n) and the right phase scale - left, each split into a table offset and a fraction `delta`;
// tap counts min(n + 1, (L - offset) / step) and min(srcLen - n - 1, (L - offset) / step) by integer division.  A weight
// is a[o] + delta * (a[o+1] - a[o]): the reference's difference table (:523-544) recomputed bit for bit, with a copy of
// the last entry appended so that the last difference is 0.  Each sum runs left taps then right taps, in order, from the
// caller's value (legacy call) or 0; the file is compiled with -fmad=false so that no multiply-add is contracted.
//
// Shared memory holds the table (L + 1 floats) when it is at most kTableSmemMax bytes (every preset: Best is 128 KB) and
// the source span of the tile, from n_first - K + 1 to n_last + K with K = L / step the most taps a side can have.  The
// tile length is chosen on the host so that the span fits; a tile whose span does not fit (a ratio near 2^-nbit, where K
// reaches L, or float positions above 2^24 that land further apart than estimated) reads its source from global memory
// instead, and a table that does not fit is read from global memory through L1.
#include "common.cuh"

namespace {

constexpr int kThreads = 1024;
constexpr int kOutPerThread = 4;                      // outputs per thread of a full tile
constexpr size_t kTableSmemMax = 160 * 1024;

struct RsParams {
    const float *data, *table;                        // table: L + 1 floats (the last entry repeated)
    float *out;
    long long inLen, srcLen;
    int outLen, tableLength, bitLength, step, K;
    float ratio, scale, scaleDiv;
    int accumulate, tile, tiles, spanCap;
};

__device__ __forceinline__ float position(long long i, float ratio) {
    return __double2float_rn((double)i / (double)ratio);                    // :483, t = i*1.0/ratio stored in a float
}

// one output; sample g of the clip is x[g - base] (kSrcSmem: the staged span, zeros beyond the clip) or x[g] (global)
template <bool kSrcSmem>
__device__ __forceinline__ float one_output(const RsParams &p, const float *__restrict__ a, const float *__restrict__ x,
                                            long long base, int i, float acc) {
    const float t = position(i, p.ratio);
    const int n = (int)floorf(t);
    const float bits = (float)p.bitLength;
    float factor = p.scale * (t - (float)n);                                 // :487-495
    float fv = factor * bits;
    int off = (int)floorf(fv);
    float delta = fv - (float)off;
    int len = min(n + 1, (p.tableLength - off) / p.step);
    for (int j = 0; j < len; j++) {
        const int o = off + j * p.step;
        const float a0 = a[o], w = a0 + delta * (a[o + 1] - a0);
        const long long g = (long long)n - j;
        float xv;
        if (kSrcSmem) xv = x[g - base];
        else xv = g < p.inLen ? __ldg(x + g) : 0.0f;
        acc = acc + w * xv;
    }
    factor = p.scale - factor;                                               // :503-515
    fv = factor * bits;
    off = (int)floorf(fv);
    delta = fv - (float)off;
    len = (int)min(p.srcLen - n - 1, (long long)((p.tableLength - off) / p.step));
    for (int j = 0; j < len; j++) {
        const int o = off + j * p.step;
        const float a0 = a[o], w = a0 + delta * (a[o + 1] - a0);
        const long long g = (long long)n + j + 1;
        const float xv = kSrcSmem ? x[g - base] : __ldg(x + g);
        acc = acc + w * xv;
    }
    return acc;
}

template <bool kTableSmem>
__global__ void __launch_bounds__(kThreads) k_resample(RsParams p) {
    extern __shared__ float smem[];
    const int clip = blockIdx.x / p.tiles, tile = blockIdx.x % p.tiles;
    const int i0 = tile * p.tile, i1 = (int)min((long long)p.outLen, (long long)i0 + p.tile);
    const float *x = p.data + (size_t)clip * (size_t)p.inLen;
    float *out = p.out + (size_t)clip * (size_t)p.outLen;
    float *xs = smem + (kTableSmem ? p.tableLength + 1 : 0);
    if (kTableSmem)
        for (int k = threadIdx.x; k <= p.tableLength; k += blockDim.x) smem[k] = __ldg(p.table + k);
    const float *a = kTableSmem ? smem : p.table;

    // the source samples the tile's taps touch: left taps reach n_first - K + 1, right taps n_last + K (< srcLen)
    const long long nFirst = (long long)floorf(position(i0, p.ratio)), nLast = (long long)floorf(position(i1 - 1, p.ratio));
    const long long lo = max(0LL, nFirst - p.K + 1);
    const long long hi = max(nLast, min(nLast + p.K, p.srcLen - 1));
    const bool staged = hi - lo + 1 <= p.spanCap;
    if (staged)
        for (long long g = lo + threadIdx.x; g <= hi; g += blockDim.x) xs[g - lo] = g < p.inLen ? __ldg(x + g) : 0.0f;
    __syncthreads();

    for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
        float acc = p.accumulate ? out[i] : 0.0f;                            // :498, dataArr2[i] += ...
        acc = staged ? one_output<true>(p, a, xs, lo, i, acc) : one_output<false>(p, a, x, 0, i, acc);
        if (p.scaleDiv != 0.0f) acc = acc / p.scaleDiv;                      // :387-396
        out[i] = acc;
    }
}

template <bool kTableSmem>
int launch(const RsParams &p, unsigned grid, size_t smem, cudaStream_t st) {
    const int rc = af_smem_optin(k_resample<kTableSmem>, smem, "k_resample");
    if (rc) return rc;
    k_resample<kTableSmem><<<grid, kThreads, smem, st>>>(p);
    AF_LAUNCH_CHECK("k_resample");
    return AF_OK;
}

}  // namespace

extern "C" int af_launch_resample(const AfResampleArgs *a, void *stream) {
    if (a->batch <= 0 || a->outLen <= 0) return AF_OK;
    if (a->step <= 0 || a->tableLength < 2 || a->inLen <= 0 || a->srcLen > a->inLen || !a->table)
        return af_fail(AF_ERR_ARG, "resample: step=%d, table %d, lengths %d / %d", a->step, a->tableLength, a->srcLen,
                       a->inLen);
    int dev = 0, optin = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    RsParams p;
    p.data = a->data; p.table = a->table; p.out = a->out;
    p.inLen = a->inLen; p.srcLen = a->srcLen; p.outLen = a->outLen;
    p.tableLength = a->tableLength; p.bitLength = a->bitLength; p.step = a->step; p.K = a->tableLength / a->step;
    p.ratio = a->ratio; p.scale = a->scale; p.scaleDiv = a->scaleDiv; p.accumulate = a->accumulate;

    const size_t tabBytes = sizeof(float) * ((size_t)a->tableLength + 1);
    const bool tabSmem = tabBytes <= kTableSmemMax && (int)tabBytes < optin;
    const long long capFloats = ((long long)optin - (tabSmem ? (long long)tabBytes : 0)) / (long long)sizeof(float);
    // source samples of a tile of T outputs: (T - 1) / ratio apart at most, plus both tap reaches, plus the rounding of the
    // float positions (half an ulp of t at each end, an ulp being 2^-23 t)
    const double tmax = (double)a->outLen / (double)a->ratio;
    const long long slack = 2 * ((long long)ceil(tmax * 0x1p-23) + 2);
    auto span = [&](long long T) { return (long long)ceil((double)(T - 1) / (double)a->ratio) + 2LL * p.K + slack; };
    long long T = (long long)kThreads * kOutPerThread;
    while (T > kThreads && span(T) > capFloats) T /= 2;
    while (T > kThreads && ((a->outLen + T - 1) / T) * (long long)a->batch < 2LL * sms) T /= 2;
    const long long need = span(T) < (long long)a->srcLen + 1 ? span(T) : (long long)a->srcLen + 1;
    p.spanCap = need <= capFloats ? (int)need : 0;                            // 0: every tile reads global memory
    p.tile = (int)T;
    p.tiles = (int)((a->outLen + T - 1) / T);
    const long long grid = (long long)p.tiles * a->batch;
    if (grid > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "resample: too many tiles in one launch");
    const size_t smem = (tabSmem ? tabBytes : 0) + sizeof(float) * (size_t)p.spanCap;
    cudaStream_t st = (cudaStream_t)stream;
    return tabSmem ? launch<true>(p, (unsigned)grid, smem, st) : launch<false>(p, (unsigned)grid, smem, st);
}
