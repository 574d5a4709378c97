// st.cu -- the Stockwell transforms (sm_90a).
//
// ST (replaces the loop of stObj_st, src/st_algorithm.c:188-207).  The clip's spectrum X comes from af_launch_stft (FULL
// planes, one frame per clip).  Row r of bin i != 0 is IFFT_N(X[(m + i) mod N] * G_i[m]) with the Gaussian
// G_i[m] = expf(v m^2) + expf(v (m - N)^2) evaluated in registers in the reference's float order (_stObj_initWinData,
// :211-256: m^2 a float product, the product with v before expf); v comes per row from the host.
//   k_st_rows   one CTA per (group of rows, clip): a group is one row, or for N <= 256 several rows one after the other.
//               The shifted spectrum is gathered through L2, the inverse transform is conj o forward FFT o conj in shared
//               memory (two Stockham buffers up to 8192 points, the one-buffer in-place passes at 16384) scaled by 1/N,
//               and the row is stored once, coalesced.  Bin 0 is the clip's mean (a block reduction) and a zero row.
// FST (replaces fstObj_fst, src/fst_algorithm.c:113-280).  Only the right half of the dyadic partition is ever shown
// (row f reads partition position N/2 - 1 + f), so only its segments are computed: the three single points at N/2 - 1,
// N/2, N/2 + 1 and the segments of 2^t points starting at N/2 + 2^t, t = 1 .. log2N - 2.
//   k_fst_segments  one CTA per (segment, clip): fftshift(ifft(ifftshift(seg))) * sqrt(len) of the centred spectrum
//                   (ifftshift(x) -> (-1)^k on the spectrum, fftshift -> an index offset, times 1/sqrt(N)), in shared
//                   memory; writes the clip's N/2+1 partition values.
//   k_fst_expand    one CTA per (column tile, chunk of rows, clip): each thread holds four columns, reloads their
//                   partition values only when the row's segment changes, and stores them to every row of the chunk
//                   with 16-byte stores (streaming when the output is larger than L2).  Bounded by the HBM writes.
#include <stdint.h>
#include "common.cuh"
#include "stockham.cuh"

namespace {

struct StParams {
    const float *data, *specRe, *specIm, *v;
    const int *bins;
    float *outRe, *outIm;
    const float2 *tw;
    int rows, n, log2n, rowsPerCta, groups;
};

// mean of the clip's n samples, in double, broadcast to every thread; `red` is shared scratch of >= 32 doubles
__device__ double clip_mean(const float *x, int n, double *red) {
    double s = 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += (double)x[j];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const int warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    if ((threadIdx.x & 31) == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        double t = threadIdx.x < nw ? red[threadIdx.x] : 0.0;
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (threadIdx.x == 0) red[0] = t / n;
    }
    __syncthreads();
    const double m = red[0];
    __syncthreads();
    return m;
}

template <bool kInplace>
__global__ void __launch_bounds__(1024) k_st_rows(StParams p) {
    extern __shared__ float2 smem[];
    const int n = p.n;
    const int clip = blockIdx.x / p.groups, g = blockIdx.x % p.groups;
    const float *xr = p.specRe + (size_t)clip * n, *xi = p.specIm + (size_t)clip * n;
    const float inv = 1.0f / (float)n;
    const int r1 = min(p.rows, (g + 1) * p.rowsPerCta);
    for (int r = g * p.rowsPerCta; r < r1; r++) {
        const size_t row = ((size_t)clip * p.rows + r) * n;
        const int bin = __ldg(p.bins + r);
        if (bin == 0) {                                            // :199-206
            const float mean = (float)clip_mean(p.data + (size_t)clip * n, n, reinterpret_cast<double *>(smem));
            for (int j = threadIdx.x; j < n; j += blockDim.x) { p.outRe[row + j] = mean; p.outIm[row + j] = 0.0f; }
            continue;
        }
        const float v = __ldg(p.v + r);
        float2 *a = smem, *b = smem + n;
        for (int m = threadIdx.x; m < n; m += blockDim.x) {
            const int k = (m + bin) & (n - 1);
            const float m1 = (float)m, m2 = (float)(m - n);
            const float gw = expf(m1 * m1 * v) + expf(m2 * m2 * v);
            a[m] = make_float2(__ldg(xr + k) * gw, -(__ldg(xi + k) * gw));      // conj of the windowed spectrum
        }
        __syncthreads();
        if (kInplace) {
            af_fft_inplace_dif(a, n, p.tw);
            for (int j = threadIdx.x; j < n; j += blockDim.x) {
                const float2 y = a[af_brev(j, p.log2n)];
                p.outRe[row + j] = y.x * inv;
                p.outIm[row + j] = -y.y * inv;
            }
        } else {
            const float2 *y = af_stockham(a, b, n, p.log2n, p.tw);
            for (int j = threadIdx.x; j < n; j += blockDim.x) {
                const float2 t = y[j];
                p.outRe[row + j] = t.x * inv;
                p.outIm[row + j] = -t.y * inv;
            }
        }
        __syncthreads();                                           // the buffers are free for the next row
    }
}

struct FstParams {
    const float *specRe, *specIm;
    float2 *part;
    const float2 *tw[14];          // Stockham twiddles by log2 of the segment length
    float norm;                    // 1/sqrtf(N), fstObj_new (:88)
    int n, log2n, segs;
};

// partition position c (0 .. N/2) = centred-spectrum position N/2 - 1 + c: the FFT of ifftshift(x) is (-1)^k X[k], and
// the fftshift puts bin k = c - 1 there (bin -1 = conj X[1], from the half spectrum)
__device__ __forceinline__ float2 fst_centred(const FstParams &p, const float *re, const float *im, int c) {
    const int k = c - 1;
    float r, i;
    if (k < 0) { r = -__ldg(re + 1); i = __ldg(im + 1); }        // (-1)^(N-1) conj X[1]
    else if (k & 1) { r = -__ldg(re + k); i = -__ldg(im + k); }
    else { r = __ldg(re + k); i = __ldg(im + k); }
    return make_float2(r * p.norm, i * p.norm);
}

__global__ void __launch_bounds__(256) k_fst_segments(FstParams p) {
    extern __shared__ float2 smem[];
    const int s = blockIdx.x % p.segs, clip = blockIdx.x / p.segs;
    const int width = p.n / 2 + 1;
    const float *re = p.specRe + (size_t)clip * width, *im = p.specIm + (size_t)clip * width;
    float2 *out = p.part + (size_t)clip * width;
    if (s == 0) {                                                  // the single points at N/2 - 1, N/2, N/2 + 1
        if (threadIdx.x < 3) out[threadIdx.x] = fst_centred(p, re, im, threadIdx.x);
        return;
    }
    const int len = 1 << s, off = len + 1, h = len / 2;
    float2 *a = smem, *b = smem + len;
    for (int j = threadIdx.x; j < len; j += blockDim.x) {          // ifftshift, conj in
        const float2 z = fst_centred(p, re, im, off + ((j + h) & (len - 1)));
        a[j] = make_float2(z.x, -z.y);
    }
    __syncthreads();
    const float2 *y = af_stockham(a, b, len, s, p.tw[s]);
    const float inv = 1.0f / (float)len, g = sqrtf((float)len);
    for (int j = threadIdx.x; j < len; j += blockDim.x) {          // conj out, 1/len, * sqrt(len), fftshift
        const float2 t = y[j];
        out[off + ((j + h) & (len - 1))] = make_float2(t.x * inv * g, -t.y * inv * g);
    }
}

constexpr int kExpandThreads = 256;
constexpr int kExpandRows = 64;    // rows per CTA (at least one per row lane)

struct ExpandParams {
    const float2 *part;
    const int *seg;
    float *outRe, *outIm;
    int n, log2n, minIndex, rows, groups, lanes, tiles, chunk, chunks, vec, stream;
};

__device__ __forceinline__ void store4(float *p, float4 v, int vec, int stream) {
    if (vec) {
        if (stream) __stcs(reinterpret_cast<float4 *>(p), v);
        else *reinterpret_cast<float4 *>(p) = v;
    } else {
        p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w;
    }
}

__global__ void __launch_bounds__(kExpandThreads) k_fst_expand(ExpandParams p) {
    // blockIdx.x = (clip * chunks + chunk) * tiles + tile
    const int tile = blockIdx.x % p.tiles, rest = blockIdx.x / p.tiles;
    const int chunk = rest % p.chunks, clip = rest / p.chunks;
    const int lane = threadIdx.x / p.groups, grp = threadIdx.x % p.groups;
    if (lane >= p.lanes) return;
    const int col = 4 * (tile * p.groups + grp);
    const float2 *part = p.part + (size_t)clip * (p.n / 2 + 1);
    const int k1 = min(p.rows, (chunk + 1) * p.chunk);
    int cur = -1;
    float4 vr = make_float4(0.f, 0.f, 0.f, 0.f), vi = vr;
    for (int k = chunk * p.chunk + lane; k < k1; k += p.lanes) {
        const int sg = __ldg(p.seg + p.minIndex + k);
        if (sg != cur) {                                           // column l of the row: element l >> (log2N - log2len)
            cur = sg;
            const int shift = p.log2n - (sg & 31);
            const float2 *q = part + (sg >> 5);
            const float2 a = q[col >> shift], b = q[(col + 1) >> shift], c = q[(col + 2) >> shift], d = q[(col + 3) >> shift];
            vr = make_float4(a.x, b.x, c.x, d.x);
            vi = make_float4(a.y, b.y, c.y, d.y);
        }
        const size_t o = ((size_t)clip * p.rows + k) * p.n + col;
        store4(p.outRe + o, vr, p.vec, p.stream);
        store4(p.outIm + o, vi, p.vec, p.stream);
    }
}

}  // namespace

extern "C" int af_launch_st(const float *data, const float *specRe, const float *specIm, const int *bins, const float *vArr,
                            int rows, int log2n, int batch, float *outRe, float *outIm, void *stream) {
    if (rows <= 0 || batch <= 0) return AF_OK;
    const int n = 1 << log2n;
    if (log2n < 1 || n > AF_ST_MAX_N) return af_fail(AF_ERR_UNSUPPORTED, "ST: %d points; 2 .. %d are supported", n, AF_ST_MAX_N);
    StParams p;
    p.data = data; p.specRe = specRe; p.specIm = specIm; p.bins = bins; p.v = vArr; p.outRe = outRe; p.outIm = outIm;
    p.rows = rows; p.n = n; p.log2n = log2n;
    p.rowsPerCta = n <= 256 ? 2048 / n : 1;
    p.groups = (rows + p.rowsPerCta - 1) / p.rowsPerCta;
    p.tw = af_twiddle_table(log2n);
    if ((long long)p.groups * batch > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "ST: too many rows in one launch");
    const int threads = af_cta_threads(n / 4, 1024);
    const bool inplace = af_fft_inplace(n);
    size_t smem = sizeof(float2) * (inplace ? 1 : 2) * (size_t)n;
    if (smem < 32 * sizeof(double)) smem = 32 * sizeof(double);     // the mean's reduction scratch
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)((long long)p.groups * batch);
    int rc;
    if (inplace) {
        if ((rc = af_smem_optin(k_st_rows<true>, smem, "k_st_rows"))) return rc;
        k_st_rows<true><<<grid, threads, smem, st>>>(p);
    } else {
        if ((rc = af_smem_optin(k_st_rows<false>, smem, "k_st_rows"))) return rc;
        k_st_rows<false><<<grid, threads, smem, st>>>(p);
    }
    AF_LAUNCH_CHECK("k_st_rows");
    return AF_OK;
}

extern "C" int af_launch_fst(const float *specRe, const float *specIm, float *part, const int *seg, int minIndex, int rows,
                             int log2n, int batch, float *outRe, float *outIm, void *stream) {
    if (rows <= 0 || batch <= 0) return AF_OK;
    const int n = 1 << log2n;
    if (log2n < 3 || n > AF_ST_MAX_N) return af_fail(AF_ERR_UNSUPPORTED, "FST: %d points; 8 .. %d are supported", n, AF_ST_MAX_N);
    cudaStream_t st = (cudaStream_t)stream;

    FstParams f;
    f.specRe = specRe; f.specIm = specIm; f.part = reinterpret_cast<float2 *>(part);
    f.norm = 1 / sqrtf((float)n);
    f.n = n; f.log2n = log2n; f.segs = log2n - 1;
    for (int l = 0; l < 14; l++) f.tw[l] = (l >= 1 && l <= log2n - 2) ? af_twiddle_table(l) : nullptr;
    if ((long long)f.segs * batch > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "FST: too many clips in one launch");
    const size_t smem = sizeof(float2) * 2 * (size_t)(n / 4);      // two buffers of the longest segment
    const int rc = af_smem_optin(k_fst_segments, smem, "k_fst_segments");
    if (rc) return rc;
    k_fst_segments<<<(unsigned)(f.segs * batch), af_cta_threads(n / 16, 256), smem, st>>>(f);
    AF_LAUNCH_CHECK("k_fst_segments");

    ExpandParams e;
    e.part = f.part; e.seg = seg; e.outRe = outRe; e.outIm = outIm;
    e.n = n; e.log2n = log2n; e.minIndex = minIndex; e.rows = rows;
    const int groups = n / 4;                                      // float4 column groups of a row
    e.groups = groups < kExpandThreads ? groups : kExpandThreads;
    e.tiles = groups / e.groups;
    e.lanes = kExpandThreads / e.groups;
    e.chunk = kExpandRows > e.lanes ? kExpandRows : e.lanes;
    e.chunks = (rows + e.chunk - 1) / e.chunk;
    e.vec = ((uintptr_t)outRe % 16 == 0) && ((uintptr_t)outIm % 16 == 0);
    const double outBytes = 8.0 * n * (double)rows * batch;
    int l2 = 0, dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev);
    e.stream = outBytes > (double)l2;
    const long long grid = (long long)e.tiles * e.chunks * batch;
    if (grid > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "FST: too many rows in one launch");
    k_fst_expand<<<(unsigned)grid, kExpandThreads, 0, st>>>(e);
    AF_LAUNCH_CHECK("k_fst_expand");
    return AF_OK;
}
