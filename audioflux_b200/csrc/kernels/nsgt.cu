// nsgt.cu -- band transforms of the non-stationary Gabor transform (sm_90a).
//
// Replaces steps 2 and 3 of nsgtObj_nsgt (src/nsgt_algorithm.c:544-604): per band a windowed, rotated slice of the
// clip's spectrum, a length-L inverse DFT (the reference: a dense float64 matrix product, src/dsp/dft_algorithm.c:106-152)
// and the band's matrix row, cell[map[j]] for every column j.  The forward FFT of the clip is af_launch_stft's.
//
// Inside a CTA the band's spectrum slice is read once, the transform runs in shared memory and the matrix row (and the
// cells, when asked for) is written once; nothing in between goes to global memory.
//   k_nsgt_bluestein  L <= 4096.  y[n] = c_n * sum_k (a_k c_k) conj(c_{n-k}) / L with c_m = e^{i pi m^2/L}: a circular
//                     convolution of size M = 2^ceil(log2(2L-1)) <= 8192 -- forward Stockham FFT, product with the
//                     precomputed spectrum of the chirp filter (scaled by 1/(L M)), inverse as conj o forward o conj.
//                     One CTA per (group of consecutive bands, clip); the groups are listed largest first.
//   k_nsgt_direct     4096 < L <= 16384.  O(L^2) float32 DFT, one CTA per (band, clip): the slice is staged in tiles,
//                     each thread accumulates 6 outputs, the twiddle index n k mod L is kept in integers.
#include "common.cuh"
#include "stockham.cuh"

namespace {

struct NsgtParams {
    AfNsgtArgs a;
    const float2 *tw[14];          // Stockham twiddles by log2 M
};

constexpr int kDirThreads = 1024;
constexpr int kDirOut = 6;         // outputs per thread and pass
constexpr int kDirTile = 1024;     // staged input points

__device__ __forceinline__ float2 af_conj(float2 v) { return make_float2(v.x, -v.y); }

// element k of the band's transform input: a[(j + L - L/2) mod L] = X[clamp(off + j, 0, N-1)] * w[j] (:553-578),
// i.e. j = (k + L/2) mod L; bins above N/2 are the conjugate mirror of the half spectrum
__device__ __forceinline__ float2 band_input(const AfNsgtArgs &a, const float *re, const float *im, const AfNsgtBand &b,
                                             int k) {
    int j = k + b.L / 2;
    if (j >= b.L) j -= b.L;
    const int N = a.fftLength;
    int s = b.off + j;
    s = s > N - 1 ? N - 1 : s;
    float xr, xi;
    if (s <= N / 2) { xr = __ldg(re + s); xi = __ldg(im + s); }
    else { xr = __ldg(re + (N - s)); xi = -__ldg(im + (N - s)); }
    const float w = __ldg(a.win + b.winOff + j);
    return make_float2(xr * w, xi * w);
}

// cells (when asked for) and the matrix row out[i][j] = cell[map[i][j]] (:585-604) from the band's result in shared memory
__device__ __forceinline__ void band_write(const AfNsgtArgs &a, const AfNsgtBand &b, int clip, const float2 *y) {
    if (a.cellRe) {
        float *cr = a.cellRe + (size_t)clip * a.totalLen + b.cellOff, *ci = a.cellIm + (size_t)clip * a.totalLen + b.cellOff;
        for (int n = threadIdx.x; n < b.L; n += blockDim.x) { const float2 v = y[n]; cr[n] = v.x; ci[n] = v.y; }
    }
    const int *map = a.map + (size_t)b.band * a.maxLen;
    const size_t row = ((size_t)clip * a.num + b.band) * a.maxLen;
    for (int j = threadIdx.x; j < a.maxLen; j += blockDim.x) {
        const int m = __ldg(map + j);
        const float2 v = m >= 0 ? y[m] : make_float2(0.0f, 0.0f);
        a.outRe[row + j] = v.x;
        a.outIm[row + j] = v.y;
    }
}

__global__ void __launch_bounds__(512) k_nsgt_bluestein(NsgtParams p) {
    extern __shared__ float2 smem[];
    const AfNsgtArgs &a = p.a;
    const int g = blockIdx.x / a.batch, clip = blockIdx.x % a.batch;
    const size_t width = (size_t)a.fftLength / 2 + 1;
    const float *re = a.specRe + clip * width, *im = a.specIm + clip * width;
    const float2 *tab = reinterpret_cast<const float2 *>(a.tab), *filt = reinterpret_cast<const float2 *>(a.filt);
    const int q1 = a.groupStart[g + 1];
    for (int q = a.groupStart[g]; q < q1; q++) {
        const AfNsgtBand b = a.bands[q];
        const int M = 1 << b.log2M, L = b.L;
        const float2 *c = tab + b.tabOff, *h = filt + b.filtOff, *tw = p.tw[b.log2M];
        float2 *x = smem, *y = smem + M;
        for (int k = threadIdx.x; k < M; k += blockDim.x)
            x[k] = k < L ? af_cmul(band_input(a, re, im, b, k), __ldg(c + k)) : make_float2(0.0f, 0.0f);
        __syncthreads();
        float2 *r = af_stockham(x, y, M, b.log2M, tw);
        float2 *o = r == x ? y : x;
        for (int k = threadIdx.x; k < M; k += blockDim.x) r[k] = af_conj(af_cmul(r[k], __ldg(h + k)));
        __syncthreads();
        float2 *z = af_stockham(r, o, M, b.log2M, tw);
        for (int n = threadIdx.x; n < L; n += blockDim.x) z[n] = af_cmul(__ldg(c + n), af_conj(z[n]));
        __syncthreads();
        band_write(a, b, clip, z);
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kDirThreads) k_nsgt_direct(NsgtParams p) {
    extern __shared__ float2 smem[];
    const AfNsgtArgs &a = p.a;
    const int d = blockIdx.x / a.batch, clip = blockIdx.x % a.batch;
    const AfNsgtBand b = a.bands[a.groupStart[a.nGroups] + d];
    const int L = b.L;
    const size_t width = (size_t)a.fftLength / 2 + 1;
    const float *re = a.specRe + clip * width, *im = a.specIm + clip * width;
    float2 *y = smem, *tile = y + a.maxDirectL, *fine = tile + kDirTile, *coarse = fine + AF_NSGT_FINE;
    const float2 *tab = reinterpret_cast<const float2 *>(a.tab) + b.tabOff;
    for (int i = threadIdx.x; i <= AF_NSGT_FINE + (L - 1) / AF_NSGT_FINE; i += blockDim.x) fine[i] = __ldg(tab + i);
    const float invL = 1.0f / (float)L;

    for (int n0 = 0; n0 < L; n0 += kDirThreads * kDirOut) {
        float accr[kDirOut], acci[kDirOut];
        unsigned idx[kDirOut], step[kDirOut];
#pragma unroll
        for (int r = 0; r < kDirOut; r++) {
            const int n = n0 + r * kDirThreads + threadIdx.x;
            step[r] = n < L ? (unsigned)n : 0u;
            idx[r] = 0u;
            accr[r] = acci[r] = 0.0f;
        }
        for (int k0 = 0; k0 < L; k0 += kDirTile) {
            __syncthreads();                               // the previous tile is consumed
            for (int kk = threadIdx.x; kk < kDirTile; kk += blockDim.x) {
                const int k = k0 + kk;
                tile[kk] = k < L ? band_input(a, re, im, b, k) : make_float2(0.0f, 0.0f);
            }
            __syncthreads();
            const int kn = L - k0 < kDirTile ? L - k0 : kDirTile;
            for (int kk = 0; kk < kn; kk++) {
                const float2 v = tile[kk];
#pragma unroll
                for (int r = 0; r < kDirOut; r++) {
                    const float2 t = af_cmul(coarse[idx[r] / AF_NSGT_FINE], fine[idx[r] % AF_NSGT_FINE]);   // e^{2 pi i nk/L}
                    accr[r] += v.x * t.x - v.y * t.y;
                    acci[r] += v.x * t.y + v.y * t.x;
                    idx[r] += step[r];
                    if (idx[r] >= (unsigned)L) idx[r] -= (unsigned)L;
                }
            }
        }
#pragma unroll
        for (int r = 0; r < kDirOut; r++) {
            const int n = n0 + r * kDirThreads + threadIdx.x;
            if (n < L) y[n] = make_float2(accr[r] * invL, acci[r] * invL);
        }
    }
    __syncthreads();
    band_write(a, b, clip, y);
}

}  // namespace

extern "C" int af_launch_nsgt(const AfNsgtArgs *a, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (a->batch <= 0) return AF_OK;
    NsgtParams p;
    p.a = *a;
    int log2MaxM = 0;
    while ((1 << log2MaxM) < a->maxM) log2MaxM++;
    for (int l = 0; l < 14; l++) p.tw[l] = (l >= 1 && l <= log2MaxM) ? af_twiddle_table(l) : nullptr;
    if (a->nGroups > 0) {
        if ((long long)a->nGroups * a->batch > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "NSGT: too many clips in one launch");
        const size_t smem = sizeof(float2) * 2 * (size_t)a->maxM;
        const int rc = af_smem_optin(k_nsgt_bluestein, smem, "k_nsgt_bluestein");
        if (rc) return rc;
        k_nsgt_bluestein<<<(unsigned)(a->nGroups * a->batch), af_cta_threads(a->maxM / 4, 512, 64), smem, st>>>(p);
        AF_LAUNCH_CHECK("k_nsgt_bluestein");
    }
    if (a->nDirect > 0) {
        if ((long long)a->nDirect * a->batch > 0x7fffffffLL) return af_fail(AF_ERR_ARG, "NSGT: too many clips in one launch");
        const size_t smem = sizeof(float2) * ((size_t)a->maxDirectL + kDirTile + AF_NSGT_FINE +
                                              (a->maxDirectL - 1) / AF_NSGT_FINE + 1);
        const int rc = af_smem_optin(k_nsgt_direct, smem, "k_nsgt_direct");
        if (rc) return rc;
        k_nsgt_direct<<<(unsigned)(a->nDirect * a->batch), kDirThreads, smem, st>>>(p);
        AF_LAUNCH_CHECK("k_nsgt_direct");
    }
    return AF_OK;
}
