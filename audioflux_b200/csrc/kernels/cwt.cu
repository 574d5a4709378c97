// cwt.cu -- continuous wavelet transform: big forward FFT of the clip, then per scale
// (wavelet(s*omega) * spectrum) -> inverse FFT, for N = 2^12 .. 2^22 points.
//
// Replaces `__cwtObj_cwt` (src/cwt_algorithm.c:361-483): reflect pad (:404-414), fftObj_fft (:417-422),
// the num x N filter-bank multiply (:426-437), num inverse FFTs fftObj_ifft (:440-459) and the crop
// (:447-452); and the num x N float table built by cwt_filterBank (src/filterbank/cwt_filterBank.c:85-290),
// which is evaluated on the fly here (closed form in s*omega) instead of being read from HBM.
//
// FFT decomposition (four-step, N = N1 * N2, both <= 4096 so each leg lives in shared memory):
//   columns kernel : N2 strided length-N1 transforms (+ inter-leg twiddle), `kCols` adjacent columns per CTA
//                    so global accesses are contiguous runs;
//   rows kernel    : N1 contiguous length-N2 transforms, `rows` adjacent rows per CTA so the strided
//                    result is written as contiguous runs.
// For N <= 4096 the columns kernel alone is the whole transform (N2 = 1).
// Shared-memory legs use the same Stockham radix-4/2 autosort passes as stft_generic.cu.
#include <math.h>
#include <stdlib.h>
#include "common.cuh"
#include "fft32_gen.cuh"

namespace {

__device__ __forceinline__ float2 cw(int k, int m, float dir) {   // exp(dir * 2 pi i k / m)
    float s, c;
    sincospif(dir * 2.0f * (float)k / (float)m, &s, &c);
    return make_float2(c, s);
}

// tw[j] = exp(dir * 2 pi i j / n), j < n: one table per CTA replaces a sincospif per butterfly
__device__ void fill_twiddles(float2 *tw, int n, float dir) {
    for (int j = threadIdx.x; j < n; j += blockDim.x) tw[j] = cw(j, n, dir);
}

// In-place-pair Stockham FFT over `cnt` independent sequences of length n = 2^log2n stored with pitch
// `pitch` (float2 units) in a / b.  All threads of the CTA cooperate; result pointer returned.
__device__ float2 *block_fft_multi(float2 *a, float2 *b, int log2n, int cnt, int pitch, float dir, const float2 *tw) {
    const int n = 1 << log2n;
    int P = 1, rem = log2n;
    while (rem >= 2) {
        const int t = n >> 2;
        for (int e = threadIdx.x; e < t * cnt; e += blockDim.x) {
            const int s = e / t, i = e - s * t;
            const float2 *src = a + (size_t)s * pitch;
            float2 *dst = b + (size_t)s * pitch;
            const int k = i & (P - 1);
            float2 u0 = src[i], u1 = src[i + t], u2 = src[i + 2 * t], u3 = src[i + 3 * t];
            if (k) {
                const int idx = k * (n / (4 * P));                 // exp(dir 2 pi i k / 4P) = tw[k n / 4P]
                const float2 w1 = tw[idx], w2 = tw[2 * idx], w3 = tw[3 * idx];
                u1 = af_cmul(u1, w1); u2 = af_cmul(u2, w2); u3 = af_cmul(u3, w3);
            }
            const float2 s02 = make_float2(u0.x + u2.x, u0.y + u2.y), d02 = make_float2(u0.x - u2.x, u0.y - u2.y);
            const float2 s13 = make_float2(u1.x + u3.x, u1.y + u3.y);
            // (u1 - u3) * (dir * i):  forward (dir=-1): (y, -x);  inverse: (-y, x)
            const float2 d13 = make_float2(-dir * (u1.y - u3.y), dir * (u1.x - u3.x));
            const int j = ((i - k) << 2) + k;
            dst[j] = make_float2(s02.x + s13.x, s02.y + s13.y);
            dst[j + P] = make_float2(d02.x + d13.x, d02.y + d13.y);
            dst[j + 2 * P] = make_float2(s02.x - s13.x, s02.y - s13.y);
            dst[j + 3 * P] = make_float2(d02.x - d13.x, d02.y - d13.y);
        }
        __syncthreads();
        float2 *tmp = a; a = b; b = tmp;
        P <<= 2; rem -= 2;
    }
    if (rem == 1) {
        const int t = n >> 1;
        for (int e = threadIdx.x; e < t * cnt; e += blockDim.x) {
            const int s = e / t, i = e - s * t;
            const float2 *src = a + (size_t)s * pitch;
            float2 *dst = b + (size_t)s * pitch;
            const int k = i & (P - 1);
            const float2 u0 = src[i];
            float2 u1 = src[i + t];
            if (k) u1 = af_cmul(u1, tw[k * (n / (2 * P))]);
            const int j = ((i - k) << 1) + k;
            dst[j] = make_float2(u0.x + u1.x, u0.y + u1.y);
            dst[j + P] = make_float2(u0.x - u1.x, u0.y - u1.y);
        }
        __syncthreads();
        float2 *tmp = a; a = b; b = tmp;
    }
    return a;
}

// psi_hat(s * omega): device twin of af_wavelet_eval (host/af_cwt_bank.c)
__device__ float wavelet_eval(int type, float g, float b, float factor, float sw) {
    if (type == WaveletContinue_Bump) {
        const float r = (sw - g) / b;
        if (!(fabsf(r) < 1.0f - 1e-6f)) return 0.0f;
        const float v = 2.0f * 2.718281828459045f * expf(-1.0f / (1.0f - r * r));
        return isnan(v) ? 0.0f : v;
    }
    if (!(sw > 0.0f)) return 0.0f;
    switch (type) {
    case WaveletContinue_Morse: {
        const float pw = (g == 3.0f) ? sw * sw * sw : powf(sw, g);
        return 2.0f * factor * expf(b * logf(sw) - pw);
    }
    case WaveletContinue_Morlet: return 2.0f * expf(-(sw - g) * (sw - g) / b);
    case WaveletContinue_Paul: return (float)((double)factor * pow((double)sw, (double)g) * exp(-(double)sw));
    case WaveletContinue_DOG: case WaveletContinue_Mexican:
        return (float)((double)factor * pow((double)sw, (double)g) * exp(-(double)sw * sw / b));
    case WaveletContinue_Hermit: {
        const double d = (double)sw - g;
        return (float)((double)factor * d * (1.0 + d) * exp(-d * d / b));
    }
    default: {  // Ricker
        const double x = sw, gg = g;
        return (float)((double)factor * x * x / (gg * gg * gg) * exp(-x * x / (gg * gg)));
    }
    }
}

struct CwtParams {
    const float *data;        // batch x dataLength
    float2 *spec;             // batch x N           (forward spectrum)
    float2 *work;             // items x N           (inter-leg buffer; items = batch or batch*num)
    float *outRe, *outIm;     // batch x num x dataLength
    const float *scaleArr;    // num
    int det;                  // 1: bank * omega * j (cwtObj_cwtDet, src/cwt_algorithm.c:485-528, 426-437)
    float omegaHi, omegaLo;   // 2 pi / N = omegaHi + omegaLo
    const float *bankTable;   // PWT: tabulated bank rows [num][bankWidth] over bins 0..bankWidth-1 instead of a wavelet
    int bankWidth;
    int log2N, log2N1, log2N2, N, N1, N2;
    int dataLength, padLength, num, batch;
    int wType; float g, b, factor;
    int cols, rows;           // adjacent columns / rows per CTA (chosen so each leg fits shared memory)
    int itemBase;             // first (clip, scale) item of this launch (fast path processes items in groups)
    const int *support;       // [lo: num | hi: num] bins [lo, hi) outside which the bank row is below 2^-28 of its peak (NULL: no pruning)
};

__device__ __forceinline__ float load_padded(const CwtParams &p, const float *x, int i) {
    // reflect padding of padLength on both sides (cwt_algorithm.c:404-414)
    int j = i - p.padLength;
    if (j < 0) j = -j - 1;
    else if (j >= p.dataLength) j = 2 * p.dataLength - 1 - j;
    return x[j];
}

// wavelet(s*omega_k) * X[k]  (cwtObj_cwt) or  j * omega_k * wavelet(s*omega_k) * X[k]  (cwtObj_cwtDet: the reference
// multiplies the bank by wArr[k] = 2 pi k / N in float and then forms (-bd * im, bd * re), src/cwt_algorithm.c:426-437,
// 500-512).  omega_k = 2 pi k / N for k <= N/2, negative above, where every wavelet family is zero.
__device__ __forceinline__ float2 bank_times_spec(const CwtParams &p, float s, int sIdx, int k, float2 x) {
    float wv = 0.0f, omega = 0.0f;
    if (k <= p.N / 2) {
        // omega_k = float(2 pi k / N) as the reference tabulates it (double product, rounded once): k * (hi + lo) with
        // hi + lo = 2 pi / N split into two floats gives the same value without the int->double->float conversion chain
        // and FP64 multiplies per element
        omega = fmaf((float)k, p.omegaHi, (float)k * p.omegaLo);
        if (p.bankTable) wv = k < p.bankWidth ? p.bankTable[(size_t)sIdx * p.bankWidth + k] : 0.0f;   // pwtObj_pwt
        else wv = wavelet_eval(p.wType, p.g, p.b, p.factor, s * omega);
    }
    if (!p.det) return make_float2(wv * x.x, wv * x.y);
    const float bd = wv * omega;
    return make_float2(-(bd * x.y), bd * x.x);
}

// MODE 0: forward, input = real clip (padded) ; MODE 1: inverse, input = wavelet(s*omega_k) * spec[k]
template <int MODE>
__global__ void k_cwt_cols(CwtParams p) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    const int N1 = p.N1, N2 = p.N2, pitch = N1 + 1;
    float2 *a = reinterpret_cast<float2 *>(smemRaw), *b = a + (size_t)p.cols * pitch;
    float2 *tw = b + (size_t)p.cols * pitch;                       // [N1] leg twiddles, then [N2] fine inter-leg twiddles
    float2 *tf = tw + N1;
    const int item = blockIdx.x;                                   // MODE 0: clip ; MODE 1: clip*num + scale
    const int clip = MODE == 0 ? item : item / p.num;
    const int sIdx = MODE == 0 ? 0 : item % p.num;
    const int col0 = blockIdx.y * p.cols;
    const int nc = min(p.cols, N2 - col0);
    const float dir = MODE == 0 ? -1.0f : 1.0f;
    const float s = MODE == 1 ? p.scaleArr[sIdx] : 0.0f;
    fill_twiddles(tw, N1, dir);
    if (N2 > 1) for (int j = threadIdx.x; j < N2; j += blockDim.x) tf[j] = cw(j, p.N, dir);

    for (int e = threadIdx.x; e < N1 * nc; e += blockDim.x) {
        const int i = e / nc, c = e - i * nc;
        const int k = i * N2 + col0 + c;                           // element of the length-N sequence
        float2 v;
        if (MODE == 0) {
            v = make_float2(load_padded(p, p.data + (size_t)clip * p.dataLength, k), 0.0f);
        } else {
            v = bank_times_spec(p, s, sIdx, k, p.spec[(size_t)clip * p.N + k]);
        }
        a[(size_t)c * pitch + i] = v;
    }
    __syncthreads();
    float2 *r = block_fft_multi(a, b, p.log2N1, nc, pitch, dir, tw);

    if (N2 == 1) {
        // whole transform done: r[0][k]
        if (MODE == 0) {
            for (int k = threadIdx.x; k < N1; k += blockDim.x) p.spec[(size_t)clip * p.N + k] = r[k];
        } else {
            const float inv = 1.0f / (float)p.N;
            float *oRe = p.outRe + (size_t)item * p.dataLength, *oIm = p.outIm + (size_t)item * p.dataLength;
            for (int k = threadIdx.x; k < p.dataLength; k += blockDim.x) {
                const float2 v = r[k + p.padLength];
                oRe[k] = v.x * inv; oIm[k] = v.y * inv;
            }
        }
        return;
    }
    // inter-leg twiddle W_N^(dir * col * k1) and store B[k1][col] (row-major k1*N2 + col)
    float2 *wk = p.work + (size_t)item * p.N;
    for (int e = threadIdx.x; e < N1 * nc; e += blockDim.x) {
        const int k1 = e / nc, c = e - k1 * nc;
        const int col = col0 + c;
        float2 v = r[(size_t)c * pitch + k1];
        const int prod = col * k1;                                 // < N;  exp(dir 2 pi i prod / N) = tw[prod / N2] * tf[prod % N2]
        v = af_cmul(v, af_cmul(tw[prod >> p.log2N2], tf[prod & (N2 - 1)]));
        wk[(size_t)k1 * N2 + col] = v;
    }
}

template <int MODE>
__global__ void k_cwt_rows(CwtParams p) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    const int N1 = p.N1, N2 = p.N2, pitch = N2 + 1;
    float2 *a = reinterpret_cast<float2 *>(smemRaw), *b = a + (size_t)p.rows * pitch;
    float2 *tw = b + (size_t)p.rows * pitch;                       // [N2]
    const int item = blockIdx.x;
    const int clip = MODE == 0 ? item : item / p.num;
    const int row0 = blockIdx.y * p.rows;
    const int nr = min(p.rows, N1 - row0);
    const float dir = MODE == 0 ? -1.0f : 1.0f;
    const float2 *wk = p.work + (size_t)item * p.N;
    fill_twiddles(tw, N2, dir);
    for (int e = threadIdx.x; e < nr * N2; e += blockDim.x) {
        const int rr = e / N2, i = e - rr * N2;
        a[(size_t)rr * pitch + i] = wk[(size_t)(row0 + rr) * N2 + i];
    }
    __syncthreads();
    float2 *r = block_fft_multi(a, b, p.log2N2, nr, pitch, dir, tw);
    // result element (row k1, k2) is sequence index k1 + N1*k2
    if (MODE == 0) {
        float2 *sp = p.spec + (size_t)clip * p.N;
        for (int e = threadIdx.x; e < nr * N2; e += blockDim.x) {
            const int k2 = e / nr, rr = e - k2 * nr;
            sp[(size_t)k2 * N1 + row0 + rr] = r[(size_t)rr * pitch + k2];
        }
    } else {
        const float inv = 1.0f / (float)p.N;
        float *oRe = p.outRe + (size_t)item * p.dataLength, *oIm = p.outIm + (size_t)item * p.dataLength;
        for (int e = threadIdx.x; e < nr * N2; e += blockDim.x) {
            const int k2 = e / nr, rr = e - k2 * nr;
            const long long n = (long long)k2 * N1 + row0 + rr - p.padLength;
            if (n < 0 || n >= p.dataLength) continue;
            const float2 v = r[(size_t)rr * pitch + k2];
            oRe[n] = v.x * inv; oIm[n] = v.y * inv;
        }
    }
}

// ---- support of every bank row: bins [lo, hi) where psi_hat(s omega_k) exceeds 2^-28 of the row's peak.  Outside, the
// fast path treats the row as zero (relative error <= 4e-9, far inside the 1e-4 tolerance): low scales touch a sliver of
// the spectrum, and loading / evaluating the wavelet over all N/2 bins would dominate their columns units.
__device__ __forceinline__ float bank_value(const CwtParams &p, int sIdx, int k) {
    if (p.bankTable) return k < p.bankWidth ? fabsf(p.bankTable[(size_t)sIdx * p.bankWidth + k]) : 0.0f;
    const float omega = fmaf((float)k, p.omegaHi, (float)k * p.omegaLo);
    return fabsf(wavelet_eval(p.wType, p.g, p.b, p.factor, p.scaleArr[sIdx] * omega));
}
__global__ void k_cwt_support_peak(CwtParams p, unsigned *peakBits) {
    const int sIdx = blockIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
    float v = k <= p.N / 2 ? bank_value(p, sIdx, k) : 0.0f;
    if (!(v < INFINITY)) v = 0.0f;
    unsigned m = __float_as_uint(v);
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(&peakBits[sIdx], m);
}
__global__ void k_cwt_support_range(CwtParams p, const unsigned *peakBits, int *support) {
    const int sIdx = blockIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > p.N / 2) return;
    const float thr = __uint_as_float(peakBits[sIdx]) * 3.7252903e-9f;          // 2^-28
    if (bank_value(p, sIdx, k) > thr) { atomicMin(&support[sIdx], k); atomicMax(&support[p.num + sIdx], k + 1); }
}

// ============================================================================================
// Fast path for N = 2^19 (BASELINE config 4): N1 = 1024 columns leg, N2 = 512 rows leg, every
// transform done by ONE WARP in registers (generated 32/16-point DFTs on (re, im) register pairs, warp-private
// shared-memory transposes, __syncwarp only) -- the CTA synchronises three times instead of once per
// radix pass, and 2-3 CTAs share an SM so the load / transform / store phases of different CTAs overlap.
// Both directions run the forward transform; the inverse is conj . DFT . conj with the conjugations
// folded into the load (MODE 1 loads conj(wavelet * X)) and the final store.
// ============================================================================================
constexpr int kWCols = 8;             // columns (= warps) per CTA in the columns kernel
constexpr int kWColPitch = 1056;      // c64 per column slot: 1024 points + room for the 33 x 32 float transpose plane
constexpr int kWRows = 16;            // rows per CTA in the rows kernel (2 per warp)
constexpr int kWRowPitch = 520;       // c64 per row slot
// Both tiles are filled / drained by threads that walk ACROSS slots (8 columns or 16 rows per index) while the FFT
// warps walk ALONG one slot.  The slot pitches are multiples of 16 c64 (the float transpose planes inside a slot
// rely on it), so the across-walk would hit one 8-byte bank pair 8 times; XOR-ing the low index bits with the slot
// number makes it conflict-free and leaves the along-walk (16 consecutive entries of one slot) a permutation of the
// same 128 bytes.
__device__ __forceinline__ int wcol_idx(int c, int i) { return c * kWColPitch + (i ^ (2 * c)); }
__device__ __forceinline__ int wrow_idx(int r, int k) { return r * kWRowPitch + (k ^ (r & 15)); }

// 32 x 32 complex transpose of a warp's register tile through a 33-padded float plane (real, then imaginary)
__device__ __forceinline__ void warp_transpose32(c64 (&z)[32], float *plane, int lane, const c64 *srcBr /* values at AF_BR5 */) {
    (void)srcBr;
    float yr[32], yi[32];
#pragma unroll
    for (int ka = 0; ka < 32; ka++) c_unpack(z[ka], yr[ka], yi[ka]);
#pragma unroll
    for (int ka = 0; ka < 32; ka++) plane[ka * 33 + lane] = yr[ka];
    __syncwarp();
#pragma unroll
    for (int n1 = 0; n1 < 32; n1++) yr[n1] = plane[lane * 33 + n1];
    __syncwarp();
#pragma unroll
    for (int ka = 0; ka < 32; ka++) plane[ka * 33 + lane] = yi[ka];
    __syncwarp();
#pragma unroll
    for (int n1 = 0; n1 < 32; n1++) z[n1] = c_pack(yr[n1], plane[lane * 33 + n1]);
    __syncwarp();
}

// twiddle tables of the columns leg: [32 ka][32 n1] W_1024^(n1 ka), [N2] W_N^j, [1024] W_1024^j
__device__ void cwt_cols_w_tables(const CwtParams &p, float2 *tw1) {
    float2 *tf = tw1 + 1024, *t1k = tf + p.N2;
    for (int j = threadIdx.x; j < 1024; j += blockDim.x) tw1[j] = cw((j >> 5) * (j & 31), 1024, -1.0f);
    for (int j = threadIdx.x; j < p.N2; j += blockDim.x) tf[j] = cw(j, p.N, -1.0f);
    for (int j = threadIdx.x; j < 1024; j += blockDim.x) t1k[j] = cw(j, 1024, -1.0f);
}

// one unit of the columns leg: kWCols adjacent columns of item `item`, result into wk (the item's inter-leg buffer)
template <int MODE>
__device__ void cwt_cols_w_unit(const CwtParams &p, c64 *tile, const float2 *tw1, int item, int by, float2 *wk) {
    const float2 *tf = tw1 + 1024, *t1k = tf + p.N2;
    const int N2 = p.N2;
    const int clip = MODE == 0 ? item : item / p.num;
    const int col0 = by * kWCols;
    const float s = MODE == 1 ? p.scaleArr[item % p.num] : 0.0f;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // rows i of the column whose input can be non-zero (k = i N2 + column): everything for the forward transform, the
    // bank row's support for the inverse
    int iLo = 0, iHi = 1023, kLo = 0, kHi = p.N;
    if (MODE == 1 && p.support) {
        kLo = p.support[item % p.num]; kHi = p.support[p.num + item % p.num];
        if (kHi <= kLo) { kLo = 0; kHi = 0; iLo = 0; iHi = -1; }
        else { iLo = kLo >> p.log2N2; iHi = (kHi - 1) >> p.log2N2; }
    }
    const bool single = MODE == 1 && p.support && iHi - iLo < 32;       // every lane of the 32 x 32 split sees at most ONE non-zero row
    c64 *colp = tile + (size_t)warp * kWColPitch;
    c64 y[32];
    if (single) {
        // row i = the member of [iLo, iHi] congruent to lane mod 32; stage 1 + its twiddle of a one-hot input collapse to
        // y[ka] = v W_1024^(i ka): no tile fill, no first FFT
        const int i = iLo + ((lane - iLo) & 31);
        const int k = i * N2 + col0 + warp;
        c64 v = 0ull;
        if (i <= iHi && k >= kLo && k < kHi && k <= p.N / 2) {
            const float2 t = bank_times_spec(p, s, item % p.num, k, p.spec[(size_t)clip * p.N + k]);
            v = c_pack(t.x, -t.y);                                             // conj: inverse transform via forward DFT
        }
#pragma unroll
        for (int ka = 0; ka < 32; ka++) y[ka] = ka ? c_mul(v, c_from(t1k[(i * ka) & 1023])) : v;
    } else {
        const int e0 = iLo * kWCols, e1 = (iHi + 1) * kWCols;
        for (int e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
            const int i = e / kWCols, c = e - i * kWCols;
            const int k = i * N2 + col0 + c;
            c64 v;
            if (MODE == 0) {
                v = c_pack(load_padded(p, p.data + (size_t)clip * p.dataLength, k), 0.0f);
            } else {
                // every wavelet family / bank is zero above N/2: do not fetch that half of the spectrum at all
                const float2 t = (k <= p.N / 2 && k >= kLo && k < kHi) ? bank_times_spec(p, s, item % p.num, k, p.spec[(size_t)clip * p.N + k]) : make_float2(0.0f, 0.0f);
                v = c_pack(t.x, -t.y);                                         // conj: inverse transform via forward DFT
            }
            tile[wcol_idx(c, i)] = v;
        }
        __syncthreads();
        // warp `warp` transforms column `warp`: 1024 points as 32 x 32, element n = lane + 32 j (rows outside the support are zero)
        c64 z[32];
#pragma unroll
        for (int j = 0; j < 32; j++) {
            const int i = lane + 32 * j;
            z[j] = (i >= iLo && i <= iHi) ? tile[wcol_idx(warp, i)] : 0ull;
        }
        __syncwarp();
        af_fft32(z);
#pragma unroll
        for (int ka = 0; ka < 32; ka++) y[ka] = ka ? c_mul(z[AF_BR5(ka)], c_from(tw1[ka * 32 + lane])) : z[AF_BR5(0)];
    }
    {
        warp_transpose32(y, reinterpret_cast<float *>(colp), lane, nullptr);
        af_fft32(y);                                                           // X[k1 = lane + 32 kb] at AF_BR5(kb)
        const int col = col0 + warp;
        // inter-leg twiddle W_N^(col k1), k1 = lane + 32 kb: W_N^(col lane) . (W_N^(32 col))^kb.  Two table products per lane
        // (W_N^j = W_1024^(j / N2) . W_N^(j % N2)) and a running product over kb in groups of 8, re-anchored at kb = 0, 8, 16, 24
        // by exact table values: 10 table look-ups per lane instead of 64, and at most 7 chained float products (relative
        // error < 1e-6).
        auto wN = [&](int j) { return c_mul(c_from(t1k[(j >> p.log2N2) & 1023]), c_from(tf[j & (N2 - 1)])); };
        const c64 step = N2 > 1 ? wN((32 * col) & (p.N - 1)) : c_pack(1.0f, 0.0f);
#pragma unroll
        for (int g8 = 0; g8 < 4; g8++) {
            c64 w = N2 > 1 ? wN((col * (lane + 256 * g8)) & (p.N - 1)) : c_pack(1.0f, 0.0f);
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int kb = 8 * g8 + u, k1 = lane + 32 * kb;
                c64 v = y[AF_BR5(kb)];
                if (N2 > 1) { v = c_mul(v, w); if (u < 7) w = c_mul(w, step); }
                tile[wcol_idx(warp, k1)] = v;
            }
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 1024 * kWCols; e += blockDim.x) {
        const int k1 = e / kWCols, c = e - k1 * kWCols;
        float re, im;
        c_unpack(tile[wcol_idx(c, k1)], re, im);
        wk[(size_t)k1 * N2 + col0 + c] = make_float2(re, im);
    }
}

template <int MODE>
__global__ void __launch_bounds__(kWCols * 32) k_cwt_cols_w(CwtParams p) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    c64 *tile = reinterpret_cast<c64 *>(smemRaw);                              // [kWCols][kWColPitch]
    float2 *tw1 = reinterpret_cast<float2 *>(tile + (size_t)kWCols * kWColPitch);
    cwt_cols_w_tables(p, tw1);
    const int item = p.itemBase + blockIdx.x;
    cwt_cols_w_unit<MODE>(p, tile, tw1, item, blockIdx.y, p.work + (size_t)item * p.N);
}

__device__ void cwt_rows_w_tables(float2 *tw) {                               // [32 ka][16 q] W_512^(q ka)
    for (int j = threadIdx.x; j < 512; j += blockDim.x) tw[j] = cw((j >> 4) * (j & 15), 512, -1.0f);
}

// one unit of the rows leg: kWRows adjacent rows of item `item`, read from wk (the item's inter-leg buffer)
template <int MODE>
__device__ void cwt_rows_w_unit(const CwtParams &p, c64 *tile, const float2 *tw, int item, int by, const float2 *wk) {
    const int N1 = p.N1;
    const int clip = MODE == 0 ? item : item / p.num;
    const int row0 = by * kWRows;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int h = lane >> 4, q = lane & 15;

    {   // each half-warp transforms one row of 512 points as 16 x 32: element n = q + 16 j
        const int r = 2 * warp + h;
        const float2 *src = wk + (size_t)(row0 + r) * 512;
        c64 z[32];
#pragma unroll
        for (int j = 0; j < 32; j++) z[j] = c_from(__ldcg(&src[q + 16 * j]));     // L2 only: the ring slot was written by other SMs
        af_fft32(z);                                                           // over j -> Y[q][ka] at AF_BR5(ka)
        float *plane = reinterpret_cast<float *>(tile + (size_t)r * kWRowPitch);   // 1040 floats >= 32 x 17
        float yr[32], yi[32];
#pragma unroll
        for (int ka = 0; ka < 32; ka++) {
            c64 y = z[AF_BR5(ka)];
            if (ka && q) y = c_mul(y, c_from(tw[ka * 16 + q]));
            c_unpack(y, yr[ka], yi[ka]);
        }
        // transpose inside the half-warp: lane q2 receives columns ka = q2 and q2 + 16 (16 values of n1 each)
        c64 u0[16], u1[16];
        float ar[16], br[16];
#pragma unroll
        for (int ka = 0; ka < 32; ka++) plane[ka * 17 + q] = yr[ka];
        __syncwarp();
#pragma unroll
        for (int n1 = 0; n1 < 16; n1++) { ar[n1] = plane[q * 17 + n1]; br[n1] = plane[(q + 16) * 17 + n1]; }
        __syncwarp();
#pragma unroll
        for (int ka = 0; ka < 32; ka++) plane[ka * 17 + q] = yi[ka];
        __syncwarp();
#pragma unroll
        for (int n1 = 0; n1 < 16; n1++) { u0[n1] = c_pack(ar[n1], plane[q * 17 + n1]); u1[n1] = c_pack(br[n1], plane[(q + 16) * 17 + n1]); }
        __syncwarp();
        af_fft16(u0);                                                          // X[k = q + 32 kb] at AF_BR4(kb)
        af_fft16(u1);                                                          // X[k = q + 16 + 32 kb]
#pragma unroll
        for (int kb = 0; kb < 16; kb++) { tile[wrow_idx(r, q + 32 * kb)] = u0[AF_BR4(kb)]; tile[wrow_idx(r, q + 16 + 32 * kb)] = u1[AF_BR4(kb)]; }
    }
    __syncthreads();
    // result element (row k1, k2) is sequence index k1 + N1 * k2
    if (MODE == 0) {
        float2 *sp = p.spec + (size_t)clip * p.N;
        for (int e = threadIdx.x; e < kWRows * 512; e += blockDim.x) {
            const int k2 = e / kWRows, rr = e - k2 * kWRows;
            float re, im;
            c_unpack(tile[wrow_idx(rr, k2)], re, im);
            sp[(size_t)k2 * N1 + row0 + rr] = make_float2(re, im);
        }
    } else {
        const float inv = 1.0f / (float)p.N;
        float *oRe = p.outRe + (size_t)item * p.dataLength, *oIm = p.outIm + (size_t)item * p.dataLength;
        // thread -> (row rr, columns k2 = k20 + 16 it): 16 consecutive output samples per half-warp and plane.
        // Shared-memory reads of 4 iterations are issued ahead of their stores.
        const int rr = threadIdx.x & (kWRows - 1), k20 = threadIdx.x / kWRows;
#pragma unroll 1
        for (int it0 = 0; it0 < 512 / 16; it0 += 4) {
            c64 v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) v[u] = tile[wrow_idx(rr, k20 + 16 * (it0 + u))];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const long long n = (long long)(k20 + 16 * (it0 + u)) * N1 + row0 + rr - p.padLength;
                if (n < 0 || n >= p.dataLength) continue;
                float re, im;
                c_unpack(v[u], re, im);
                __stcs(&oRe[n], re * inv); __stcs(&oIm[n], -im * inv);         // conj back; streaming (evict-first) stores: the
                                                                               // 352 MB / clip of results must not push the ring out of L2
            }
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(kWRows * 16) k_cwt_rows_w(CwtParams p) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    c64 *tile = reinterpret_cast<c64 *>(smemRaw);                              // [kWRows][kWRowPitch]
    float2 *tw = reinterpret_cast<float2 *>(tile + (size_t)kWRows * kWRowPitch);
    cwt_rows_w_tables(tw);
    __syncthreads();
    const int item = p.itemBase + blockIdx.x;
    cwt_rows_w_unit<MODE>(p, tile, tw, item, blockIdx.y, p.work + (size_t)item * p.N);
}

// ============================================================================================
// Both inverse legs in ONE persistent kernel (N = 2^19 fast path).  The inter-leg buffer of an item (4 MB) used to be
// written by a columns launch over ALL items of the chunk and read back by a rows launch: 352 MB per clip to HBM and
// back, about three times the 354 MB of results per clip.  Here the (clip, scale) items are taken in
// groups of `groupItems`; a group's inter-leg data lives in one slot of a small ring (kRing slots, tens of MB: it stays
// in the 50 MB L2), the rows units of group g are queued right behind the columns units of group g + 1, and a slot is
// rewritten -- in L2, before its dirty lines are ever evicted -- as soon as the rows units of its previous group are
// done.  CTAs claim units from one global counter; two per-group counters carry the dependencies (columns done -> rows
// may start; rows done -> the slot may be reused).  Unit order guarantees progress: whatever a unit waits for was
// claimed earlier by a resident CTA.
// ============================================================================================
constexpr int kRing = 3;
struct FusedParams {
    CwtParams p;
    int items, groupItems, groups, cb, rb;      // items = batch * num; cb / rb = column / row units per item
    unsigned *counters;                         // [0] next unit, [1 + g] columns done of group g, [1 + groups + g] rows done
};

__device__ __forceinline__ unsigned ld_acquire(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(256, 2) k_cwt_fused_w(FusedParams f) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    const CwtParams &p = f.p;
    c64 *tile = reinterpret_cast<c64 *>(smemRaw);                              // max(cols tile, rows tile)
    float2 *tw1 = reinterpret_cast<float2 *>(tile + (size_t)kWCols * kWColPitch);   // columns tables (1024 + N2 + 1024)
    float2 *twr = tw1 + 2048 + p.N2;                                           // rows table (512)
    __shared__ unsigned sUnit;
    cwt_cols_w_tables(p, tw1);
    cwt_rows_w_tables(twr);
    __syncthreads();
    const unsigned colsPerGroup = (unsigned)f.groupItems * f.cb, rowsPerGroup = (unsigned)f.groupItems * f.rb;
    // unit sequence: cols(0) | cols(1) rows(0) | cols(2) rows(1) | ... | rows(groups - 1); the last group may be short
    const unsigned span = colsPerGroup + rowsPerGroup;
    const unsigned total = (unsigned)f.groups * span;
    for (;;) {
        __syncthreads();                                                        // previous unit's tile fully consumed
        if (threadIdx.x == 0) sUnit = atomicAdd(&f.counters[0], 1u);
        __syncthreads();
        const unsigned u = sUnit;
        if (u >= total) break;
        bool isRows;
        unsigned g, r;
        if (u < colsPerGroup) { isRows = false; g = 0; r = u; }
        else {
            const unsigned v = u - colsPerGroup, blk = v / span, w = v - blk * span;
            if (blk + 1 < (unsigned)f.groups) { if (w < colsPerGroup) { isRows = false; g = blk + 1; r = w; } else { isRows = true; g = blk; r = w - colsPerGroup; } }
            else { isRows = true; g = blk; r = w; if (w >= rowsPerGroup) continue; }      // tail: only rows(groups - 1)
        }
        const int perItem = isRows ? f.rb : f.cb;
        const int li = (int)(r / perItem), by = (int)(r % perItem);
        const int item = (int)g * f.groupItems + li;
        const int itemsInGroup = min(f.groupItems, f.items - (int)g * f.groupItems);
        float2 *wk = p.work + ((size_t)(g % kRing) * f.groupItems + li) * p.N;
        if (li < itemsInGroup) {
            if (threadIdx.x == 0) {
                if (isRows) {                                                   // every columns unit of this group has landed
                    const unsigned need = (unsigned)itemsInGroup * f.cb;
                    while (ld_acquire(&f.counters[1 + g]) < need) __nanosleep(200);
                } else if (g >= kRing) {                                        // the slot's previous group has been read out
                    const int prevItems = min(f.groupItems, f.items - (int)(g - kRing) * f.groupItems);
                    const unsigned need = (unsigned)prevItems * f.rb;
                    while (ld_acquire(&f.counters[1 + f.groups + (g - kRing)]) < need) __nanosleep(200);
                }
            }
            __syncthreads();
            if (isRows) cwt_rows_w_unit<1>(p, tile, twr, item, by, wk);
            else cwt_cols_w_unit<1>(p, tile, tw1, item, by, wk);
            __syncthreads();                                                    // every thread's global writes of this unit are done ...
            if (threadIdx.x == 0) {                                             // ... and ordered before the release below (the fence is
                __threadfence();                                                // cumulative over the barrier: one per unit instead of 256)
                atomicAdd(&f.counters[1 + (isRows ? f.groups : 0) + g], 1u);
            }
        }
    }
}

__global__ void k_cwt_bank_table(CwtParams p, float *bank) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)p.num * p.N) return;
    const int sIdx = (int)(i / p.N), k = (int)(i % p.N);
    float wv = 0.0f;
    if (k <= p.N / 2) {
        const float omega = (float)((double)k * 2.0 * M_PI / (double)p.N);
        wv = wavelet_eval(p.wType, p.g, p.b, p.factor, p.scaleArr[sIdx] * omega);
    }
    bank[i] = wv;
}

void fill_params(const AfCwtArgs *a, CwtParams *p) {
    p->log2N = a->log2n; p->N = 1 << a->log2n;
    p->log2N1 = a->log2n <= 12 ? a->log2n : (a->log2n + 1) / 2;
    p->log2N2 = a->log2n - p->log2N1;
    p->N1 = 1 << p->log2N1; p->N2 = 1 << p->log2N2;
    p->dataLength = a->dataLength; p->padLength = a->padLength; p->num = a->num; p->batch = a->batch;
    p->scaleArr = a->scaleArr;
    p->det = a->det;
    p->support = NULL;
    { const double w = 2.0 * M_PI / (double)p->N; p->omegaHi = (float)w; p->omegaLo = (float)(w - (double)p->omegaHi); }
    p->bankTable = a->bankTable; p->bankWidth = a->bankWidth;
    p->itemBase = 0;
    p->wType = a->wavelet.waveletType; p->g = a->wavelet.gamma; p->b = a->wavelet.beta; p->factor = (float)a->wavelet.factor;
    const size_t budget = (size_t)(getenv("AFB200_CWT_LEG_KB") ? atoi(getenv("AFB200_CWT_LEG_KB")) : 72) * 1024;   // per-CTA leg buffers: small enough for 2-3 CTAs per SM so load / FFT / store phases of different CTAs overlap
    p->cols = p->N2 == 1 ? 1 : 8;
    while (p->cols > 1 && sizeof(float2) * 2 * (size_t)p->cols * (p->N1 + 1) > budget) p->cols >>= 1;
    p->rows = 16;
    while (p->rows > 1 && sizeof(float2) * 2 * (size_t)p->rows * (p->N2 + 1) > budget) p->rows >>= 1;
}

template <typename K>
int set_smem(K kernel, size_t bytes, const char *name) {
    if (bytes <= 48 * 1024) return AF_OK;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    return e == cudaSuccess ? AF_OK : af_cuda_check(e, name);
}

}  // namespace

// fast path (N = 2^19): persistent fused inverse legs over a small ring of inter-leg slots
static int cwt_fused_enabled(const AfCwtArgs *a) {
    const char *e = getenv("AFB200_CWT_FUSED");
    return a->log2n == 19 && !getenv("AFB200_CWT_GENERIC") && !(e && e[0] == '0');
}
static int cwt_group_items(void) {
    const char *e = getenv("AFB200_CWT_GROUP");
    const int g = e ? atoi(e) : 0;
    return g > 0 && g <= 64 ? g : 2;                     // 3 slots x 2 items x 4 MB = 24 MB: half of the 50 MB L2 of an H100
}

// workspace = forward spectrum (batch x N float2) + inter-leg buffer: batch x num x N float2 when N > 4096, or -- fused
// fast path -- a ring of kRing x groupItems item slots plus the unit counters
extern "C" size_t af_cwt_workspace_bytes(const AfCwtArgs *a) {
    const size_t N = (size_t)1 << a->log2n;
    size_t bytes = sizeof(float2) * N * (size_t)a->batch;
    if (cwt_fused_enabled(a)) {
        // the forward transform of the chunk uses one inter-leg slot per clip, the fused inverse the ring
        size_t slots = (size_t)kRing * cwt_group_items();
        if ((size_t)a->batch > slots) slots = (size_t)a->batch;
        return bytes + sizeof(float2) * N * slots + 65536;
    }
    if (a->log2n > 12) bytes += sizeof(float2) * N * (size_t)a->batch * a->num;
    return bytes;
}

extern "C" int af_launch_cwt(const AfCwtArgs *a, const float *data, void *workspace, float *outRe, float *outIm, void *stream) {
    if (a->log2n < 2 || a->log2n > 24) return af_fail(AF_ERR_UNSUPPORTED, "CWT length 2^%d is outside [2^2, 2^24]", a->log2n);
    CwtParams p;
    fill_params(a, &p);
    p.data = data; p.outRe = outRe; p.outIm = outIm;
    p.spec = static_cast<float2 *>(workspace);
    p.work = p.spec + (size_t)p.N * a->batch;
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if (p.log2N1 == 10 && p.log2N2 == 9 && !getenv("AFB200_CWT_GENERIC")) {
        // warp-level transforms (see k_cwt_cols_w / k_cwt_rows_w)
        const size_t smC = sizeof(c64) * (size_t)kWCols * kWColPitch + sizeof(float2) * (1024 + p.N2 + 1024);
        const size_t smR = sizeof(c64) * (size_t)kWRows * kWRowPitch + sizeof(float2) * 512;
        if ((rc = set_smem(k_cwt_cols_w<0>, smC, "smem k_cwt_cols_w<0>")) || (rc = set_smem(k_cwt_cols_w<1>, smC, "smem k_cwt_cols_w<1>")) ||
            (rc = set_smem(k_cwt_rows_w<0>, smR, "smem k_cwt_rows_w<0>")) || (rc = set_smem(k_cwt_rows_w<1>, smR, "smem k_cwt_rows_w<1>"))) return rc;
        const unsigned cb = (unsigned)(p.N2 / kWCols), rb = (unsigned)(p.N1 / kWRows), items = (unsigned)(a->batch * a->num);
        if (a->support && a->supportReady && !getenv("AFB200_CWT_NOPRUNE")) {
            if (!*a->supportReady) {                       // once per object: peak and [lo, hi) of every bank row
                cudaError_t e = cudaMemsetAsync(a->support, 0x7f, sizeof(int) * (size_t)a->num, st);
                if (e == cudaSuccess) e = cudaMemsetAsync(a->support + a->num, 0, sizeof(int) * 2 * (size_t)a->num, st);
                if (e != cudaSuccess) return af_cuda_check(e, "cudaMemsetAsync(cwt support)");
                const dim3 g((unsigned)((p.N / 2 + 1 + 255) / 256), (unsigned)a->num);
                unsigned *peak = reinterpret_cast<unsigned *>(a->support + 2 * a->num);
                k_cwt_support_peak<<<g, 256, 0, st>>>(p, peak);
                AF_LAUNCH_CHECK("k_cwt_support_peak");
                k_cwt_support_range<<<g, 256, 0, st>>>(p, peak, a->support);
                AF_LAUNCH_CHECK("k_cwt_support_range");
                *a->supportReady = 1;
            }
            p.support = a->support;
        }
        if (data) {                                        // NULL: reuse the spectra already in the workspace
            k_cwt_cols_w<0><<<dim3((unsigned)a->batch, cb), kWCols * 32, smC, st>>>(p);
            AF_LAUNCH_CHECK("k_cwt_cols_w<0>");
            k_cwt_rows_w<0><<<dim3((unsigned)a->batch, rb), kWRows * 16, smR, st>>>(p);
            AF_LAUNCH_CHECK("k_cwt_rows_w<0>");
        }
        if (a->forwardOnly) return AF_OK;
        if (cwt_fused_enabled(a)) {
            FusedParams f;
            f.p = p;
            f.items = (int)items; f.groupItems = cwt_group_items(); f.groups = (f.items + f.groupItems - 1) / f.groupItems;
            f.cb = (int)cb; f.rb = (int)rb;
            {
                size_t slots = (size_t)kRing * f.groupItems;
                if ((size_t)a->batch > slots) slots = (size_t)a->batch;
                f.counters = reinterpret_cast<unsigned *>(p.work + (size_t)p.N * slots);
            }
            if ((size_t)(1 + 2 * f.groups) * sizeof(unsigned) > 65536) return af_fail(AF_ERR_UNSUPPORTED, "CWT: %d item groups exceed the counter block", f.groups);
            cudaError_t e = cudaMemsetAsync(f.counters, 0, (size_t)(1 + 2 * f.groups) * sizeof(unsigned), st);
            if (e != cudaSuccess) return af_cuda_check(e, "cudaMemsetAsync(cwt counters)");
            const size_t smF = sizeof(c64) * (size_t)kWCols * kWColPitch + sizeof(float2) * (2048 + p.N2 + 512);
            if ((rc = set_smem(k_cwt_fused_w, smF, "smem k_cwt_fused_w"))) return rc;
            int sms = af_sm_count();
            if (sms <= 0) sms = 132;
            // Optional (AFB200_CWT_L2PERSIST=1): pin the ring in L2 with a persisting access-policy window on this stream.  The
            // set-aside takes L2 away from the spectrum reads and the result stores, so the default is off: streaming result
            // stores already keep the ring's lines in L2 for most of their life.
            const char *pe = getenv("AFB200_CWT_L2PERSIST");
            const bool persist = pe && pe[0] == '1';
            const size_t ringBytes = sizeof(float2) * (size_t)p.N * kRing * f.groupItems;
            if (persist) {
                static int limitSet = 0;
                int dev = 0, maxPersist = 0, maxWindow = 0;
                cudaGetDevice(&dev);
                cudaDeviceGetAttribute(&maxPersist, cudaDevAttrMaxPersistingL2CacheSize, dev);
                cudaDeviceGetAttribute(&maxWindow, cudaDevAttrMaxAccessPolicyWindowSize, dev);
                if (maxPersist > 0 && maxWindow > 0) {
                    if (!limitSet) { cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, (size_t)maxPersist); limitSet = 1; }
                    cudaStreamAttrValue av;
                    memset(&av, 0, sizeof(av));
                    av.accessPolicyWindow.base_ptr = p.work;
                    av.accessPolicyWindow.num_bytes = ringBytes < (size_t)maxWindow ? ringBytes : (size_t)maxWindow;
                    av.accessPolicyWindow.hitRatio = ringBytes <= (size_t)maxPersist ? 1.0f : (float)((double)maxPersist / (double)ringBytes);
                    av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
                    av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
                    cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &av);
                    cudaGetLastError();
                }
            }
            k_cwt_fused_w<<<(unsigned)(2 * sms), 256, smF, st>>>(f);
            AF_LAUNCH_CHECK("k_cwt_fused_w");
            if (persist) {
                cudaStreamAttrValue av;
                memset(&av, 0, sizeof(av));                          // num_bytes = 0: window off for whatever follows on this stream
                cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &av);
                cudaGetLastError();
            }
            return AF_OK;
        }
        for (unsigned i0 = 0; i0 < items; i0 += items) {
            CwtParams q = p;
            q.itemBase = (int)i0;
            k_cwt_cols_w<1><<<dim3(items, cb), kWCols * 32, smC, st>>>(q);
            AF_LAUNCH_CHECK("k_cwt_cols_w<1>");
            k_cwt_rows_w<1><<<dim3(items, rb), kWRows * 16, smR, st>>>(q);
            AF_LAUNCH_CHECK("k_cwt_rows_w<1>");
        }
        return AF_OK;
    }
    const int threads = 512;
    const size_t smemC = sizeof(float2) * (2 * (size_t)p.cols * (p.N1 + 1) + p.N1 + p.N2);
    const size_t smemR = sizeof(float2) * (2 * (size_t)p.rows * (p.N2 + 1) + p.N2);
    if (smemC > 220 * 1024 || smemR > 220 * 1024) return af_fail(AF_ERR_UNSUPPORTED, "CWT length 2^%d does not fit the shared-memory FFT legs", a->log2n);
    if ((rc = set_smem(k_cwt_cols<0>, smemC, "smem k_cwt_cols<0>")) || (rc = set_smem(k_cwt_cols<1>, smemC, "smem k_cwt_cols<1>")) ||
        (rc = set_smem(k_cwt_rows<0>, smemR, "smem k_cwt_rows<0>")) || (rc = set_smem(k_cwt_rows<1>, smemR, "smem k_cwt_rows<1>"))) return rc;
    const unsigned colBlocks = (unsigned)((p.N2 + p.cols - 1) / p.cols);
    const unsigned rowBlocks = (unsigned)((p.N1 + p.rows - 1) / p.rows);
    // forward transform of every clip
    if (data) {                                            // NULL: reuse the spectra already in the workspace
        k_cwt_cols<0><<<dim3((unsigned)a->batch, colBlocks), threads, smemC, st>>>(p);
        AF_LAUNCH_CHECK("k_cwt_cols<0>");
        if (p.N2 > 1) {
            k_cwt_rows<0><<<dim3((unsigned)a->batch, rowBlocks), threads, smemR, st>>>(p);
            AF_LAUNCH_CHECK("k_cwt_rows<0>");
        }
    }
    if (a->forwardOnly) return AF_OK;
    // per (clip, scale): wavelet * spectrum -> inverse transform -> planes
    const unsigned items = (unsigned)(a->batch * a->num);
    k_cwt_cols<1><<<dim3(items, colBlocks), threads, smemC, st>>>(p);
    AF_LAUNCH_CHECK("k_cwt_cols<1>");
    if (p.N2 > 1) {
        k_cwt_rows<1><<<dim3(items, rowBlocks), threads, smemR, st>>>(p);
        AF_LAUNCH_CHECK("k_cwt_rows<1>");
    }
    return AF_OK;
}

extern "C" int af_launch_cwt_bank_table(const AfCwtArgs *a, float *bank, void *stream) {
    CwtParams p;
    fill_params(a, &p);
    const long long total = (long long)p.num * p.N;
    k_cwt_bank_table<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, bank);
    AF_LAUNCH_CHECK("k_cwt_bank_table");
    return AF_OK;
}
