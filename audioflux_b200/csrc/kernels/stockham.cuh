// stockham.cuh -- block-cooperative radix-4 (+ one radix-2) Stockham autosort FFT in shared memory, forward
// direction (e^{-2 pi i k n / nc}), any power of two nc.  `a` holds the input, `b` is scratch of the same size; the
// function returns whichever of the two holds the result.  All threads of the block must call it.
#pragma once
#include "common.cuh"

__device__ __forceinline__ float2 af_twiddle(int k, int m) {   // exp(-2 pi i k / m)
    float s, c;
    sincospif(-2.0f * (float)k / (float)m, &s, &c);
    return make_float2(c, s);
}

// `tw` (may be null): device table tw[j] = exp(-2 pi i j / nc), j < nc, built once per (device, nc) on the host in double
// precision (af_twiddle_table).  With it every butterfly twiddle is one cached load instead of a sincospif evaluation.
__device__ __forceinline__ float2 af_tw(const float2 *tw, int k, int shift, int m) {
    return tw ? __ldg(tw + ((size_t)k << shift)) : af_twiddle(k, m);
}

__device__ __forceinline__ float2 *af_stockham(float2 *a, float2 *b, int nc, int log2nc, const float2 *tw = nullptr) {
    // Stockham autosort passes: P = product of radices already applied
    int P = 1, rem = log2nc;
    while (rem >= 2) {
        const int t = nc >> 2;
        for (int i = threadIdx.x; i < t; i += blockDim.x) {
            const int k = i & (P - 1);
            float2 u0 = a[i], u1 = a[i + t], u2 = a[i + 2 * t], u3 = a[i + 3 * t];
            if (k) {
                float2 w1 = af_tw(tw, k, rem - 2, 4 * P);              // nc / (4P) = 2^(rem-2)
                float2 w2 = af_cmul(w1, w1), w3 = af_cmul(w2, w1);
                u1 = af_cmul(u1, w1); u2 = af_cmul(u2, w2); u3 = af_cmul(u3, w3);
            }
            float2 s02 = make_float2(u0.x + u2.x, u0.y + u2.y), d02 = make_float2(u0.x - u2.x, u0.y - u2.y);
            float2 s13 = make_float2(u1.x + u3.x, u1.y + u3.y);
            float2 d13 = make_float2(u1.y - u3.y, -(u1.x - u3.x));          // (u1-u3) * (-i)
            const int j = ((i - k) << 2) + k;
            b[j] = make_float2(s02.x + s13.x, s02.y + s13.y);
            b[j + P] = make_float2(d02.x + d13.x, d02.y + d13.y);
            b[j + 2 * P] = make_float2(s02.x - s13.x, s02.y - s13.y);
            b[j + 3 * P] = make_float2(d02.x - d13.x, d02.y - d13.y);
        }
        __syncthreads();
        float2 *tmp = a; a = b; b = tmp;
        P <<= 2; rem -= 2;
    }
    if (rem == 1) {
        const int t = nc >> 1;
        for (int i = threadIdx.x; i < t; i += blockDim.x) {
            const int k = i & (P - 1);
            float2 u0 = a[i], u1 = a[i + t];
            if (k) u1 = af_cmul(u1, af_tw(tw, k, 0, 2 * P));           // last pass: 2P = nc
            const int j = ((i - k) << 1) + k;
            b[j] = make_float2(u0.x + u1.x, u0.y + u1.y);
            b[j + P] = make_float2(u0.x - u1.x, u0.y - u1.y);
        }
        __syncthreads();
        float2 *tmp = a; a = b; b = tmp;
    }

    return a;
}

// same forward transform over ONE buffer, for sizes whose two Stockham buffers do not fit shared memory (16384 points:
// 2 x 128 KB): in-place radix-2 decimation-in-frequency passes.  The result is in bit-reversed order: element j of the
// transform is a[__brev(j) >> (32 - log2nc)].  All threads of the block must call it.
__device__ __forceinline__ void af_fft_inplace_dif(float2 *a, int nc, const float2 *tw = nullptr) {
    for (int half = nc >> 1, shift = 0; half >= 1; half >>= 1, shift++) {
        for (int i = threadIdx.x; i < (nc >> 1); i += blockDim.x) {
            const int k = i & (half - 1), base = ((i - k) << 1) + k;
            const float2 u = a[base], v = a[base + half];
            a[base] = make_float2(u.x + v.x, u.y + v.y);
            float2 d = make_float2(u.x - v.x, u.y - v.y);
            if (k) d = af_cmul(d, af_tw(tw, k, shift, 2 * half));               // exp(-2 pi i k / (2 half)) = tw[k << shift]
            a[base + half] = d;
        }
        __syncthreads();
    }
}

// the companion of af_fft_inplace_dif: the same forward transform over one buffer by in-place radix-2
// decimation-in-time passes, from bit-reversed input (a[__brev(j) >> (32 - log2nc)] holds element j) to natural-order
// output.  After af_fft_inplace_dif, pointwise work in bit-reversed order and conj -> this -> conj / nc invert without
// a permutation.  All threads of the block must call it.
__device__ __forceinline__ void af_fft_inplace_dit(float2 *a, int nc, int log2nc, const float2 *tw = nullptr) {
    for (int half = 1, shift = log2nc - 1; half < nc; half <<= 1, shift--) {
        for (int i = threadIdx.x; i < (nc >> 1); i += blockDim.x) {
            const int k = i & (half - 1), base = ((i - k) << 1) + k;
            const float2 u = a[base];
            float2 v = a[base + half];
            if (k) v = af_cmul(v, af_tw(tw, k, shift, 2 * half));              // exp(-2 pi i k / (2 half)) = tw[k << shift]
            a[base] = make_float2(u.x + v.x, u.y + v.y);
            a[base + half] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
    }
}

// the one-buffer in-place passes replace the two Stockham buffers from 16384 points (2 x 128 KB) up
static inline bool af_fft_inplace(int nc) { return nc > 8192; }

// position of element j in the bit-reversed order that af_fft_inplace_dif leaves and af_fft_inplace_dit reads
__device__ __forceinline__ int af_brev(int j, int log2nc) { return log2nc ? (int)(__brev((unsigned)j) >> (32 - log2nc)) : 0; }

// ---- real sequences: an N-point real FFT as an nc = N/2-point complex FFT of z[j] = x[2j] + i x[2j+1] ----

// W_N^k = exp(-2 pi i k / N), k <= nc: from the second half of af_twiddle_table(log2 nc), or evaluated without a table
__device__ __forceinline__ float2 af_real_tw(const float2 *tw, int nc, int k) {
    return tw ? __ldg(tw + nc + k) : af_twiddle(k, 2 * nc);
}

// post-pass: X[k] (k = 0 .. nc) from zk = Z[k mod nc], zp = Z[(nc - k) mod nc] of the packed transform Z and w = W_N^k,
// X[k] = E[k] + W_N^k O[k]; X[0] and X[nc] are real
__device__ __forceinline__ float2 af_real_post(float2 zk, float2 zp, float2 w, int k, int nc) {
    const float er = 0.5f * (zk.x + zp.x), ei = 0.5f * (zk.y - zp.y);
    const float orr = 0.5f * (zk.y + zp.y), oi = -0.5f * (zk.x - zp.x);
    float xr = er + (w.x * orr - w.y * oi), xi = ei + (w.x * oi + w.y * orr);
    if (k == 0 || k == nc) xi = 0.0f;
    return make_float2(xr, xi);
}

// the post-pass over a packed transform Z in natural order (af_stockham)
__device__ __forceinline__ float2 af_real_bin(const float2 *Z, float2 w, int k, int nc) {
    return af_real_post(Z[k == nc ? 0 : k], Z[k == 0 ? 0 : nc - k], w, k, nc);
}

// pre-pass of the inverse, conjugated: packed point k of the inverse real transform of the Hermitian X, from pk = X[k],
// pm = X[nc - k] and w = W_N^k: conj(E + i O), E = (pk + conj pm) / 2, O = (pk - conj pm) / 2 * conj(w)
__device__ __forceinline__ float2 af_real_pre_conj(float2 pk, float2 pm, float2 w) {
    const float er = 0.5f * (pk.x + pm.x), ei = 0.5f * (pk.y - pm.y);
    const float dr = 0.5f * (pk.x - pm.x), di = 0.5f * (pk.y + pm.y);
    const float orr = dr * w.x + di * w.y, oi = di * w.x - dr * w.y;
    return make_float2(er - oi, -(ei + orr));
}

// ---- in-place real correlation: af_fft_inplace_dif, a product per bin, af_real_inverse, af_real_at ----

// bin k (0 .. nc) of the real FFT whose nc-point packed transform z is in bit-reversed order (af_fft_inplace_dif)
__device__ __forceinline__ float2 af_real_bin_brev(const float2 *z, const float2 *tw, int k, int nc, int log2nc) {
    const float2 zk = z[af_brev(k == nc ? 0 : k, log2nc)], zp = z[af_brev(k == 0 ? 0 : nc - k, log2nc)];
    return af_real_post(zk, zp, af_real_tw(tw, nc, k), k, nc);
}

// nc times the real inverse IFFT_N (1/N included, N = 2 nc) of the Hermitian spectrum X[k] = spectrum(k), in place in
// the nc points of a: per pair (k, nc - k), the conjugated pre-pass written at the pair's bit-reversed positions, then
// af_fft_inplace_dit leaves the packed result in natural order (read it with af_real_at).
// Each thread owns its pairs and overwrites their positions: spectrum(k) may read a only at the bit-reversed positions
// of bins k and nc - k (as af_real_bin_brev does), never another pair's.  All threads of the block must call it.
template <class Spectrum>
__device__ __forceinline__ void af_real_inverse(float2 *a, int nc, int log2nc, const float2 *tw, Spectrum spectrum) {
    for (int k = threadIdx.x; k <= nc / 2; k += blockDim.x) {
        const int m = nc - k;
        const float2 pk = spectrum(k), pm = spectrum(m);
        a[af_brev(k, log2nc)] = af_real_pre_conj(pk, pm, af_real_tw(tw, nc, k));
        if (k > 0 && m != k) a[af_brev(m, log2nc)] = af_real_pre_conj(pm, pk, af_real_tw(tw, nc, m));
    }
    __syncthreads();
    af_fft_inplace_dit(a, nc, log2nc, tw);
}

// value m (0 .. 2 nc - 1) of the real result af_real_inverse leaves in y: r[2j] + i r[2j+1] = conj(y[j])
__device__ __forceinline__ float af_real_at(const float2 *y, int m) {
    const float2 v = y[m >> 1];
    return (m & 1) ? -v.y : v.x;
}

// value v at position k (0 .. N/2) of a real even N-sequence, in the float view f of a packed buffer
__device__ __forceinline__ void af_put_even(float *f, int n, int k, float v) {
    f[k] = v;
    if (k > 0 && k < n / 2) f[n - k] = v;
}

// host side (stockham.cu): cached device tables per (device, log2 n): [0, n) exp(-2 pi i j / n) and, behind it,
// [0, n] exp(-2 pi i j / (2n)) (the real-FFT twiddles of a 2n-point real transform packed into n complex points)
const float2 *af_twiddle_table(int log2n);
