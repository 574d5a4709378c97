// cqt.cu -- constant-Q transform kernels: fixed /2 decimator and per-octave kernel correlation.
//
// Replaces the reference's recursive-octave loop `_cqtObj_cqt` (src/cqt_algorithm.c:845-1061):
//   per octave: resampleObj_resample (/2, src/dsp/resample_algorithm.c:430-521) ; stftObj_stft with a
//   rect window and centre zero padding (src/stft_algorithm.c:601-694) ; compaction ; `__mcdot1` of the
//   half spectrum with the thresholded spectral kernels ; scaling (:972-989, 1020-1041).
//
// GPU restatement: for a real frame x, sum_k X[k] K_b[k] == sum_n x[n] kappa_b[n] with
// kappa_b = DFT of the (thresholded, half-spectrum) kernel row, so one octave is a strided complex
// correlation  out[t][b] = sum_n xpad[t*hop + n] * kappa_b[n]  -- dense FP32 FMA work on data that
// stays in shared memory, with no per-frame FFT, no T x 512 spectra in HBM and no compaction pass.
// The signal tile is staged polyphase-major (xs[r][u] = x[hop*u + r]) so that the 32 lanes of a warp
// (32 consecutive frames) read consecutive words for every (r, a) step whatever the hop is.
#include <math.h>
#include <string.h>
#include "common.cuh"
#include "c64.cuh"

namespace {

constexpr int kDecThreads = 256;
constexpr int kDecPer = 8;                       // outputs per thread (register sliding window)
constexpr int kDecTile = kDecThreads * kDecPer;  // outputs per CTA
constexpr int kDecSpan = 2 * kDecTile + 64;      // staged input samples per CTA
__constant__ float c_decTaps[64];                // [0..31] left taps (x[2i-j]), [32..62] right taps (x[2i+1+j])

// shared-memory slot of staged sample i: 4 pad floats after every 32 samples keep the 16-byte alignment and spread the
// per-thread windows (64-byte stride) over all banks: the LDS.128 of a quarter-warp are conflict-free
__device__ __forceinline__ int dec_slot(int i) { return i + 4 * (i >> 5); }

// out[i] = (sum_{j<32} L[j] x[2i-j] + sum_{j<31} R[j] x[2i+1+j]) / sqrt(1/2), zero outside the clip: a 64-tap FIR
// h[k] over the window x[2i-32+k] (h[0] = 0, h[32-j] = L[j], h[33+j] = R[j] = c_decTaps[32+j]).  Each thread keeps an 80-sample window in
// registers (20 LDS.128) and produces 8 outputs; the taps are consumed as (even, odd) PAIRS against the aligned sample
// pairs of the window with (even, odd) pair FMAs (c64.cuh) -- 32 per output, the two halves of the accumulator added at the end.
__global__ void __launch_bounds__(kDecThreads, 2) k_decimate2(const float *__restrict__ in, int inLength, long long inStride,
                                                              float *__restrict__ out, long long outStride) {
    __shared__ __align__(16) float sx[kDecSpan + 4 * (kDecSpan / 32) + 8];
    const int outLength = inLength / 2;
    const int o0 = blockIdx.x * kDecTile;
    const float *x = in + (long long)blockIdx.y * inStride;
    const int m0 = 2 * o0 - 32;                               // staged sample i = x[m0 + i]
    __shared__ __align__(16) float sh[64];                    // the FIR in window order
    if (threadIdx.x < 64) {
        const int k = threadIdx.x;
        sh[k] = k == 0 ? 0.0f : (k <= 32 ? c_decTaps[32 - k] : c_decTaps[k - 1]);
    }
    const bool vec = ((inStride & 3) == 0) && ((reinterpret_cast<uintptr_t>(in) & 15) == 0);
    if (vec && m0 >= 0 && m0 + kDecSpan <= inLength) {
        constexpr int kV = kDecSpan / 4, kPer = (kV + kDecThreads - 1) / kDecThreads;
        float4 q[kPer];
#pragma unroll
        for (int b = 0; b < kPer; b++) {
            const int v = threadIdx.x + b * kDecThreads;
            if (v < kV) q[b] = __ldg(reinterpret_cast<const float4 *>(x + m0) + v);
        }
#pragma unroll
        for (int b = 0; b < kPer; b++) {
            const int v = threadIdx.x + b * kDecThreads;
            if (v < kV) *reinterpret_cast<float4 *>(sx + dec_slot(4 * v)) = q[b];
        }
    } else {
        for (int i = threadIdx.x; i < kDecSpan; i += kDecThreads) {
            const int m = m0 + i;
            sx[dec_slot(i)] = (m >= 0 && m < inLength) ? x[m] : 0.0f;
        }
    }
    __syncthreads();
    c64 w[kDecPer + 32];                                      // aligned sample pairs (x[2o0 - 32 + 2 (8 t + n)], next)
    // slot of sample 16 t + 4 v = slot(16 t) + 4 v + 4 ((16 (t & 1) + 4 v) >> 5): two base pointers (the odd threads' second
    // one is a pad further) and compile-time offsets -> LDS.128 with immediate offsets
    const float *baseA = sx + dec_slot(2 * kDecPer * threadIdx.x), *baseB = baseA + 4 * (threadIdx.x & 1);
#pragma unroll
    for (int v = 0; v < (kDecPer + 32) / 2; v++) {
        const float4 q = *reinterpret_cast<const float4 *>(((4 * v) & 31) >= 16 ? baseB + 4 * v + 4 * ((4 * v) >> 5) : baseA + 4 * v + 4 * ((4 * v) >> 5));
        w[2 * v] = c_pack(q.x, q.y);
        w[2 * v + 1] = c_pack(q.z, q.w);
    }
    c64 acc[kDecPer];
#pragma unroll
    for (int q = 0; q < kDecPer; q++) acc[q] = 0ull;
#pragma unroll
    for (int u = 0; u < 32; u++) {
        const c64 h = reinterpret_cast<const c64 *>(sh)[u];   // (h[2u], h[2u+1])
#pragma unroll
        for (int q = 0; q < kDecPer; q++) acc[q] = v_fma(h, w[q + u], acc[q]);
    }
    const float scale = 1.4142135623730951f;                  // 1 / sqrt(0.5)
    float r[kDecPer];
#pragma unroll
    for (int q = 0; q < kDecPer; q++) {
        float a, b;
        c_unpack(acc[q], a, b);
        r[q] = (a + b) * scale;
    }
    const int o = o0 + kDecPer * threadIdx.x;
    float *dst = out + (long long)blockIdx.y * outStride + o;
    if (o + kDecPer <= outLength && ((outStride & 3) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0)) {
#pragma unroll
        for (int v = 0; v < kDecPer / 4; v++)
            reinterpret_cast<float4 *>(dst)[v] = make_float4(r[4 * v], r[4 * v + 1], r[4 * v + 2], r[4 * v + 3]);
    } else {
#pragma unroll
        for (int q = 0; q < kDecPer; q++)
            if (o + q < outLength) dst[q] = r[q];
    }
}

struct OctParams {
    const float *sig; long long sigStride; int sigLength, validLength;
    int N, hop, T, bpo;
    const float2 *kappa;          // [bpo][N] (re, im)
    const float *scale;           // [bpo]
    float *outRe, *outIm; long long outStride; int num, colOff;
    int padLeft;                  // zero samples logically in front of the clip: N/2 (centre padding) or 0 (streaming: right padding)
    int TT;                       // frames per CTA (multiple of kFT)
    int rowLen;                   // polyphase row pitch (floats)
    int rowsA;                    // ceil(N / hop)
    int nChunk;                   // kernel taps resident in shared memory at a time
    int segs;                     // tap segments worked on by different threads (large hops: few frames fit in shared
                                  // memory, so the taps of one frame are split to get enough threads), summed at the end
};

constexpr int kBinsPerPass = 12;  // bins whose kernels sit in shared memory together
constexpr int kFT = 4;            // frames per thread
constexpr int kJG = 2;            // thread groups over bins
constexpr int kBT = 6;            // bins per thread: 4 x 6 complex accumulators, 10 shared loads per 48 FMAs

__global__ void k_cqt_octave(OctParams p) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    float2 *sk = reinterpret_cast<float2 *>(smemRaw);                       // [kBinsPerPass][nChunk]
    float *xs = reinterpret_cast<float *>(smemRaw + sizeof(float2) * (size_t)kBinsPerPass * p.nChunk);
    const int clip = blockIdx.y;
    const int t0 = blockIdx.x * p.TT;
    const float *sig = p.sig + (long long)clip * p.sigStride;
    const int h = p.hop, N = p.N;

    // stage the tile's span of the zero-padded signal, polyphase-major
    const int span = (p.TT - 1) * h + N;
    const long long m0 = (long long)t0 * h - p.padLeft;      // signal index of padded position t0*h
    // (4 independent loads in flight per thread: at the top octave the staging moves 3x more data per MAC than
    //  lower down and is load-latency bound; hop is a power of two in every default configuration, then the
    //  polyphase split is a shift and a mask)
    const int hShift = (h & (h - 1)) == 0 ? __ffs(h) - 1 : -1;
    for (int i0 = threadIdx.x; i0 < span; i0 += 4 * blockDim.x) {
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + u * blockDim.x;
            const long long m = m0 + i;
            v[u] = (i < span && m >= 0 && m < p.validLength) ? sig[m] : 0.0f;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + u * blockDim.x;
            if (i >= span) continue;
            const int r = hShift >= 0 ? (i & (h - 1)) : i % h, a = hShift >= 0 ? (i >> hShift) : i / h;
            xs[r * p.rowLen + a] = v[u];
        }
    }

    const int quarter = p.TT / kFT;
    const int tl = threadIdx.x % quarter;                    // frame lane inside the tile
    const int jg = (threadIdx.x / quarter) % kJG;            // bin group 0..kJG-1
    const int seg = threadIdx.x / (quarter * kJG);           // tap segment 0..segs-1: taps a in [aLo, aHi) of every phase r
    const int aLo = (int)((long long)p.rowsA * seg / p.segs), aHi = (int)((long long)p.rowsA * (seg + 1) / p.segs);

    for (int j0 = 0; j0 < p.bpo; j0 += kBinsPerPass) {
        const int nb = min(kBinsPerPass, p.bpo - j0);
        float ar[kFT][kBT], ai[kFT][kBT];
#pragma unroll
        for (int f = 0; f < kFT; f++)
#pragma unroll
            for (int u = 0; u < kBT; u++) { ar[f][u] = 0.0f; ai[f][u] = 0.0f; }
        // the kernels of this pass are streamed through shared memory in chunks of p.nChunk taps
        for (int n0 = 0; n0 < N; n0 += p.nChunk) {
            const int n1 = min(N, n0 + p.nChunk), cw = n1 - n0;
            __syncthreads();                                   // xs staged / previous chunk consumed
            for (int i = threadIdx.x; i < kBinsPerPass * cw; i += blockDim.x) {
                const int j = i / cw, n = i - j * cw;
                sk[(size_t)j * p.nChunk + n] = j < nb ? p.kappa[(size_t)(j0 + j) * N + n0 + n] : make_float2(0.f, 0.f);
            }
            __syncthreads();
            const float2 *kb = sk + (size_t)(jg * kBT) * p.nChunk - n0;
            // taps n of this chunk and of this thread's segment, in ascending n: tap n = a*h + r reads polyphase row r at
            // column a.  One flat loop with (r, a) advanced incrementally: no per-phase set-up (a division and ~50
            // instructions per phase, which dominated at the top octaves where a phase holds only N/hop = 4 taps).
            const int nBeg = max(n0, aLo * h), nEnd = min(n1, aHi * h);
            if (nBeg < nEnd) {
                int a = hShift >= 0 ? (nBeg >> hShift) : nBeg / h;
                int r = nBeg - a * h;
                const float *row = xs + r * p.rowLen + tl + a;
#pragma unroll 2
                for (int n = nBeg; n < nEnd; n++) {
                    float x[kFT];
#pragma unroll
                    for (int f = 0; f < kFT; f++) x[f] = row[f * quarter];
#pragma unroll
                    for (int u = 0; u < kBT; u++) {
                        const float2 c = kb[(size_t)u * p.nChunk + n];
#pragma unroll
                        for (int f = 0; f < kFT; f++) {
                            ar[f][u] = fmaf(x[f], c.x, ar[f][u]);
                            ai[f][u] = fmaf(x[f], c.y, ai[f][u]);
                        }
                    }
                    row += p.rowLen;
                    if (++r == h) { r = 0; row -= (long long)h * p.rowLen - 1; }
                }
            }
        }
        if (p.segs > 1) {
            // sum the tap segments: partial accumulators go through the kernel buffer (dead until the next pass reloads it;
            // the signal tile must survive for that pass)
            __syncthreads();
            float *red = reinterpret_cast<float *>(sk);
            const int slot = (jg * quarter + tl) * (2 * kFT * kBT);
            for (int sgm = 1; sgm < p.segs; sgm++) {
                if (seg == sgm) {
#pragma unroll
                    for (int f = 0; f < kFT; f++)
#pragma unroll
                        for (int u = 0; u < kBT; u++) { red[slot + (f * kBT + u) * 2] = ar[f][u]; red[slot + (f * kBT + u) * 2 + 1] = ai[f][u]; }
                }
                __syncthreads();
                if (seg == 0) {
#pragma unroll
                    for (int f = 0; f < kFT; f++)
#pragma unroll
                        for (int u = 0; u < kBT; u++) { ar[f][u] += red[slot + (f * kBT + u) * 2]; ai[f][u] += red[slot + (f * kBT + u) * 2 + 1]; }
                }
                __syncthreads();
            }
        }
#pragma unroll
        for (int f = 0; f < kFT; f++) {
            const int t = t0 + tl + f * quarter;
            if (t >= p.T || seg != 0) continue;
#pragma unroll
            for (int u = 0; u < kBT; u++) {
                const int j = j0 + jg * kBT + u;
                if (j >= p.bpo || jg * kBT + u >= nb) continue;
                const float s = p.scale[j];
                const long long o = (long long)clip * p.outStride + (long long)t * p.num + p.colOff + j;
                p.outRe[o] = ar[f][u] * s;
                p.outIm[o] = ai[f][u] * s;
            }
        }
    }
}

// Last resort for geometries whose polyphase tile does not fit shared memory at all (hops in the thousands: long kernels
// -- large factor, many bins per octave -- over few octaves): one warp per (frame, bin), the lanes stride over the taps
// straight from global memory (coalesced signal and kernel reads), warp-shuffle reduction.  Same sums as k_cqt_octave in
// another order (float32, <= 2^14 terms in 32 partial sums).
__global__ void __launch_bounds__(256) k_cqt_octave_direct(OctParams p) {
    const int lane = threadIdx.x & 31;
    const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);     // (frame, bin) of this warp
    const int clip = blockIdx.y;
    if (w >= (long long)p.T * p.bpo) return;
    const int t = (int)(w / p.bpo), j = (int)(w - (long long)t * p.bpo);
    const float *sig = p.sig + (long long)clip * p.sigStride;
    const long long m0 = (long long)t * p.hop - p.padLeft;
    const float2 *kap = p.kappa + (size_t)j * p.N;
    float ar = 0.0f, ai = 0.0f;
    for (int n = lane; n < p.N; n += 32) {
        const long long m = m0 + n;
        const float x = (m >= 0 && m < p.validLength) ? sig[m] : 0.0f;
        const float2 c = kap[n];
        ar = fmaf(x, c.x, ar);
        ai = fmaf(x, c.y, ai);
    }
    for (int o = 16; o; o >>= 1) {
        ar += __shfl_xor_sync(0xffffffffu, ar, o);
        ai += __shfl_xor_sync(0xffffffffu, ai, o);
    }
    if (lane == 0) {
        const float sc = p.scale[j];
        const long long o = (long long)clip * p.outStride + (long long)t * p.num + p.colOff + j;
        p.outRe[o] = ar * sc;
        p.outIm[o] = ai * sc;
    }
}


// ---- tensor-core octave kernel ---------------------------------------------------------------------------------
// One octave is a GEMM  out[T x 24] = A[T x N] . B[N x 24]  with a Hankel A operand, A[t][n] = xpad[t*hop + n]
// (never materialised: the mma A fragments are read straight from the staged signal tile) and B = the 12 time-domain
// kernels kappa_b as interleaved (re, im) columns.  mma.sync.m16n8k8 TF32 with the 3xTF32 split (x = hi + lo, hi by
// truncation, lo = x - hi exact; hi*hi + lo*hi + hi*lo) keeps fp32-level accuracy (measured against the oracle in
// tests/test_gpu_parity.py); the kappa fragments arrive pre-split from a host-built table, chunk by chunk.
//   * signal tile: polyphase-major xs[r][u] = x[hop*u + r] with row pitch == 8 (mod 32) for hop >= 8 -> the fragment
//     element (frame g, tap t4) sits in bank 8*t4 + g: conflict-free; plain linear for hop <= 4 (4g + t4, or equal
//     addresses for hop 2: broadcast);
//   * warp w owns kTcMT m-tiles (16 frames each); per k-step it reads 3 LDS.128 of B fragments (shared by its m-tiles)
//     and, per m-tile, 4 LDS.32 + 8 ALU (split) + 9 HMMA: ~140 MAC per issued instruction (FP32 loop: ~26).
constexpr int kTcMT = 2;                          // m-tiles (16 frames) per warp
constexpr int kTcKC = 16;                         // k-steps (8 taps) of kernel fragments resident in shared memory at a time

struct OctTcParams {
    const float *sig; long long sigStride; int validLength;
    int N, hop, hs, T;
    const float4 *bfrag;          // [N/8 k-steps][3 n-tiles][32 lanes] (hi0, hi1, lo0, lo1)
    const float *scale;           // [12]
    float *outRe, *outIm; long long outStride; int num, colOff;
    int TT, rowLen, warps, padLeft;
};

__global__ void k_cqt_octave_tc(OctTcParams p) {
    extern __shared__ __align__(16) unsigned char smemRaw[];
    float4 *sB = reinterpret_cast<float4 *>(smemRaw);                        // [kTcKC][3][32]
    float *xs = reinterpret_cast<float *>(smemRaw + sizeof(float4) * kTcKC * 96);
    const int clip = blockIdx.y;
    const int t0 = blockIdx.x * p.TT;
    const float *sig = p.sig + (long long)clip * p.sigStride;
    const int h = p.hop, N = p.N, hs = p.hs;
    const bool poly = h >= 8;

    // stage the tile's span of the zero-padded signal
    const int span = (p.TT - 1) * h + N;
    const long long m0 = (long long)t0 * h - p.padLeft;
    for (int i0 = threadIdx.x; i0 < span; i0 += 4 * blockDim.x) {
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + u * blockDim.x;
            const long long m = m0 + i;
            v[u] = (i < span && m >= 0 && m < p.validLength) ? sig[m] : 0.0f;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + u * blockDim.x;
            if (i >= span) continue;
            xs[poly ? (i & (h - 1)) * p.rowLen + (i >> hs) : i] = v[u];
        }
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t4 = lane & 3;
    float acc[kTcMT][3][4];
#pragma unroll
    for (int m = 0; m < kTcMT; m++)
#pragma unroll
        for (int n = 0; n < 3; n++) acc[m][n][0] = acc[m][n][1] = acc[m][n][2] = acc[m][n][3] = 0.0f;
    const int tb = warp * (16 * kTcMT);                                     // first frame (within the tile) of this warp
    const int rowStep = poly ? 8 : 8 * h;                                   // address step from frame g to frame g + 8
    const int colStep = poly ? 4 * p.rowLen : 4;                            // address step from tap t4 to tap t4 + 4

#define AF_MMA_TF32(ACC, A0, A1, A2, A3, B0, B1)                                                              \
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" \
        : "+f"(ACC[0]), "+f"(ACC[1]), "+f"(ACC[2]), "+f"(ACC[3])                                              \
        : "r"(A0), "r"(A1), "r"(A2), "r"(A3), "r"(B0), "r"(B1))

    const int kSteps = N >> 3;
    for (int kc = 0; kc < kSteps; kc += kTcKC) {
        __syncthreads();                                                    // signal staged / previous chunk consumed
        const int nk = min(kTcKC, kSteps - kc);
        for (int i = threadIdx.x; i < nk * 96; i += blockDim.x) sB[i] = p.bfrag[(size_t)kc * 96 + i];
        __syncthreads();
#pragma unroll 2
        for (int ks = 0; ks < nk; ks++) {
            const int n0 = (kc + ks) << 3;
            const float4 b0 = sB[(ks * 3 + 0) * 32 + lane], b1 = sB[(ks * 3 + 1) * 32 + lane], b2 = sB[(ks * 3 + 2) * 32 + lane];
            const int base = poly ? ((n0 & (h - 1)) + t4) * p.rowLen + (n0 >> hs) + tb + g : (tb + g) * h + n0 + t4;
#pragma unroll
            for (int m = 0; m < kTcMT; m++) {
                const float *a = xs + base + m * (poly ? 16 : 16 * h);
                const float af[4] = {a[0], a[rowStep], a[colStep], a[colStep + rowStep]};
                uint32_t ah[4], al[4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    ah[i] = __float_as_uint(af[i]) & 0xffffe000u;
                    al[i] = __float_as_uint(af[i] - __uint_as_float(ah[i]));
                }
                AF_MMA_TF32(acc[m][0], al[0], al[1], al[2], al[3], __float_as_uint(b0.x), __float_as_uint(b0.y));
                AF_MMA_TF32(acc[m][1], al[0], al[1], al[2], al[3], __float_as_uint(b1.x), __float_as_uint(b1.y));
                AF_MMA_TF32(acc[m][2], al[0], al[1], al[2], al[3], __float_as_uint(b2.x), __float_as_uint(b2.y));
                AF_MMA_TF32(acc[m][0], ah[0], ah[1], ah[2], ah[3], __float_as_uint(b0.z), __float_as_uint(b0.w));
                AF_MMA_TF32(acc[m][1], ah[0], ah[1], ah[2], ah[3], __float_as_uint(b1.z), __float_as_uint(b1.w));
                AF_MMA_TF32(acc[m][2], ah[0], ah[1], ah[2], ah[3], __float_as_uint(b2.z), __float_as_uint(b2.w));
                AF_MMA_TF32(acc[m][0], ah[0], ah[1], ah[2], ah[3], __float_as_uint(b0.x), __float_as_uint(b0.y));
                AF_MMA_TF32(acc[m][1], ah[0], ah[1], ah[2], ah[3], __float_as_uint(b1.x), __float_as_uint(b1.y));
                AF_MMA_TF32(acc[m][2], ah[0], ah[1], ah[2], ah[3], __float_as_uint(b2.x), __float_as_uint(b2.y));
            }
        }
    }
#undef AF_MMA_TF32
    // C fragment: rows g / g + 8 = frames, columns 2 t4, 2 t4 + 1 = (re, im) of bin 4 nt + t4
#pragma unroll
    for (int m = 0; m < kTcMT; m++)
#pragma unroll
        for (int n = 0; n < 3; n++) {
            const int j = 4 * n + t4;
            const float s = p.scale[j];
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                const int t = t0 + tb + 16 * m + g + 8 * hf;
                if (t >= p.T) continue;
                const long long o = (long long)clip * p.outStride + (long long)t * p.num + p.colOff + j;
                p.outRe[o] = acc[m][n][2 * hf] * s;
                p.outIm[o] = acc[m][n][2 * hf + 1] * s;
            }
        }
}

}  // namespace

extern "C" int af_launch_decimate2(const float *in, int inLength, int inStride, int batch, const float *left32,
                                   const float *right31, float *out, int outStride, void *stream) {
    const int outLength = inLength / 2;
    if (outLength <= 0 || batch <= 0) return AF_OK;
    if (batch > 65535) return af_fail(AF_ERR_ARG, "decimate2: batch %d > 65535 per launch", batch);
    // taps are the same for every object (fixed "Fast" resampler): put them in constant memory once per device
    static int tapsReady[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !tapsReady[dev]) {
        cudaError_t e = cudaMemcpyToSymbolAsync(c_decTaps, left32, 32 * sizeof(float), 0, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
        if (e == cudaSuccess) e = cudaMemcpyToSymbolAsync(c_decTaps, right31, 31 * sizeof(float), 32 * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);   // first use only: visible to every stream afterwards
        if (e != cudaSuccess) return af_cuda_check(e, "cudaMemcpyToSymbolAsync(c_decTaps)");
        if (dev >= 0 && dev < 64) tapsReady[dev] = 1;
    }
    dim3 grid((unsigned)((outLength + kDecTile - 1) / kDecTile), (unsigned)batch);
    k_decimate2<<<grid, kDecThreads, 0, (cudaStream_t)stream>>>(in, inLength, inStride, out, outStride);
    AF_LAUNCH_CHECK("k_decimate2");
    return AF_OK;
}

extern "C" int af_launch_cqt_octave(const float *sig, int sigLength, int sigStride, int batch, int validLength,
                                    int fftLength, int hop, int padLeft, int timeLength, int bpo, const float *kappa2,
                                    const float *scale, int num, int colOff,
                                    float *outRe, float *outIm, void *stream) {
    if (batch <= 0 || timeLength <= 0) return AF_OK;
    if (hop < 1) return af_fail(AF_ERR_ARG, "cqt octave: hop < 1");
    if (batch > 65535) return af_fail(AF_ERR_ARG, "cqt octave: batch %d > 65535 per launch", batch);
    OctParams p;
    p.sig = sig; p.sigStride = sigStride; p.sigLength = sigLength; p.validLength = validLength;
    p.N = fftLength; p.hop = hop; p.T = timeLength; p.bpo = bpo; p.padLeft = padLeft;
    p.kappa = reinterpret_cast<const float2 *>(kappa2); p.scale = scale;
    p.outRe = outRe; p.outIm = outIm; p.outStride = (long long)timeLength * num; p.num = num; p.colOff = colOff;
    p.rowsA = (fftLength + hop - 1) / hop;
    p.nChunk = fftLength < 512 ? fftLength : 512;
    const size_t kBytes = sizeof(float2) * (size_t)kBinsPerPass * p.nChunk;
    // frames per CTA: the largest tile that still lets two CTAs share an SM (<= 100 KB); if that would drop below
    // 256 frames (large hops: the polyphase signal tile is hop x TT floats) take the largest tile that fits at all
    static const int ttChoices[] = {512, 256, 128, 64, 32, 16, 8};
    int TT = 0;
    size_t smem = 0;
    for (int pass = 0; pass < 2 && TT == 0; pass++) {
        for (int c = 0; c < 7; c++) {
            const int tt = ttChoices[c];
            if (pass == 0 && tt < 256) break;
            int rowLen = tt + p.rowsA + 1;
            // pitch chosen so consecutive samples (r fastest) land in different banks while staging
            if (hop >= 32) rowLen |= 1; else { int want = 32 / hop; rowLen = ((rowLen + 31) / 32) * 32 + want; }
            const size_t bytes = kBytes + sizeof(float) * (size_t)hop * rowLen;
            if (bytes <= (size_t)(pass == 0 ? 100 : 200) * 1024) { TT = tt; p.rowLen = rowLen; smem = bytes; break; }
        }
    }
    if (TT == 0) {
        // no tile of the polyphase kernel fits (hop x (8 + fftLength / hop) floats > 150 KB): warp-per-output kernel
        p.TT = 0; p.rowLen = 0; p.segs = 1;
        const long long outs = (long long)timeLength * bpo;
        const dim3 g((unsigned)((outs + 7) / 8), (unsigned)batch);
        k_cqt_octave_direct<<<g, 256, 0, (cudaStream_t)stream>>>(p);
        AF_LAUNCH_CHECK("k_cqt_octave_direct");
        return AF_OK;
    }
    p.TT = TT;
    // enough threads per CTA: split the taps of a frame over up to rowsA segments until the CTA has >= 512 threads
    p.segs = 1;
    while (p.segs * 2 <= p.rowsA && (TT / kFT) * kJG * p.segs * 2 <= 512) p.segs *= 2;
    if ((size_t)(TT / kFT) * kJG * 2 * kFT * kBT * sizeof(float) > kBytes) p.segs = 1;   // reduction scratch must fit the kernel buffer
    cudaError_t e = cudaFuncSetAttribute(k_cqt_octave, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return af_cuda_check(e, "cudaFuncSetAttribute(k_cqt_octave)");
    dim3 grid((unsigned)((timeLength + TT - 1) / TT), (unsigned)batch);
    k_cqt_octave<<<grid, (TT / kFT) * kJG * p.segs, smem, (cudaStream_t)stream>>>(p);
    AF_LAUNCH_CHECK("k_cqt_octave");
    return AF_OK;
}

// Host side of the tensor-core octave kernel: the B-fragment table [N/8][3][32] float4 of the 12 kernels
// (column 2 b = Re kappa_b, 2 b + 1 = Im kappa_b), pre-split into TF32 hi (truncated) and lo (= x - hi) parts.
extern "C" void af_cqt_tc_fragments(const float *kappa2 /* [12][N] (re, im) */, int N, float *out /* N/8 * 96 * 4 */) {
    for (int ks = 0; ks < N / 8; ks++)
        for (int nt = 0; nt < 3; nt++)
            for (int lane = 0; lane < 32; lane++) {
                const int g = lane >> 2, t4 = lane & 3;
                const int col = nt * 8 + g, b = col >> 1, part = col & 1;
                float v[2], hi[2], lo[2];
                for (int i = 0; i < 2; i++) {
                    v[i] = kappa2[((size_t)b * N + ks * 8 + t4 + 4 * i) * 2 + part];
                    uint32_t u;
                    memcpy(&u, &v[i], 4);
                    u &= 0xffffe000u;
                    memcpy(&hi[i], &u, 4);
                    lo[i] = v[i] - hi[i];
                }
                float *o = out + (((size_t)ks * 3 + nt) * 32 + lane) * 4;
                o[0] = hi[0]; o[1] = hi[1]; o[2] = lo[0]; o[3] = lo[1];
            }
}

// tile geometry of the tensor-core kernel: 8 warps x 2 m-tiles = 256 frames when the signal tile fits ~100 KB (two CTAs
// per SM), else fewer warps; returns the dynamic shared-memory bytes, 0 when even one warp does not fit
static size_t cqt_tc_geometry(int fftLength, int hop, int *warpsOut, int *ttOut, int *rowLenOut) {
    const size_t bBytes = sizeof(float4) * kTcKC * 96;
    for (int warps = 8; warps >= 1; warps /= 2) {
        const int TT = warps * 16 * kTcMT;
        int rowLen = TT + fftLength / hop + 1;
        rowLen = ((rowLen + 31) / 32) * 32 + 8;                      // == 8 (mod 32): conflict-free fragment reads
        const size_t sigFloats = hop >= 8 ? (size_t)hop * rowLen : (size_t)(TT - 1) * hop + fftLength;
        const size_t smem = bBytes + sizeof(float) * sigFloats;
        if (smem <= (size_t)100 * 1024 || (warps == 1 && smem <= (size_t)227 * 1024)) {
            *warpsOut = warps; *ttOut = TT; *rowLenOut = rowLen;
            return smem;
        }
    }
    return 0;
}

extern "C" int af_cqt_tc_supported(int fftLength, int hop, int bpo) {
    int w, tt, rl;
    return bpo == 12 && fftLength >= 64 && fftLength % 64 == 0 && hop >= 2 && (hop & (hop - 1)) == 0 &&
           cqt_tc_geometry(fftLength, hop, &w, &tt, &rl) > 0;
}

extern "C" int af_launch_cqt_octave_tc(const float *sig, int sigStride, int batch, int validLength, int fftLength, int hop,
                                       int padLeft, int timeLength, const float *bfrag, const float *scale, int num, int colOff,
                                       float *outRe, float *outIm, void *stream) {
    if (batch <= 0 || timeLength <= 0) return AF_OK;
    if (!af_cqt_tc_supported(fftLength, hop, 12)) return af_fail(AF_ERR_UNSUPPORTED, "cqt octave (tensor core): fftLength %d hop %d", fftLength, hop);
    if (batch > 65535) return af_fail(AF_ERR_ARG, "cqt octave: batch %d > 65535 per launch", batch);
    OctTcParams p;
    p.sig = sig; p.sigStride = sigStride; p.validLength = validLength;
    p.N = fftLength; p.hop = hop; p.T = timeLength; p.padLeft = padLeft;
    p.hs = 0; while ((1 << p.hs) < hop) p.hs++;
    p.bfrag = reinterpret_cast<const float4 *>(bfrag); p.scale = scale;
    p.outRe = outRe; p.outIm = outIm; p.outStride = (long long)timeLength * num; p.num = num; p.colOff = colOff;
    const size_t smem = cqt_tc_geometry(fftLength, hop, &p.warps, &p.TT, &p.rowLen);
    cudaError_t e = cudaFuncSetAttribute(k_cqt_octave_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return af_cuda_check(e, "cudaFuncSetAttribute(k_cqt_octave_tc)");
    dim3 grid((unsigned)((timeLength + p.TT - 1) / p.TT), (unsigned)batch);
    k_cqt_octave_tc<<<grid, p.warps * 32, smem, (cudaStream_t)stream>>>(p);
    AF_LAUNCH_CHECK("k_cqt_octave_tc");
    return AF_OK;
}
