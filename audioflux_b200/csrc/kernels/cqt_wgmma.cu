// cqt_wgmma.cu -- one CQT octave on the Hopper warpgroup tensor cores (wgmma.mma_async, TF32).
//
// Same restatement as cqt.cu (reference: src/cqt_algorithm.c:951-1048, the per-octave STFT + sparse spectral dot,
// rewritten as the strided correlation out[t][b] = sum_n xpad[t*hop + n] kappa_b[n]):
//     D[64 frames x 56] = A[64 x N] . B[N x 56] per warpgroup m-tile,   A[t][n] = xpad[(t0 + t) hop + n]  (a Hankel matrix),
//     B = the 12 time-domain kernels as interleaved (re, im) columns (24 used), TF32 hi parts in rows 0-31, lo in 32-63.
// The Hankel operand is never materialised: each thread loads its A fragment (the mma.m16n8k8 layout, per warp of the
// warpgroup) straight from the staged signal tile into registers, where it is split into TF32 hi / lo.  B is streamed
// chunk by chunk (128 taps, 32 KB: hi and lo) from the host-built image by TMA bulk copies into 128B-swizzled K-major
// shared memory, double-buffered behind an mbarrier each, and read by the tensor cores through matrix descriptors.
// fp32 accuracy with TF32 tensor cores: x = hi + lo (hi = top 19 bits, lo = x - hi exact); per 8 taps one N = 56 wgmma
// A_hi . [B_hi | B_lo] (columns 0-23 and 32-55 used) and one N = 24 wgmma A_lo . B_hi, summed in the epilogue.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "common.cuh"

namespace {

constexpr int kWgChunkK = AF_CQT_WG_CHUNK_K;             // taps per kernel chunk in shared memory
constexpr int kWgChunkBytes = 64 * kWgChunkK * 4;        // one chunk image: 64 rows (32 hi + 32 lo) x 128 taps = 32 KB
constexpr int kWgMT = AF_CQT_WG_MT;                      // 64-frame m-tiles per warpgroup

struct WgParams {
    const float *sig; long long sigStride; int validLength;
    int N, hop, hs, T, padLeft;    // padLeft: N/2 (centre padding) or 0 (streaming)
    const unsigned char *bimg;     // [N / 128 chunks][32 KB] pre-swizzled shared-memory images of B
    const float *scale;            // [12]
    float *outRe, *outIm; long long outStride; int num, colOff;
    int TT, rowLen;                // frames per CTA; polyphase row pitch (hop >= 8)
};

// sm_90 shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 bytes apart
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smemAddr) {
    uint64_t d = 0;
    d |= (uint64_t)((smemAddr >> 4) & 0x3fffu);
    d |= (uint64_t)1 << 16;                      // leading byte offset (unused by swizzled K-major layouts)
    d |= (uint64_t)(1024 >> 4) << 32;            // stride byte offset
    d |= (uint64_t)1 << 62;                      // layout: 128B swizzle
    return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 56] += A[64 x 8] (registers) . B[8 x 56] (descriptor)
__device__ __forceinline__ void wg_n56(float (&d)[28], const uint32_t (&a)[4], uint64_t descB, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %33, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n56k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27}, "
        "{%28, %29, %30, %31}, %32, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(descB), "r"(accumulate));
}

// D[64 x 24] += A[64 x 8] (registers) . B[8 x 24] (descriptor)
__device__ __forceinline__ void wg_n24(float (&d)[12], const uint32_t (&a)[4], uint64_t descB, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %17, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n24k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, "
        "{%12, %13, %14, %15}, %16, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(descB), "r"(accumulate));
}

// Two warpgroups per CTA, kWgMT m-tiles of 64 frames each (TT = 256 frames, or fewer warpgroups / m-tiles when the
// signal tile of a large hop does not fit).  Signal tile layout as in k_cqt_octave_tc: polyphase-major with a row pitch
// == 8 (mod 32) for hop >= 8, linear for hop <= 4, so the fragment loads are conflict-free.
template <int MT>
__global__ void __launch_bounds__(256, 2) k_cqt_octave_wgmma(WgParams p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *sB = smem;                                                      // [2 slots][32 KB]
    float *xs = reinterpret_cast<float *>(smem + 2 * kWgChunkBytes);
    const int h = p.hop, N = p.N, hs = p.hs;
    const bool poly = h >= 8;
    const int span = (p.TT - 1) * h + N;
    const size_t sigFloats = poly ? (size_t)h * p.rowLen : (size_t)span;
    uint64_t *bFull = reinterpret_cast<uint64_t *>(smem + 2 * kWgChunkBytes + ((sigFloats * 4 + 15) & ~(size_t)15));
    const int chunks = N / kWgChunkK;
    const int clip = blockIdx.y;
    const int t0 = blockIdx.x * p.TT;
    const float *sig = p.sig + (long long)clip * p.sigStride;

    if (threadIdx.x == 0) {
        af_mbar_init(&bFull[0], 1);
        af_mbar_init(&bFull[1], 1);
        af_fence_barrier_init();
        af_mbar_arrive_expect_tx(&bFull[0], kWgChunkBytes);
        af_tma_load_1d(sB, p.bimg, kWgChunkBytes, &bFull[0]);
    }

    // stage the tile's span of the zero-padded signal (overlaps the first kernel chunk's copy)
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
    __syncthreads();

    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int g = lane >> 2, t4 = lane & 3;
    const int tb = wg * 64 * MT + warp * 16;                                       // first frame (within the tile) of this warp
    const int rowStep = poly ? 8 : 8 * h;                                          // address step from frame g to frame g + 8
    const int colStep = poly ? 4 * p.rowLen : 4;                                   // address step from tap t4 to tap t4 + 4
    const int mStep = poly ? 64 : 64 * h;                                          // address step from one m-tile to the next
    float dHH[MT][28], dLH[MT][12];
#pragma unroll
    for (int m = 0; m < MT; m++) {
#pragma unroll
        for (int i = 0; i < 28; i++) dHH[m][i] = 0.0f;
#pragma unroll
        for (int i = 0; i < 12; i++) dLH[m][i] = 0.0f;
    }

    for (int c = 0; c < chunks; c++) {
        af_mbar_wait(&bFull[c & 1], (uint32_t)(c >> 1) & 1u);
        // the other slot held chunk c - 1, whose MMAs every warpgroup has waited for before the barrier that ended it
        if (threadIdx.x == 0 && c + 1 < chunks) {
            af_mbar_arrive_expect_tx(&bFull[(c + 1) & 1], kWgChunkBytes);
            af_tma_load_1d(sB + (size_t)((c + 1) & 1) * kWgChunkBytes, p.bimg + (size_t)(c + 1) * kWgChunkBytes, kWgChunkBytes,
                           &bFull[(c + 1) & 1]);
        }
        const uint32_t bBase = af_smem_u32(sB + (size_t)(c & 1) * kWgChunkBytes);
#pragma unroll 4
        for (int ks = 0; ks < kWgChunkK / 8; ks++) {
            const int n0 = c * kWgChunkK + ks * 8;
            const int base = poly ? ((n0 & (h - 1)) + t4) * p.rowLen + (n0 >> hs) + tb + g : (tb + g) * h + n0 + t4;
            uint32_t ah[MT][4], al[MT][4];
#pragma unroll
            for (int m = 0; m < MT; m++) {
                const float *a = xs + base + m * mStep;
                const float af[4] = {a[0], a[rowStep], a[colStep], a[colStep + rowStep]};
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    ah[m][i] = __float_as_uint(af[i]) & 0xffffe000u;
                    al[m][i] = __float_as_uint(af[i] - __uint_as_float(ah[m][i]));
                }
            }
            // K atom ks / 4 of the chunk image (64 rows x 128 B), 8-tap step ks % 4 inside it (+32 bytes)
            const uint64_t dB = wg_desc_sw128(bBase + (uint32_t)(ks >> 2) * 8192u + (uint32_t)(ks & 3) * 32u);
            wg_fence();
#pragma unroll
            for (int m = 0; m < MT; m++) {
                wg_n56(dHH[m], ah[m], dB, 1u);
                wg_n24(dLH[m], al[m], dB, 1u);
            }
            wg_commit();
            wg_wait0();
        }
        __syncthreads();                                                           // slot c & 1 may be refilled
    }

    // D fragment: rows g / g + 8 of the warp's 16 = frames, columns 8 i + 2 t4 (+1) = (re, im) of bin 4 i + t4;
    // columns 32 + 8 i + 2 t4 (+1) of the N = 56 accumulator hold the A_hi . B_lo part of the same bin
#pragma unroll
    for (int m = 0; m < MT; m++)
#pragma unroll
        for (int i = 0; i < 3; i++) {
            const int j = 4 * i + t4;
            const float s = p.scale[j];
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                const int t = t0 + tb + 64 * m + g + 8 * hf;
                if (t >= p.T) continue;
                const int e = 4 * i + 2 * hf;
                const long long o = (long long)clip * p.outStride + (long long)t * p.num + p.colOff + j;
                p.outRe[o] = (dHH[m][e] + dLH[m][e] + dHH[m][e + 16]) * s;
                p.outIm[o] = (dHH[m][e + 1] + dLH[m][e + 1] + dHH[m][e + 17]) * s;
            }
        }
}

}  // namespace

// Pre-swizzled shared-memory images of the B operand: per 128-tap chunk ONE K-major 128B-swizzled [64 rows][128 k] matrix
// whose rows 0-31 are the TF32 hi parts of the 24 (+8 zero) columns and rows 32-63 the lo parts; a K atom (32 taps) is
// 64 rows x 128 B = 8192 B (8 groups of 8 rows).  A_hi . [B_hi | B_lo] is then one N = 56 MMA and A_lo . B_hi an N = 24
// MMA on the first 24 rows of the same image.
extern "C" void af_cqt_wgmma_bimage(const float *kappa2 /* [12][N] (re, im) */, int N, unsigned char *out /* N/128 * 32 KB */) {
    memset(out, 0, (size_t)(N / kWgChunkK) * kWgChunkBytes);
    for (int c = 0; c < N / kWgChunkK; c++)
        for (int n = 0; n < 24; n++)
            for (int k = 0; k < kWgChunkK; k++) {
                const int b = n >> 1, part = n & 1;
                const float v = kappa2[((size_t)b * N + c * kWgChunkK + k) * 2 + part];
                uint32_t u;
                memcpy(&u, &v, 4);
                u &= 0xffffe000u;
                float hi;
                memcpy(&hi, &u, 4);
                const float lo = v - hi;
                const int ka = k >> 5, kk = k & 31;
                for (int half = 0; half < 2; half++) {
                    const int row = n + 32 * half, g = row >> 3, r = row & 7;
                    const size_t off = (size_t)ka * 8192 + (size_t)g * 1024 + (size_t)r * 128 + (size_t)(((kk >> 2) ^ r) * 16) + (size_t)(kk & 3) * 4;
                    memcpy(out + (size_t)c * kWgChunkBytes + off, half ? &lo : &hi, 4);
                }
            }
}

// tile geometry from af_cqt_octave_plan (host/af_cqt.c): two warpgroups x kWgMT m-tiles (256 frames) when the CTA fits
// ~113 KB (two CTAs per SM), else smaller tiles
extern "C" int af_launch_cqt_octave_wgmma(const AfCqtOctPlan *plan, const float *sig, int sigStride, int batch, int validLength,
                                          int fftLength, int hop, int padLeft, int timeLength, const unsigned char *bimg,
                                          const float *scale, int num, int colOff, float *outRe, float *outIm, void *stream) {
    if (batch <= 0 || timeLength <= 0) return AF_OK;
    if (plan->kernel != AF_CQT_WGMMA || !bimg)
        return af_fail(AF_ERR_UNSUPPORTED, "cqt octave (wgmma): fftLength %d hop %d", fftLength, hop);
    if (batch > 65535) return af_fail(AF_ERR_ARG, "cqt octave: batch %d > 65535 per launch", batch);
    WgParams p;
    p.sig = sig; p.sigStride = sigStride; p.validLength = validLength;
    p.N = fftLength; p.hop = hop; p.T = timeLength; p.padLeft = padLeft;
    p.hs = 0; while ((1 << p.hs) < hop) p.hs++;
    p.bimg = bimg; p.scale = scale;
    p.outRe = outRe; p.outIm = outIm; p.outStride = (long long)timeLength * num; p.num = num; p.colOff = colOff;
    p.rowLen = plan->rowLen;
    p.TT = plan->TT;
    const dim3 grid((unsigned)((timeLength + p.TT - 1) / p.TT), (unsigned)batch);
    int rc;
    if (plan->mt == kWgMT) {
        if ((rc = af_smem_optin(k_cqt_octave_wgmma<kWgMT>, plan->smem, "k_cqt_octave_wgmma"))) return rc;
        k_cqt_octave_wgmma<kWgMT><<<grid, plan->threads, plan->smem, (cudaStream_t)stream>>>(p);
    } else {
        if ((rc = af_smem_optin(k_cqt_octave_wgmma<1>, plan->smem, "k_cqt_octave_wgmma"))) return rc;
        k_cqt_octave_wgmma<1><<<grid, plan->threads, plan->smem, (cudaStream_t)stream>>>(p);
    }
    AF_LAUNCH_CHECK("k_cqt_octave_wgmma");
    return AF_OK;
}
