// mfcc_fused.cu -- fused framed-STFT(2048) -> |X|^2 / |X| -> banded filter bank -> log10 / cbrt ->
// ortho DCT-II -> first ccNum coefficients, one persistent kernel, samples read from HBM once.
//
// Replaces, for fftLength = 2048, the whole chain
//   stftObj_stft  (src/stft_algorithm.c:696-715, 790-801)  -> __mccut (src/reassign_algorithm.c:600-604)
//   -> __mcsquare / sqrtf (src/bft_algorithm.c:489-497) -> __mdot1 (:515-518)
//   -> log10f clamp / powf(1/3) (src/feature/xxcc_algorithm.c:124-140) -> fftObj_dct (:142-149) -> cut (:151-155)
// of the reference, which makes 6 passes over T x 2048 floats per clip plus a dense 1025 x 128 dot.
//
// Structure (one CTA per SM, persistent, static tile schedule => bit-identical results for any
// batch size / GPU count):
//   * warp W (of kFrameWarps) owns frame f0+W of the current tile; a tile is `framesPerTile`
//     consecutive frames of one clip whose sample span [(f0*hop), (f0+F-1)*hop + 2048) is brought
//     into shared memory ONCE by a 1-D TMA bulk copy (cp.async.bulk + mbarrier complete_tx),
//     double buffered through a full/empty mbarrier ring fed by a dedicated producer warp;
//   * the 2048 real samples are packed as 1024 complex points and transformed as 32 x 32:
//     lane n1 holds z[n1 + 32*n2] in registers (one complex value per 64-bit register pair, all
//     butterflies on (re, im) register pairs, c64.cuh), a generated straight-line 32-point DFT runs over n2,
//     twiddles W_1024^(n1*k) come half from a conflict-free transposed shared table and half from one
//     extra multiply by W_64^n1, a 33-padded shared transpose regroups the data (warp-private,
//     __syncwarp only), a second 32-point DFT runs over n1;  lane l then holds Z[l + 32*kb];
//   * real-FFT post-pass pairs bin k with 1024-k through one warp shuffle per component (both
//     powers |E +- W*O|^2 come from one evaluation);
//   * the banded bank is applied lane-per-filter from a zero-padded transposed weight table whose
//     per-filter start bins are shifted down (host planner) until the 32 lanes of a group read 32
//     different banks -> conflict-free;
//   * DCT-II is the one dense GEMM-shaped piece ([frames x 128] . [128 x cc]): the frame warps drop their
//     log-mel rows into a multi-buffered (kLBufs) 16 x 128 shared tile and a dedicated epilogue warp contracts the
//     whole tile on the tensor cores (mma.sync m16n8k8 TF32, 3xTF32 split so the result keeps fp32 accuracy)
//     while the frame warps are already transforming the next tile.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "common.cuh"
#include "fft32_gen.cuh"

namespace {

constexpr int kN = 2048;            // fftLength
constexpr int kNC = 1024;           // packed complex points
#ifndef AF_FRAME_WARPS
#define AF_FRAME_WARPS 13
#endif
constexpr int kFrameWarps = AF_FRAME_WARPS;     // consumer warps = max frames per tile (<= 16: one mma M tile); 13 by default
#ifndef AF_ABLATE
#define AF_ABLATE 0     // diagnostic timing builds: 1 no bank loop, 2 no post-pass, 4 no FFTs, 8 no transposes, 16 no window/sample loads
#endif
#ifndef AF_EPI_WARPS
#define AF_EPI_WARPS 2
#endif
#ifndef AF_CTAS_PER_SM
#define AF_CTAS_PER_SM 1
#endif
constexpr int kEpiWarps = AF_EPI_WARPS;   // DCT epilogue warps; tile `it` is served by warp it % kEpiWarps
constexpr int kCtasPerSm = AF_CTAS_PER_SM;   // independent CTAs per SM drift apart, so their phases (LSU-heavy load /
                                             // transpose / bank vs FMA-heavy FFT) overlap instead of queueing on one pipe
constexpr int kThreads = (kFrameWarps + 1 + kEpiWarps) * 32;   // + TMA producer warp + DCT epilogue warps
constexpr int kMaxPeers = 15;      // extra destinations of the output tile (P2P stores to peer GPUs)
constexpr int kLPitch = 132;        // log-mel tile row pitch (floats): 4g + t -> 32 distinct banks for mma A fragments
constexpr int kLRows = kFrameWarps <= 8 ? 8 : 16;   // stored rows of the mma M=16 tile (rows beyond are zeros)
constexpr int kStages = 2;
#ifndef AF_LBUFS
#define AF_LBUFS 3
#endif
constexpr int kLBufs = AF_LBUFS;    // log-mel tiles in flight between the frame warps and the DCT epilogue (2 leaves frame
                                    // warps waiting for the epilogue)
constexpr int kMaxNum = 128;        // filters (padded)
constexpr int kScratchFloats = 1152;            // per warp: 33x32 float transpose plane, later Ps[0..1024] + zero pad
constexpr int kPsPad = 1152;        // Ps[0..1024], zeros up to kPsPad (padded band reads)
constexpr int kTailMax = 512;       // bins above the last filter's peak (interval mode)
constexpr int kStageBytes = 16 * 64 * 4;   // result tile of one epilogue warp (<= 16 frames x 64 coefficients), source of the bulk stores

struct Plan {                       // host-side descriptor of the device tables
    float *dWindowHalf;             // 2048, window * 0.5
    float2 *dTw1;                   // [17 ka][32 n1]  W_1024^(n1*ka), ka = 0..16
    float2 *dTw2;                   // [32]            W_2048^lane (post-pass base twiddle)
    float *dMelW;                   // transposed zero-padded weights, group after group: [len_g][32]
    int *dMelStart;                 // 128
    float *dDct;                    // [128 m][dctPitch] ortho DCT-II, B operand of the epilogue mma (pitch % 32 == 8)
    int melGroupLen[4];
    int melGroups;
    int melWFloats;
    int num, ccNum, ct, dataType;
    // interval ("shared product") form of a triangular bank, see build_intervals()
    int melMode;                    // 0: lane per filter over its whole support; 1: lane per interval
    float *dMelAux;                 // [128 gains][kTailMax tail weights]
    int tailStart, tailLen;
};

struct Params {
    const float *data;
    float *out;
    const float *windowHalf;
    const float2 *tw1, *tw2;
    const float *melW;
    const int *melStart;
    const float *dct;
    long long dataStride;
    int batch, timeLength, hop;
    int framesPerTile, tilesPerClip;
    long long totalTiles;
    int spanFloats;                 // floats per stage buffer
    int melGroups, melWFloats;
    int melGroupLen[4];
    int melMode, num, tailStart, tailLen;
    const float *melAux;
    int ccNum, rectify, dataType;
    int rawMel;                     // 1: stop after the bank: out[frame][num] = bank . |X|^2 (bftObj_bft real mode), no log / DCT
    int bulkStore;                  // 1: the result tile leaves as one TMA bulk store per destination (16-byte aligned rows)
    // fused all-gather: every finished tile is also stored at the same offset of up to kMaxPeers other buffers
    // (peer GPUs' gathered arrays mapped over NVLink, opened with cudaIpcOpenMemHandle by the host side)
    int nPeer;
    float *peerOut[kMaxPeers];
};

// shared-memory carve-up (bytes), all 16-byte aligned
struct Smem {
    int spanOff, scratchOff, windowOff, tw1Off, tw2Off, melWOff, melStartOff, melAuxOff, dctOff, lOff, stageOff, barOff, total;
};

__host__ __device__ inline Smem carve(int spanFloats, int melWFloats, int ct) {
    Smem s; int o = 0;
    s.spanOff = o;     o += kStages * spanFloats * 4;
    s.scratchOff = o;  o += kFrameWarps * kScratchFloats * 4;
    s.windowOff = o;   o += kN * 4;
    s.tw1Off = o;      o += 17 * 32 * 8;
    s.tw2Off = o;      o += 32 * 8;
    s.melWOff = o;     o += ((melWFloats * 4 + 15) / 16) * 16;
    s.melStartOff = o; o += kMaxNum * 4;
    s.melAuxOff = o;   o += (kMaxNum + kTailMax) * 4;
    s.dctOff = o;      o += kMaxNum * (ct <= 5 ? 40 : 72) * 4;
    s.lOff = o;        o += kLBufs * kLRows * kLPitch * 4;
    s.stageOff = o;    o += kEpiWarps * kStageBytes;
    s.barOff = o;      o += (2 * kStages + 2 * kLBufs) * 8;
    s.total = o;
    return s;
}

template <int CT, int MODE>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) k_mfcc_fused(Params p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const Smem L = carve(p.spanFloats, p.melWFloats, CT);
    float *span = reinterpret_cast<float *>(smem + L.spanOff);
    float *scratchAll = reinterpret_cast<float *>(smem + L.scratchOff);
    float2 *sWin2 = reinterpret_cast<float2 *>(smem + L.windowOff);
    float2 *sTw1 = reinterpret_cast<float2 *>(smem + L.tw1Off);
    float2 *sTw2 = reinterpret_cast<float2 *>(smem + L.tw2Off);
    float *sMelW = reinterpret_cast<float *>(smem + L.melWOff);
    int *sMelStart = reinterpret_cast<int *>(smem + L.melStartOff);
    float *sMelAux = reinterpret_cast<float *>(smem + L.melAuxOff);     // interval mode: [128 gains][tail weights]
    float *sDct = reinterpret_cast<float *>(smem + L.dctOff);
    float *sL = reinterpret_cast<float *>(smem + L.lOff);                 // [kLBufs][kLRows][kLPitch] log-mel tiles
    uint64_t *fullBar = reinterpret_cast<uint64_t *>(smem + L.barOff);
    uint64_t *emptyBar = fullBar + kStages;
    uint64_t *lFull = emptyBar + kStages;                                  // [kLBufs] frame warps -> epilogue
    uint64_t *lEmpty = lFull + kLBufs;                                     // [kLBufs] epilogue -> frame warps
    constexpr int kDctPitch = CT <= 5 ? 40 : 72;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // ---- one-time: tables -> shared, barriers ----
    for (int i = threadIdx.x; i < kN; i += kThreads) reinterpret_cast<float *>(sWin2)[i] = p.windowHalf[i];
    for (int i = threadIdx.x; i < 17 * 32; i += kThreads) sTw1[i] = p.tw1[i];
    for (int i = threadIdx.x; i < 32; i += kThreads) sTw2[i] = p.tw2[i];
    for (int i = threadIdx.x; i < p.melWFloats; i += kThreads) sMelW[i] = p.melW[i];
    for (int i = threadIdx.x; i < kMaxNum; i += kThreads) sMelStart[i] = p.melStart[i];
    for (int i = threadIdx.x; i < kMaxNum + kTailMax; i += kThreads) sMelAux[i] = MODE ? p.melAux[i] : 0.0f;
    for (int i = threadIdx.x; i < kMaxNum * kDctPitch; i += kThreads) sDct[i] = p.dct[i];
    for (int i = threadIdx.x; i < kLBufs * kLRows * kLPitch; i += kThreads) sL[i] = 0.0f;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; s++) { af_mbar_init(&fullBar[s], 1); af_mbar_init(&emptyBar[s], kFrameWarps); }
        for (int s = 0; s < kLBufs; s++) { af_mbar_init(&lFull[s], kFrameWarps); af_mbar_init(&lEmpty[s], 1); }
        af_fence_barrier_init();
    }
    __syncthreads();

    const int F = p.framesPerTile;

    if (warp == kFrameWarps) {
        // ================= producer: one lane streams tile spans with TMA =================
        if (lane == 0) {
            int it = 0;
            for (long long tile = blockIdx.x; tile < p.totalTiles; tile += gridDim.x, ++it) {
                const int stage = it % kStages;
                const uint32_t round = (uint32_t)(it / kStages);
                af_mbar_wait_sleepy(&emptyBar[stage], (round & 1u) ^ 1u);
                const long long clip = tile / p.tilesPerClip;
                const int f0 = (int)(tile % p.tilesPerClip) * F;
                const int nf = min(F, p.timeLength - f0);
                const uint32_t bytes = (uint32_t)(((nf - 1) * p.hop + kN) * 4);
                af_mbar_arrive_expect_tx(&fullBar[stage], bytes);
                af_tma_load_1d(span + (size_t)stage * p.spanFloats,
                               p.data + clip * p.dataStride + (long long)f0 * p.hop, bytes, &fullBar[stage]);
            }
        }
        return;
    }

    if (warp > kFrameWarps) {
        // ================= epilogue: DCT-II of a whole tile on the tensor cores =================
        // out[16 x 8*CT] = L[16 x 128] . D^T[128 x 8*CT], mma.sync.m16n8k8 TF32 with the 3xTF32 split
        // (x = hi + lo, hi = tf32(x), lo = tf32(x - hi);  lo*hi + hi*lo + hi*hi) -> fp32-level accuracy.
        if (p.rawMel) return;                                  // filter-bank output only: no cepstral epilogue
        const int g = lane >> 2, t = lane & 3;
        const int epi = warp - (kFrameWarps + 1);
        int it = 0;
        for (long long tile = blockIdx.x; tile < p.totalTiles; tile += gridDim.x, ++it) {
            if (it % kEpiWarps != epi) continue;
            const int buf = it % kLBufs;
            const long long clip = tile / p.tilesPerClip;
            const int f0 = (int)(tile % p.tilesPerClip) * F;
            const int nf = min(F, p.timeLength - f0);
            af_mbar_wait_sleepy(&lFull[buf], (uint32_t)(it / kLBufs) & 1u);
            const float *A = sL + (size_t)buf * kLRows * kLPitch;
            // two accumulator sets (hi*hi and the two cross terms) and term-major issue order: consecutive HMMAs
            // never touch the same accumulator, so the in-order warp is not serialised on the mma latency
            float acc[CT][4], acx[CT][4];
#pragma unroll
            for (int n = 0; n < CT; n++) {
                acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.0f;
                acx[n][0] = acx[n][1] = acx[n][2] = acx[n][3] = 0.0f;
            }
#define AF_MMA_TF32(ACC, A0, A1, A2, A3, B0, B1)                                                              \
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" \
        : "+f"(ACC[0]), "+f"(ACC[1]), "+f"(ACC[2]), "+f"(ACC[3])                                              \
        : "r"(A0), "r"(A1), "r"(A2), "r"(A3), "r"(B0), "r"(B1))
#pragma unroll 2
            for (int k0 = 0; k0 < kMaxNum; k0 += 8) {
                const float af[4] = {A[g * kLPitch + k0 + t], kLRows > 8 ? A[(g + 8) * kLPitch + k0 + t] : 0.0f,
                                     A[g * kLPitch + k0 + t + 4], kLRows > 8 ? A[(g + 8) * kLPitch + k0 + t + 4] : 0.0f};
                // TF32 split by truncation: hi = top 19 bits, lo = (x - hi) (exact), again cut to 19 bits
                uint32_t ah[4], al[4], bh[CT][2], bl[CT][2];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    ah[i] = __float_as_uint(af[i]) & 0xffffe000u;
                    al[i] = __float_as_uint(af[i] - __uint_as_float(ah[i])) & 0xffffe000u;
                }
#pragma unroll
                for (int n = 0; n < CT; n++) {
                    const float bf[2] = {sDct[(k0 + t) * kDctPitch + n * 8 + g], sDct[(k0 + t + 4) * kDctPitch + n * 8 + g]};
#pragma unroll
                    for (int i = 0; i < 2; i++) {
                        bh[n][i] = __float_as_uint(bf[i]) & 0xffffe000u;
                        bl[n][i] = __float_as_uint(bf[i] - __uint_as_float(bh[n][i])) & 0xffffe000u;
                    }
                }
#pragma unroll
                for (int n = 0; n < CT; n++) AF_MMA_TF32(acx[n], al[0], al[1], al[2], al[3], bh[n][0], bh[n][1]);
#pragma unroll
                for (int n = 0; n < CT; n++) AF_MMA_TF32(acc[n], ah[0], ah[1], ah[2], ah[3], bh[n][0], bh[n][1]);
#pragma unroll
                for (int n = 0; n < CT; n++) AF_MMA_TF32(acx[n], ah[0], ah[1], ah[2], ah[3], bl[n][0], bl[n][1]);
            }
#undef AF_MMA_TF32
#pragma unroll
            for (int n = 0; n < CT; n++)
#pragma unroll
                for (int i = 0; i < 4; i++) acc[n][i] += acx[n][i];
            __syncwarp();
            if (lane == 0) af_mbar_arrive(&lEmpty[buf]);           // tile consumed: frame warps may overwrite it
            // C fragment: rows g and g+8, columns n*8 + 2t, +1.  Destination 0 is this GPU's buffer, 1..nPeer the
            // peers' (the all-gather of the result rides on the epilogue, tile by tile).  The tile is a contiguous run of
            // nf * ccNum floats in every destination: it is staged in shared memory and leaves as ONE TMA bulk store per
            // destination (full lines over NVLink rather than 32-bit scalars).
            const long long tileOff = ((long long)clip * p.timeLength + f0) * p.ccNum;
            if (p.bulkStore) {
                float *stage = reinterpret_cast<float *>(smem + L.stageOff + epi * kStageBytes);
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");       // this warp's previous stores have read the staging tile
                __syncwarp();
#pragma unroll
                for (int n = 0; n < CT; n++) {
                    const int c = n * 8 + 2 * t;
                    if (g < nf) {
                        if (c < p.ccNum) stage[g * p.ccNum + c] = acc[n][0];
                        if (c + 1 < p.ccNum) stage[g * p.ccNum + c + 1] = acc[n][1];
                    }
                    if (g + 8 < nf) {
                        if (c < p.ccNum) stage[(g + 8) * p.ccNum + c] = acc[n][2];
                        if (c + 1 < p.ccNum) stage[(g + 8) * p.ccNum + c + 1] = acc[n][3];
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane <= p.nPeer) {
                    float *o = (lane == 0 ? p.out : p.peerOut[lane - 1]) + tileOff;
                    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                                 ::"l"(o), "r"(af_smem_u32(stage)), "r"((uint32_t)(nf * p.ccNum * 4)) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            } else {
                for (int d = 0; d <= p.nPeer; d++) {
                    float *o = (d == 0 ? p.out : p.peerOut[d - 1]) + tileOff;
#pragma unroll
                    for (int n = 0; n < CT; n++) {
                        const int c = n * 8 + 2 * t;
                        if (g < nf) {
                            if (c < p.ccNum) o[(long long)g * p.ccNum + c] = acc[n][0];
                            if (c + 1 < p.ccNum) o[(long long)g * p.ccNum + c + 1] = acc[n][1];
                        }
                        if (g + 8 < nf) {
                            if (c < p.ccNum) o[(long long)(g + 8) * p.ccNum + c] = acc[n][2];
                            if (c + 1 < p.ccNum) o[(long long)(g + 8) * p.ccNum + c + 1] = acc[n][3];
                        }
                    }
                }
            }
        }
        if (p.bulkStore) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        return;
    }

    // ================= consumers: warp `warp` computes frame f0 + warp of every tile =================
    float *scratch = scratchAll + (size_t)warp * kScratchFloats;
    const int partner = (32 - lane) & 31;
    const c64 w16 = c_from(sTw1[16 * 32 + lane]);            // W_1024^(16*lane) = W_64^lane
    const c64 wBase = c_from(sTw2[lane]);                    // W_2048^lane
    const c64 *sWinC = reinterpret_cast<const c64 *>(sWin2);
    const c64 *sTw1C = reinterpret_cast<const c64 *>(sTw1);

    int it = 0;
    for (long long tile = blockIdx.x; tile < p.totalTiles; tile += gridDim.x, ++it) {
        const int stage = it % kStages;
        const uint32_t round = (uint32_t)(it / kStages);
        const int f0 = (int)(tile % p.tilesPerClip) * F;
        const int nf = min(F, p.timeLength - f0);
        const bool active = warp < nf;

        af_mbar_wait(&fullBar[stage], round & 1u);

        c64 z[32];
        if (active) {
            // ---- A: load 2048 samples (1024 packed pairs), apply 0.5*window ----
            const c64 *sp = reinterpret_cast<const c64 *>(span + (size_t)stage * p.spanFloats + warp * p.hop);
#pragma unroll
            for (int j = 0; j < 32; j++) z[j] = (AF_ABLATE & 16) ? c_pack(1.0f + j, lane) : v_mul(sp[lane + 32 * j], sWinC[lane + 32 * j]);
        }
        __syncwarp();
        if (lane == 0) af_mbar_arrive(&emptyBar[stage]);     // span slot may be refilled
        const int lbuf = it % kLBufs;
        float *lrow = sL + ((size_t)lbuf * kLRows + warp) * kLPitch;
        float *melRow = p.out + ((tile / p.tilesPerClip) * p.timeLength + f0 + warp) * (long long)p.num;   // rawMel destination
        if (!active && p.rawMel) continue;
        if (!active) {
            // keep the log-mel tile protocol in step: one arrival per warp per tile, never before the
            // epilogue released this buffer (tile it-2), else an early arrival would complete the wrong phase
            af_mbar_wait(&lEmpty[lbuf], ((uint32_t)(it / kLBufs) & 1u) ^ 1u);
            if (lane == 0) af_mbar_arrive(&lFull[lbuf]);
            continue;
        }

        // ---- B: 1024-point FFT as 32 x 32 ----
        if (!(AF_ABLATE & 4)) af_fft32(z);                    // over n2; Y[n1=lane][ka] at AF_BR5(ka)
        {
            float yr[32], yi[32];
#pragma unroll
            for (int ka = 0; ka < 32; ka++) {                 // times W_1024^(lane*ka) = W^(lane*(ka&15)) * W^(16*lane*(ka>>4))
                c64 y = z[AF_BR5(ka)];
                if (ka >= 16) y = c_mul(y, w16);
                if (ka & 15) y = c_mul(y, sTw1C[(ka & 15) * 32 + lane]);
                c_unpack(y, yr[ka], yi[ka]);
            }
            // 32 x 32 transpose, real plane then imaginary plane, through one 33-padded float buffer
            if (!(AF_ABLATE & 8)) {
#pragma unroll
            for (int ka = 0; ka < 32; ka++) scratch[ka * 33 + lane] = yr[ka];
            __syncwarp();
#pragma unroll
            for (int n1 = 0; n1 < 32; n1++) yr[n1] = scratch[lane * 33 + n1];
            __syncwarp();
#pragma unroll
            for (int ka = 0; ka < 32; ka++) scratch[ka * 33 + lane] = yi[ka];
            __syncwarp();
#pragma unroll
            for (int n1 = 0; n1 < 32; n1++) z[n1] = c_pack(yr[n1], scratch[lane * 33 + n1]);
            __syncwarp();
            } else {
#pragma unroll
                for (int n1 = 0; n1 < 32; n1++) z[n1] = c_pack(yr[n1], yi[n1]);
            }
        }
        if (!(AF_ABLATE & 4)) af_fft32(z);                    // over n1; Z[lane + 32*kb] at AF_BR5(kb)

        // ---- C: real-FFT post-pass + power / magnitude -> Ps[0..1024] ----
        // (window pre-scaled by 1/2, so E' = Z[k] + conj Z[N-k] and O' = -i (Z[k] - conj Z[N-k]) need no halving;
        //  X[k] = E' + W O', conj X[N-k] = E' - W O' with W = W_2048^k = W_2048^lane * W_64^kb)
#pragma unroll
        for (int kb = 0; kb < ((AF_ABLATE & 2) ? 1 : 16); kb++) {
            const c64 zk = z[AF_BR5(kb)];
            float pr, pi;
            c_unpack(z[AF_BR5(31 - kb)], pr, pi);
            pr = __shfl_sync(0xffffffffu, pr, partner);
            pi = __shfl_sync(0xffffffffu, pi, partner);
            c64 zp = c_pack(pr, pi);
            if (lane == 0) zp = z[AF_BR5((32 - kb) & 31)];
            const c64 zc = c_conj(zp);
            const c64 e = c_add(zk, zc);
            c64 o = c_mul_mi(c_sub(zk, zc));
            o = af_mul_w64(o, kb);                             // compile-time constant twiddle
            const c64 wo = c_mul(o, wBase);
            float pk = c_norm2(c_add(e, wo)), pn = c_norm2(c_sub(e, wo));
            if (p.dataType == SpectralData_Mag) { pk = sqrtf(pk); pn = sqrtf(pn); }
            const int k = lane + 32 * kb;
            scratch[k] = pk;
            scratch[kNC - k] = pn;
        }
        if (lane == 0) {                                       // k = 512 pairs with itself
            float pk = 4.0f * c_norm2(z[AF_BR5(16)]);
            if (p.dataType == SpectralData_Mag) pk = sqrtf(pk);
            scratch[512] = pk;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {                          // zero pad behind Ps for padded band reads
            const int idx = kNC + 1 + lane + 32 * i;
            if (idx < kPsPad) scratch[idx] = 0.0f;
        }
        __syncwarp();

        // ---- D: banded filter bank (lane = filter within group, bank-conflict-free starts) + rectify ----
        if (!p.rawMel) af_mbar_wait(&lEmpty[lbuf], ((uint32_t)(it / kLBufs) & 1u) ^ 1u);   // epilogue done with tile it-kLBufs
        if (MODE) {
            // Interval form of a triangular bank (two filters overlap on every bin and their weights there sum to the
            // filters' gains: fall_m(k) = g_m (1 - r_{m+1}(k))).  Lane j owns interval j = the bins between the peaks
            // of filters j-1 and j and accumulates A_j = sum r_j P and S_j = sum P ONCE; then
            //     mel_m = g_m (A_m + (S_{m+1} - A_{m+1})),
            // i.e. every bin is read and multiplied once instead of twice (half the shared-memory traffic of the
            // filter-per-lane loop).  Padded slots carry r = 0 and are masked out of S by the (r > 0) test.
            const float4 *wg4 = reinterpret_cast<const float4 *>(sMelW) + lane;
            float A[4], U[4];
#pragma unroll
            for (int g = 0; g < 4; g++) {
                A[g] = 0.0f; U[g] = 0.0f;
                if (g >= p.melGroups) continue;
                const int len4 = (AF_ABLATE & 1) ? 0 : p.melGroupLen[g] >> 2;
                const float2 *ps2 = reinterpret_cast<const float2 *>(scratch + sMelStart[g * 32 + lane]);
                float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f, s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
                float4 w = wg4[0];
                float2 p0 = ps2[0], p1 = ps2[1];
#pragma unroll 2
                for (int i = 0; i < len4; i++) {
                    const float4 wn = wg4[(i + 1) * 32];
                    const float2 q0 = ps2[2 * i + 2], q1 = ps2[2 * i + 3];
                    a0 = fmaf(p0.x, w.x, a0); a1 = fmaf(p0.y, w.y, a1); a2 = fmaf(p1.x, w.z, a2); a3 = fmaf(p1.y, w.w, a3);
                    if (!(AF_ABLATE & 32)) {
                        s0 = fmaf(p0.x, w.x > 0.0f ? 1.0f : 0.0f, s0); s1 = fmaf(p0.y, w.y > 0.0f ? 1.0f : 0.0f, s1);
                        s2 = fmaf(p1.x, w.z > 0.0f ? 1.0f : 0.0f, s2); s3 = fmaf(p1.y, w.w > 0.0f ? 1.0f : 0.0f, s3);
                    }
                    w = wn; p0 = q0; p1 = q1;
                }
                A[g] = (a0 + a1) + (a2 + a3);
                U[g] = ((s0 + s1) + (s2 + s3)) - A[g];
                wg4 += len4 * 32;
            }
            // tail interval (above the last filter's peak): its falling weights directly, one bin per lane
            float ut = 0.0f;
            if (!(AF_ABLATE & 64)) for (int i = lane; i < p.tailLen; i += 32) ut = fmaf(scratch[p.tailStart + i], sMelAux[kMaxNum + i], ut);
            if (!(AF_ABLATE & 64))
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) ut += __shfl_xor_sync(0xffffffffu, ut, o);
#pragma unroll
            for (int g = 0; g < 4; g++) {
                if (g >= p.melGroups) { lrow[g * 32 + lane] = 0.0f; continue; }
                float un = U[g];
                if (!(AF_ABLATE & 64)) {
                    un = __shfl_down_sync(0xffffffffu, U[g], 1);
                    const float nextFirst = __shfl_sync(0xffffffffu, U[g < 3 ? g + 1 : 3], 0);
                    if (lane == 31) un = nextFirst;
                }
                const int m = g * 32 + lane;
                if (m + 1 == p.num) un = ut;
                float v = m < p.num ? sMelAux[m] * (A[g] + un) : 0.0f;
                if (p.rectify == CepstralRectify_CubicRoot) v = powf(v, 1.0f / 3.0f);
                else v = __log2f(v < 1e-8f ? 1e-8f : v) * 0.30102999566398120f;
                lrow[m] = m < p.num ? v : 0.0f;
            }
        } else
        {
            // weights: per group [len/4][32 lanes] float4 (LDS.128); P: two LDS.64 per 4 taps (starts are even and
            // spread over distinct 8-byte bank pairs per half-warp by the host planner)
            const float4 *wg4 = reinterpret_cast<const float4 *>(sMelW) + lane;
            for (int g = 0; g < p.melGroups; g++) {
                const int len4 = (AF_ABLATE & 1) ? 0 : p.melGroupLen[g] >> 2;
                const float2 *ps2 = reinterpret_cast<const float2 *>(scratch + sMelStart[g * 32 + lane]);
                float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f, acc3 = 0.0f;
                // software pipelined: the loads of stage i+1 are in flight while stage i is accumulated
                // (the final prefetch over-reads one stage: the tables carry the padding).  A two-stage-deep
                // pipeline needs 128 registers and a longer prologue per group.
                float4 w = wg4[0];
                float2 p0 = ps2[0], p1 = ps2[1];
#pragma unroll 2
                for (int i = 0; i < len4; i++) {
                    const float4 wn = wg4[(i + 1) * 32];
                    const float2 q0 = ps2[2 * i + 2], q1 = ps2[2 * i + 3];
                    acc0 = fmaf(p0.x, w.x, acc0);
                    acc1 = fmaf(p0.y, w.y, acc1);
                    acc2 = fmaf(p1.x, w.z, acc2);
                    acc3 = fmaf(p1.y, w.w, acc3);
                    w = wn; p0 = q0; p1 = q1;
                }
                float v = (acc0 + acc1) + (acc2 + acc3);
                if (p.rawMel) {                                  // coalesced: one 128-byte row segment per group
                    if (g * 32 + lane < p.num) melRow[g * 32 + lane] = v;
                    wg4 += len4 * 32;
                    continue;
                }
                if (p.rectify == CepstralRectify_CubicRoot) v = powf(v, 1.0f / 3.0f);
                else v = __log2f(v < 1e-8f ? 1e-8f : v) * 0.30102999566398120f;   // log10 via MUFU.LG2
                lrow[g * 32 + lane] = v;
                wg4 += len4 * 32;
            }
            if (!p.rawMel) for (int g = p.melGroups; g < 4; g++) lrow[g * 32 + lane] = 0.0f;
        }
        __syncwarp();
        if (!p.rawMel && lane == 0) af_mbar_arrive(&lFull[lbuf]);           // row ready for the tensor-core DCT epilogue

    }
}

void free_plan(Plan *pl) {
    if (!pl) return;
    af_dev_free(pl->dWindowHalf); af_dev_free(pl->dTw1); af_dev_free(pl->dTw2);
    af_dev_free(pl->dMelW); af_dev_free(pl->dMelStart); af_dev_free(pl->dDct); af_dev_free(pl->dMelAux);
    free(pl);
}

}  // namespace

// Mel plan: filters are processed in groups of 32 (lane = filter).  Each filter's first tap may be moved down by
// delta (extra taps get zero weight): delta makes the start bin even (LDS.64 reads of the power spectrum) and,
// where the group's length budget allows, spreads the 16 starts of a half-warp over different 8-byte bank
// pairs.  The budget is the longest filter of the group (+1 for parity) rounded up to 4 taps, so short groups
// of adjacent filters accept a 2-way conflict instead of padding; longest filters are placed first.
static int plan_rows(const int *rowStart, const int *rowLen, int num, int *startShifted /* kMaxNum */, int *groupLen /* 4 */) {
    int total = 0;
    for (int m = 0; m < kMaxNum; m++) startShifted[m] = 0;
    for (int g = 0; g < 4; g++) groupLen[g] = 0;
    for (int g = 0; g * 32 < num; g++) {
        int gmax = 0;
        for (int m = g * 32; m < num && m < g * 32 + 32; m++) if (rowLen[m] > gmax) gmax = rowLen[m];
        const int cap = (gmax + 1 + 3) & ~3;
        int len = 0;
        for (int h = 0; h < 2; h++) {                         // half-warps: lanes 16h .. 16h+15
            int order[16], cnt = 0, used[16] = {0};
            for (int m = g * 32 + 16 * h; m < num && m < g * 32 + 16 * h + 16; m++) order[cnt++] = m;
            for (int i = 1; i < cnt; i++)
                for (int j = i; j > 0 && rowLen[order[j]] > rowLen[order[j - 1]]; j--) { int t = order[j]; order[j] = order[j - 1]; order[j - 1] = t; }
            for (int i = 0; i < cnt; i++) {
                const int m = order[i], s0 = rowStart[m];
                int best = -1, bestUsed = 1 << 30;
                for (int d = s0 & 1; d < 34 && s0 - d >= 0 && rowLen[m] + d <= cap; d += 2) {
                    const int u = used[((s0 - d) >> 1) & 15];
                    if (u < bestUsed) { bestUsed = u; best = d; }
                }
                if (best < 0) best = (s0 & 1) && s0 > 0 ? 1 : 0;
                used[((s0 - best) >> 1) & 15]++;
                startShifted[m] = s0 - best;
                if (rowLen[m] + best > len) len = rowLen[m] + best;
            }
        }
        len = (len + 3) & ~3;
        groupLen[g] = len;
        total += len * 32;
    }
    return total + 8 * 32;                                    // two stages of padding for the pipelined prefetch
}

static int plan_mel(const AfBands *bands, int num, int *startShifted, int *groupLen) {
    return plan_rows(bands->start, bands->len, num, startShifted, groupLen);
}

// ---- interval form of a triangular bank ---------------------------------------------------------------------
// Accepts a bank in which (i) every bin is covered by at most two filters, consecutive ones, and (ii) where filters
// m-1 and m overlap, bank[m-1][k] / g_{m-1} + bank[m][k] / g_m = 1 (g = per-filter gain of the normalisation; the
// Slaney and ETSI triangles of auditory_filterBank.c:373-500 have this form by construction).  Then bin k belongs to
// exactly one interval j(k) (between the peaks of filters j-1 and j) with rising weight r[k] = bank[j][k] / g_j, and
//     mel_m = g_m ( sum_{I_m} r P  +  sum_{I_{m+1}} (1 - r) P ).
// Interval `num` (above the last peak) keeps the last filter's own falling weights (tail).  Verified numerically
// against the actual table with tolerance kTriTol; any violation -> the generic filter-per-lane path is used.
constexpr float kTriTol = 2e-6f;
struct Intervals {
    int start[kMaxNum + 1], len[kMaxNum + 1];
    float r[kNC + 1];
    int owner[kNC + 1];             // interval of each bin, -1 = none
    float tailW[kTailMax];
    int tailStart, tailLen;
};

static bool build_intervals(const float *bank, const AfBands *bands, int num, const float *gain, Intervals *iv) {
    const int width = kNC + 1;
    if (num < 2 || num > kMaxNum) return false;
    int peak[kMaxNum];
    for (int m = 0; m < num; m++) {
        peak[m] = -1;
        if (!(gain[m] > 0.0f)) return false;
        if (bands->len[m] <= 0) continue;                    // a triangle narrower than the bin spacing: no bins, mel = 0
        int best = bands->start[m];
        for (int k = bands->start[m]; k < bands->start[m] + bands->len[m]; k++)
            if (bank[(size_t)m * width + k] > bank[(size_t)m * width + best]) best = k;
        peak[m] = best;
    }
    for (int k = 0; k < width; k++) { iv->r[k] = 0.0f; iv->owner[k] = -1; }
    int lo = 0;                                              // filters are ordered: first candidate cover of bin k
    int prevOwner = -1;
    for (int k = 0; k < width; k++) {
        int cover[3], nc = 0;
        while (lo < num && bands->start[lo] + bands->len[lo] <= k) lo++;
        for (int m = lo; m < num && bands->start[m] <= k && nc < 3; m++)
            if (k < bands->start[m] + bands->len[m] && bank[(size_t)m * width + k] != 0.0f) cover[nc++] = m;
        if (nc == 0) continue;
        if (nc > 2 || (nc == 2 && cover[1] != cover[0] + 1)) return false;
        int j; float r;
        if (nc == 2) {
            const int a = cover[0];
            j = a + 1;
            r = bank[(size_t)j * width + k] / gain[j];
            if (fabsf(bank[(size_t)a * width + k] / gain[a] - (1.0f - r)) > kTriTol) return false;
        } else {
            // a bin under one filter only: the filter's centre bin (weight = gain), or the outer flank of the first /
            // last filter (an inner flank would be shared with the neighbouring filter)
            const int m = cover[0];
            const float w = bank[(size_t)m * width + k] / gain[m];
            if (fabsf(1.0f - w) <= kTriTol) { j = m; r = 1.0f; }
            else if (m == 0 && k <= peak[0]) { j = 0; r = w; }
            else if (m == num - 1 && k >= peak[m]) { j = num; r = 1.0f - w; }
            else return false;
        }
        if (!(r > 0.0f) && j < num) r = 1e-30f;
        if (j < prevOwner) return false;                     // intervals must be runs of consecutive bins
        prevOwner = j;
        iv->owner[k] = j;
        iv->r[k] = r;
    }
    for (int j = 0; j <= num; j++) { iv->start[j] = 0; iv->len[j] = 0; }
    for (int k = 0; k < width; k++) {
        const int j = iv->owner[k];
        if (j < 0) continue;
        if (iv->len[j] == 0) iv->start[j] = k;
        iv->len[j] = k - iv->start[j] + 1;
    }
    iv->tailStart = iv->start[num]; iv->tailLen = iv->len[num];
    if (iv->tailLen > kTailMax) return false;
    for (int i = 0; i < kTailMax; i++) iv->tailW[i] = 0.0f;
    for (int i = 0; i < iv->tailLen; i++) {
        const int k = iv->tailStart + i;
        iv->tailW[i] = iv->owner[k] == num ? bank[(size_t)(num - 1) * width + k] / gain[num - 1] : 0.0f;
    }
    // empty intervals read (and ignore) the bins where they would sit, keeping the lanes' starts monotone
    int last = 0;
    for (int j = 0; j < num; j++) { if (iv->len[j] == 0) iv->start[j] = last; else last = iv->start[j] + iv->len[j]; }
    return true;
}

extern "C" int af_mfcc_fused_supported(int fftLength, int num, int ccNum, const AfBands *bands) {
    if (fftLength != kN || num < 1 || num > kMaxNum || ccNum < 1 || ccNum > 64 || !bands) return 0;
    int starts[kMaxNum], groupLen[4];
    const int floats = plan_mel(bands, num, starts, groupLen);
    for (int g = 0; g < 4; g++) if (groupLen[g] + 8 > kPsPad - (kNC + 1)) return 0;   // padded (and prefetched) reads stay inside the zero pad
    return floats * 4 <= 24 * 1024;                              // weight table budget in shared memory
}

extern "C" void af_mfcc_plan_free(void *plan) { free_plan(static_cast<Plan *>(plan)); }
extern "C" int af_mfcc_plan_mode(void *plan) { return plan ? static_cast<Plan *>(plan)->melMode : -1; }

extern "C" int af_mfcc_plan_build(void **planOut, int fftLength, int num, int ccNum, const float *window,
                                  const float *bank, const AfBands *bands, const float *dct /* ccNum x num */,
                                  int dataType, const float *gain /* num per-filter normalisation gains, or NULL */) {
    *planOut = NULL;
    if (!af_mfcc_fused_supported(fftLength, num, ccNum, bands)) return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC plan: unsupported configuration");
    Plan *pl = static_cast<Plan *>(calloc(1, sizeof(Plan)));
    if (!pl) return AF_ERR_NOMEM;
    pl->num = num; pl->ccNum = ccNum; pl->dataType = dataType;
    pl->ct = ccNum <= 16 ? 2 : ccNum <= 24 ? 3 : ccNum <= 40 ? 5 : 8;
    int rc = AF_OK;

    float *wh = static_cast<float *>(malloc(sizeof(float) * kN));
    for (int i = 0; i < kN; i++) wh[i] = 0.5f * window[i];
    rc = af_dev_upload(reinterpret_cast<void **>(&pl->dWindowHalf), wh, sizeof(float) * kN);
    free(wh);

    float2 *tw = static_cast<float2 *>(malloc(sizeof(float2) * 1024));
    for (int ka = 0; ka < 17 && rc == AF_OK; ka++)
        for (int n1 = 0; n1 < 32; n1++) {
            double a = -2.0 * M_PI * (double)(ka * n1) / 1024.0;
            tw[ka * 32 + n1] = make_float2((float)cos(a), (float)sin(a));
        }
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dTw1), tw, sizeof(float2) * 17 * 32);
    for (int k = 0; k < 32; k++) {
        double a = -2.0 * M_PI * (double)k / 2048.0;
        tw[k] = make_float2((float)cos(a), (float)sin(a));
    }
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dTw2), tw, sizeof(float2) * 32);
    free(tw);

    // zero-padded band weights: group g -> [len_g/4][32 lanes][4 taps], starts shifted for conflict-free reads
    const int width = kNC + 1;
    pl->melGroups = (num + 31) / 32;
    int starts[kMaxNum];
    Intervals *iv = static_cast<Intervals *>(malloc(sizeof(Intervals)));
    // The interval loop is opt-in (AFB200_MFCC_BANK_MODE=1): it halves the bank loop's shared-memory traffic, but the
    // kernel is bound by the latency of queued MIO operations per warp, and the interval form adds a serial tail (warp
    // reduction of the last interval + neighbour exchange by shuffles) that can outweigh the shorter loop.
    const char *force = getenv("AFB200_MFCC_BANK_MODE");
    float ones[kMaxNum];
    for (int m = 0; m < kMaxNum; m++) ones[m] = 1.0f;
    pl->melMode = 0;
    if (iv && force && force[0] == '1' && build_intervals(bank, bands, num, gain ? gain : ones, iv)) {
        int glen[4];
        const int tot = plan_rows(iv->start, iv->len, num, starts, glen);
        bool fits = tot * 4 <= 24 * 1024;
        for (int g = 0; g < 4; g++) if (glen[g] + 8 > kPsPad - (kNC + 1)) fits = false;
        if (fits) {
            pl->melMode = 1;
            pl->melWFloats = tot;
            for (int g = 0; g < 4; g++) pl->melGroupLen[g] = glen[g];
            pl->tailStart = iv->tailStart; pl->tailLen = iv->tailLen;
        }
    }
    if (pl->melMode == 1) {
        const int total = pl->melWFloats;
        float *mw = static_cast<float *>(calloc((size_t)total, sizeof(float)));
        int off = 0;
        for (int g = 0; g < pl->melGroups; g++) {
            for (int l = 0; l < 32; l++) {
                const int j = g * 32 + l;
                if (j >= num) continue;
                const int delta = iv->start[j] - starts[j];
                for (int i = 0; i < iv->len[j]; i++) {
                    const int k = iv->start[j] + i;
                    if (iv->owner[k] == j) mw[off + ((i + delta) >> 2) * 128 + l * 4 + ((i + delta) & 3)] = iv->r[k];
                }
            }
            off += pl->melGroupLen[g] * 32;
        }
        float aux[kMaxNum + kTailMax];
        for (int m = 0; m < kMaxNum; m++) aux[m] = m < num ? (gain ? gain[m] : 1.0f) : 0.0f;
        for (int i = 0; i < kTailMax; i++) aux[kMaxNum + i] = iv->tailW[i];
        if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dMelW), mw, sizeof(float) * (size_t)total);
        if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dMelAux), aux, sizeof(aux));
        free(mw);
    } else {
        const int total = plan_mel(bands, num, starts, pl->melGroupLen);
        pl->melWFloats = total;
        float *mw = static_cast<float *>(calloc((size_t)(total > 0 ? total : 1), sizeof(float)));
        int off = 0;
        for (int g = 0; g < pl->melGroups; g++) {
            for (int l = 0; l < 32; l++) {
                const int m = g * 32 + l;
                if (m >= num) continue;
                const int delta = bands->start[m] - starts[m];
                for (int i = 0; i < bands->len[m]; i++)
                    mw[off + ((i + delta) >> 2) * 128 + l * 4 + ((i + delta) & 3)] = bank[(size_t)m * width + bands->start[m] + i];
            }
            off += pl->melGroupLen[g] * 32;
        }
        if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dMelW), mw, sizeof(float) * (size_t)(total > 0 ? total : 1));
        free(mw);
    }
    free(iv);
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dMelStart), starts, sizeof(int) * kMaxNum);

    // DCT table as the mma B operand: D^T[m][c] with row pitch 40 (72 for cc > 40): pitch % 32 == 8 makes the
    // (k0 + t, n0 + g) fragment reads hit 32 different banks; rows m >= num and columns c >= ccNum are zero
    const int ct = pl->ct, pitch = ct <= 5 ? 40 : 72;
    float *dt = static_cast<float *>(calloc((size_t)kMaxNum * pitch, sizeof(float)));
    for (int m = 0; m < num; m++)
        for (int c = 0; c < ccNum; c++) dt[(size_t)m * pitch + c] = dct[(size_t)c * num + m];
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dDct), dt, sizeof(float) * (size_t)kMaxNum * pitch);
    free(dt);

    if (rc != AF_OK) { free_plan(pl); return rc; }
    *planOut = pl;
    return AF_OK;
}

static int launch_fused(void *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                        int rectifyType, float *out, int nPeer, float *const *peerOut, int rawMel, void *stream) {
    Plan *pl = static_cast<Plan *>(plan);
    if (!pl) return af_fail(AF_ERR_ARG, "fused MFCC: no plan");
    if (batch <= 0 || timeLength <= 0) return AF_OK;
    if (slideLength % 4 || dataLength % 4 || (reinterpret_cast<uintptr_t>(data) & 15))
        return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC needs 16-byte aligned clips and slideLength %% 4 == 0 (TMA bulk copy)");

    Params p;
    memset(&p, 0, sizeof(p));
    p.data = data; p.out = out; p.windowHalf = pl->dWindowHalf; p.tw1 = pl->dTw1; p.tw2 = pl->dTw2;
    p.melW = pl->dMelW; p.melStart = pl->dMelStart; p.dct = pl->dDct;
    p.dataStride = dataLength; p.batch = batch; p.timeLength = timeLength; p.hop = slideLength;
    p.melGroups = pl->melGroups; p.melWFloats = pl->melWFloats;
    p.melMode = pl->melMode; p.num = pl->num; p.tailStart = pl->tailStart; p.tailLen = pl->tailLen; p.melAux = pl->dMelAux;
    for (int g = 0; g < 4; g++) p.melGroupLen[g] = pl->melGroupLen[g];
    p.ccNum = pl->ccNum; p.rectify = rectifyType; p.dataType = pl->dataType;
    p.rawMel = rawMel;
    if (rawMel && pl->melMode) return af_fail(AF_ERR_UNSUPPORTED, "fused filter-bank output needs the filter-per-lane plan");
    if (nPeer < 0 || nPeer > kMaxPeers || (nPeer > 0 && !peerOut)) return af_fail(AF_ERR_ARG, "fused MFCC: nPeer=%d outside [0, %d]", nPeer, kMaxPeers);
    p.nPeer = nPeer;
    for (int d = 0; d < nPeer; d++) p.peerOut[d] = peerOut[d];
    {   // one bulk store per destination needs 16-byte aligned tiles: ccNum % 4 == 0 and aligned bases
        int bulk = !rawMel && pl->ccNum % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
        for (int d = 0; d < nPeer; d++) if (reinterpret_cast<uintptr_t>(peerOut[d]) & 15) bulk = 0;
        const char *sv = getenv("AFB200_MFCC_STORE");
        if (sv && !strcmp(sv, "plain")) bulk = 0;
        p.bulkStore = bulk;
    }

    // frames per tile: as many as fit the shared-memory budget (<= kFrameWarps)
    const int budget = kCtasPerSm == 1 ? 227 * 1024 : (233472 - kCtasPerSm * 1024) / kCtasPerSm;
    int F = kFrameWarps;
    for (; F >= 1; F--) {
        int spanFloats = (F - 1) * slideLength + kN;
        if (carve(spanFloats, pl->melWFloats, pl->ct).total <= budget) break;
    }
    if (F < 1) return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC: slideLength %d too large for shared memory", slideLength);
    if (F > timeLength) F = timeLength;
    p.framesPerTile = F;
    p.spanFloats = (F - 1) * slideLength + kN;
    p.tilesPerClip = (timeLength + F - 1) / F;
    p.totalTiles = (long long)p.tilesPerClip * batch;
    const int smemBytes = carve(p.spanFloats, pl->melWFloats, pl->ct).total;

    int sms = af_sm_count();
    if (sms <= 0) sms = 132;
    long long grid = p.totalTiles < (long long)sms * kCtasPerSm ? p.totalTiles : (long long)sms * kCtasPerSm;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaSuccess;
#define AF_MFCC_LAUNCH2(CT_, MODE_)                                                                               \
    e = cudaFuncSetAttribute(k_mfcc_fused<CT_, MODE_>, cudaFuncAttributeMaxDynamicSharedMemorySize, smemBytes);  \
    if (e != cudaSuccess) return af_cuda_check(e, "cudaFuncSetAttribute(k_mfcc_fused)");                          \
    k_mfcc_fused<CT_, MODE_><<<(unsigned)grid, kThreads, smemBytes, st>>>(p)
#define AF_MFCC_LAUNCH(CT_) if (pl->melMode) { AF_MFCC_LAUNCH2(CT_, 1); } else { AF_MFCC_LAUNCH2(CT_, 0); }
    switch (pl->ct) {
    case 2: AF_MFCC_LAUNCH(2); break;
    case 3: AF_MFCC_LAUNCH(3); break;
    case 5: AF_MFCC_LAUNCH(5); break;
    default: AF_MFCC_LAUNCH(8); break;
    }
#undef AF_MFCC_LAUNCH2
#undef AF_MFCC_LAUNCH
    AF_LAUNCH_CHECK("k_mfcc_fused");
    return AF_OK;
}

extern "C" int af_launch_mfcc_fused(void *plan, const float *data, int dataLength, int batch, int timeLength,
                                    int slideLength, int rectifyType, float *out, int nPeer, float *const *peerOut,
                                    void *stream) {
    return launch_fused(plan, data, dataLength, batch, timeLength, slideLength, rectifyType, out, nPeer, peerOut, 0, stream);
}

// same kernel stopped after the filter bank: out[batch][T][num] = bank . |X|^2 (or |X|), i.e. bftObj_bft in real mode
extern "C" int af_launch_mel_fused(void *plan, const float *data, int dataLength, int batch, int timeLength,
                                   int slideLength, float *out, void *stream) {
    return launch_fused(plan, data, dataLength, batch, timeLength, slideLength, 0, out, 0, NULL, 1, stream);
}

// Diagnostic / test hook (host only, no device needed): the interval form the planner derives from a bank.
// Returns 1 when the bank has the triangular two-overlap structure (then owner/r/tail/starts/groupLen are filled), else 0.
extern "C" int afb200_mfccIntervalPlan(const float *bank, int num, const float *gain, int *owner /* 1025 */,
                                       float *r /* 1025 */, int *ivStart /* num+1 */, int *ivLen /* num+1 */,
                                       float *tailW /* 512 */, int *groupLen /* 4 */, int *startShifted /* 128 */) {
    if (!bank || num < 2 || num > kMaxNum) return 0;
    AfBands bands;
    if (af_bands_build(bank, num, kNC + 1, &bands)) return 0;
    Intervals *iv = static_cast<Intervals *>(malloc(sizeof(Intervals)));
    float ones[kMaxNum];
    for (int m = 0; m < kMaxNum; m++) ones[m] = 1.0f;
    int ok = iv && build_intervals(bank, &bands, num, gain ? gain : ones, iv) ? 1 : 0;
    if (ok) {
        for (int k = 0; k <= kNC; k++) { if (owner) owner[k] = iv->owner[k]; if (r) r[k] = iv->r[k]; }
        for (int j = 0; j <= num; j++) { if (ivStart) ivStart[j] = iv->start[j]; if (ivLen) ivLen[j] = iv->len[j]; }
        if (tailW) for (int i = 0; i < kTailMax; i++) tailW[i] = iv->tailW[i];
        int st[kMaxNum], gl[4];
        plan_rows(iv->start, iv->len, num, st, gl);
        if (groupLen) for (int g = 0; g < 4; g++) groupLen[g] = gl[g];
        if (startShifted) for (int m = 0; m < kMaxNum; m++) startShifted[m] = st[m];
    }
    free(iv);
    af_bands_free(&bands);
    return ok;
}
