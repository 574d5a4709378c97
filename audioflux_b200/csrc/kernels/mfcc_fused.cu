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
#include <string.h>
#include "mfcc_common.cuh"
#include "fft32_gen.cuh"

namespace {

constexpr int kN = 2048;            // fftLength
constexpr int kNC = 1024;           // packed complex points
constexpr int kFrameWarps = 13;     // consumer warps = max frames per tile (<= 16: one mma M tile)
constexpr int kEpiWarps = 2;        // DCT epilogue warps; tile `it` is served by warp it % kEpiWarps
constexpr int kThreads = (kFrameWarps + 1 + kEpiWarps) * 32;   // + TMA producer warp + DCT epilogue warps
constexpr int kLPitch = 132;        // log-mel tile row pitch (floats): 4g + t -> 32 distinct banks for mma A fragments
constexpr int kLRows = 16;          // stored rows of the mma M=16 tile (rows >= kFrameWarps are zeros)
constexpr int kStages = 2;
constexpr int kLBufs = 3;           // log-mel tiles in flight between the frame warps and the DCT epilogue (2 leaves frame
                                    // warps waiting for the epilogue)
constexpr int kMaxNum = 128;        // filters (padded)
constexpr int kScratchFloats = 1152;            // per warp: 33x32 float transpose plane, later Ps[0..1024] + zero pad
constexpr int kPsPad = 1152;        // Ps[0..1024], zeros up to kPsPad (padded band reads)
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
    int num, ccNum, rectify, dataType;
    int rawMel;                     // 1: stop after the bank: out[frame][num] = bank . |X|^2 (bftObj_bft real mode), no log / DCT
    int bulkStore;                  // 1: the result tile leaves as one TMA bulk store per destination (16-byte aligned rows)
    // fused all-gather: every finished tile is also stored at the same offset of up to kMaxPeers other buffers
    // (peer GPUs' gathered arrays mapped over NVLink, opened with cudaIpcOpenMemHandle by the host side)
    int nPeer;
    float *peerOut[kMfccMaxPeers];
};

// shared-memory carve-up (bytes), all 16-byte aligned
struct Smem {
    int spanOff, scratchOff, windowOff, tw1Off, tw2Off, melWOff, melStartOff, dctOff, lOff, stageOff, barOff, total;
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
    s.dctOff = o;      o += kMaxNum * af_mfcc_dct_pitch(ct) * 4;
    s.lOff = o;        o += kLBufs * kLRows * kLPitch * 4;
    s.stageOff = o;    o += kEpiWarps * kStageBytes;
    s.barOff = o;      o += (2 * kStages + 2 * kLBufs) * 8;
    s.total = o;
    return s;
}

template <int CT>
__global__ void __launch_bounds__(kThreads, 1) k_mfcc_fused(Params p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const Smem L = carve(p.spanFloats, p.melWFloats, CT);
    float *span = reinterpret_cast<float *>(smem + L.spanOff);
    float *scratchAll = reinterpret_cast<float *>(smem + L.scratchOff);
    float2 *sWin2 = reinterpret_cast<float2 *>(smem + L.windowOff);
    float2 *sTw1 = reinterpret_cast<float2 *>(smem + L.tw1Off);
    float2 *sTw2 = reinterpret_cast<float2 *>(smem + L.tw2Off);
    float *sMelW = reinterpret_cast<float *>(smem + L.melWOff);
    int *sMelStart = reinterpret_cast<int *>(smem + L.melStartOff);
    float *sDct = reinterpret_cast<float *>(smem + L.dctOff);
    float *sL = reinterpret_cast<float *>(smem + L.lOff);                 // [kLBufs][kLRows][kLPitch] log-mel tiles
    uint64_t *fullBar = reinterpret_cast<uint64_t *>(smem + L.barOff);
    uint64_t *emptyBar = fullBar + kStages;
    uint64_t *lFull = emptyBar + kStages;                                  // [kLBufs] frame warps -> epilogue
    uint64_t *lEmpty = lFull + kLBufs;                                     // [kLBufs] epilogue -> frame warps
    constexpr int kDctPitch = af_mfcc_dct_pitch(CT);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // ---- one-time: tables -> shared, barriers ----
    for (int i = threadIdx.x; i < kN; i += kThreads) reinterpret_cast<float *>(sWin2)[i] = p.windowHalf[i];
    for (int i = threadIdx.x; i < 17 * 32; i += kThreads) sTw1[i] = p.tw1[i];
    for (int i = threadIdx.x; i < 32; i += kThreads) sTw2[i] = p.tw2[i];
    for (int i = threadIdx.x; i < p.melWFloats; i += kThreads) sMelW[i] = p.melW[i];
    for (int i = threadIdx.x; i < kMaxNum; i += kThreads) sMelStart[i] = p.melStart[i];
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
#pragma unroll 2
            for (int k0 = 0; k0 < kMaxNum; k0 += 8) {
                const float af[4] = {A[g * kLPitch + k0 + t], A[(g + 8) * kLPitch + k0 + t],
                                     A[g * kLPitch + k0 + t + 4], A[(g + 8) * kLPitch + k0 + t + 4]};
                uint32_t ah[4], al[4], bh[CT][2], bl[CT][2];
#pragma unroll
                for (int i = 0; i < 4; i++) af_tf32_split(af[i], ah[i], al[i]);
#pragma unroll
                for (int n = 0; n < CT; n++) {
                    const float bf[2] = {sDct[(k0 + t) * kDctPitch + n * 8 + g], sDct[(k0 + t + 4) * kDctPitch + n * 8 + g]};
#pragma unroll
                    for (int i = 0; i < 2; i++) af_tf32_split(bf[i], bh[n][i], bl[n][i]);
                }
#pragma unroll
                for (int n = 0; n < CT; n++) AF_MMA_TF32(acx[n], al[0], al[1], al[2], al[3], bh[n][0], bh[n][1]);
#pragma unroll
                for (int n = 0; n < CT; n++) AF_MMA_TF32(acc[n], ah[0], ah[1], ah[2], ah[3], bh[n][0], bh[n][1]);
#pragma unroll
                for (int n = 0; n < CT; n++) AF_MMA_TF32(acx[n], ah[0], ah[1], ah[2], ah[3], bl[n][0], bl[n][1]);
            }
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
                af_bulk_wait_read0();                                        // this warp's previous stores have read the staging tile
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
                af_fence_proxy_async_smem();
                __syncwarp();
                if (lane <= p.nPeer) {
                    float *o = (lane == 0 ? p.out : p.peerOut[lane - 1]) + tileOff;
                    af_bulk_store(o, stage, (uint32_t)(nf * p.ccNum * 4));
                    af_bulk_commit();
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
        if (p.bulkStore) af_bulk_wait0();
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
            for (int j = 0; j < 32; j++) z[j] = v_mul(sp[lane + 32 * j], sWinC[lane + 32 * j]);
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
        af_fft32(z);                                          // over n2; Y[n1=lane][ka] at AF_BR5(ka)
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
        }
        af_fft32(z);                                          // over n1; Z[lane + 32*kb] at AF_BR5(kb)

        // ---- C: real-FFT post-pass + power / magnitude -> Ps[0..1024] ----
        // (window pre-scaled by 1/2, so E' = Z[k] + conj Z[N-k] and O' = -i (Z[k] - conj Z[N-k]) need no halving;
        //  X[k] = E' + W O', conj X[N-k] = E' - W O' with W = W_2048^k = W_2048^lane * W_64^kb)
#pragma unroll
        for (int kb = 0; kb < 16; kb++) {
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
        // weights: per group [len/4][32 lanes] float4 (LDS.128); P: two LDS.64 per 4 taps (starts are even and
        // spread over distinct 8-byte bank pairs per half-warp by the host planner)
        const float4 *wg4 = reinterpret_cast<const float4 *>(sMelW) + lane;
        for (int g = 0; g < p.melGroups; g++) {
            const int len4 = p.melGroupLen[g] >> 2;
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
            lrow[g * 32 + lane] = af_mfcc_rectify(v, p.rectify);
            wg4 += len4 * 32;
        }
        if (!p.rawMel) for (int g = p.melGroups; g < 4; g++) lrow[g * 32 + lane] = 0.0f;
        __syncwarp();
        if (!p.rawMel && lane == 0) af_mbar_arrive(&lFull[lbuf]);           // row ready for the tensor-core DCT epilogue

    }
}

void free_plan(Plan *pl) {
    if (!pl) return;
    af_dev_free(pl->dWindowHalf); af_dev_free(pl->dTw1); af_dev_free(pl->dTw2);
    af_dev_free(pl->dMelW); af_dev_free(pl->dMelStart); af_dev_free(pl->dDct);
    free(pl);
}

}  // namespace

// Mel plan: filters are processed in groups of 32 (lane = filter).  Each filter's first tap may be moved down by
// delta (extra taps get zero weight): delta makes the start bin even (LDS.64 reads of the power spectrum) and,
// where the group's length budget allows, spreads the 16 starts of a half-warp over different 8-byte bank
// pairs.  The budget is the longest filter of the group (+1 for parity) rounded up to 4 taps, so short groups
// of adjacent filters accept a 2-way conflict instead of padding; longest filters are placed first.
static int plan_mel(const AfBands *bands, int num, int *startShifted /* kMaxNum */, int *groupLen /* 4 */) {
    const int *rowStart = bands->start, *rowLen = bands->len;
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

int af_mfcc1_supported(int fftLength, int num, int ccNum, const AfBands *bands) {
    if (fftLength != kN || num < 1 || num > kMaxNum || ccNum < 1 || ccNum > 64 || !bands) return 0;
    int starts[kMaxNum], groupLen[4];
    const int floats = plan_mel(bands, num, starts, groupLen);
    for (int g = 0; g < 4; g++) if (groupLen[g] + 8 > kPsPad - (kNC + 1)) return 0;   // padded (and prefetched) reads stay inside the zero pad
    return floats * 4 <= 24 * 1024;                              // weight table budget in shared memory
}

void af_mfcc1_plan_free(void *plan) { free_plan(static_cast<Plan *>(plan)); }

int af_mfcc1_plan_build(void **planOut, int fftLength, int num, int ccNum, const float *window, const float *bank,
                        const AfBands *bands, const float *dct /* ccNum x num */, int dataType) {
    *planOut = NULL;
    if (!af_mfcc1_supported(fftLength, num, ccNum, bands)) return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC plan: unsupported configuration");
    Plan *pl = static_cast<Plan *>(calloc(1, sizeof(Plan)));
    if (!pl) return AF_ERR_NOMEM;
    pl->num = num; pl->ccNum = ccNum; pl->dataType = dataType;
    pl->ct = af_mfcc_ct(ccNum);
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
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dMelStart), starts, sizeof(int) * kMaxNum);
    if (rc == AF_OK) rc = af_mfcc_dct_upload(&pl->dDct, dct, num, ccNum, pl->ct);

    if (rc != AF_OK) { free_plan(pl); return rc; }
    *planOut = pl;
    return AF_OK;
}

int af_mfcc1_launch(void *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                    int rectifyType, float *out, int nPeer, float *const *peerOut, int rawMel, void *stream) {
    Plan *pl = static_cast<Plan *>(plan);
    Params p;
    memset(&p, 0, sizeof(p));
    p.data = data; p.out = out; p.windowHalf = pl->dWindowHalf; p.tw1 = pl->dTw1; p.tw2 = pl->dTw2;
    p.melW = pl->dMelW; p.melStart = pl->dMelStart; p.dct = pl->dDct;
    p.dataStride = dataLength; p.batch = batch; p.timeLength = timeLength; p.hop = slideLength;
    p.melGroups = pl->melGroups; p.melWFloats = pl->melWFloats;
    p.num = pl->num;
    for (int g = 0; g < 4; g++) p.melGroupLen[g] = pl->melGroupLen[g];
    p.ccNum = pl->ccNum; p.rectify = rectifyType; p.dataType = pl->dataType;
    p.rawMel = rawMel;
    p.nPeer = nPeer;
    for (int d = 0; d < nPeer; d++) p.peerOut[d] = peerOut[d];
    p.bulkStore = !rawMel && af_mfcc_bulk_store_ok(pl->ccNum, out, nPeer, peerOut);   // (the bank output leaves row by row)

    // frames per tile: as many as fit the shared-memory budget (<= kFrameWarps)
    const int budget = 227 * 1024;
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
    static void (*const kernels[4])(Params) = {k_mfcc_fused<2>, k_mfcc_fused<3>, k_mfcc_fused<5>, k_mfcc_fused<8>};
    return af_mfcc_launch_ct(kernels, "k_mfcc_fused", pl->ct, p.totalTiles, kThreads, smemBytes, stream, p);
}
