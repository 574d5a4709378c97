// mfcc_fused2.cu -- second-generation fused framed-STFT(2048) -> |X|^2 / |X| -> banded filter bank -> log10 / cbrt
// -> ortho DCT-II -> first ccNum coefficients.  One persistent kernel, samples read from HBM once (1-D TMA bulk copies
// through an mbarrier ring), results leave as whole tiles (TMA bulk stores, also to peer GPUs).
//
// Replaces, for fftLength = 2048, the same reference chain as mfcc_fused.cu (v1):
//   stftObj_stft (src/stft_algorithm.c:696-715, 790-801) -> __mccut (src/reassign_algorithm.c:600-604)
//   -> __mcsquare / sqrtf (src/bft_algorithm.c:489-497) -> __mdot1 (:515-518, src/vector/flux_vector.c:55-86)
//   -> log10f clamp / powf(1/3) (src/feature/xxcc_algorithm.c:124-140) -> fftObj_dct (:142-149) -> cut (:151-155)
//
// What changed against v1 (whose frame warps spend most of their time in the bank loop and the post-pass shuffles):
//  * the real 2048-point FFT is split as 64 (real, in registers) x 32 (complex, in registers): lane n2 transforms the
//    64 real samples x[32 n1 + n2] (packed complex 32-point DFT + an IN-LANE post-pass, compile-time twiddles), the
//    columns k1 = 1..31 are twiddled, transposed through shared memory and transformed again; lane k1 then holds the
//    bins k1 + 64 k2 and (by Hermitian symmetry) 2048 - (k1 + 64 k2): all 1025 bins without any cross-lane exchange
//    (v1: 32 shuffles + a second twiddle pass per frame);
//  * the two "half" columns k1 = 0 and k1 = 32 (real-valued after stage 1) are collected for the whole tile and
//    transformed by the TMA producer warp, one lane per (frame, column): 1/13 of a frame's work instead of a
//    divergent second pass in every frame warp;
//  * the filter bank is applied per TILE by the helper warps, not per frame by the frame warps: the power spectra of
//    the tile's frames sit in shared memory as [bin pair][frame], lane = frame, and every bin pair is multiplied
//    ONCE for the two filters that overlap on it (interval form: rising slope of filter i, falling slope of filter
//    i-1, the reference's own float weights, no re-normalisation) with two FMAs per lane.  The intervals are cut into PIECES of
//    at most Lmax bin pairs (host-planned, Lmax = 3 for the 128-band mel bank) so that the 128 helper lanes carry equal
//    work (the longest interval is 15 pairs, the mean 4.5); a piece's partial sums go into a slot that ALIASES the power
//    tile rows its pass has finished reading, and are added up per band in a fixed order (bit-stable);
//  * the 13 x cc result tile is staged in shared memory and leaves as one TMA bulk store per destination (this GPU and,
//    for the fused all-gather, every peer GPU): full lines over NVLink instead of 32-bit stores.
#include <string.h>
#include "mfcc_common.cuh"
#include "fft32_gen.cuh"

namespace {

constexpr int kN = 2048;
constexpr int kBins = 1025;
constexpr int kPairs = 513;         // bin pairs of the power-spectrum tile
constexpr int kFW = 13;             // frame warps = max frames per tile (<= 16: one mma M tile)
constexpr int kBW = 4;              // filter-bank warps (one interval per lane)
constexpr int kDW = 2;              // DCT (tensor-core) + store warps, one tile behind the bank warps
constexpr int kEW = kBW;                        // (planner: helper lanes that walk intervals)
constexpr int kThreads = (kFW + 1 + kBW + kDW) * 32;  // + producer / special-column warp: 20 warps at <= 96 registers
// Warp roles.  Warps w and w + 4 issue from the same SM sub-partition, so frame warps 0..12 put four frames on the
// sub-partition of warp 16 and three on each of the others.  Warp 16 is a DCT warp: the DCT warps issue the fewest
// instructions per tile (dependent tensor-core steps, not FP32 work).  No bank warp, the critical path, shares a
// sub-partition with four frames: the producer is warp 13, the bank warps 14, 15, 17 and 18, the other DCT warp 19.
constexpr int kProducerWarp = 13;
__device__ __forceinline__ int bank_warp_index(int warp) { return warp >= 14 && warp <= 18 && warp != 16 ? warp - 14 - (warp > 16) : -1; }
__device__ __forceinline__ int dct_warp_index(int warp) { return warp == 16 || warp == 19 ? (warp - 16) / 3 : -1; }
constexpr int kMaxNum = 128;
constexpr int kLPitch = 132;        // log-mel tile row pitch (floats): 4g + t -> 32 distinct banks for mma A fragments
constexpr int kMaxTab = 1408;       // bank table entries (one float4 per bin pair of an interval) in the parameter block
constexpr int kMaxPieces = 256;     // pieces the intervals may be cut into (slots = rows of the power tile)
constexpr int kMaxPass = kMaxPieces / (kEW * 32);   // bank passes: one piece per helper lane and pass
constexpr int kSpecPitch = 17;      // c64 slots per n2 row of the special-column buffer (odd -> conflict-free both ways)
constexpr int kPitchPairs = kFW | 1;   // power-tile row pitch (frames): odd -> conflict-free column walks; always kFW wide
constexpr int kTileFloats = kPairs * kPitchPairs * 2;   // one power tile; there are two, used by alternate tiles
// Stage C transposes through frame w's own column of the power tile (float2 slot 13 s + w, s < 513), which is free from
// the bank's release of the buffer until the frame's power stores.  Element pair j = n2 / 2 of plane row r = k1 - 1
// sits at slot s = r + 31 j: the writers' 32-bit stores hit words 26 r + 6 j + 2 w + (n2 & 1) (mod 32), 32 banks; the
// readers' float2 loads hit bank pairs 13 r + 13 * 31 j + w (mod 16), 16 per half-warp.  Both: one wavefront.
constexpr int kTrRows = 31;
static_assert(kPitchPairs == 13 && (kTrRows - 1) + kTrRows * 15 < kPairs, "the transpose slot map fits a power-tile column");
constexpr int kBarBytes = 128;      // 16 mbarriers at the start of shared memory (128 keeps the TMA span aligned)
constexpr int kTwRows = 31;         // stage-D twiddles W_2048^(n2 k1) = g (1 - i t), n2 = 1..31 (row n2 - 1), lane k1

struct Plan {
    float2 *dWinPairs;              // [32 m][32 lane]  0.5 * (w[64 m + lane], w[64 m + 32 + lane])
    float2 *dTw;                    // [kTwRows][32 k1]  (g, t) of W_2048^(n2 k1) = g (1 - i t), n2 = 1..31 (row n2 - 1)
    float *dDct;                    // [128 m][dctPitch]
    int num, ccNum, ct, dataType;
    unsigned ivDesc[kMaxNum + 4];   // (first bin pair << 16) | table offset; entries num+1.. = end sentinels
    int nPass;                      // bank passes
    int nPieces, lmax, firstPass2;  // pieces 0 .. firstPass2-1 run in pass 0
    unsigned pieceDesc[kMaxPieces];                  // (first bin pair << 20) | (pairs << 16) | table offset
    unsigned short piecePrefix[kMaxNum + 4];         // first piece of interval i; [num + 1 ..] = nPieces
    unsigned short assign[kMaxPass * kEW * 32];      // piece of helper lane (pass, warp * 32 + lane), 0xffff = none
    int tabLen;
    float4 *tab;                    // host copy of the bank table
    float4 *dTab;                   // device copy, staged into shared memory by every CTA
    unsigned *dDesc;
    unsigned short *dAssign, *dPrefix;
};

struct Params {
    const float *data;
    float *out;
    const float2 *winPairs, *tw;
    const float *dct;
    long long dataStride;
    unsigned totalTiles;            // (< 2^31: checked by the launcher) 32-bit tile arithmetic in the kernel
    int batch, timeLength, hop, framesPerTile, tilesPerClip, spanFloats, stages;
    int num, ccNum, rectify, dataType, rawMel, bulkStore, dctPitch;
    int nPeer;
    float *peerOut[kMfccMaxPeers];
    int offSpan, offP, offWin, offTw, offSpec, offDct, offL, offStage, offTab, offDesc, offAssign, offPrefix, stageBytes;   // offL: two log-mel tiles
    int nPass;
    const unsigned short *assign;
    int tabLen;
    const float4 *bankTab;          // [tabLen] (rise[2q], rise[2q+1], fall[2q], fall[2q+1]) per bin pair of an interval
    const unsigned *pieceDesc;      // [kMaxPieces]
    const unsigned short *piecePrefix;   // [kMaxNum + 4]
};

__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

template <int CT>
__global__ void __launch_bounds__(kThreads, 1) k_mfcc_fused2(const __grid_constant__ Params p) {
    extern __shared__ __align__(128) unsigned char smem[];
    float *span = reinterpret_cast<float *>(smem + p.offSpan);
    float *sP = reinterpret_cast<float *>(smem + p.offP);                 // [2][kPairs][kPitchPairs][2]
    float2 *sWin = reinterpret_cast<float2 *>(smem + p.offWin);
    float2 *sTw = reinterpret_cast<float2 *>(smem + p.offTw);
    c64 *sSpec = reinterpret_cast<c64 *>(smem + p.offSpec);               // [2][32 n2][kSpecPitch]
    float *sDct = reinterpret_cast<float *>(smem + p.offDct);
    float *sL = reinterpret_cast<float *>(smem + p.offL);                 // [16][kLPitch]
    float *sStage = reinterpret_cast<float *>(smem + p.offStage);         // result tile(s), dense rows
    uint64_t *fullBar = reinterpret_cast<uint64_t *>(smem);               // [2] TMA landed (barriers at offset 0: fixed addresses)
    uint64_t *emptyBar = fullBar + 2;                                     // [2] frame warps took their samples
    uint64_t *specFull = fullBar + 4;                                     // [2] special columns of a tile stored
    uint64_t *pFull = fullBar + 6;                                        // [2] power-spectrum tile complete
    uint64_t *pEmpty = fullBar + 8;                                       // [2] bank done with it
    uint64_t *cDone = fullBar + 10;                                       // [2] frame warps' transposes read out of it
    uint64_t *lFull = fullBar + 12;                                       // [2] log-mel tile written by the bank warps
    uint64_t *lEmpty = fullBar + 14;                                      // [2] ... consumed by the DCT warps
    float4 *sTab = reinterpret_cast<float4 *>(smem + p.offTab);           // interval-form bank weights
    unsigned *sDesc = reinterpret_cast<unsigned *>(smem + p.offDesc);
    unsigned short *sAssign = reinterpret_cast<unsigned short *>(smem + p.offAssign);
    unsigned short *sPrefix = reinterpret_cast<unsigned short *>(smem + p.offPrefix);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int pitch = kPitchPairs;        // compile-time: the power-tile stores and walks take immediate offsets

    // ---- one-time: tables -> shared, zero the tiles (pad slots are multiplied by zero weights), barriers ----
    for (int i = threadIdx.x; i < 32 * 32; i += kThreads) sWin[i] = p.winPairs[i];
    for (int i = threadIdx.x; i < kTwRows * 32; i += kThreads) sTw[i] = p.tw[i];
    for (int i = threadIdx.x; i < p.tabLen; i += kThreads) sTab[i] = p.bankTab[i];
    for (int i = threadIdx.x; i < kMaxPieces; i += kThreads) sDesc[i] = p.pieceDesc[i];
    for (int i = threadIdx.x; i < kMaxNum + 4; i += kThreads) sPrefix[i] = p.piecePrefix[i];
    for (int i = threadIdx.x; i < kMaxPass * kEW * 32; i += kThreads) sAssign[i] = p.assign[i];
    for (int i = threadIdx.x; i < 2 * kTileFloats; i += kThreads) sP[i] = 0.0f;
    for (int i = threadIdx.x; i < 2 * 32 * kSpecPitch; i += kThreads) sSpec[i] = 0ull;
    for (int i = threadIdx.x; i < 2 * 16 * kLPitch; i += kThreads) sL[i] = 0.0f;
    if (!p.rawMel)
        for (int i = threadIdx.x; i < kMaxNum * p.dctPitch; i += kThreads) sDct[i] = p.dct[i];
    for (int i = threadIdx.x; i < p.stageBytes / 4; i += kThreads) sStage[i] = 0.0f;
    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; s++) {
            af_mbar_init(&fullBar[s], 1);
            af_mbar_init(&emptyBar[s], kFW);
            af_mbar_init(&specFull[s], kFW);
            af_mbar_init(&pFull[s], kFW + 1);
            af_mbar_init(&pEmpty[s], kBW);
            af_mbar_init(&cDone[s], kFW);
            af_mbar_init(&lFull[s], kBW);
            af_mbar_init(&lEmpty[s], kDW);
        }
        af_fence_barrier_init();
    }
    __syncthreads();

    const int F = p.framesPerTile;

    if (warp == kProducerWarp) {
        // ================= producer (TMA) + special columns k1 = 0 / 32 of every frame of the tile =================
        const int S = p.stages;
        auto issue = [&](unsigned tile, int stage) {
            const unsigned clip = tile / (unsigned)p.tilesPerClip;
            const int f0 = (int)(tile - clip * (unsigned)p.tilesPerClip) * F;
            const int nf = min(F, p.timeLength - f0);
            const uint32_t bytes = (uint32_t)(((nf - 1) * p.hop + kN) * 4);
            af_mbar_arrive_expect_tx(&fullBar[stage], bytes);
            af_tma_load_1d(span + (size_t)stage * p.spanFloats, p.data + (long long)clip * p.dataStride + (long long)f0 * p.hop, bytes,
                           &fullBar[stage]);
        };
        if (lane == 0)
            for (int s = 0; s < S; s++) {
                const unsigned tile = blockIdx.x + (unsigned)s * gridDim.x;
                if (tile < p.totalTiles) issue(tile, s);
            }
        const int f = lane & 15, kind = lane >> 4;              // lane = (frame, column kind)
        int it = 0;
        for (unsigned tile = blockIdx.x; tile < p.totalTiles; tile += gridDim.x, ++it) {
            const int stage = it % S;
            if (lane == 0) {
                af_mbar_wait_sleepy(&emptyBar[stage], (uint32_t)(it / S) & 1u);       // tile `it` taken: refill the slot
                const unsigned next = tile + (unsigned)S * gridDim.x;
                if (next < p.totalTiles) issue(next, stage);
            }
            __syncwarp();
            const int f0 = (int)(tile % (unsigned)p.tilesPerClip) * F;
            const int nf = min(F, p.timeLength - f0);
            const int sb = it & 1;
            af_mbar_wait(&specFull[sb], (uint32_t)(it >> 1) & 1u);
            // a[n2] = R_n2[0], b[n2] = R_n2[32] (both real).  kind 0: X[64 k2] = DFT32(a)[k2], k2 = 0..16;
            // kind 1: X[32 + 64 k2] = DFT32(b[n2] W_64^n2)[k2], k2 = 0..15
            c64 u[32];
            const c64 *sp = sSpec + (size_t)sb * 32 * kSpecPitch + min(f, nf - 1);
#pragma unroll
            for (int n2 = 0; n2 < 32; n2++) {
                float a, b;
                c_unpack(sp[n2 * kSpecPitch], a, b);
                const float v = kind ? b : a;
                u[n2] = kind ? af_mul_w64_real(v, n2 & 15) : c_pack(v, 0.0f);
                if (n2 >= 16 && kind) u[n2] = c_mul_mi(u[n2]);                        // W_64^16 = -i
            }
            af_fft32_fma(u);
            af_mbar_wait(&cDone[sb], (uint32_t)(it >> 1) & 1u);          // the frames' transposes are out of these columns
            if (f < nf) {
                float *dst = sP + sb * kTileFloats + 2 * f + (kind ? 32 * pitch : 0);   // bin 64 k2 + 32 kind -> pair 32 k2 + 16 kind
#pragma unroll
                for (int k2 = 0; k2 < 16; k2++) {
                    float pw = c_norm2_fma(u[AF_BR5(k2)]);
                    if (p.dataType == SpectralData_Mag) pw = sqrtf(pw);
                    dst[(size_t)k2 * 64 * pitch] = pw;
                }
                if (!kind) {
                    float pw = c_norm2_fma(u[AF_BR5(16)]);
                    if (p.dataType == SpectralData_Mag) pw = sqrtf(pw);
                    dst[(size_t)16 * 64 * pitch] = pw;                                // bin 1024
                }
            }
            __syncwarp();
            if (lane == 0) af_mbar_arrive(&pFull[sb]);
        }
        return;
    }

    if (bank_warp_index(warp) >= 0) {
        // ================= bank warps: interval-form filter bank over the whole tile =================
        const int e = bank_warp_index(warp);
        const int rowFloats = p.num;
        int it = 0;
        for (unsigned tile = blockIdx.x; tile < p.totalTiles; tile += gridDim.x, ++it) {
            const int lbuf = it & 1;                               // (power tile and log-mel tile alike)
            float *P = sP + lbuf * kTileFloats;
            af_mbar_wait(&pFull[lbuf], (uint32_t)(it >> 1) & 1u);
            if (!p.rawMel) af_mbar_wait(&lEmpty[lbuf], ((uint32_t)(it >> 1) & 1u) ^ 1u);    // DCT done with tile it - 2
            // ---- phase 1: ONE PIECE (<= Lmax bin pairs of one interval) PER LANE AND PASS, all frames of the tile in
            // registers: one LDS.128 of weights (rise of filter i, fall of filter i-1) and, per frame, one LDS.64 of the
            // power pair + two complex-pair FMAs -- kFW independent accumulator chains per lane.  Pass 0 walks the low rows of the
            // power tile, pass 1 the rest; once every helper warp is through a pass the rows it read are dead and take
            // the pieces' partial sums S[piece][frame] = (rise part, fall part), piece index = row index.
            c64 *sS = reinterpret_cast<c64 *>(P);
            for (int ps = 0; ps < p.nPass; ps++) {
                const unsigned piece = sAssign[(ps * kBW + e) * 32 + lane];
                const bool have = piece != 0xffffu;
                const unsigned d0 = sDesc[have ? piece : 0];
                const int len = have ? (int)((d0 >> 16) & 15u) : 0;
                const float4 *wt = sTab + (d0 & 0xffffu);
                const c64 *q = reinterpret_cast<const c64 *>(P) + (size_t)(d0 >> 20) * pitch;
                c64 aR[kFW], aF[kFW];
#pragma unroll
                for (int f = 0; f < kFW; f++) { aR[f] = 0ull; aF[f] = 0ull; }
                for (int j = 0; j < len; j++) {
                    const float4 w = wt[j];
                    const c64 wr = c_pack(w.x, w.y), wf = c_pack(w.z, w.w);
#pragma unroll
                    for (int f = 0; f < kFW; f++) {
                        const c64 v = q[f];
                        aR[f] = v_fma(v, wr, aR[f]);
                        aF[f] = v_fma(v, wf, aF[f]);
                    }
                    q += pitch;
                }
                named_bar_sync(3, kBW * 32);                   // every helper warp has read this pass's rows
                if (have) {
#pragma unroll
                    for (int f = 0; f < kFW; f++) {
                        float r0, r1, f0_, f1_;
                        c_unpack(aR[f], r0, r1);
                        c_unpack(aF[f], f0_, f1_);
                        sS[(size_t)piece * pitch + f] = c_pack(r0 + r1, f0_ + f1_);
                    }
                }
            }
            // (tile geometry after phase 1: nothing of it stays live across the accumulator loop)
            const unsigned clip = tile / (unsigned)p.tilesPerClip;
            const int f0 = (int)(tile - clip * (unsigned)p.tilesPerClip) * F;
            const int nf = min(F, p.timeLength - f0);
            float *L = sL + (size_t)lbuf * 16 * kLPitch;
            float *stage = sStage + (size_t)lbuf * (p.stageBytes / 8);   // (filter-bank output mode: two staging tiles)
            const int stagePitch = p.num + 4;                              // padded rows (bank conflicts)
            if (p.rawMel && e == 0) af_bulk_wait_read0();             // the store of tile it - 2 has read this staging tile
            named_bar_sync(1, kBW * 32);                           // every partial sum of the tile is in shared memory
            // ---- phase 2: mel_m = sum of the rise parts of interval m + the fall parts of interval m + 1 (pieces in
            // ascending order), rectified (cepstra) or staged as the result row (filter bank) ----
            static_assert(kBW * 32 >= kMaxNum, "one band per helper lane");
            const int m = e * 32 + lane;
            float v[kFW];
#pragma unroll
            for (int f = 0; f < kFW; f++) v[f] = 0.0f;
            if (m < p.num) {
                const int a0 = sPrefix[m], a1 = sPrefix[m + 1], a2 = sPrefix[m + 2];
                for (int s = a0; s < a1; s++) {
                    const c64 *row = sS + (size_t)s * pitch;
#pragma unroll
                    for (int f = 0; f < kFW; f++) v[f] += c_re(row[f]);
                }
                for (int s = a1; s < a2; s++) {
                    const c64 *row = sS + (size_t)s * pitch;
#pragma unroll
                    for (int f = 0; f < kFW; f++) v[f] += c_im(row[f]);
                }
            }
            __syncwarp();
            if (lane == 0) af_mbar_arrive(&pEmpty[lbuf]);          // frame warps may overwrite the power tile (and the sums in it)
            if (m < p.num) {
#pragma unroll
                for (int f = 0; f < kFW; f++) {
                    if (p.rawMel) { if (f < nf) stage[f * stagePitch + m] = v[f]; }
                    else L[f * kLPitch + m] = af_mfcc_rectify(v[f], p.rectify);
                }
            }
            if (!p.rawMel) {
                __syncwarp();
                if (lane == 0) af_mbar_arrive(&lFull[lbuf]);       // the DCT warps take the tile from here
                continue;
            }
            af_fence_proxy_async_smem();
            named_bar_sync(3, kBW * 32);                           // the result rows are staged
            const long long tileOff = ((long long)clip * p.timeLength + f0) * rowFloats;
            if (p.bulkStore) {
                if (e == 0) {                                       // one row per lane (padded staging rows)
                    if (lane < nf) af_bulk_store(p.out + tileOff + (long long)lane * rowFloats, stage + lane * stagePitch, (uint32_t)(rowFloats * 4));
                    af_bulk_commit();
                }
            } else {
                for (int r = 0; r < nf; r++)
                    for (int i = e * 32 + lane; i < rowFloats; i += kBW * 32) p.out[tileOff + (long long)r * rowFloats + i] = stage[r * stagePitch + i];
            }
        }
        if (e == 0) af_bulk_wait0();
        return;
    }

    if (dct_warp_index(warp) >= 0) {
        // ================= DCT warps: ortho DCT-II of the log-mel tile on the tensor cores, then the tile leaves =================
        if (p.rawMel) return;
        const int d = dct_warp_index(warp);
        const int g = lane >> 2, t = lane & 3;
        constexpr int kNB = (CT + kDW - 1) / kDW;                  // n-blocks of the DCT per warp
        float *stage = sStage;
        int it = 0;
        for (unsigned tile = blockIdx.x; tile < p.totalTiles; tile += gridDim.x, ++it) {
            const unsigned clip = tile / (unsigned)p.tilesPerClip;
            const int f0 = (int)(tile - clip * (unsigned)p.tilesPerClip) * F;
            const int nf = min(F, p.timeLength - f0);
            const int lbuf = it & 1;
            const float *L = sL + (size_t)lbuf * 16 * kLPitch;
            af_mbar_wait(&lFull[lbuf], (uint32_t)(it >> 1) & 1u);
            // out[16 x 8 CT] = L[16 x 128] . D^T[128 x 8 CT]: mma.sync m16n8k8 TF32, 3xTF32 split (hi by truncation,
            // lo = x - hi exact), separate accumulators for hi*hi and the cross terms
            float acc[kNB][4], acx[kNB][4];
#pragma unroll
            for (int n = 0; n < kNB; n++) {
                acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.0f;
                acx[n][0] = acx[n][1] = acx[n][2] = acx[n][3] = 0.0f;
            }
#pragma unroll 2
            for (int k0 = 0; k0 < kMaxNum; k0 += 8) {
                const float af[4] = {L[g * kLPitch + k0 + t], L[(g + 8) * kLPitch + k0 + t],
                                     L[g * kLPitch + k0 + t + 4], L[(g + 8) * kLPitch + k0 + t + 4]};
                uint32_t ah[4], al[4];
#pragma unroll
                for (int i = 0; i < 4; i++) af_tf32_split(af[i], ah[i], al[i]);
#pragma unroll
                for (int n = 0; n < kNB; n++) {
                    const int nb = d + n * kDW;
                    if (nb < CT) {
                        const float bf[2] = {sDct[(k0 + t) * p.dctPitch + nb * 8 + g], sDct[(k0 + t + 4) * p.dctPitch + nb * 8 + g]};
                        uint32_t bh[2], bl[2];
#pragma unroll
                        for (int i = 0; i < 2; i++) af_tf32_split(bf[i], bh[i], bl[i]);
                        AF_MMA_TF32(acx[n], al[0], al[1], al[2], al[3], bh[0], bh[1]);
                        AF_MMA_TF32(acc[n], ah[0], ah[1], ah[2], ah[3], bh[0], bh[1]);
                        AF_MMA_TF32(acx[n], ah[0], ah[1], ah[2], ah[3], bl[0], bl[1]);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) af_mbar_arrive(&lEmpty[lbuf]);          // the bank warps may refill this log-mel tile
            if (d == 0) af_bulk_wait_read0();                         // the previous tile's bulk stores have read the staging tile
            named_bar_sync(2, kDW * 32);
            // C fragment: rows g and g+8, columns nb*8 + 2t, +1 -> dense staging tile [nf][ccNum]
#pragma unroll
            for (int n = 0; n < kNB; n++) {
                const int nb = d + n * kDW;
                if (nb >= CT) continue;
                const int c = nb * 8 + 2 * t;
                const float v0 = acc[n][0] + acx[n][0], v1 = acc[n][1] + acx[n][1];
                const float v2 = acc[n][2] + acx[n][2], v3 = acc[n][3] + acx[n][3];
                if (g < nf) {
                    if (c < p.ccNum) stage[g * p.ccNum + c] = v0;
                    if (c + 1 < p.ccNum) stage[g * p.ccNum + c + 1] = v1;
                }
                if (g + 8 < nf) {
                    if (c < p.ccNum) stage[(g + 8) * p.ccNum + c] = v2;
                    if (c + 1 < p.ccNum) stage[(g + 8) * p.ccNum + c + 1] = v3;
                }
            }
            af_fence_proxy_async_smem();
            named_bar_sync(4, kDW * 32);                           // the result tile is staged
            // ---- the tile leaves: destination 0 is this GPU's buffer, 1..nPeer the peers' gathered arrays (NVLink) ----
            const long long tileOff = ((long long)clip * p.timeLength + f0) * p.ccNum;
            if (p.bulkStore) {
                if (d == 0 && lane <= p.nPeer) {                   // one destination per lane, the whole tile at once
                    float *o = (lane == 0 ? p.out : p.peerOut[lane - 1]) + tileOff;
                    af_bulk_store(o, stage, (uint32_t)(nf * p.ccNum * 4));
                    af_bulk_commit();
                }
            } else {
                const int n = nf * p.ccNum;
                for (int dst = 0; dst <= p.nPeer; dst++) {
                    float *o = (dst == 0 ? p.out : p.peerOut[dst - 1]) + tileOff;
                    for (int i = d * 32 + lane; i < n; i += kDW * 32) o[i] = stage[i];
                }
                named_bar_sync(2, kDW * 32);                       // staging tile read before the next tile's fragments land
            }
        }
        if (d == 0) af_bulk_wait0();
        return;
    }

    // ================= frame warps: warp w transforms frame f0 + w of every tile =================
    const c64 *sWinC = reinterpret_cast<const c64 *>(sWin);
    const c64 *sTwC = reinterpret_cast<const c64 *>(sTw);
    // addresses (floats) in this frame's column: power of bin = lane + 64 k2 (k2 < 16) and 64 (32 - k2) - lane (k2 >= 16);
    // transposes: lane n2 writes pair n2 / 2 of every row, lane k1 reads row k1 - 1 (lane 0 has no column: it reads
    // row 0 with lane 1, and its spectrum is never stored)
    const int strideK2 = 64 * pitch;
    const int offLo = (lane >> 1) * (2 * pitch) + (lane & 1);
    const int offHi = -((lane + 1) >> 1) * (2 * pitch) + (lane & 1);
    const int trWrite = (lane >> 1) * (kTrRows * 2 * pitch) + (lane & 1);
    const int trRead = (lane ? lane - 1 : 0) * pitch;

    int it = 0, stage = 0;
    uint32_t stagePhase = 0;
    // position of the tile inside its clip, advanced by gridDim.x tiles per iteration (no division in the loop)
    unsigned tIn = blockIdx.x % (unsigned)p.tilesPerClip;
    const unsigned tStep = gridDim.x % (unsigned)p.tilesPerClip;
    for (unsigned tile = blockIdx.x; tile < p.totalTiles; tile += gridDim.x, ++it) {
        const int f0 = (int)tIn * F;
        tIn += tStep;
        if (tIn >= (unsigned)p.tilesPerClip) tIn -= (unsigned)p.tilesPerClip;
        const int nf = min(F, p.timeLength - f0);
        const bool active = warp < nf;
        const int sb = it & 1;                                     // spectrum buffer and power tile of this tile
        float *col = sP + sb * kTileFloats + 2 * warp;              // this frame's column of the power tile

        af_mbar_wait(&fullBar[stage], stagePhase);

        c64 z[32];
        if (active) {
            // ---- A: x[32 n1 + lane], n1 = 0..63; packed z[m] = (s[2m], s[2m+1]) (0.5 w is applied in B) ----
            const float *sp = span + (size_t)stage * p.spanFloats + warp * p.hop + lane;
#pragma unroll
            for (int m = 0; m < 32; m++) z[m] = c_pack(sp[64 * m], sp[64 * m + 32]);
        }
        __syncwarp();
        if (lane == 0) af_mbar_arrive(&emptyBar[stage]);           // span slot may be refilled
        if (++stage == p.stages) { stage = 0; stagePhase ^= 1u; }
        if (!active) {
            // keep the tile protocols in step (one arrival per warp per tile and barrier, after the release of tile it - 2)
            af_mbar_wait(&pEmpty[sb], ((uint32_t)(it >> 1) & 1u) ^ 1u);
            if (lane == 0) {
                af_mbar_arrive(&specFull[sb]);
                af_mbar_arrive(&cDone[sb]);
                af_mbar_arrive(&pFull[sb]);
            }
            continue;
        }

        // ---- B: 64-point real DFT of the windowed column: packed complex 32-point DFT + in-lane post-pass ----
        af_fft32_fma_win(z, sWinC + lane);                         // Z[k] at AF_BR5(k)
        // R[k] = (Z[k] + conj Z[32-k]) - i W_64^k (Z[k] - conj Z[32-k]) at AF_BR5(k), (R[0], R[32]) in z[0]
        af_rfft64_post_fma(z);
        // the bank is done with tile it - 2, so the producer has read that tile's special columns out of this spectrum
        // buffer, and this frame's column of the power tile is free
        af_mbar_wait(&pEmpty[sb], ((uint32_t)(it >> 1) & 1u) ^ 1u);
        sSpec[((size_t)sb * 32 + lane) * kSpecPitch + warp] = z[0];
        __syncwarp();
        if (lane == 0) af_mbar_arrive(&specFull[sb]);

        // ---- C: columns k1 = 1..31, 32 x 32 transpose (real plane, then imaginary plane) through this frame's column
        // of the power tile (slot map at kTrRows): 32-bit stores, lane k1 reads its row as 16 float2 (n2, n2 + 1). ----
        {
            float yr[32], yi[32];
            float *tw = col + trWrite;
            const float2 *row = reinterpret_cast<const float2 *>(col) + trRead;
#pragma unroll
            for (int k1 = 1; k1 < 32; k1++) c_unpack(z[AF_BR5(k1)], yr[k1], yi[k1]);
#pragma unroll
            for (int k1 = 1; k1 < 32; k1++) tw[(k1 - 1) * 2 * pitch] = yr[k1];
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 16; j++) { const float2 v = row[j * kTrRows * pitch]; yr[2 * j] = v.x; yr[2 * j + 1] = v.y; }
            __syncwarp();
#pragma unroll
            for (int k1 = 1; k1 < 32; k1++) tw[(k1 - 1) * 2 * pitch] = yi[k1];
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 16; j++) {
                const float2 v = row[j * kTrRows * pitch];
                z[2 * j] = c_pack(yr[2 * j], v.x);
                z[2 * j + 1] = c_pack(yr[2 * j + 1], v.y);
            }
            __syncwarp();
            if (lane == 0) af_mbar_arrive(&cDone[sb]);             // the producer may store the special bins
        }
        // ---- D: 32-point DFT over n2 of the column times W_2048^(n2 k1), in lane k1: bins k1 + 64 k2 and, mirrored,
        // 64 (32 - k2) - k1.  The twiddle is applied as (1 - i t) and a gain g inside the first butterflies. ----
        af_fft32_fma_tw(z, sTwC + lane);
        if (lane) {
            if (p.dataType == SpectralData_Mag) {                  // (uniform branch: no sqrt sequence in the power path)
#pragma unroll
                for (int k2 = 0; k2 < 32; k2++) {
                    const float pw = sqrtf(c_norm2_fma(z[AF_BR5(k2)]));
                    if (k2 < 16) col[offLo + k2 * strideK2] = pw;
                    else col[offHi + (32 - k2) * strideK2] = pw;
                }
            } else {
#pragma unroll
                for (int k2 = 0; k2 < 32; k2++) {
                    const float pw = c_norm2_fma(z[AF_BR5(k2)]);
                    if (k2 < 16) col[offLo + k2 * strideK2] = pw;
                    else col[offHi + (32 - k2) * strideK2] = pw;
                }
            }
        }
        __syncwarp();
        if (lane == 0) af_mbar_arrive(&pFull[sb]);
    }
}

void free_plan(Plan *pl) {
    if (!pl) return;
    af_dev_free(pl->dWinPairs); af_dev_free(pl->dTw); af_dev_free(pl->dDct); af_dev_free(pl->dTab); af_dev_free(pl->dDesc); af_dev_free(pl->dAssign); af_dev_free(pl->dPrefix);
    free(pl->tab);
    free(pl);
}

// ---- interval form of a banded bank in which at most two consecutive filters overlap on any bin ------------------
// Every bin k with a non-zero weight is given to ONE interval i in [0, num]: on interval i filter i contributes its
// weight as "rise" and filter i-1 as "fall", so   mel_m = sum_{k in I_m} bank[m][k] P[k] + sum_{k in I_{m+1}} bank[m][k] P[k]
// with the bank's own float weights (the same products as the direct form, each bin read once for both filters).
struct Intervals {
    int owner[kBins];               // interval of each bin, -1 = no filter covers it
    int first[kMaxNum + 1], last[kMaxNum + 1];     // bin range of interval i (last < first: empty)
};

bool build_intervals2(const float *bank, int num, Intervals *iv) {
    if (num < 1 || num > kMaxNum) return false;
    int cur = 0;
    int peak[kMaxNum];
    for (int m = 0; m < num; m++) peak[m] = -1;
    for (int i = 0; i <= num; i++) { iv->first[i] = 1; iv->last[i] = 0; }
    for (int k = 0; k < kBins; k++) {
        int cover[3], nc = 0;
        for (int m = 0; m < num && nc < 3; m++)
            if (bank[(size_t)m * kBins + k] != 0.0f) cover[nc++] = m;
        iv->owner[k] = -1;
        if (nc == 0) continue;
        if (nc > 2 || (nc == 2 && cover[1] != cover[0] + 1)) return false;
        int i;
        if (nc == 2) i = cover[1];
        else {
            // one filter only: its rising side (interval m) up to its peak, its falling side (interval m + 1) after it --
            // keeps the two outer slopes of the bank in intervals of their own instead of one double-length interval
            const int m = cover[0];
            if (peak[m] < 0) {
                int best = k;
                for (int kk = k; kk < kBins && bank[(size_t)m * kBins + kk] != 0.0f; kk++)
                    if (bank[(size_t)m * kBins + kk] > bank[(size_t)m * kBins + best]) best = kk;
                peak[m] = best;
            }
            i = (cur <= m && k <= peak[m]) ? m : m + 1;
        }
        if (i < cur || i > cover[0] + 1) return false;             // intervals must be monotone runs of bins
        cur = i;
        iv->owner[k] = i;
        if (iv->last[i] < iv->first[i]) iv->first[i] = k;
        iv->last[i] = k;
    }
    return true;
}

// table: per interval the float4 (rise[2q], rise[2q+1], fall[2q], fall[2q+1]) of its bin pairs q; returns entries or -1
int build_table(const float *bank, int num, const Intervals *iv, unsigned *desc /* num+2 */, float4 *tab /* kMaxTab */) {
    int off = 0;
    for (int i = 0; i <= num; i++) {
        const bool empty = iv->last[i] < iv->first[i];
        const int q0 = empty ? 0 : iv->first[i] >> 1, q1 = empty ? -1 : iv->last[i] >> 1;
        desc[i] = ((unsigned)q0 << 16) | (unsigned)off;
        for (int q = q0; q <= q1; q++) {
            if (off >= kMaxTab) return -1;
            float w[4] = {0, 0, 0, 0};
            for (int h = 0; h < 2; h++) {
                const int k = 2 * q + h;
                if (k >= kBins || iv->owner[k] != i) continue;
                if (i < num) w[h] = bank[(size_t)i * kBins + k];
                if (i > 0) w[2 + h] = bank[(size_t)(i - 1) * kBins + k];
            }
            tab[off++] = make_float4(w[0], w[1], w[2], w[3]);
        }
    }
    desc[num + 1] = (unsigned)off;
    return off;
}

// Pieces: every interval is cut into runs of at most lmax bin pairs (interval order = ascending rows of the power tile).
// Pass q takes pieces [q W, (q + 1) W), W = helper lanes; a piece's partial sums are stored in row `piece index` of the
// power tile once its pass is over, so pass q must not read rows below q W.  lmax is the smallest value for which the
// pieces fit the passes (at most kMaxPieces pieces) and that condition holds.  Inside a pass the pieces are dealt to half-warps
// (16 lanes) such that their first rows differ mod 16 where possible: with the odd tile pitch the 16 lanes then read 16
// different 8-byte bank pairs for every frame and every step of the walk (conflict-free LDS.64).
// Returns the number of passes or -1 when no lmax <= 15 works.
struct PiecePlan {
    int nPieces, lmax, firstPass2, nPass, passLen[kMaxPass];
    unsigned pieceDesc[kMaxPieces];
    unsigned short prefix[kMaxNum + 4];
    unsigned short assign[kMaxPass * kEW * 32];
};

int plan_pieces(int num, const unsigned *desc /* num + 2 */, PiecePlan *pp) {
    const int W = kEW * 32, n = num + 1;
    for (int lmax = 1; lmax <= 15; lmax++) {
        int cnt = 0;
        bool fits = true;
        for (int i = 0; i < n && fits; i++) {
            const int off = (int)(desc[i] & 0xffffu), len = (int)(desc[i + 1] & 0xffffu) - off, q0 = (int)(desc[i] >> 16);
            pp->prefix[i] = (unsigned short)cnt;
            for (int j = 0; j < len; j += lmax) {
                if (cnt >= kMaxPieces) { fits = false; break; }
                const int l = len - j < lmax ? len - j : lmax;
                pp->pieceDesc[cnt++] = ((unsigned)(q0 + j) << 20) | ((unsigned)l << 16) | (unsigned)(off + j);
            }
        }
        if (!fits) continue;
        for (int i = n; i < kMaxNum + 4; i++) pp->prefix[i] = (unsigned short)cnt;
        for (int i = cnt; i < kMaxPieces; i++) pp->pieceDesc[i] = 0;
        if (cnt > kPairs || cnt > kMaxPass * W) continue;                    // (slots are rows of the power tile)
        const int nPass = (cnt + W - 1) / W;
        bool ok = true;                                                      // pass q must not read a row that holds a sum of passes < q
        for (int q = 1; q < nPass && ok; q++) ok = (int)(pp->pieceDesc[q * W] >> 20) >= q * W;
        if (!ok) continue;
        const int n0 = cnt < W ? cnt : W;
        pp->nPieces = cnt; pp->lmax = lmax; pp->firstPass2 = n0; pp->nPass = nPass;
        for (int i = 0; i < kMaxPass * W; i++) pp->assign[i] = 0xffffu;
        for (int ps = 0; ps < kMaxPass; ps++) pp->passLen[ps] = 0;
        for (int ps = 0; ps < pp->nPass; ps++) {
            const int base = ps * W, m = cnt - base < W ? cnt - base : W;
            unsigned short *row = pp->assign + (size_t)ps * W;
            int used[2 * kEW][16], fill[2 * kEW];
            memset(used, 0, sizeof(used)); memset(fill, 0, sizeof(fill));
            int later[kMaxPieces], nLater = 0;
            for (int c = 0; c < m; c++) {                                    // first round: a half-warp whose residue slot is free
                const int pc = base + c, r = (int)(pp->pieceDesc[pc] >> 20) & 15, l = (int)(pp->pieceDesc[pc] >> 16) & 15;
                if (l > pp->passLen[ps]) pp->passLen[ps] = l;
                int best = -1;
                for (int h = 0; h < 2 * kEW; h++)
                    if (fill[h] < 16 && !used[h][r] && (best < 0 || fill[h] < fill[best])) best = h;
                if (best < 0) { later[nLater++] = pc; continue; }
                used[best][r] = 1;
                row[best * 16 + fill[best]++] = (unsigned short)pc;
            }
            for (int c = 0; c < nLater; c++) {                               // the rest: wherever there is room (a 2-way conflict)
                int best = -1;
                for (int h = 0; h < 2 * kEW; h++) if (fill[h] < 16 && (best < 0 || fill[h] < fill[best])) best = h;
                row[best * 16 + fill[best]++] = (unsigned short)later[c];
            }
        }
        return pp->nPass;
    }
    return -1;
}

constexpr int kSmemBudget = 227 * 1024;

// Shared-memory carve-up: as many frames per tile as fit (<= kFW), two TMA stages when they fit, else one.  Fills the
// offsets, framesPerTile, stages, spanFloats and stageBytes of *pp (dctPitch must be set); returns the bytes, or -1
// when not even one frame fits.
int carve_smem(Params *pp, int timeLength, int hop, int num, int ccNum, int tabLen, int rawMel) {
    int F = kFW < timeLength ? kFW : timeLength, stages = 2;
    for (;;) {
        int o = kBarBytes;                                      // the mbarriers come first
        const int spanFloats = (F - 1) * hop + kN;
        pp->offSpan = o;    o += stages * spanFloats * 4;
        pp->offP = o;       o += (2 * kTileFloats * 4 + 15) & ~15;
        pp->offWin = o;     o += 32 * 32 * 8;
        pp->offTw = o;      o += kTwRows * 32 * 8;
        pp->offSpec = o;    o += 2 * 32 * kSpecPitch * 8;
        pp->offDct = o;     o += rawMel ? 0 : kMaxNum * pp->dctPitch * 4;
        pp->offL = o;       o += 2 * 16 * kLPitch * 4;
        pp->stageBytes = rawMel ? 2 * ((F * (num + 4) * 4 + 15) & ~15) : ((F * ccNum * 4 + 15) & ~15);
        pp->offStage = o;   o += pp->stageBytes;
        pp->offTab = o;     o += tabLen * 16;
        pp->offDesc = o;    o += kMaxPieces * 4;
        pp->offAssign = o;  o += (kMaxPass * kEW * 32 * 2 + 15) & ~15;
        pp->offPrefix = o;  o += ((kMaxNum + 4) * 2 + 15) & ~15;
        pp->spanFloats = spanFloats;
        pp->framesPerTile = F; pp->stages = stages;
        if (o <= kSmemBudget) return o;
        if (stages == 2) { stages = 1; continue; }
        stages = 2;
        if (--F < 1) return -1;
    }
}

}  // namespace

int af_mfcc2_supported(int fftLength, int num, int ccNum, const float *bank) {
    if (fftLength != kN || num < 1 || num > kMaxNum || ccNum < 1 || ccNum > 64 || !bank) return 0;
    Intervals *iv = static_cast<Intervals *>(malloc(sizeof(Intervals)));
    float4 *tab = static_cast<float4 *>(malloc(sizeof(float4) * kMaxTab));
    unsigned desc[kMaxNum + 4];
    PiecePlan *pc = static_cast<PiecePlan *>(malloc(sizeof(PiecePlan)));
    const int ok = iv && tab && pc && build_intervals2(bank, num, iv) && build_table(bank, num, iv, desc, tab) >= 0 &&
                   plan_pieces(num, desc, pc) > 0;
    free(iv); free(tab); free(pc);
    return ok;
}

void af_mfcc2_plan_free(void *plan) { free_plan(static_cast<Plan *>(plan)); }

int af_mfcc2_plan_build(void **planOut, int fftLength, int num, int ccNum, const float *window, const float *bank,
                        const float *dct /* ccNum x num */, int dataType) {
    *planOut = NULL;
    if (!af_mfcc2_supported(fftLength, num, ccNum, bank)) return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC v2 plan: unsupported configuration");
    Plan *pl = static_cast<Plan *>(calloc(1, sizeof(Plan)));
    if (!pl) return AF_ERR_NOMEM;
    pl->num = num; pl->ccNum = ccNum; pl->dataType = dataType;
    pl->ct = af_mfcc_ct(ccNum);
    int rc = AF_OK;

    float2 *wp = static_cast<float2 *>(malloc(sizeof(float2) * 1024));
    for (int m = 0; m < 32; m++)
        for (int l = 0; l < 32; l++) wp[m * 32 + l] = make_float2(0.5f * window[64 * m + l], 0.5f * window[64 * m + 32 + l]);
    rc = af_dev_upload(reinterpret_cast<void **>(&pl->dWinPairs), wp, sizeof(float2) * 1024);
    // g = cos, t = tan for every entry (u = 1): the factor u in {1, -i} that would keep |t| <= 1 differs between the
    // lanes of one instruction.  n2 k1 <= 961 never hits 512 (cos = 0); |t| <= 326, and g (x + t y) still rounds as c x + s y.
    for (int n2 = 1; n2 <= kTwRows; n2++)
        for (int k1 = 0; k1 < 32; k1++) {
            const double a = 2.0 * M_PI * (double)(n2 * k1) / 2048.0;
            wp[(n2 - 1) * 32 + k1] = make_float2((float)cos(a), (float)tan(a));
        }
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dTw), wp, sizeof(float2) * kTwRows * 32);
    free(wp);

    Intervals *iv = static_cast<Intervals *>(malloc(sizeof(Intervals)));
    pl->tab = static_cast<float4 *>(malloc(sizeof(float4) * kMaxTab));
    if (!iv || !pl->tab) { free(iv); free_plan(pl); return AF_ERR_NOMEM; }
    build_intervals2(bank, num, iv);
    pl->tabLen = build_table(bank, num, iv, pl->ivDesc, pl->tab);
    free(iv);
    for (int i = num + 2; i < kMaxNum + 4; i++) pl->ivDesc[i] = pl->ivDesc[num + 1];
    {
        PiecePlan *pc = static_cast<PiecePlan *>(malloc(sizeof(PiecePlan)));
        if (!pc || plan_pieces(num, pl->ivDesc, pc) <= 0) { free(pc); free_plan(pl); return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC v2 plan: no piece plan"); }
        pl->nPass = pc->nPass; pl->nPieces = pc->nPieces; pl->lmax = pc->lmax; pl->firstPass2 = pc->firstPass2;
        memcpy(pl->pieceDesc, pc->pieceDesc, sizeof(pl->pieceDesc));
        memcpy(pl->piecePrefix, pc->prefix, sizeof(pl->piecePrefix));
        memcpy(pl->assign, pc->assign, sizeof(pl->assign));
        free(pc);
    }
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dAssign), pl->assign, sizeof(pl->assign));
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dTab), pl->tab, sizeof(float4) * (size_t)(pl->tabLen > 0 ? pl->tabLen : 1));
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dDesc), pl->pieceDesc, sizeof(pl->pieceDesc));
    if (rc == AF_OK) rc = af_dev_upload(reinterpret_cast<void **>(&pl->dPrefix), pl->piecePrefix, sizeof(pl->piecePrefix));
    if (rc == AF_OK) rc = af_mfcc_dct_upload(&pl->dDct, dct, num, ccNum, pl->ct);
    if (rc != AF_OK) { free_plan(pl); return rc; }
    *planOut = pl;
    return AF_OK;
}

int af_mfcc2_launch(void *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                    int rectifyType, float *out, int nPeer, float *const *peerOut, int rawMel, void *stream) {
    Plan *pl = static_cast<Plan *>(plan);
    Params *pp = static_cast<Params *>(malloc(sizeof(Params)));     // 24 KB: off the stack
    if (!pp) return AF_ERR_NOMEM;
    memset(pp, 0, sizeof(Params));
    pp->data = data; pp->out = out; pp->winPairs = pl->dWinPairs; pp->tw = pl->dTw; pp->dct = pl->dDct;
    pp->dataStride = dataLength; pp->batch = batch; pp->timeLength = timeLength; pp->hop = slideLength;
    pp->num = pl->num; pp->ccNum = pl->ccNum; pp->rectify = rectifyType; pp->dataType = pl->dataType; pp->rawMel = rawMel;
    pp->dctPitch = af_mfcc_dct_pitch(pl->ct);
    pp->nPeer = nPeer;
    for (int d = 0; d < nPeer; d++) pp->peerOut[d] = peerOut[d];
    pp->nPass = pl->nPass; pp->assign = pl->dAssign;
    pp->bankTab = pl->dTab; pp->pieceDesc = pl->dDesc; pp->piecePrefix = pl->dPrefix; pp->tabLen = pl->tabLen;
    pp->bulkStore = af_mfcc_bulk_store_ok(rawMel ? pl->num : pl->ccNum, out, nPeer, peerOut);

    const int total = carve_smem(pp, timeLength, slideLength, pl->num, pl->ccNum, pl->tabLen, rawMel);
    if (total < 0) { free(pp); return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC: slideLength %d too large for shared memory", slideLength); }
    const int F = pp->framesPerTile;
    pp->tilesPerClip = (timeLength + F - 1) / F;
    if ((long long)pp->tilesPerClip * batch >= (1ll << 31)) { free(pp); return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC: more than 2^31 tiles in one launch"); }
    pp->totalTiles = (unsigned)((long long)pp->tilesPerClip * batch);
    static void (*const kernels[4])(Params) = {k_mfcc_fused2<2>, k_mfcc_fused2<3>, k_mfcc_fused2<5>, k_mfcc_fused2<8>};
    const int launched = af_mfcc_launch_ct(kernels, "k_mfcc_fused2", pl->ct, (long long)pp->totalTiles, kThreads, total, stream, *pp);
    free(pp);
    return launched;
}

// Test hook (host only): the shared-memory carve-up af_mfcc2_launch makes for a clip of timeLength frames at hop `hop`,
// a bank of `num` bands with tabLen table entries and ccNum coefficients (rawMel: the filter-bank output instead).
// Returns the bytes (-1: no frame fits); info = {frames per tile, TMA stages, offSpan, offP, offWin, offTw, offSpec,
// offDct, offL, offStage, offTab, offDesc, offAssign, offPrefix, stageBytes, spanFloats}.
extern "C" int afb200_mfccCarve2(int timeLength, int hop, int num, int ccNum, int tabLen, int rawMel, int *info /* 16 */) {
    if (timeLength < 1 || hop < 1 || num < 1 || num > kMaxNum || ccNum < 1 || ccNum > 64 || tabLen < 0 || tabLen > kMaxTab) return -1;
    Params pp;
    memset(&pp, 0, sizeof(pp));
    pp.dctPitch = af_mfcc_dct_pitch(af_mfcc_ct(ccNum));
    const int total = carve_smem(&pp, timeLength, hop, num, ccNum, tabLen, rawMel);
    if (info) {
        const int v[16] = {pp.framesPerTile, pp.stages, pp.offSpan, pp.offP, pp.offWin, pp.offTw, pp.offSpec, pp.offDct, pp.offL,
                           pp.offStage, pp.offTab, pp.offDesc, pp.offAssign, pp.offPrefix, pp.stageBytes, pp.spanFloats};
        memcpy(info, v, sizeof(v));
    }
    return total;
}

// Diagnostic / test hook (host only): the interval form the planner derives from a bank [num][1025], its cut into pieces
// and the lane assignment of the bank passes.  Returns the number of table entries (>= 0) or -1 when the bank does not
// have the two-overlap structure / no piece plan exists.  desc: per interval (first bin pair << 16) | table offset;
// pieceDesc [256]: (first bin pair << 20) | (pairs << 16) | table offset; prefix [num + 2]: first piece of interval i;
// assign: [passes][helper lanes] piece per lane (0xffff = none); info = {passes, helper lanes, pieces, lmax, pieces of
// pass 0, passLen[0..passes)}.
extern "C" int afb200_mfccBankPlan2(const float *bank, int num, int *owner /* 1025 */, unsigned *desc /* num+2 */,
                                    float *table /* 4 * 1408 */, unsigned *pieceDesc /* 256 */, unsigned short *prefix /* num+2 */,
                                    unsigned short *assign /* 2 * 128 */, int *info /* 16 */) {
    if (!bank || num < 1 || num > kMaxNum) return -1;
    Intervals *iv = static_cast<Intervals *>(malloc(sizeof(Intervals)));
    float4 *tab = static_cast<float4 *>(malloc(sizeof(float4) * kMaxTab));
    PiecePlan *pc = static_cast<PiecePlan *>(malloc(sizeof(PiecePlan)));
    unsigned d[kMaxNum + 4];
    int n = -1;
    if (iv && tab && pc && build_intervals2(bank, num, iv)) {
        n = build_table(bank, num, iv, d, tab);
        if (n >= 0 && plan_pieces(num, d, pc) <= 0) n = -1;
        if (n >= 0) {
            if (owner) memcpy(owner, iv->owner, sizeof(int) * kBins);
            if (desc) memcpy(desc, d, sizeof(unsigned) * (size_t)(num + 2));
            if (table) memcpy(table, tab, sizeof(float4) * (size_t)n);
            if (pieceDesc) memcpy(pieceDesc, pc->pieceDesc, sizeof(pc->pieceDesc));
            if (prefix) memcpy(prefix, pc->prefix, sizeof(unsigned short) * (size_t)(num + 2));
            if (assign) memcpy(assign, pc->assign, sizeof(unsigned short) * (size_t)pc->nPass * kEW * 32);
            if (info) {
                info[0] = pc->nPass; info[1] = kEW * 32; info[2] = pc->nPieces; info[3] = pc->lmax; info[4] = pc->firstPass2;
                for (int i = 0; i < pc->nPass; i++) info[5 + i] = pc->passLen[i];
            }
        }
    }
    free(iv); free(tab); free(pc);
    return n;
}
