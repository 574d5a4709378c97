/* af_internal.h -- private declarations shared by the host C files and the CUDA launchers. */
#ifndef AF_INTERNAL_H
#define AF_INTERNAL_H

#include <stddef.h>
#include "../../include/afb200_ext.h"

#ifdef __cplusplus
extern "C" {
#endif

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

/* ---------------- errors / device context (host/af_ctx.c) ---------------- */
#define AF_OK 0
#define AF_ERR_ARG 10
#define AF_ERR_CUDA 11
#define AF_ERR_NOGPU 12
#define AF_ERR_UNSUPPORTED 13
#define AF_ERR_NOMEM 14

int af_fail(int code, const char *fmt, ...);      /* records message, prints to stderr, returns code */
void af_clear_error(void);
int af_cuda_check(int cudaError, const char *what);   /* 0 ok, else AF_ERR_CUDA (message recorded) */
int af_device_ready(void);                        /* 0 when a usable GPU is selected, else error */

typedef struct {          /* growable device buffer */
    void *ptr;
    size_t bytes;
} AfDevBuf;
int af_devbuf_reserve(AfDevBuf *b, size_t bytes);
void af_devbuf_free(AfDevBuf *b);
int af_dev_upload(void **dptr, const void *host, size_t bytes);   /* cudaMalloc + H2D */
void af_dev_free(void *dptr);
int af_stream_sync(void *stream);
int af_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream);
int af_memset_d(void *dst, int v, size_t bytes, void *stream);
size_t af_dev_free_bytes(void);

/* Every batched entry point runs through af_run_batch, which holds the memKind rule:
 * - AFB200_MEM_DEVICE: the chunk function runs once on the caller's pointers and stream, without synchronising.
 * - AFB200_MEM_HOST: items flow through two device slots on three streams -- copy-in of chunk k+1, the transform of
 *   chunk k and copy-out of chunk k-1 overlap (H2D and D2H are opposite PCIe directions) -- and the call returns
 *   synchronised, with no copy into or out of caller memory still in flight, whether it succeeded or not.  With
 *   page-locked caller buffers a call runs at the speed of the larger transfer and needs at most two chunks of device
 *   memory instead of the batch; pageable buffers work too (the driver stages them synchronously).
 * A chunk is about `chunkBytes` of the larger side (in + in-out planes, or out + in-out planes), a multiple of 16
 * items when it holds at least 16, and at least one item.  Items must be independent of one another. */
enum { AF_IN = 1, AF_OUT = 2, AF_INOUT = 3 };
#define AF_PIPE_MAX_PLANES 7
#define AF_PIPE_CHUNK_BYTES ((size_t)64 << 20)
typedef struct {
    const void *ptr;      /* caller's pointer (host or device, as memKind says); NULL: the plane is not used in this call */
    size_t per;           /* floats per item */
    int dir;              /* AF_IN, AF_OUT or AF_INOUT: in-out planes are copied in before the chunk and back after it */
    int layers;           /* > 1: `layers` planes of batch x per floats one after the other (device chunk: layers x nb x per) */
} AfPlane;
typedef struct {
    int ready;
    void *stream, *inStream, *outStream, *evIn[2], *evDone[2], *evOut[2];
    AfDevBuf slot[2][AF_PIPE_MAX_PLANES];
} AfPipe;
/* transform of `nb` items on the device: d[i] is plane i (NULL when it is not used), ctx the entry point's arguments */
typedef int (*AfChunkFn)(void *ctx, int nb, float *const *d, void *stream);
int af_run_batch(AfPipe *pipe, int memKind, void *stream, AfChunkFn fn, void *ctx, const AfPlane *planes, int nPlanes,
                 int batch, size_t chunkBytes);
void af_pipe_free(AfPipe *pipe);
/* host-side ordering of a table rebuild after the kernels that read the old table: *ev records the end of the last
 * launch on `stream` (created on first use); af_fence_wait blocks until it has passed (no-op when NULL) */
int af_fence_record(void **ev, void *stream);
int af_fence_wait(void *ev);
/* device-side ordering: later work on `stream` waits for the launch *ev last recorded (no-op when NULL).  An object
 * whose device state is written and read from several streams brackets each use with af_fence_order(fence, st) and
 * af_fence_record(&fence, st): the fence then chains every use, whatever stream it ran on. */
int af_fence_order(void *ev, void *stream);
void af_fence_free(void *ev);
/* clips per group of a device workspace of perClip bytes per clip: a quarter of the free memory, at most cap bytes,
 * at least one clip and at most `batch` */
int af_chunk_clips(size_t perClip, size_t cap, int batch);

/* streaming bookkeeping shared by STFT, CQT and SpectrogramObj (stft_algorithm.c:474-599, cqt_algorithm.c:346-456):
 * the samples that did not complete a hop are carried to the next call */
typedef struct {
    float *buf;           /* fftLength + slideLength floats */
    int length;           /* may be negative when slideLength > fftLength: samples of the next call to skip */
    float *cur; size_t curCap;   /* tail ++ new samples */
} AfTail;
/* 1: *cur / *curLength hold the carried samples followed by `data`; 0: not a whole frame yet (or out of memory) */
int af_tail_assemble(AfTail *t, int fftLength, int slideLength, const float *data, int dataLength,
                     const float **cur, int *curLength);
void af_tail_free(AfTail *t);
int af_sm_count(void);

/* The frame-wise pitch trackers' core (host/af_pitch_frames.c), the first member of the PitchPEF, PitchYIN, PitchNCF
 * and PitchCEP objects: frames of n = 2^log2n samples every slideLength, the streaming carry and the staging pipe. */
typedef struct { int samplate, log2n, n, slideLength, isContinue; AfTail tail; AfPipe pipe; } AfPitchFrames;
/* a tracker's constructor constants: its name, largest radix2Exp and what limits it, lowFre's default, highFre's
 * default (NULL highFre) and the highFre that replaces a rejected one (lowFre then takes its default) */
typedef struct { const char *who; int maxExp; const char *why; float lowFre, highFre, highReset; } AfPitchRules;
/* samplate, lowFre, highFre, radix2Exp, slideLength and isContinue resolved in the reference's order into *f (no carry,
 * no pipe) and *lf / *hf; 0, or -2 above maxExp */
int af_pitch_frames_init(AfPitchFrames *f, float *lf, float *hf, const AfPitchRules *r, const int *samplate,
                         const float *lowFre, const float *highFre, const int *radix2Exp, const int *slideLength,
                         const int *isContinue);
int af_pitch_frames(const AfPitchFrames *f, int dataLength);        /* frames in dataLength samples */
int af_pitch_time_length(const AfPitchFrames *f, int dataLength);   /* calTimeLength: with the carry; 0 for NULL f */
/* the batched call's argument check ("<who>: bad argument") and device; *T the frames per clip, 0 for an empty batch */
int af_pitch_batch_begin(const AfPitchFrames *f, const char *who, const float *data, int dataLength, int batch,
                         const float *fre, int *T);
/* the legacy call's input in *x / *len (error cleared, carry assembled); returns its frames, 0: nothing to do */
int af_pitch_legacy_input(AfPitchFrames *f, const float *data, int dataLength, const float **x, int *len);
void af_pitch_frames_free(AfPitchFrames *f);                       /* the pipe and the carry */

/* ---------------- setup-time tables (host/af_window.c, af_filterbank.c, ...) ---------------- */
int af_window_symmetric(int windowType, int length, const float *value, double *out);
int af_window_fft(int windowType, int length, float *out);
int af_window_create(int windowType, int length, int periodic, float *out);

typedef struct {
    float low, high;      /* after the range rules of bftObj_new / cwtObj_new */
    int lowIndex, highIndex;   /* linear scale only */
} AfRange;
/* range defaults + Linear/Octave revisions shared by bftObj_new and cwtObj_new; returns 0 or -1 */
int af_revise_range(int num, int fftLength, int samplate, const float *lowFre, const float *highFre,
                    int scaleType, int binPerOctave, AfRange *out);
/* num+2 band edges (Hz) and their bins (isEdge=1: the num centres themselves, gammatone);
 * slaneyBins: 1 = first grid point above the edge */
void af_band_edges(int num, int fftLength, int samplate, float lowFre, float highFre, int scaleType,
                   int binPerOctave, int slaneyBins, int isEdge, float *freEdge, int *binEdge);
int af_auditory_filterbank(int num, int fftLength, int samplate, int scaleType, int styleType,
                           int normType, float lowFre, float highFre, int binPerOctave,
                           float *bank, float *freBandArr, int *binBandArr);

/* banded view of a dense row-major bank[num][width]: per row first non-zero and count */
typedef struct {
    int num, width;
    int *start, *len;     /* num each */
    int nnz, maxLen;
} AfBands;
int af_bands_build(const float *bank, int num, int width, AfBands *b);
void af_bands_free(AfBands *b);

void af_decimator_taps(float *left32, float *right31);

typedef struct {
    int num, binPerOctave, octaveNum, fftLength, samplate;
    int vqt, rows;       /* beta != 0: one kernel row per bin (rows = num), else the top octave's rows shared (rows = bpo) */
    float *freBandArr;   /* num+2 */
    float *sLenArr;      /* num: sqrt(kernel length) */
    float *kr, *ki;      /* rows x (fftLength/2+1) spectral kernels, thresholded */
} AfCqtBank;
int af_cqt_bank_build(AfCqtBank *b, int num, int samplate, float minFre, int binPerOctave, float factor,
                      float beta, float thresh, int windowType, int normType);
void af_cqt_bank_free(AfCqtBank *b);
/* time-domain kernels kappa[b][n] = sum_{k<=N/2} K[b][k] e^{-2 pi i k n/N}  -> 2 x rows x N floats */
int af_cqt_time_kernels(const AfCqtBank *b, float *kappaRe, float *kappaIm);
/* chroma folding matrix [num][cqtLength] of cqtObj_chroma; -1 when num does not divide binPerOctave */
int af_chroma_cqt_bank(int num, int cqtLength, int binPerOctave, float minFre, float *bank);

typedef struct {
    int waveletType;
    float gamma, beta, cf;
    double factor;       /* per-wavelet constant */
} AfWavelet;
int af_wavelet_setup(AfWavelet *w, int waveletType, const float *gamma, const float *beta);
float af_wavelet_eval(const AfWavelet *w, float sw);   /* psi_hat(s*omega), host reference of the device fn */
void af_cwt_scales(int num, int dataLength, int samplate, float lowFre, float highFre, int scaleType,
                   int binPerOctave, float cf, float *freBandArr, int *binBandArr, float *scaleArr);

void af_dct2_matrix(int num, int ccNum, float *out /* ccNum x num, ortho scaled */);
int af_dct2_upload_transposed(float **dDctT, int n);   /* device [n][n]: the transpose of af_dct2_matrix(n, n) */
void af_fft_twiddles(int n, float *cosArr, float *sinArr /* n/2 each: cos, -sin (2 pi i/n) */);

/* ---------------- kernel launchers (kernels directory), all asynchronous on `stream` ---------------- */
typedef struct {
    int fftLength, slideLength;
    int dataLength;       /* samples per clip */
    int timeLength;       /* frames per clip */
    int batch;
    int padLeft;          /* samples logically prepended (CQT / STFT padding) */
    int padMode;          /* PaddingMode_Constant (0) | Reflect | Wrap: content of the logical samples outside the clip */
    float padValue1, padValue2;   /* constant mode: value left / right of the clip (0 for CQT) */
    int validLength;      /* samples of the clip actually used (dataLength minus dropped tail) */
    const float *window;  /* device, fftLength (NULL = rect) */
    const float *data;    /* device, batch x dataLength */
} AfFrameSrc;

enum { AF_STFT_FULL = 0, AF_STFT_HALF = 1, AF_STFT_POWER = 2, AF_STFT_MAG = 3, AF_STFT_SQUARE = 4 };
/* generic framed real FFT.  FULL: planes T x n mirrored; HALF: planes T x (n/2+1);
 * POWER/MAG: outRe = |X|^2 or |X| (optionally ^normValue when POWER), T x (n/2+1);
 * SQUARE: (re,im) <- X^2 complex square, T x (n/2+1). */
int af_launch_stft(const AfFrameSrc *src, int mode, float normValue, float *outRe, float *outIm, void *stream);

/* inverse STFT: planes [batch*T][width] (width = n or n/2+1) -> data[batch][(T-1)*hop+n] (accumulating, then
 * divided by the window sum); frames = scratch batch*T*n floats; window NULL = rect */
int af_launch_istft(const float *re, const float *im, int width, int fftLength, int slideLength, int timeLength,
                    int batch, const float *window, int methodType, float *frames, float *data, void *stream);

typedef struct {
    int num, width;               /* width = fftLength/2+1 */
    const float *dense;           /* device num x width */
    const int *start, *len;       /* device, num each */
    const float *packed;          /* device, band weights row after row */
    const int *packedOff;         /* device, num each */
    int banded;                   /* 1: use band kernels */
    int maxLen;
} AfBankDev;
/* out[r][m] = sum_k in[r][k] * bank[m][k]  (rows = batch*T); optional out <- out^postPow */
int af_launch_bank(const AfBankDev *bank, const float *in, int rows, float postPow, float *out, void *stream);
/* in-place SQUARE / POWER / MAG of half-spectrum planes (modes of af_launch_stft) */
int af_launch_spec_post(float *re, float *im, long long cells, int mode, float normValue, void *stream);
int af_launch_copy_cols(const float *in, int rows, int width, int lo, int count, float *out, void *stream);
/* rectify (0 log10 clamp 1e-8 | 1 cube root) then out[r][c] = sum_m D[c][m] * rect(in[r][m]) */
int af_launch_xxcc(const float *in, int rows, int num, int ccNum, int rectifyType, const float *dct,
                   float *out, void *stream);
/* cepstra + log-energy replace/append + the reference's per-frame delta FIRs (xxcc_algorithm.c:168-296) */
int af_launch_xxcc_standard(const float *in, const float *energy, int rows, int num, int ccNum,
                            int rectifyType, int energyType, int order, const float *dctT,
                            float *coe, float *d1, float *d2, void *stream);

/* out[r][c] = normalise_c( sum_j bank[c][j] * (re^2+im^2 | sqrt) ) (cqt_algorithm.c:484-600) */
int af_launch_chroma(const float *re, const float *im, int rows, int num, int chromaNum, int isMag,
                     int normType, const float *bank, float *out, void *stream);

/* Fused MFCC at fftLength 2048: framed STFT -> |X|^2 / |X| -> banded bank (-> log10 / cbrt -> DCT-II) in one kernel.
 * v2 (kernels/mfcc_fused2.cu) serves banks in which at most two consecutive filters overlap on a bin, v1
 * (kernels/mfcc_fused.cu) the other banks its weight table holds; everything else takes the composed kernels. */
enum { AF_MFCC_COMPOSED = -1, AF_MFCC_V1 = 0, AF_MFCC_V2 = 1 };
typedef struct {
    int bankOnly, realMode, ccNum;    /* bftObj_bft's bank output (fused only in real mode), or ccNum cepstral coefficients */
    int reassign, linear, banded;     /* the object: reassigned spectrum, Linear scale, banded device bank */
    float normValue;
    int fftLength, num, slideLength, dataLength;
    const float *data, *bank;         /* device clips; host bank num x (fftLength/2+1) */
    const AfBands *bands;
    int *v2Bank;                      /* the object's cache of v2's verdict on its bank: 0 unknown, 1 accepted, -1 rejected */
} AfMfccCall;
/* AF_MFCC_V2 / AF_MFCC_V1 / AF_MFCC_COMPOSED for one call (host only); reads the test hooks AFB200_MFCC_KERNEL=v1 and
 * AFB200_BFT_GENERAL (bank output through the composed kernels) */
int af_mfcc_route(const AfMfccCall *call);
typedef struct AfMfccPlan AfMfccPlan;   /* device tables of one kernel (AF_MFCC_V1 | AF_MFCC_V2), bank-only or ccNum coefficients */
int af_mfcc_plan_build(AfMfccPlan **plan, int kernel, int bankOnly, int fftLength, int num, int ccNum, const float *window,
                       const float *bank, const AfBands *bands, int dataType);
int af_mfcc_plan_kind(const AfMfccPlan *plan);     /* its kernel, AF_MFCC_COMPOSED for NULL */
void af_mfcc_plan_free(AfMfccPlan *plan);
/* out: batch x T x num (bank-only plan) or batch x T x ccNum, the latter also stored at the same offset of every
 * peerOut[0..nPeer) (fused all-gather) */
int af_launch_mfcc(const AfMfccPlan *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                   int rectifyType, float *out, int nPeer, float *const *peerOut, void *stream);

int af_launch_decimate2(const float *in, int inLength, int inStride, int batch, const float *left32,
                        const float *right31, float *out, int outStride, void *stream);

/* CQT octave plan (host/af_cqt.c): the one function that picks the kernel and tile of an octave, shared by the compute
 * path and the cqtObj_octavePlan query.  Tile constants the kernels are compiled with (cqt.cu, cqt_wgmma.cu): */
#define AF_CQT_BINS_PER_PASS 12   /* FP32 loop: bins whose kernels sit in shared memory together */
#define AF_CQT_FT 4               /* FP32 loop: frames per thread */
#define AF_CQT_JG 2               /* FP32 loop: thread groups over bins */
#define AF_CQT_BT 6               /* FP32 loop: bins per thread */
#define AF_CQT_TC_MT 2            /* mma.sync: 16-frame m-tiles per warp */
#define AF_CQT_TC_KC 16           /* mma.sync: k-steps (8 taps) of kernel fragments resident in shared memory */
#define AF_CQT_WG_CHUNK_K 128     /* wgmma: taps per kernel chunk in shared memory */
#define AF_CQT_WG_MT 2            /* wgmma: 64-frame m-tiles per warpgroup, at most */
enum { AF_CQT_WGMMA = 0, AF_CQT_TC = 1, AF_CQT_LOOP = 2, AF_CQT_DIRECT = 3 };
typedef struct {
    int kernel;           /* AF_CQT_* */
    int TT;               /* frames per CTA (0: direct kernel) */
    int threads;          /* threads per CTA */
    int segs;             /* FP32 loop: tap segments summed through shared memory (else 1) */
    int smem;             /* dynamic shared-memory bytes */
    int rowLen;           /* polyphase row pitch in floats (FP32 loop; mma.sync / wgmma with hop >= 8) */
    int rowsA, nChunk;    /* FP32 loop: ceil(fftLength / hop), kernel taps resident in shared memory at a time */
    int warps;            /* mma.sync: warps per CTA */
    int wg, mt;           /* wgmma: warpgroups per CTA, m-tiles per warpgroup */
} AfCqtOctPlan;
/* device kernel tables an object of this shape uploads: mma.sync B fragments / wgmma B images */
int af_cqt_tc_tables(int fftLength, int bpo);
int af_cqt_wgmma_tables(int fftLength, int bpo);
/* kernel and tile of one octave with hop `hop`: wgmma where the hop allows it, else mma.sync 3xTF32, else the FP32 loop,
 * else (no polyphase tile fits) the direct kernel.  Host only. */
void af_cqt_octave_plan(int fftLength, int hop, int bpo, AfCqtOctPlan *plan);

/* out[b][t][colOff + j] (row stride num) = scale[j] * sum_n xpad[t*hop + n] * kappa[j][n];
 * kappa2 = interleaved (re, im) pairs [bpo][fftLength]; plan: AF_CQT_LOOP or AF_CQT_DIRECT */
int af_launch_cqt_octave(const AfCqtOctPlan *plan, const float *sig, int sigLength, int sigStride, int batch, int validLength,
                         int fftLength, int hop, int padLeft, int timeLength, int bpo, const float *kappa2,
                         const float *scale, int num, int colOff,
                         float *outRe, float *outIm, void *stream);

/* tensor-core octave kernel (3xTF32 mma.sync): 12 bins per octave, power-of-two hop >= 2; plan: AF_CQT_TC */
void af_cqt_tc_fragments(const float *kappa2, int fftLength, float *out /* fftLength/8 * 96 * 4 floats */);
int af_launch_cqt_octave_tc(const AfCqtOctPlan *plan, const float *sig, int sigStride, int batch, int validLength, int fftLength,
                            int hop, int padLeft, int timeLength, const float *bfrag, const float *scale, int num, int colOff,
                            float *outRe, float *outIm, void *stream);

/* wgmma octave kernel (kernels/cqt_wgmma.cu): Hankel A fragments from the staged signal, B images in swizzled shared
 * memory; power-of-two hops 2 .. 128; plan: AF_CQT_WGMMA */
void af_cqt_wgmma_bimage(const float *kappa2, int fftLength, unsigned char *out /* fftLength/128 * 32768 bytes */);
int af_launch_cqt_octave_wgmma(const AfCqtOctPlan *plan, const float *sig, int sigStride, int batch, int validLength, int fftLength,
                               int hop, int padLeft, int timeLength, const unsigned char *bimg, const float *scale, int num,
                               int colOff, float *outRe, float *outIm, void *stream);

typedef struct {
    int log2n, num, batch, padLength, dataLength;
    AfWavelet wavelet;
    const float *scaleArr;   /* device, num */
    int det;                 /* 1: multiply the bank by j*omega (cwtObj_cwtDet) */
    const float *bankTable;  /* device, num x bankWidth: tabulated bank (PWT) instead of the closed-form wavelet */
    int bankWidth;
    int *support;            /* device, 3 x num ints: per bank row the bins [lo, hi) above 2^-28 of its peak (+ scratch); NULL = no pruning */
    int *supportReady;       /* host flag of the owning object: 0 until the launcher has filled `support` */
} AfCwtArgs;
size_t af_cwt_workspace_bytes(const AfCwtArgs *a);
/* data == NULL: skip the forward transform and reuse the spectra a previous call left in `workspace` */
int af_launch_cwt(const AfCwtArgs *a, const float *data, void *workspace, float *outRe, float *outIm, void *stream);
/* forward FFT of `rows` real sequences x [rows][2^log2n], 2^15 <= 2^log2n <= 2^20, by the CWT's four-step forward legs
 * (kernels/cwt.cu): the spectra [rows][2^log2n] float2 at the start of `workspace`, which has
 * af_fft_rows_workspace_bytes(log2n, rows) bytes */
size_t af_fft_rows_workspace_bytes(int log2n, int rows);
int af_launch_fft_rows(const float *x, int log2n, int rows, void *workspace, void *stream);
/* rows per chunk of a long-row pass whose workspace (its real rows and af_fft_rows_workspace_bytes) stays within 512 MB */
long long af_fft_rows_chunk(int log2n, long long rows);
int af_launch_cwt_bank_table(const AfCwtArgs *a, float *bank /* device num x n */, void *stream);

/* ---------------- BFT core shared with the SpectrogramObj front door (host/af_bft.c) ---------------- */
typedef struct {
    int num, radix2Exp, samplate, binPerOctave, slideLength, lowIndex, highIndex;
    float lowFre, highFre;
    int windowType, dataType, scaleType, styleType, normalType;
} AfBftSpec;
int af_filterbank_clipped(void);   /* non-zero weights the last af_auditory_filterbank call (this thread) dropped above the Nyquist bin */
int af_bft_create(const AfBftSpec *spec, BFTObj *out);      /* 0, -1 (memory), -2 (unsupported bank) */
int af_bft_device(BFTObj b);      /* lazy device set-up of the object's tables */
/* device clips -> spect [batch x T x num] (real mode) and, when dPhase is given, the phase of the STFT bins
 * lowIndex .. lowIndex+count-1 [batch x T x count] (spectrogramObj_spectrogramBatch) */
int af_bft_spectrogram(BFTObj b, const float *dData, int dataLength, int batch, float *dSpect, int lowIndex, int count,
                       float *dPhase, void *stream);
int af_launch_phase(const float *re, const float *im, int rows, int width, int lo, int count, float *out, void *stream);

/* synchrosqueezing (kernels/squeeze.cu): row index of the instantaneous frequency, row scatter */
int af_launch_wsst_index(const float *wr, const float *wi, const float *dr, const float *di, int num, int n, int scaleType,
                         float fre0, float freLast, int samplate, const float *dNorm, int *idx, void *stream);
int af_launch_synsq_index(const float *re, const float *im, int num, int n, int scaleType, float fre0, float freLast,
                          int samplate, const float *dNorm, int *idx, void *stream);
int af_launch_squeeze_scatter(const float *re, const float *im, const int *idx, int num, int n, float thresh,
                              float *outRe, float *outIm, void *stream);

/* reassignment (kernels/reassign.cu): coordinates -> cell indices -> order-independent 64-bit fixed-point scatter.
 * S_h / S_dh / S_th: half-spectrum planes [batch][T][n/2+1]; out planes are ADDED to (reassign_algorithm.c:374-381). */
typedef struct {
    int fftLength, slideLength, samplate, timeLength, batch;
    int reType, order, resultType;
    float thresh;
} AfReassignArgs;
int af_launch_reassign(const AfReassignArgs *a, const float *r1, const float *i1, const float *r2, const float *i2,
                       const float *r3, const float *i3, int *tIdx, int *fIdx, unsigned *maxBits,
                       unsigned long long *accRe, unsigned long long *accIm, float *outRe, float *outIm, void *stream);

/* cepstral deconvolution of rows x num constant-Q magnitudes (kernels/deconv.cu): mode 0 cqhc, 1 deconv */
int af_launch_cq_deconv(const float *in, int rows, int num, int mode, int hcNum, int bpo, float *out0, float *out1, void *stream);
/* the same rows through af_run_batch (cqtObj_cqhcBatch / cqtObj_deconvBatch / spectrogramObj_deconvBatch, af_cqt.c) */
int af_deconv_batch(AfPipe *pipe, const float *in, int rows, int num, int mode, int hcNum, int bpo, float *out0, float *out1,
                    int memKind, void *stream);
/* af_launch_xxcc through af_run_batch, rows as items (xxccObj_xxccBatch / cqtObj_cqccBatch, af_xxcc.c) */
int af_xxcc_batch(AfPipe *pipe, const float *in, int rows, int num, int ccNum, int rectifyType, const float *dctT,
                  float *out, int memKind, void *stream);

/* energy / rms / zero-crossing rate of the windowed frames of ONE clip (src/temporal_algorithm.c:93-146); device arrays [T] */
int af_launch_temporal(const float *data, int fftLength, int slideLength, int timeLength, const float *window,
                       float *energy, float *rms, float *zcr, void *stream);

/* spectral descriptors (kernels/spectral.cu): all requests of one spectralObj_spectralBatch call in one launch */
typedef struct {
    const float *spec, *phase;    /* device, batch x T x num */
    const float *fre;             /* device, num (NULL when no frequency feature is requested) */
    const int *idx;               /* device bin list (NULL: the contiguous range start .. start+nb-1) */
    float *out;                   /* device, planes of batch x T */
    int num, T, batch, start, nb, nReq;
    float meanFre;                /* float mean of fre over the bins, summed in list order (spectral_algorithm.c:1124-1130) */
    int req[AFB200_SPECTRAL_MAX_REQ], plane[AFB200_SPECTRAL_MAX_REQ];
    float par[4 * AFB200_SPECTRAL_MAX_REQ];
    int fresh;                    /* onset (0 for spectralObj_*): frame 1 of PD / WPD / NWPD is written as 0 and BROADBAND
                                     stores its counts, instead of leaving / adding to what `out` holds */
} AfSpectralArgs;
int af_launch_spectral(const AfSpectralArgs *a, void *stream);

/* onset detection (kernels/onset.cu).  Max filter over bins: out[r][k] = max of in[r][k - order/2 .. k - 1 + order -
 * order/2] clipped to [0, num), rows = clips x T.  Peak picking: one CTA per clip normalises evn [clips][T] in place
 * and writes points [clips][T] (0 after the clip's count) and counts [clips]; postMax, postAvg >= 1. */
int af_launch_onset_maxfilter(const float *in, long long rows, int num, int order, float *out, void *stream);
typedef struct {
    float *evn;
    int *points, *counts;
    int clips, T, preMax, postMax, preAvg, postAvg, wait;
    float delta;
} AfOnsetPickArgs;
int af_launch_onset_pick(const AfOnsetPickArgs *a, void *stream);

/* NSGT band transforms (kernels/nsgt.cu).  Bands with L <= AF_NSGT_BLUESTEIN_MAX run as Bluestein FFTs of size
 * M = 2^ceil(log2(2L-1)) (k_nsgt_bluestein, one CTA per (group of bands, clip)); longer bands, up to AF_NSGT_MAX_LEN,
 * as a direct DFT (k_nsgt_direct, one CTA per (band, clip)). */
#define AF_NSGT_BLUESTEIN_MAX 4096
#define AF_NSGT_MAX_LEN 16384
#define AF_NSGT_GROUP_BUDGET 8192     /* sum of M over the bands of one Bluestein group */
#define AF_NSGT_FINE 64               /* direct path: twiddle e^{2 pi i idx/L} = coarse[idx / 64] * fine[idx % 64] */
typedef struct {
    int L, log2M;
    int off;        /* first spectrum bin of the window (clamped at 0) */
    int winOff;     /* window offset in the concatenated windows */
    int cellOff;    /* first cell of the band */
    int tabOff;     /* float2 offset in `tab`: Bluestein chirp c_m = e^{i pi m^2/L} (L), direct: fine (64) then coarse */
    int filtOff;    /* float2 offset in `filt`: FFT_M of the chirp filter, divided by L*M (Bluestein only) */
    int band;
} AfNsgtBand;
typedef struct {
    int fftLength, num, maxLen, totalLen, batch;
    const float *specRe, *specIm;  /* device, batch x (fftLength/2+1) */
    const float *win;              /* device, totalLen */
    const int *map;                /* device, num x maxLen: cell index of every matrix column, -1 = none */
    const AfNsgtBand *bands;       /* device, num: Bluestein bands group after group, then the direct bands */
    const int *groupStart;         /* device, nGroups+1 offsets into `bands` */
    const float *tab, *filt;       /* device, interleaved complex */
    int nGroups, maxM;             /* Bluestein: groups, largest M */
    int nDirect, maxDirectL;       /* direct: bands[groupStart[nGroups] ..] */
    float *outRe, *outIm;          /* device, batch x num x maxLen */
    float *cellRe, *cellIm;        /* device, batch x totalLen, or NULL */
} AfNsgtArgs;
int af_launch_nsgt(const AfNsgtArgs *a, void *stream);

/* Stockwell transforms (kernels/st.cu), N = 2^log2n <= AF_ST_MAX_N.
 * ST: spec = FULL spectrum planes batch x N (af_launch_stft); per row r of `bins`, out[clip][r] = IFFT_N(X[(m + bin) mod N]
 * * (expf(v m^2) + expf(v (m-N)^2))), v = vArr[r]; bin 0 gives the clip's mean and an imaginary row of 0.
 * FST: spec = HALF spectrum planes batch x (N/2+1); part = scratch batch x (N/2+1) complex (the right half of the dyadic
 * partition, from position N/2-1); out row k (frequency minIndex+k) column l = part[(seg[f] >> 5) + (l >> (log2n - (seg[f] & 31)))]
 * with seg[f] = (offset << 5) | log2 of the segment length, f = minIndex + k. */
#define AF_ST_MAX_EXP 14
#define AF_ST_MAX_N (1 << AF_ST_MAX_EXP)
int af_launch_st(const float *data, const float *specRe, const float *specIm, const int *bins, const float *vArr, int rows,
                 int log2n, int batch, float *outRe, float *outIm, void *stream);
int af_launch_fst(const float *specRe, const float *specIm, float *part, const int *seg, int minIndex, int rows, int log2n,
                  int batch, float *outRe, float *outIm, void *stream);

/* Cepstrogram (kernels/cepstrogram.cu), N = 2^log2n <= AF_CEPS_MAX_N, one launch per call.  Frames come either from
 * clips (data batch x dataLength, frame t at t * hop, times `window` unless NULL) or from STFT planes (specRe / specIm
 * rows x specWidth, specWidth N or N/2+1; data == NULL).  Per frame L = logf(max(|X|^2, 1e-16)) (the even part over N
 * bins at specWidth N), y = Re IFFT_N(L): cep = y[0 .. N/2], env = Re FFT_N(y liftered to quefrencies {0..c, N-c..N-1}),
 * det = Re FFT_N(y on {c+1 .. N-c}); each output rows x (N/2+1) and skipped when NULL. */
#define AF_CEPS_MAX_EXP 14
#define AF_CEPS_MAX_N (1 << AF_CEPS_MAX_EXP)
typedef struct {
    int log2n, cepNum;
    const float *data, *window;   /* clips: batch x dataLength; window device N floats or NULL (Rect) */
    int dataLength, hop, timeLength, batch;
    const float *specRe, *specIm; /* planes: rows x specWidth (data == NULL) */
    int rows, specWidth;
    float *cep, *env, *det;       /* device, frames x (N/2+1) each, or NULL */
} AfCepsArgs;
int af_launch_cepstrogram(const AfCepsArgs *a, void *stream);

/* Resampler (kernels/resample.cu), one launch per call: out[b][i] for i < outLen of every clip b of `data` (batch x inLen),
 * the windowed-sinc sum of src/dsp/resample_algorithm.c:430-521 in its order and rounding; the sum starts from out[b][i]
 * when `accumulate` (the legacy call adds into the caller's buffer), else from 0, and is divided by `scaleDiv` when it is
 * not 0.  `table` holds the float32 table (tableLength floats); the weight of entry o is
 * table[o] + delta * (table[o+1] - table[o]), with 0 for the last entry's difference.  Taps read x[0 .. srcLen-1];
 * left-tap positions at or beyond inLen read 0. */
typedef struct {
    const float *data, *table;
    float *out;
    int inLen, srcLen, outLen, batch, tableLength, bitLength, step;
    float ratio, scale, scaleDiv;
    int accumulate;
} AfResampleArgs;
int af_launch_resample(const AfResampleArgs *a, void *stream);

/* Masks of harmonic-percussive separation (kernels/hpss.cu), one launch: from the half-spectrum planes re / im
 * [clips * timeLength][width] the masked planes of H (hRe / hIm) and P (pRe / pIm) in the same layout, either pair NULL
 * to skip it.  Medians over hOrder frames of one clip (zeros beyond its first and last frame) and over pOrder bins (zeros
 * beyond the plane), orders odd, 1 .. AFB200_HPSS_MAX_ORDER; an order of 1 gives a median of 0. */
typedef struct {
    const float *re, *im;
    float *hRe, *hIm, *pRe, *pIm;
    int clips, timeLength, width, hOrder, pOrder;
} AfHpssArgs;
int af_launch_hpss_mask(const AfHpssArgs *a, void *stream);

/* Harmonic ratio (kernels/harmonic_ratio.cu), W = 2^log2w (1 .. AFB200_HARMONIC_RATIO_MAX_EXP), two launches per call:
 * every frame t of every clip b (samples b * dataLength + t * hop .. + W-1, times `window`) gets its crossing index in
 * minIdx[b * T + t] (-1 for none) and, when it has one, its value in value[b * T + t]; then the frames without one take
 * the index of the last earlier frame of their clip that has one (0 when none) and get their value.
 * 1 <= maxLength <= W-1. */
typedef struct {
    const float *data, *window;   /* device: clips batch x dataLength, window W floats */
    float *value;                 /* device, batch x timeLength */
    int *minIdx;                  /* device workspace, batch x timeLength */
    int log2w, maxLength, dataLength, hop, timeLength, batch;
} AfHarmonicRatioArgs;
int af_launch_harmonic_ratio(const AfHarmonicRatioArgs *a, void *stream);

/* Pitch by the pitch estimation filter (kernels/pitch_pef.cu), n = 2^log2n (1 .. AFB200_PITCH_PEF_MAX_EXP), one launch:
 * every frame t of every clip b (samples b * dataLength + t * hop .. + n-1) gets fre[b * T + t] = logFre[k], k the first
 * arg-max over minIndex .. maxIndex of the correlation of the weighted log-frequency power with the filter (see
 * include/afb200_pitch_pef.h), computed with an L = 2^log2L-point real transform.  `tables` (device) holds, in order:
 * window n, lin n+1, logFre 2n, bandWidth 2n (floats), interpIndex 2n (ints), filter spectrum L/2 + 1 (float pairs). */
typedef struct {
    const float *data;            /* device: clips batch x dataLength */
    const float *tables;
    float *fre;                   /* device, batch x timeLength */
    int log2n, log2L, padNum, minIndex, maxIndex, dataLength, hop, timeLength, batch;
} AfPitchPefArgs;
/* float offsets of the parts of `tables` */
#define AF_PEF_LIN(n) (n)
#define AF_PEF_LOG(n) (2 * (n) + 1)
#define AF_PEF_BW(n) (4 * (n) + 1)
#define AF_PEF_IDX(n) (6 * (n) + 1)
#define AF_PEF_SPEC(n) (8 * (n) + 2)      /* even: float2-aligned */
#define AF_PEF_TABLE_FLOATS(n, L) (8 * (size_t)(n) + 2 + (size_t)(L) + 2)
int af_launch_pitch_pef(const AfPitchPefArgs *a, void *stream);
/* Pitch by YIN (kernels/pitch_yin.cu), n = 2^log2n (1 .. AFB200_PITCH_YIN_MAX_EXP), one launch: every frame t of every
 * clip b (samples b * dataLength + t * hop .. + n-1) gets, with f = b * T + t, the outputs of
 * include/afb200_pitch_yin.h: fre[f] and value1[f] (only in frames with a trough), value2[f], and the trough rows
 * mFre / mTrough [f][yinLength/2 + 1] (zero past the count) with their count lens[f].  Each output but fre may be
 * NULL.  1 <= minIndex <= maxIndex <= n - 1 - autoLength. */
typedef struct {
    const float *data;            /* device: clips batch x dataLength */
    float *fre, *value1, *value2, *mFre, *mTrough;
    int *lens;
    int log2n, autoLength, minIndex, maxIndex, samplate, dataLength, hop, timeLength, batch;
    float thresh;
} AfPitchYinArgs;
int af_launch_pitch_yin(const AfPitchYinArgs *a, void *stream);
/* Pitch by the normalised correlation (mode AF_PITCH_NCF) or the cepstrum (AF_PITCH_CEP) (kernels/pitch_ncf_cep.cu),
 * n = 2^log2n (1 .. 14), one launch: every frame t of every clip b (samples b * dataLength + t * hop .. + n-1) gets
 * fre[b * T + t] = samplate / (index + 1), index __vmax's first arg-max over minIndex .. maxIndex of the row of
 * include/afb200_pitch_ncf.h or include/afb200_pitch_cep.h.  NCF: 1 <= minIndex <= maxIndex < n; CEP:
 * 0 <= minIndex <= maxIndex < 2n. */
enum { AF_PITCH_NCF = 0, AF_PITCH_CEP = 1 };
typedef struct {
    const float *data, *window;   /* device: clips batch x dataLength, window n floats */
    float *fre;                   /* device, batch x timeLength */
    int mode, log2n, minIndex, maxIndex, samplate, dataLength, hop, timeLength, batch;
} AfPitchLagArgs;
int af_launch_pitch_ncf_cep(const AfPitchLagArgs *a, void *stream);
/* in-place iterative radix-2 forward FFT in double, n a power of two (host/af_cqt_bank.c; setup only) */
void af_fft_double(double *re, double *im, int n);

/* Discrete wavelet transforms (kernels/wavelet.cu).  One split level of DWT / WPT: node k (0 .. nodes-1) of L samples
 * at in + b*inStride + k*L, periodically indexed, gives a[i] = sum_j loD[j] x[(2i + dec - dec/2 - j) mod L] and d[i]
 * likewise with hiD, i < L/2; a goes to lo + b*loStride + k*L + i and d to hi + b*hiStride + k*L + L/2 + i, the two
 * halves exchanged when wpt and the node's tree index nodeBase + k is even and non-zero.  L is a power of two. */
typedef struct {
    const float *in, *loD, *hiD;  /* device; filters dec floats */
    float *lo, *hi;
    long long inStride, loStride, hiStride;
    int L, nodes, nodeBase, wpt, dec, batch;
} AfWaveletLevel;
int af_launch_wavelet_level(const AfWaveletLevel *a, void *stream);
/* out[b][r][j] = coef[b][base(r) + (j >> shift(r))], r < rows, j < N = 2^log2n: DWT (wpt = 0) base = 2^(r+1),
 * shift = log2n - r - 1; WPT base = r * N / rows, shift = log2(rows) */
int af_launch_wavelet_expand(const float *coef, int log2n, int rows, int wpt, int batch, float *out, void *stream);
/* One SWT level: out[b][t] = sum_j f[j] x[(t + off - j*s) mod n] for loD -> lo and hiD -> hi, x = in + b*inStride,
 * t < n, s = dilation, off = dec*s/2 */
int af_launch_swt_level(const float *in, long long inStride, const float *loD, const float *hiD, int dec, int n, int s,
                        int batch, float *lo, float *hi, long long outStride, void *stream);

/* Non-negative matrix factorisation (kernels/nmf.cu), 1 + 4 maxIter launches whatever the batch: for each matrix b of
 * V [batch][n][m], W [batch][n][k] and H [batch][k][m] (in place) the iterations of src/classic/nmf.c, each matrix
 * stopping on its own.  type 0 KL, 1 IS, 2 Euclidean (the caller maps every other type to 2); norm 1 | 2 column p-norm,
 * other column max.  iters (device, batch ints, or NULL) receives the iterations each matrix ran.  The workspace (one
 * n x m plane per matrix, two for IS, and the previous W and H) is allocated and freed in stream order on `stream`. */
typedef struct {
    const float *V;
    float *W, *H;
    int *iters;
    int n, m, k, batch, maxIter, type, norm;
    float thresh;
} AfNmfArgs;
int af_launch_nmf(const AfNmfArgs *a, void *stream);

/* Cross-correlation (kernels/xcorr.cu) of `batch` pairs of rows a, b [batch][n] (b NULL: the autocorrelation of each row
 * of a), M = the smallest power of two >= 2n: out [batch][2n-1] = IFFT_M(FFT_M(a) conj(FFT_M(b))) at lags -(n-1) .. n-1,
 * divided by sqrtf(float(sum a^2) float(sum b^2)) when coeff; maxValue / maxIndex (batch each, either NULL) receive the
 * row's __vmax.  M <= AF_XCORR_SHORT_MAX: one launch (k_xcorr, one CTA per pair).  Longer: the four-step forward legs of
 * the CWT path in groups of pairs over the object's workspace `work` (grown as needed, at most about 512 MB a group),
 * every use of it bracketed by the object's fence (af_fence_order / af_fence_record). */
#define AF_XCORR_SHORT_MAX (1 << 14)
typedef struct {
    const float *a, *b;
    float *out, *maxValue;
    int *maxIndex;
    int n, batch, coeff;
    AfDevBuf *work;
    void **fence;
} AfXcorrArgs;
int af_launch_xcorr(const AfXcorrArgs *a, void *stream);

/* Chirp z-transform (kernels/czt.cu), N = 2^log2n, M = 2N <= 2^(AFB200_CZT_MAX_EXP + 1), one launch (k_czt, one CTA per
 * row): g = x * pre over the N inputs (re / im either NULL), zero-padded to M; y = IFFT_M(FFT_M(g) H);
 * re3 / im3 [batch][M]: y[N-1+k] post[k] for k < N, then y[N .. M-1].  `tables`: pre (N complex), post (N complex) and H
 * (M complex, bit-reversed order), interleaved float pairs.  af_launch_czt_filter turns the chirp filter h, uploaded in
 * the H slot in natural order, into H in place (one launch). */
typedef struct {
    const float *re, *im;
    float *re3, *im3;
    const float *tables;
    int log2n, batch;
} AfCztArgs;
int af_launch_czt(const AfCztArgs *a, void *stream);
int af_launch_czt_filter(float *H, int log2m, void *stream);

void af_count_launch(int n);

#ifdef __cplusplus
}
#endif
#endif
