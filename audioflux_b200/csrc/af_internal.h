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
int af_stream_create(void **stream);
void af_stream_destroy(void *stream);
int af_stream_sync(void *stream);
int af_event_create(void **ev);
void af_event_destroy(void *ev);
int af_event_record(void *ev, void *stream);
int af_stream_wait_event(void *stream, void *ev);
int af_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream);
int af_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream);
int af_memset_d(void *dst, int v, size_t bytes, void *stream);
size_t af_dev_free_bytes(void);

/* Host-pointer batches: items flow through two device slots on three streams -- copy-in of chunk k+1, the transform
 * of chunk k and copy-out of chunk k-1 overlap (H2D and D2H are opposite PCIe directions).  With page-locked caller
 * buffers a call runs at the speed of the larger transfer and needs two chunks of device memory instead of the
 * batch; pageable buffers work too (the driver stages them synchronously). */
typedef struct {
    int ready;
    void *inStream, *outStream, *evIn[2], *evDone[2], *evOut[2];
    AfDevBuf in[2], out0[2], out1[2];
} AfPipe;
/* transform of `nb` items already on the device: dIn -> dOut0 (and dOut1 when the entry point has two planes) */
typedef int (*AfChunkFn)(void *obj, const float *dIn, int nb, float *dOut0, float *dOut1, void *stream);
int af_pipe_run(AfPipe *pipe, AfChunkFn fn, void *obj, const float *hIn, size_t inFloatsPerItem, int batch,
                float *hOut0, float *hOut1, size_t outFloatsPerItem, void *computeStream);
void af_pipe_free(AfPipe *pipe);
int af_sm_count(void);

/* ---------------- setup-time tables (host/af_window.c, af_filterbank.c, ...) ---------------- */
int af_window_symmetric(int windowType, int length, const float *value, double *out);
int af_window_fft(int windowType, int length, float *out);

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

typedef struct {
    int fftLength, slideLength, num, ccNum, rectifyType, dataType;
    float normValue;
    const float *window, *dct;    /* device */
    AfBankDev bank;
    /* fused-kernel specific tables (device), built by af_mfcc_plan_build */
    void *plan;
} AfMfccArgs;
int af_mfcc_fused_supported(int fftLength, int num, int ccNum, const AfBands *bands);
int af_mfcc_plan_build(void **plan, int fftLength, int num, int ccNum, const float *window,
                       const float *bank, const AfBands *bands, const float *dct, int dataType,
                       const float *gain /* per-filter normalisation gains (NULL = 1) */);
int af_launch_mel_fused(void *plan, const float *data, int dataLength, int batch, int timeLength,
                        int slideLength, float *out, void *stream);   /* stops after the bank: batch x T x num */
int af_mfcc_plan_mode(void *plan);      /* 1: interval (shared product) bank loop, 0: filter-per-lane */
void af_mfcc_plan_free(void *plan);
int af_launch_mfcc_fused(void *plan, const float *data, int dataLength, int batch, int timeLength,
                         int slideLength, int rectifyType, float *out, int nPeer, float *const *peerOut,
                         void *stream);

/* second-generation fused kernel (kernels/mfcc_fused2.cu): banks in which at most two consecutive filters overlap */
int af_mfcc2_supported(int fftLength, int num, int ccNum, const float *bank /* num x (fftLength/2+1) */);
int af_mfcc2_plan_build(void **plan, int fftLength, int num, int ccNum, const float *window, const float *bank,
                        const float *dct, int dataType);
void af_mfcc2_plan_free(void *plan);
int af_launch_mfcc2(void *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                    int rectifyType, float *out, int nPeer, float *const *peerOut, void *stream);
int af_launch_mel2(void *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                   float *out, void *stream);

int af_launch_decimate2(const float *in, int inLength, int inStride, int batch, const float *left32,
                        const float *right31, float *out, int outStride, void *stream);
/* out[b][t][colOff + j] (row stride num) = scale[j] * sum_n xpad[t*hop + n] * kappa[j][n];
 * kappa2 = interleaved (re, im) pairs [bpo][fftLength] */
int af_launch_cqt_octave(const float *sig, int sigLength, int sigStride, int batch, int validLength,
                         int fftLength, int hop, int padLeft, int timeLength, int bpo, const float *kappa2,
                         const float *scale, int num, int colOff,
                         float *outRe, float *outIm, void *stream);

/* tensor-core octave kernel (3xTF32 mma.sync): 12 bins per octave, power-of-two hop >= 2 */
int af_cqt_tc_supported(int fftLength, int hop, int bpo);
void af_cqt_tc_fragments(const float *kappa2, int fftLength, float *out /* fftLength/8 * 96 * 4 floats */);
int af_launch_cqt_octave_tc(const float *sig, int sigStride, int batch, int validLength, int fftLength, int hop,
                            int padLeft, int timeLength, const float *bfrag, const float *scale, int num, int colOff,
                            float *outRe, float *outIm, void *stream);

/* wgmma octave kernel (kernels/cqt_wgmma.cu): Hankel A fragments from the staged signal, B images in swizzled shared
 * memory; power-of-two hops 2 .. 128 */
int af_cqt_wgmma_supported(int fftLength, int hop, int bpo);
void af_cqt_wgmma_bimage(const float *kappa2, int fftLength, unsigned char *out /* fftLength/128 * 32768 bytes */);
int af_launch_cqt_octave_wgmma(const float *sig, int sigStride, int batch, int validLength, int fftLength, int hop,
                               int padLeft, int timeLength, const unsigned char *bimg, const float *scale, int num, int colOff,
                               float *outRe, float *outIm, void *stream);

typedef struct {
    int log2n, num, batch, padLength, dataLength;
    AfWavelet wavelet;
    const float *scaleArr;   /* device, num */
    int det;                 /* 1: multiply the bank by j*omega (cwtObj_cwtDet) */
    const float *bankTable;  /* device, num x bankWidth: tabulated bank (PWT) instead of the closed-form wavelet */
    int bankWidth;
    int *support;            /* device, 3 x num ints: per bank row the bins [lo, hi) above 2^-28 of its peak (+ scratch); NULL = no pruning */
    int *supportReady;       /* host flag of the owning object: 0 until the launcher has filled `support` */
    int forwardOnly;         /* 1: only the forward transform of the `batch` real sequences -> workspace[batch][N] float2 (long-frame STFT) */
} AfCwtArgs;
size_t af_cwt_workspace_bytes(const AfCwtArgs *a);
/* data == NULL: skip the forward transform and reuse the spectra a previous call left in `workspace` */
int af_launch_cwt(const AfCwtArgs *a, const float *data, void *workspace, float *outRe, float *outIm, void *stream);
int af_launch_cwt_bank_table(const AfCwtArgs *a, float *bank /* device num x n */, void *stream);

/* ---------------- BFT core shared with the SpectrogramObj front door (host/af_bft.c) ---------------- */
typedef struct {
    int num, radix2Exp, samplate, binPerOctave, slideLength, lowIndex, highIndex;
    float lowFre, highFre;
    int windowType, dataType, scaleType, styleType, normalType;
} AfBftSpec;
/* streaming bookkeeping of an STFT object (af_stft.c): tail of the earlier calls ++ data -> *cur / *curLength; 0 = no frame yet */
int af_stft_continue_assemble(STFTObj s, const float *data, int dataLength, const float **cur, int *curLength);
int af_filterbank_clipped(void);   /* non-zero weights the last af_auditory_filterbank call (this thread) dropped above the Nyquist bin */
int af_bft_create(const AfBftSpec *spec, BFTObj *out);      /* 0, -1 (memory), -2 (unsupported bank) */
int af_bft_phase(BFTObj b, const float *data, int dataLength, int batch, int lowIndex, int count, float *phase,
                 int memKind, void *stream);
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

/* energy / rms / zero-crossing rate of the windowed frames of ONE clip (src/temporal_algorithm.c:93-146); device arrays [T] */
int af_launch_temporal(const float *data, int fftLength, int slideLength, int timeLength, const float *window,
                       float *energy, float *rms, float *zcr, void *stream);

void af_count_launch(int n);

#ifdef __cplusplus
}
#endif
#endif
