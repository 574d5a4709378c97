/* afb200_ext.h -- ADDITIVE entry points of libaudioflux_b200.so (no reference counterpart).
 *
 * The reference API is one clip per call with host pointers (python/audioflux/bft.py:349-365
 * loops channels in Python); fed that way a GPU is PCIe/launch bound.  These entry points
 * take a whole batch and either host or device pointers.
 *
 *   memKind 0: host pointers (pageable or pinned) -- the call stages the batch through the device in
 *              bounded chunks (about 64 MB, copies overlapping the compute) and returns synchronised;
 *              it never holds the whole batch on the device.
 *   memKind 1: device pointers on the current device -- asynchronous on `stream`
 *              (a cudaStream_t passed as void*; NULL = the CUDA default stream).  The call
 *              returns without synchronising; results are ordered on that stream.
 * All return 0 on success, non-zero on failure with afb200_lastError() describing it.
 * Layouts are the reference's: row-major, time-major, separate real/imag float planes.
 */
#ifndef AFB200_EXT_H
#define AFB200_EXT_H
#include "afb200_stft.h"
#include "afb200_bft.h"
#include "afb200_xxcc.h"
#include "afb200_cqt.h"
#include "afb200_cwt.h"
#include "afb200_spectrogram.h"
#include "afb200_pwt.h"
#include "afb200_spectral.h"
#include "afb200_nsgt.h"
#include "afb200_st.h"
#include "afb200_cepstrogram.h"
#include "afb200_resample.h"
#include "afb200_hpss.h"
#include "afb200_onset.h"
#include "afb200_harmonic_ratio.h"
#include "afb200_pitch_pef.h"
#include "afb200_pitch_yin.h"
#include "afb200_pitch_ncf.h"
#include "afb200_pitch_cep.h"
#include "afb200_dwt.h"
#include "afb200_wpt.h"
#include "afb200_swt.h"
#include "afb200_nmf.h"
#include "afb200_xcorr.h"
#include "afb200_czt.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Memory kinds of the batched entry points.  AFB200_MEM_DEVICE calls are asynchronous on the caller's stream.
 * An object is NOT thread-safe and is SINGLE-STREAM: its tables are bound to the device that was current at its first
 * compute call, and the general (non-fused) paths use per-object scratch buffers (spectrum planes, frame buffers, the CWT
 * workspace), so two calls on the same object must be ordered on one stream (or by events).  Different objects may run
 * concurrently on different streams / threads. */
#define AFB200_MEM_HOST 0
#define AFB200_MEM_DEVICE 1

int afb200_version(void);
int afb200_deviceCount(void);              /* 0 when no usable GPU (compute calls then fail loudly) */
int afb200_setDevice(int device);          /* device used by objects created / run from this thread */
int afb200_getDevice(void);
const char *afb200_lastError(void);        /* thread-local message of the last failure */
long long afb200_kernelLaunchCount(void);  /* kernels launched by this library since load */
int afb200_deviceSynchronize(void);

/* data: batch x dataLength; out planes: batch x T x (fftLength/2+1) */
int stftObj_stftBatch(STFTObj stftObj, const float *data, int dataLength, int batch,
                      float *mReal, float *mImag, int memKind, void *stream);
/* inverse: planes batch x T x specWidth (specWidth = fftLength, or fftLength/2+1 = the layout stftObj_stftBatch
 * writes) -> data batch x ((T-1)*slide + fftLength), pre-zeroed by the caller */
int stftObj_istftBatch(STFTObj stftObj, const float *mReal, const float *mImag, int timeLength, int batch,
                       int specWidth, int methodType, float *data, int memKind, void *stream);
/* out: batch x T x num (mImag3 may be NULL when resultType=1) */
int bftObj_bftBatch(BFTObj bftObj, const float *data, int dataLength, int batch,
                    float *mReal3, float *mImag3, int memKind, void *stream);
/* fused BFT(real mode) -> rectify -> ortho DCT-II -> first ccNum.  out: batch x T x ccNum */
int bftObj_mfccBatch(BFTObj bftObj, const float *data, int dataLength, int batch, int ccNum,
                     int rectifyType, float *out, int memKind, void *stream);
/* SpectrogramObj front door: spect batch x T x bandNum (+ phase for the Linear scale, may be NULL);
 * mfcc = the fused kernel of bftObj_mfccBatch */
int spectrogramObj_spectrogramBatch(SpectrogramObj spectrogramObj, const float *data, int dataLength, int batch,
                                    float *spect, float *phase, int memKind, void *stream);
int spectrogramObj_mfccBatch(SpectrogramObj spectrogramObj, const float *data, int dataLength, int batch, int ccNum,
                             int rectifyType, float *out, int memKind, void *stream);
/* spectrogramObj_deconv for any number of rows (frames of any number of clips): in, timbre, pitch rows x bandNum */
int spectrogramObj_deconvBatch(SpectrogramObj spectrogramObj, const float *in, int rows, float *timbre, float *pitch,
                               int memKind, void *stream);
/* MFCC + all-gather as ONE kernel (multi-GPU, one process per GPU).  Device pointers only: `out` is this GPU's
 * destination, peerOut[0..nPeer) (nPeer <= 15) the same logical location inside the other GPUs' gathered buffers,
 * mapped with afb200_ipcOpenHandle.  The kernel epilogue stores every finished tile to all of them (NVLink P2P
 * stores), so the exchange overlaps the transform tile by tile; the caller fences across ranks afterwards. */
int bftObj_mfccBatchScatter(BFTObj bftObj, const float *data, int dataLength, int batch, int ccNum, int rectifyType,
                            float *out, int nPeer, void **peerOut, void *stream);
/* cudaMalloc'ed buffers other processes can map (cudaIpc*; handle = 64 opaque bytes) */
int afb200_peerAlloc(void **devPtr, size_t bytes);
int afb200_peerFree(void *devPtr);
int afb200_ipcGetHandle(void *devPtr, void *handle64);
int afb200_ipcOpenHandle(const void *handle64, void **devPtr);
int afb200_ipcCloseHandle(void *devPtr);
/* diagnostics: the kernel that served the object's last bftObj_mfccBatch call: 1 fused v2, 0 fused v1, -1 composed (or none yet) */
int bftObj_mfccPlanMode(BFTObj bftObj);
int bftObj_getFilterBankArr(BFTObj bftObj, float *bank /* num x (fftLength/2+1) host */);
/* in: rows x num; out: rows x ccNum */
int xxccObj_xxccBatch(XXCCObj xxccObj, const float *in, int rows, int ccNum, int rectifyType,
                      float *out, int memKind, void *stream);
/* xxccObj_xxccStandard over `rows` frames; energy: rows (NULL allowed when energyType = Ignore);
 * coe / delta1 / delta2: rows x (ccNum, +1 when energyType = Append) */
int xxccObj_xxccStandardBatch(XXCCObj xxccObj, const float *in, const float *energy, int rows, int ccNum,
                              int deltaWindowLength, int energyType, int rectifyType,
                              float *coe, float *delta1, float *delta2, int memKind, void *stream);
/* out planes: batch x T x num */
int cqtObj_cqtBatch(CQTObj cqtObj, const float *data, int dataLength, int batch,
                    float *mReal3, float *mImag3, int memKind, void *stream);
/* CQT planes rows x num -> rows x chromaNum / rows x ccNum (rows = batch*T) */
int cqtObj_chromaBatch(CQTObj cqtObj, const float *mReal, const float *mImag, int rows, int chromaNum,
                       int dataType, int normType, float *out, int memKind, void *stream);
int cqtObj_cqccBatch(CQTObj cqtObj, const float *in, int rows, int ccNum, int rectifyType, float *out,
                     int memKind, void *stream);
int cqtObj_getKernelBank(CQTObj cqtObj, float *kr, float *ki /* binPerOctave x (fftLength/2+1) host */);
/* diagnostics: per octave, top octave first -- kernel (0 wgmma, 1 mma.sync, 2 FP32 loop, 3 direct), the octave's hop,
   frames per CTA (0 for direct), threads per CTA, tap segments (FP32 loop; else 1), dynamic shared memory bytes.
   Each array holds octaveNum ints; any may be NULL.  Returns octaveNum, or < 0 on error.  Host only: needs no device. */
int cqtObj_octavePlan(CQTObj cqtObj, int *kernel, int *hop, int *framesPerCta, int *threadsPerCta, int *segs,
                      int *smemBytes);
/* data: batch x 2^radix2Exp; out planes: batch x num x 2^radix2Exp */
int cwtObj_cwtBatch(CWTObj cwtObj, const float *data, int batch, float *mReal4, float *mImag4,
                    int memKind, void *stream);
/* derivative transform (after cwtObj_enableDet); data may be NULL with batch = 1 to reuse the last spectrum */
int cwtObj_cwtDetBatch(CWTObj cwtObj, const float *data, int batch, float *mReal4, float *mImag4,
                       int memKind, void *stream);
int cwtObj_getFilterBankArr(CWTObj cwtObj, float *bank /* num x fftLength host; fftLength = the TRANSFORM length: 2^radix2Exp, twice that with isPad */);
/* PWT: data batch x 2^radix2Exp -> planes batch x num x 2^radix2Exp */
int pwtObj_pwtBatch(PWTObj pwtObj, const float *data, int batch, float *mReal3, float *mImag3, int memKind, void *stream);
int pwtObj_pwtDetBatch(PWTObj pwtObj, const float *data, int batch, float *mReal3, float *mImag3, int memKind, void *stream);
int pwtObj_getFilterBankArr(PWTObj pwtObj, float *bank /* num x fftLength host; fftLength as for cwtObj_getFilterBankArr */);

/* setup-time table builders, exported for parity tests against the reference's
 * window_calFFTWindow (src/dsp/flux_window.c:890-940), auditory_filterBank
 * (src/filterbank/auditory_filterBank.c:56-207) and the /2 resampler taps
 * (src/dsp/resample_algorithm.c:546-634). */
int afb200_window(int windowType, int length, float *out);
int afb200_auditoryFilterBank(int num, int fftLength, int samplate, int scaleType, int styleType,
                              int normType, float lowFre, float highFre, int binPerOctave,
                              float *bank, float *freBandArr /* num */, int *binBandArr /* num */);
int afb200_decimatorTaps(float *left32, float *right31);
/* planner of the second-generation fused kernel (kernels/mfcc_fused2.cu, host only): every bin of `bank` (num x 1025)
 * is given to one interval i in [0, num] on which filter i "rises" and filter i-1 "falls" (the bank's own weights);
 * returns the number of float4 table entries (rise[2q], rise[2q+1], fall[2q], fall[2q+1]) or -1 when some bin is
 * covered by more than two, or by non-consecutive, filters (or no piece plan exists).  desc[i] = (first bin pair << 16) |
 * table offset.  The intervals are cut into pieces of at most lmax bin pairs, one per helper lane and pass:
 * pieceDesc[p] = (first bin pair << 20) | (pairs << 16) | table offset, prefix[i] = first piece of interval i,
 * assign = piece of each lane (0xffff = none), info = {passes, helper lanes, pieces, lmax, pieces of pass 0,
 * longest piece of each pass}. */
int afb200_mfccBankPlan2(const float *bank, int num, int *owner /* 1025 */, unsigned *desc /* num + 2 */,
                         float *table /* 4 x 1408 */, unsigned *pieceDesc /* 256 */, unsigned short *prefix /* num + 2 */,
                         unsigned short *assign /* passes x helper lanes */, int *info /* 16 */);
/* shared-memory carve-up of the second-generation fused kernel (host only, what its launcher computes): frames per tile
 * and TMA stages for a clip of timeLength frames at hop `hop`, a bank of num bands with tabLen table entries and ccNum
 * coefficients (rawMel != 0: filter-bank output).  Returns the bytes of shared memory, or -1 when not one frame fits.
 * info = {frames per tile, stages, byte offsets of the TMA span, the two power tiles, window, twiddles, special columns,
 * DCT matrix, log-mel tiles, staging, bank table, piece descriptors, lane assignment, piece prefix; staging bytes,
 * span floats}. */
int afb200_mfccCarve2(int timeLength, int hop, int num, int ccNum, int tabLen, int rawMel, int *info /* 16 */);
/* cepstral deconvolution of rows x num constant-Q magnitudes (cqtObj_cqhc / cqtObj_deconv for any number of rows) */
int cqtObj_cqhcBatch(CQTObj cqtObj, const float *in, int rows, int hcNum, float *out /* rows x hcNum */, int memKind, void *stream);
int cqtObj_deconvBatch(CQTObj cqtObj, const float *in, int rows, float *timbre, float *pitch /* rows x num each */,
                       int memKind, void *stream);
/* chroma_cqtFilterBank (src/filterbank/chroma_filterBank.c:176-262): bank num x cqtLength */
int afb200_chromaCqtFilterBank(int num, int cqtLength, int binPerOctave, float minFre, float *bank);

/* Feature ids of spectralObj_spectralBatch and their parameters par[4*i .. 4*i+3] = {step, p, threshold, flags}
 * (unused slots ignored; flags is an integer held in a float):
 *   FLUX       step, p, -, flags bit0 isPositive, bit1 isExp, bit2 type (mean)
 *   ROLLOFF    threshold                          ENTROPY / EEF   flags bit0 isNorm
 *   BANDWIDTH  p                                  ENERGY          p = gamma, flags bit0 isLog
 *   SD / SF    step, flags bit0 isPositive        MKL             flags bit2 type (mean)
 *   BROADBAND  threshold                          EER             p = gamma, flags bit0 isNorm
 *   NOVELTY    step, threshold, flags bits0-1 methodType, bit2 dataType (Number)
 * MAX / MEAN / VAR write two consecutive planes: value, then frequency. */
enum {
    AFB200_SPECTRAL_FLATNESS = 0, AFB200_SPECTRAL_FLUX, AFB200_SPECTRAL_ROLLOFF, AFB200_SPECTRAL_CENTROID,
    AFB200_SPECTRAL_SPREAD, AFB200_SPECTRAL_SKEWNESS, AFB200_SPECTRAL_KURTOSIS, AFB200_SPECTRAL_ENTROPY,
    AFB200_SPECTRAL_CREST, AFB200_SPECTRAL_SLOPE, AFB200_SPECTRAL_DECREASE, AFB200_SPECTRAL_BANDWIDTH,
    AFB200_SPECTRAL_RMS, AFB200_SPECTRAL_ENERGY, AFB200_SPECTRAL_HFC, AFB200_SPECTRAL_SD, AFB200_SPECTRAL_SF,
    AFB200_SPECTRAL_MKL, AFB200_SPECTRAL_PD, AFB200_SPECTRAL_WPD, AFB200_SPECTRAL_NWPD, AFB200_SPECTRAL_CD,
    AFB200_SPECTRAL_RCD, AFB200_SPECTRAL_BROADBAND, AFB200_SPECTRAL_NOVELTY, AFB200_SPECTRAL_EEF,
    AFB200_SPECTRAL_EER, AFB200_SPECTRAL_MAX, AFB200_SPECTRAL_MEAN, AFB200_SPECTRAL_VAR,
    AFB200_SPECTRAL_COUNT
};
#define AFB200_SPECTRAL_MAX_REQ 64
/* spec (and phase, NULL unless PD / WPD / NWPD / CD / RCD is requested): batch x timeLength x num, time-major.
 * req[i]: AFB200_SPECTRAL_* id, par[4*i .. 4*i+3] its parameters; 1 <= nReq <= AFB200_SPECTRAL_MAX_REQ.
 * out: one plane of batch x timeLength per request (two for MAX / MEAN / VAR), in request order.  Frames that the
 * reference leaves unwritten stay as they were in `out` (frame 1 of PD / WPD / NWPD, VAR with fewer than 2 bins) and
 * BROADBAND adds its counts to what `out` holds.  req / par are host arrays; one kernel launch per call.  Each clip's
 * temporal features start afresh (frame 0 of clip b never looks at clip b-1). */
int spectralObj_spectralBatch(SpectralObj spectralObj, const float *spec, const float *phase, int timeLength, int batch,
                              int nReq, const int *req, const float *par, float *out, int memKind, void *stream);

/* NSGT of a batch: data batch x 2^radix2Exp -> matrix planes batch x num x maxTimeLength, and (when cellReal / cellImag
 * are not NULL) the cells batch x totalTimeLength.  Columns the reference's time grids map to no cell are 0.
 * Each clip's result is bit-identical to nsgtObj_nsgt on that clip, whatever the batch. */
int nsgtObj_nsgtBatch(NSGTObj nsgtObj, const float *data, int batch, float *mReal, float *mImag,
                      float *cellReal, float *cellImag, int memKind, void *stream);

/* S-transform of a batch: data batch x 2^radix2Exp -> planes batch x binLength x 2^radix2Exp, rows in the order of the
 * object's bin list.  Each clip's result is bit-identical to stObj_st on that clip, whatever the batch. */
int stObj_stBatch(STObj stObj, const float *data, int batch, float *mReal, float *mImag, int memKind, void *stream);
/* rows of the current bin list (stObj_useBinArr may change it) */
int stObj_getBinLength(STObj stObj);
/* fast S-transform of a batch: planes batch x rows x 2^radix2Exp, rows = maxIndex - minIndex + 1 after the range rules of
 * fstObj_fst.  Each clip's result is bit-identical to fstObj_fst on that clip, whatever the batch. */
int fstObj_fstBatch(FSTObj fstObj, const float *data, int batch, int minIndex, int maxIndex, float *mReal, float *mImag,
                    int memKind, void *stream);

/* cepstrogram of a batch: data batch x dataLength -> cep / env / det batch x T x (N/2+1), T = cepstrogramObj_calTimeLength.
 * Any of the three may be NULL (its work is skipped), not all three.  Each clip's result is bit-identical to
 * cepstrogramObj_cepstrogram on that clip, whatever the batch. */
int cepstrogramObj_cepstrogramBatch(CepstrogramObj cepstrogramObj, int cepNum, const float *data, int dataLength, int batch,
                                    float *cep, float *env, float *det, int memKind, void *stream);
/* the same from STFT planes rows x specWidth, one frame per row -> rows x (N/2+1).  specWidth = N (the mirrored layout of
 * stftObj_stft: the even part of log S is used) or N/2+1 (the layout stftObj_stftBatch writes: taken as Hermitian).
 * The planes are read only.  Each row's result is bit-identical to cepstrogramObj_cepstrogram2 on that row. */
int cepstrogramObj_cepstrogram2Batch(CepstrogramObj cepstrogramObj, int cepNum, const float *mReal, const float *mImag,
                                     int rows, int specWidth, float *cep, float *env, float *det, int memKind, void *stream);

/* resampler of a batch: data batch x dataLength -> out batch x resampleObj_calDataLength(dataLength); out is overwritten.
 * Each clip's result is bit-identical to resampleObj_resample on that clip into a zeroed buffer, whatever the batch.
 * Refused while the object is in continue mode (a mode for one stream fed chunk by chunk through resampleObj_resample),
 * and wherever resampleObj_resample refuses.  One kernel launch per staging chunk. */
int resampleObj_resampleBatch(ResampleObj resampleObj, const float *data, int dataLength, int batch, float *out,
                              int memKind, void *stream);

/* harmonic-percussive separation of a batch: data batch x dataLength -> h and p, each batch x
 * hpssObj_calDataLength(dataLength), both overwritten.  Either output may be NULL (its inverse STFT is skipped), not
 * both.  Each clip's result is bit-identical to hpssObj_hpss on that clip into zeroed buffers, whatever the batch.
 * Refused wherever hpssObj_hpss refuses.  The device workspace (six half-spectrum planes and the inverse STFT's frames)
 * is bounded by processing the clips in groups; per group, up to fftLength 2^14: one STFT launch, one mask launch and
 * two inverse STFT launches per requested output. */
int hpssObj_hpssBatch(HPSSObj hpssObj, const float *data, int dataLength, int batch, float *h, float *p, int memKind,
                      void *stream);

/* onset detection of a batch: spec (and phase, NULL unless the object's type is PD / WPD / NWPD / CD / RCD)
 * batch x nLength x mLength -> evn batch x nLength, points batch x nLength (each clip's points first, 0 after them)
 * and counts batch (points per clip).  param and indexArr are host memory (param NULL: the defaults of onsetObj_onset).
 * Each clip's results are bit-identical to onsetObj_onset on that clip, whatever the batch.  Refused wherever
 * onsetObj_onset refuses.  Per group of clips (the filtered matrix is a workspace bounded by grouping): the max filter
 * when filterOrder >= 2, one novelty launch and one peak-picking launch. */
int onsetObj_onsetBatch(OnsetObj onsetObj, const float *spec, const float *phase, int batch, const NoveltyParam *param,
                        const int *indexArr, int indexLength, float *evn, int *points, int *counts, int memKind,
                        void *stream);

/* harmonic ratio of a batch: data batch x dataLength -> value batch x T, T = harmonicRatioObj_calTimeLength(dataLength).
 * The minIndex carry of a frame without a crossing starts afresh at every clip.  Each clip's row is bit-identical to
 * harmonicRatioObj_harmonicRatio on that clip, whatever the batch.  Two kernel launches per staging chunk: every frame,
 * then the frames without a crossing of their own. */
int harmonicRatioObj_harmonicRatioBatch(HarmonicRatioObj harmonicRatioObj, const float *data, int dataLength, int batch,
                                        float *value, int memKind, void *stream);

/* pitch (PEF) of a batch: data batch x dataLength -> freArr batch x T, T = (dataLength - n) / slideLength + 1 (0 below n
 * samples).  Each clip is computed on its own: the call neither reads nor updates the streaming carry of isContinue.
 * Each clip's row is bit-identical to pitchPEFObj_pitch on that clip without streaming, whatever the batch.  One kernel
 * launch per staging chunk. */
int pitchPEFObj_pitchBatch(PitchPEFObj pitchPEFObj, const float *data, int dataLength, int batch, float *freArr,
                           int memKind, void *stream);

/* pitch (YIN) of a batch: data batch x dataLength -> freArr, valueArr1, valueArr2 batch x T, mFreArr, mTroughArr
 * batch x T x mLen (mLen = yinLength/2 + 1, entries past lenArr zero) and lenArr batch x T ints, T =
 * (dataLength - n) / slideLength + 1 (0 below n samples).  Every output but freArr may be NULL: it is then neither
 * computed nor written.  In frames without a trough freArr and valueArr1 are left as they are, on the device as well.
 * Each clip is computed on its own: the call neither reads nor updates the streaming carry of isContinue.  Each clip's
 * row is bit-identical to pitchYINObj_pitch on that clip without streaming, whatever the batch.  One kernel launch per
 * staging chunk. */
int pitchYINObj_pitchBatch(PitchYINObj pitchYINObj, const float *data, int dataLength, int batch, float *freArr,
                           float *valueArr1, float *valueArr2, float *mFreArr, float *mTroughArr, int *lenArr,
                           int memKind, void *stream);

/* pitch (NCF, CEP) of a batch: data batch x dataLength -> freArr batch x T, T = (dataLength - n) / slideLength + 1 (0
 * below n samples).  Each clip is computed on its own: the call neither reads nor updates the streaming carry of
 * isContinue.  Each clip's row is bit-identical to pitchNCFObj_pitch / pitchCEPObj_pitch on that clip without
 * streaming, whatever the batch.  One kernel launch per staging chunk. */
int pitchNCFObj_pitchBatch(PitchNCFObj pitchNCFObj, const float *data, int dataLength, int batch, float *freArr,
                           int memKind, void *stream);
int pitchCEPObj_pitchBatch(PitchCEPObj pitchCEPObj, const float *data, int dataLength, int batch, float *freArr,
                           int memKind, void *stream);

/* discrete wavelet transforms of a batch of clips (data batch x N): coef batch x N and mData batch x rows x N (rows =
 * num for DWT, 2^num for WPT; NULL: not written); SWT: mData1, mData2 batch x num x fftLength.  One kernel launch per
 * level per staging chunk (and one for mData); each clip's rows are bit-identical to the legacy call on that clip. */
int dwtObj_dwtBatch(DWTObj dwtObj, const float *data, int batch, float *coef, float *mData, int memKind, void *stream);
int wptObj_wptBatch(WPTObj wptObj, const float *data, int batch, float *coef, float *mData, int memKind, void *stream);
int swtObj_swtBatch(SWTObj swtObj, const float *data, int batch, float *mData1, float *mData2, int memKind,
                    void *stream);

/* non-negative matrix factorisation of a batch (afb200_nmf.h): V batch x n x m; W batch x n x k and H batch x k x m in/out,
 * initialised by the caller; iters (batch ints, NULL: not written) receives the iterations each matrix ran.  maxIter,
 * type, thresh and norm apply to every matrix, NULL giving nmf's defaults.  Each matrix stops on its own and gives the
 * same bits as nmf on it, whatever the batch.  Returns -1 when n, m, k or batch is below 1 or an array is NULL.
 * 1 + 4 maxIter kernel launches per staging chunk (per call with device pointers), however many matrices it holds; the
 * host never waits between iterations.  The call allocates a device workspace for the matrices it runs at once (with
 * device pointers the whole batch) of (P n m + n k + k m + k + 1) floats each, P = 2 for IS and 1 otherwise: 4096
 * IS matrices of 513 x 431 need about 7.3 GB.  When that allocation fails the call returns an error and writes nothing. */
int nmfBatch(const float *V, int batch, int n, int m, int k, float *W, float *H, const int *maxIter, const int *type,
             const float *thresh, const int *norm, int *iters, int memKind, void *stream);

/* cross-correlation of a batch of pairs (afb200_xcorr.h): a, b batch x length (b NULL: the autocorrelation of each row of
 * a) -> out batch x (2 length - 1); maxValue and maxIndex (batch each, either may be NULL) receive each row's maximum and
 * its first index.  normType NULL means XcorrNormal_Coeff, as in xcorrObj_xcorr.  Each row is bit-identical to
 * xcorrObj_xcorr on that pair, whatever the batch.  Returns -1 for length < 1 or batch < 0 and -2 for length above
 * AFB200_XCORR_MAX_LENGTH.  Up to 8192 samples (transforms of up to 2^14 points) one kernel launch per staging chunk;
 * longer rows run the four-step transforms of the CWT path in bounded groups of pairs. */
int xcorrObj_xcorrBatch(XcorrObj xcorrObj, const float *a, const float *b, int length, int batch,
                        XcorrNormalType *normType, float *out, float *maxValue, int *maxIndex, int memKind, void *stream);

/* chirp z-transform of a batch of rows (afb200_czt.h): re, im batch x N (either may be NULL, not both) -> re3, im3
 * batch x 2N, each row bit-identical to cztObj_czt on it.  The band rule of cztObj_czt applies once per call.  One kernel
 * launch per staging chunk, plus one per change of the object's tables; a table change waits for the object's earlier
 * launches. */
int cztObj_cztBatch(CZTObj cztObj, const float *re, const float *im, int batch, float lowW, float highW,
                    float *re3, float *im3, int memKind, void *stream);

#ifdef __cplusplus
}
#endif
#endif
