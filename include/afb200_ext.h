/* afb200_ext.h -- ADDITIVE entry points of libaudioflux_b200.so (no reference counterpart).
 *
 * The reference API is one clip per call with host pointers (python/audioflux/bft.py:349-365
 * loops channels in Python); fed that way a GPU is PCIe/launch bound.  These entry points
 * take a whole batch and either host or device pointers.
 *
 *   memKind 0: host pointers (pageable or pinned) -- copies + sync happen inside the call.
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
/* diagnostics: bank loop of the fused MFCC plan built by the last bftObj_mfccBatch call
 * (1 interval / shared-product form of a triangular bank, 0 filter-per-lane, -1 no fused plan) */
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
/* planner of the fused MFCC kernel's bank loop (host only): 1 when `bank` (num x 1025) has the triangular
 * two-overlap structure and the interval form applies; fills the per-bin interval owner / rising weight etc. */
int afb200_mfccIntervalPlan(const float *bank, int num, const float *gain, int *owner, float *r, int *ivStart,
                            int *ivLen, float *tailW, int *groupLen, int *startShifted);
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
/* cepstral deconvolution of rows x num constant-Q magnitudes (cqtObj_cqhc / cqtObj_deconv for any number of rows) */
int cqtObj_cqhcBatch(CQTObj cqtObj, const float *in, int rows, int hcNum, float *out /* rows x hcNum */, int memKind, void *stream);
int cqtObj_deconvBatch(CQTObj cqtObj, const float *in, int rows, float *timbre, float *pitch /* rows x num each */,
                       int memKind, void *stream);
/* chroma_cqtFilterBank (src/filterbank/chroma_filterBank.c:176-262): bank num x cqtLength */
int afb200_chromaCqtFilterBank(int num, int cqtLength, int binPerOctave, float minFre, float *bank);

#ifdef __cplusplus
}
#endif
#endif
