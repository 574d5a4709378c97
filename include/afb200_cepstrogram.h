/* afb200_cepstrogram.h -- the cepstrogram: per frame of a windowed STFT (no padding), the real cepstrum of the log power
 * spectrum and its split by a lifter into a spectral envelope (the first cepNum quefrencies) and details (the rest).
 * Replaces include/cepstrogram_algorithm.h:14-39 (src/cepstrogram_algorithm.c).
 *
 * Differences from the reference, all on purpose:
 *   - cepstrogramObj_new returns -2 with a message for radix2Exp > 14 (one CTA holds a whole frame in shared memory);
 *   - every compute call refuses cepNum < 1 or cepNum > N/2 and leaves the outputs untouched (the reference reads and
 *     writes out of bounds there);
 *   - cepstrogramObj_cepstrogram2 computes from the caller's STFT planes and never writes them (the reference copies its
 *     own buffers INTO them, so its result depends on the object's previous call, not on the input);
 *   - at N = 2 without a slide length the hop is 1 (the reference's default N/4 is 0 there, and its calTimeLength
 *     divides by zero);
 *   - no T x N scratch plane is kept on the host: a frame's spectrum, log spectrum and cepstrum stay in shared memory. */
#ifndef AFB200_CEPSTROGRAM_H
#define AFB200_CEPSTROGRAM_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueCepstrogram *CepstrogramObj;

/* include/cepstrogram_algorithm.h:21, src/cepstrogram_algorithm.c:55-102.  windowType NULL: Rect; slideLength NULL or
 * <= 0: N/4, 1 at N = 2 (any positive value is taken, also one above N).  Returns 0, -100 (radix2Exp outside 1 .. 30) or -2
 * (radix2Exp > 14).  Needs no GPU. */
int cepstrogramObj_new(CepstrogramObj *cepstrogramObj, int radix2Exp, WindowType *windowType, int *slideLength);

/* :23, src :104-109: frames of a clip, the STFT rule without padding: (dataLength - N) / slideLength + 1, 0 when the
 * clip is shorter than N */
int cepstrogramObj_calTimeLength(CepstrogramObj cepstrogramObj, int dataLength);

/* :31-32, src :127-298.  Per frame: S = |STFT|^2 clamped below at 1e-16, y = Re IFFT_N(log S);
 *   mDataArr1 (cepstrums) = y[0 .. N/2];
 *   mDataArr2 (envelope)  = Re FFT_N(y on {0 .. cepNum} and {N-cepNum .. N-1});
 *   mDataArr3 (details)   = Re FFT_N(y on {cepNum+1 .. N-cepNum}).
 * Each is timeLength x (N/2+1) and may be NULL (not computed).  cepNum 1 .. N/2.  On failure (bad cepNum, no GPU, ...)
 * the outputs are left untouched and afb200_lastError() holds the message. */
void cepstrogramObj_cepstrogram(CepstrogramObj cepstrogramObj, int cepNum, float *dataArr, int dataLength,
                                float *mDataArr1, float *mDataArr2, float *mDataArr3);

/* :34-35, src :119-125: the same from the caller's STFT planes, nLength x N each (one frame per row).  Every bin is used:
 * y = Re IFFT_N(log S) is the inverse transform of the even part of log S.  The planes are read only. */
void cepstrogramObj_cepstrogram2(CepstrogramObj cepstrogramObj, int cepNum, float *mRealArr, float *mImageArr, int nLength,
                                 float *mDataArr1, float *mDataArr2, float *mDataArr3);

void cepstrogramObj_enableDebug(CepstrogramObj cepstrogramObj, int flag);     /* :37: no-op */

void cepstrogramObj_free(CepstrogramObj cepstrogramObj);                      /* :39 */

#ifdef __cplusplus
}
#endif
#endif
