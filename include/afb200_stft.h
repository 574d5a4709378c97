/* afb200_stft.h -- framed STFT object.  Replaces src/stft_algorithm.h:14-40
 * (implementation src/stft_algorithm.c).  Host pointers, one clip per call, caller-allocated
 * outputs that are fully overwritten. */
#ifndef AFB200_STFT_H
#define AFB200_STFT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueSTFT *STFTObj;

/* stft_algorithm.c:84-168.  radix2Exp in [1,30] else -100; NULL pointers = defaults
 * (rect window, slide = fftLength/4, isContinue 0).  isContinue=1 (streaming, :474-599): every stftObj_stft call
 * transforms the samples carried over from the previous calls followed by the new ones and keeps the rest that did not
 * complete a hop (non-padding mode only, as in the reference; the batched / device-pointer entry points are stateless).
 * Transforms run for fftLength up to 2^20 (one CTA per frame up to 16384 points, the four-step kernels above that). */
int stftObj_new(STFTObj *stftObj, int radix2Exp, WindowType *windowType, int *slideLength, int *isContinue);
void stftObj_setSlideLength(STFTObj stftObj, int slideLength);                 /* :171-178 */
void stftObj_enablePadding(STFTObj stftObj, int flag);                         /* :186-189 */
void stftObj_enableContinue(STFTObj stftObj, int flag);                        /* :180-183 */
void stftObj_setPadding(STFTObj stftObj, PaddingPositionType *positionType, PaddingModeType *modeType,
                        float *value1, float *value2);                         /* :192-213 */
void stftObj_useWindowDataArr(STFTObj stftObj, float *winDataArr);             /* :215-218 */
float *stftObj_getWindowDataArr(STFTObj stftObj);                              /* :220-223, borrowed */
int stftObj_calTimeLength(STFTObj stftObj, int dataLength);                    /* :225-262 */
int stftObj_calDataLength(STFTObj stftObj, int timeLength);                    /* :289-301 */
/* :264-287.  mRealArr/mImageArr: timeLength x fftLength, full mirrored spectrum. */
void stftObj_stft(STFTObj stftObj, float *dataArr, int dataLength, float *mRealArr, float *mImageArr);
/* :304-409.  mRealArr/mImageArr: timeLength x fftLength (full spectrum); dataArr: (timeLength-1)*slide + fftLength
 * samples, pre-zeroed by the caller (frames are added to its content, then divided by the window sum).
 * methodType 0 'weight' (synthesis window w, normaliser sum w^2), else 'overlap-add' (normaliser sum w).
 * fftLength up to 2^20: one CTA per frame up to 16384 points (16384 takes an in-place shared-memory path), above that
 * Re(IFFT) comes from one real-input forward transform of the four-step kernels (Hartley identity, kernels/istft.cu). */
void stftObj_istft(STFTObj stftObj, float *mRealArr, float *mImageArr, int timeLength, int methodType, float *dataArr);
void stftObj_free(STFTObj stftObj);                                            /* :411-467, NULL-safe */
void stftObj_debug(STFTObj stftObj);                                           /* :837-849 */

#ifdef __cplusplus
}
#endif
#endif
