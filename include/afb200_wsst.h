/* afb200_wsst.h -- synchrosqueezing objects: drop-in for src/wsst_algorithm.h:12-49 and
 * src/synsq_algorithm.h:12-33 (same names, argument meaning and defaults). */
#ifndef AFB200_WSST_H
#define AFB200_WSST_H

#include "afb200_types.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueWSST *WSSTObj;
typedef struct OpaqueSynsq *SynsqObj;

/* wsst_algorithm.c:64-160.  Defaults: samplate 32000, morlet, octave scale, thresh 0.001, isPadding as cwtObj_new. */
int wsstObj_new(WSSTObj *wsstObj, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre, int *binPerOctave,
                WaveletContinueType *waveletType, SpectralFilterBankScaleType *scaleType, float *gamma, float *beta,
                float *thresh, int *isPadding);
float *wsstObj_getFreBandArr(WSSTObj wsstObj);                    /* :162-165 */
int *wsstObj_getBinBandArr(WSSTObj wsstObj);                      /* :167-170 */
/* :172-176.  order > 1 is refused loudly: the reference dereferences an unallocated scratch array there. */
void wsstObj_setOrder(WSSTObj wsstObj, int order);
/* :178-352.  dataArr: 2^radix2Exp samples.  mRealArr1 / mImageArr1 [num x N]: the squeezed transform is ADDED to their
 * content (callers pass zeros); mRealArr2 / mImageArr2 (may be NULL): the plain CWT. */
void wsstObj_wsst(WSSTObj wsstObj, float *dataArr, float *mRealArr1, float *mImageArr1, float *mRealArr2, float *mImageArr2);
void wsstObj_free(WSSTObj wsstObj);

/* synsq_algorithm.c:38-127.  thresh is only taken when > 1 (as in the reference); order > 1 -> -2. */
int synsqObj_new(SynsqObj *synsqObj, int num, int radix2Exp, int *samplate, int *order, float *thresh);
/* :129-300.  freArr [num] ascending Hz; planes [num x N] of any time-frequency transform; result ADDED to mRealArr2 / mImageArr2. */
void synsqObj_synsq(SynsqObj synsqObj, float *freArr, SpectralFilterBankScaleType scaleType, float *mRealArr1,
                    float *mImageArr1, float *mRealArr2, float *mImageArr2);
void synsqObj_free(SynsqObj synsqObj);

/* additive: device-pointer forms (asynchronous on `stream`; planes [num x N] on the device) */
int wsstObj_wsstDevice(WSSTObj wsstObj, const float *dData, float *dOutRe, float *dOutIm, float *dCwtRe, float *dCwtIm, void *stream);
int synsqObj_synsqDevice(SynsqObj synsqObj, const float *freArr, int scaleType, const float *dRe, const float *dIm,
                         float *dOutRe, float *dOutIm, void *stream);

#ifdef __cplusplus
}
#endif
#endif
