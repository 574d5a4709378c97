/* afb200_cwt.h -- continuous wavelet transform.  Replaces src/cwt_algorithm.h:14-45
 * (src/cwt_algorithm.c); cwtDet is a "next" row. */
#ifndef AFB200_CWT_H
#define AFB200_CWT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueCWT *CWTObj;

/* cwt_algorithm.c:73-334.  -100 bad radix2Exp; 1 bad scale; -1 bad num / range;
 * -2 when isPad yields a non power-of-two length (2^radix2Exp > 1e5), which the reference
 * serves with an O(N^2) dense DFT. */
int cwtObj_new(CWTObj *cwtObj, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre,
               int *binPerOctave, WaveletContinueType *waveletType, SpectralFilterBankScaleType *scaleType,
               float *gamma, float *beta, int *isPad);
float *cwtObj_getFreBandArr(CWTObj cwtObj);                       /* :336-339 */
int *cwtObj_getBinBandArr(CWTObj cwtObj);                         /* :341-344 */
/* :346-350.  dataArr: exactly 2^radix2Exp samples; outputs num x 2^radix2Exp, row 0 = highest band. */
void cwtObj_cwt(CWTObj cwtObj, float *dataArr, float *mRealArr4, float *mImageArr4);
/* :485-528 / :352-358.  Derivative transform W' = IFFT(j * omega * wavelet * X) for synchrosqueezing.  enableDet(1)
 * must be called once; dataArr may be NULL to reuse the spectrum of the preceding single-clip cwtObj_cwt / cwtDet. */
void cwtObj_enableDet(CWTObj cwtObj, int flag);
void cwtObj_cwtDet(CWTObj cwtObj, float *dataArr, float *mRealArr4, float *mImageArr4);
void cwtObj_free(CWTObj cwtObj);

#ifdef __cplusplus
}
#endif
#endif
