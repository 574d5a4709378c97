/* afb200_pwt.h -- pseudo wavelet transform: FFT -> auditory filter bank x spectrum -> IFFT per band.
 * Replaces src/pwt_algorithm.h:16-31 (src/pwt_algorithm.c). */
#ifndef AFB200_PWT_H
#define AFB200_PWT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaquePWT *PWTObj;

/* pwt_algorithm.c:63-270.  Defaults: samplate 32000, Octave scale (C1..B7), binPerOctave 12, Slaney triangles, no
 * normalisation, no padding.  -100 bad radix2Exp; 1 bad scale; -1 bad num / range overflow; -2 when isPadding
 * yields a non power-of-two length (2^radix2Exp > 1e5; the reference then uses an O(N^2) dense DFT). */
int pwtObj_new(PWTObj *pwtObj, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre,
               int *binPerOctave, SpectralFilterBankScaleType *scaleType, SpectralFilterBankStyleType *styleType,
               SpectralFilterBankNormalType *normalType, int *isPadding);
float *pwtObj_getFreBandArr(PWTObj pwtObj);                       /* :323-326, borrowed */
int *pwtObj_getBinBandArr(PWTObj pwtObj);                         /* :328-331, borrowed */
/* :333-336.  dataArr: exactly 2^radix2Exp samples; outputs num x 2^radix2Exp.  The transform runs for radix2Exp
 * 1 .. 24 (isPadding doubles the FFT length, and is only accepted up to radix2Exp 16); an object built with radix2Exp
 * 25 .. 30 constructs, but every transform call on it fails (non-zero status, message in afb200_lastError()) and leaves the
 * outputs untouched. */
void pwtObj_pwt(PWTObj pwtObj, float *dataArr, float *mRealArr3, float *mImageArr3);
void pwtObj_enableDet(PWTObj pwtObj, int flag);                   /* :350-390 */
/* :338-344.  Derivative transform (bank x j omega); dataArr may be NULL to reuse the preceding call's spectrum. */
void pwtObj_pwtDet(PWTObj pwtObj, float *dataArr, float *mRealArr3, float *mImageArr3);
void pwtObj_free(PWTObj pwtObj);

#ifdef __cplusplus
}
#endif
#endif
