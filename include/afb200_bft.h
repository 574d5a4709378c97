/* afb200_bft.h -- BFT object: STFT -> power/magnitude -> mel/bark/erb/... filter bank.
 * Replaces src/bft_algorithm.h:14-57 (implementation src/bft_algorithm.c). */
#ifndef AFB200_BFT_H
#define AFB200_BFT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueBFT *BFTObj;

/* bft_algorithm.c:87-276.  Returns 0 ok; -100 bad radix2Exp; 1 scale > Log; -1 bad num /
 * range overflow.  isTemporal = 1: bftObj_bft also computes energy / rms / zero-crossing rate of the windowed frames
 * (src/temporal_algorithm.c:93-146), read with bftObj_getTemporalData.  isReassign = 1: the bank is applied to the
 * reassigned spectrum (include/afb200_reassign.h, Reassign_All); every call starts from zeroed planes -- the reference
 * keeps adding into its cached planes from the second call on (bft_algorithm.c:441-455), which is not reproduced. */
int bftObj_new(BFTObj *bftObj, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre,
               int *binPerOctave, WindowType *windowType, int *slideLength,
               SpectralFilterBankScaleType *filterScaleType, SpectralFilterBankStyleType *filterStyleType,
               SpectralFilterBankNormalType *filterNormalType, SpectralDataType *dataType,
               int *isReassign, int *isTemporal);
int bftObj_calTimeLength(BFTObj bftObj, int dataLength);          /* :550-555 */
float *bftObj_getFreBandArr(BFTObj bftObj);                       /* :557-560, borrowed, num floats */
int *bftObj_getBinBandArr(BFTObj bftObj);                         /* :562-565, borrowed, num ints */
void bftObj_setResultType(BFTObj bftObj, int type);               /* :568-571, 0 complex 1 real */
void bftObj_setDataNormValue(BFTObj bftObj, float normValue);     /* :573-578 */
/* :397-540.  mRealArr3/mImageArr3: timeLength x num (mImageArr3 untouched when resultType=1). */
void bftObj_bft(BFTObj bftObj, float *dataArr, int dataLength, float *mRealArr3, float *mImageArr3);
void bftObj_getTemporalData(BFTObj bftObj, float **eArr, float **rArr, float **zArr); /* :541-547, arrays of the last bftObj_bft call (isTemporal = 1) */
void bftObj_free(BFTObj bftObj);                                  /* :580-626 */

#ifdef __cplusplus
}
#endif
#endif
