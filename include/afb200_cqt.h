/* afb200_cqt.h -- constant-Q transform.  Replaces src/cqt_algorithm.h:14-62
 * (src/cqt_algorithm.c).   */
#ifndef AFB200_CQT_H
#define AFB200_CQT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueCQT *CQTObj;

int cqtObj_new(CQTObj *cqtObj, int num, int samplate, float minFre, int *isContinue);  /* cqt_algorithm.c:110-120 */
/* :123-247.  -1 if binPerOctave%12 or num%binPerOctave.  beta != 0 (VQT): every octave gets its own kernel rows. */
int cqtObj_newWith(CQTObj *cqtObj, int num, int *samplate, float *minFre, int *binPerOctave,
                   float *factor, float *beta, float *thresh, WindowType *windowType, int *slideLength,
                   int *isContinue, SpectralFilterBankNormalType *normalType, int *isScale);
int cqtObj_calTimeLength(CQTObj cqtObj, int dataLength);          /* :266-299 */
int cqtObj_getFFTLength(CQTObj cqtObj);                           /* :333-338 */
float *cqtObj_getFreBandArr(CQTObj cqtObj);                       /* :340-343, borrowed */
void cqtObj_setScale(CQTObj cqtObj, int flag);                    /* :458-461 */
/* :463-478.  mRealArr3/mImageArr3: timeLength x num. */
void cqtObj_cqt(CQTObj cqtObj, float *dataArr, int dataLength, float *mRealArr3, float *mImageArr3);
/* :484-600.  Planes of the last cqtObj_cqt call (timeLength x num) -> mDataArr3: timeLength x chromaNum.
 * Defaults: chromaNum 12 (must divide binPerOctave), dataType Power, normType Max. */
void cqtObj_chroma(CQTObj cqtObj, int *chromaNum, SpectralDataType *dataType, ChromaDataNormalType *normType,
                   float *mRealArr1, float *mImageArr1, float *mDataArr3);
/* :602-660.  mDataArr1: timeLength x num (power or magnitude) -> mDataArr2: timeLength x ccNum. */
void cqtObj_cqcc(CQTObj cqtObj, float *mDataArr1, int ccNum, CepstralRectifyType *rectifyType, float *mDataArr2);
/* :662-714.  mDataArr1 [timeLength x num] magnitudes / powers of the last cqtObj_cqt call -> mDataArr2 [timeLength x hcNum]:
 * the cepstral timbre sequence Re IFFT(|FFT(row)|) (length ceilPow2(2 num)) at round(binPerOctave log2(j + 1)). */
void cqtObj_cqhc(CQTObj cqtObj, float *mDataArr1, int hcNum, float *mDataArr2);
/* :716-781.  mDataArr2 = timbre (formant), mDataArr3 = pitch = Re IFFT(FFT(row) / |FFT(row)|), first num samples each. */
void cqtObj_deconv(CQTObj cqtObj, float *mDataArr1, float *mDataArr2, float *mDataArr3);
void cqtObj_free(CQTObj cqtObj);

#ifdef __cplusplus
}
#endif
#endif
