/* afb200_spectrogram.h -- SpectrogramObj: the reference's general spectrogram front door (the class its own
 * benchmark times, benchmark/run_audioflux.py:14-29).  Replaces the part of
 * src/spectrogram_algorithm.h:40-119 that lies on the time-frequency path:
 * construction, spectrogram (STFT -> power/magnitude -> Linear slice or mel/bark/erb/... bank) and the cepstral
 * calls and the cepstral deconvolution.  Chroma / Deep scale types and the spectral-descriptor functions (flatness,
 * centroid, ...) are outside the path: `_new` rejects those scale types with -2, the functions are not exported. */
#ifndef AFB200_SPECTROGRAM_H
#define AFB200_SPECTROGRAM_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueSpectrogram *SpectrogramObj;

/* spectrogram_algorithm.c:326-583.  Defaults: samplate 32000, lowFre 0 (Octave/Log: C1..B7), highFre samplate/2,
 * binPerOctave 12, radix2Exp 12, hann, slideLength fftLength/4, power, Linear, Slaney, no normalisation.
 * Linear: num is ignored and becomes round(highFre/det)-round(lowFre/det)+1 (spectrogramObj_getBandNum).
 * Returns 0; -100 bad radix2Exp; -1 bad num / Octave overflow; -2 unsupported (Chroma/Deep scales).
 * isContinue = 1: samples that did not complete a frame wait for the next spectrogramObj_spectrogram call (:655-664). */
int spectrogramObj_new(SpectrogramObj *spectrogramObj, int num, int *samplate, float *lowFre, float *highFre,
                       int *binPerOctave, int *radix2Exp, WindowType *windowType, int *slideLength,
                       int *isContinue, SpectralDataType *dataType,
                       SpectralFilterBankScaleType *filterScaleType, SpectralFilterBankStyleType *filterStyleType,
                       SpectralFilterBankNormalType *filterNormalType);
int spectrogramObj_newLinear(SpectrogramObj *spectrogramObj, int samplate, int radix2Exp, int *isContinue); /* :186-203 */
int spectrogramObj_newMel(SpectrogramObj *spectrogramObj, int num, int samplate, int radix2Exp, int *isContinue);  /* :205-222 */
int spectrogramObj_newBark(SpectrogramObj *spectrogramObj, int num, int samplate, int radix2Exp, int *isContinue); /* :224-242 */
int spectrogramObj_newErb(SpectrogramObj *spectrogramObj, int num, int samplate, int radix2Exp, int *isContinue);  /* :244-262 */
/* :264-324.  Chroma / Deep families: refused loudly (-2), exported so the symbols resolve */
int spectrogramObj_newChroma(SpectrogramObj *spectrogramObj, int samplate, int radix2Exp, int *isContinue);
int spectrogramObj_newDeep(SpectrogramObj *spectrogramObj, int num, int samplate, int radix2Exp, int *isContinue);
int spectrogramObj_newDeepChroma(SpectrogramObj *spectrogramObj, int samplate, int radix2Exp, int *isContinue);
void spectrogramObj_enableDebug(SpectrogramObj spectrogramObj, int flag);                    /* :3171, no-op */
void spectrogramObj_setDataNormValue(SpectrogramObj spectrogramObj, float normValue);       /* :841-846 */
int spectrogramObj_calTimeLength(SpectrogramObj spectrogramObj, int dataLength);            /* :848-853 */
float *spectrogramObj_getFreBandArr(SpectrogramObj spectrogramObj);                         /* :3176, borrowed */
int *spectrogramObj_getBinBandArr(SpectrogramObj spectrogramObj);                           /* :3181, borrowed */
int spectrogramObj_getBandNum(SpectrogramObj spectrogramObj);                               /* :3187 */
int spectrogramObj_getBinBandLength(SpectrogramObj spectrogramObj);                         /* :3192 */
/* :864-1395.  mSpectArr: timeLength x bandNum.  mPhaseArr (may be NULL) is written only for the Linear scale:
 * timeLength x bandNum of atan2f(im, max(re, 1e-16)) exactly as the reference computes it. */
void spectrogramObj_spectrogram(SpectrogramObj spectrogramObj, float *dataArr, int dataLength, float *mSpectArr,
                                float *mPhaseArr);
/* :1409-1525.  mDataArr1: timeLength x bandNum of the LAST spectrogram call; mDataArr2: timeLength x ccNum.
 * mfcc / bfcc / gtcc / lfcc act only for Mel scale / Bark scale / Gammatone style / Linear scale (else no-op). */
void spectrogramObj_xxcc(SpectrogramObj spectrogramObj, float *mDataArr1, int ccNum, CepstralRectifyType *rectifyType,
                         float *mDataArr2);
void spectrogramObj_mfcc(SpectrogramObj spectrogramObj, float *mDataArr1, int ccNum, float *mDataArr2);
void spectrogramObj_bfcc(SpectrogramObj spectrogramObj, float *mDataArr1, int ccNum, float *mDataArr2);
void spectrogramObj_gtcc(SpectrogramObj spectrogramObj, float *mDataArr1, int ccNum, float *mDataArr2);
void spectrogramObj_lfcc(SpectrogramObj spectrogramObj, float *mDataArr1, int ccNum, float *mDataArr2);
/* :1527-1537 -- empty bodies in the reference; kept as no-ops */
void spectrogramObj_mfccStandard(SpectrogramObj spectrogramObj, float *mDataArr1, int *deltaWindowLength,
                                 CepstralEnergyType *energyType, CepstralRectifyType *rectifyType, float *mDataArr2);
void spectrogramObj_xxccStandard(SpectrogramObj spectrogramObj, float *mDataArr1, int *deltaWindowLength,
                                 CepstralEnergyType *energyType, CepstralRectifyType *rectifyType, float *mDataArr2);
/* :1545-1612.  mDataArr1: timeLength x bandNum of the last spectrogram call -> mDataArr2 (timbre / tone) and mDataArr3
 * (pitch), same shape: per frame, zero-padded to ceilPow2(2 bandNum), Re IFFT(|FFT|) and Re IFFT(FFT / max(|FFT|, 1e-16)).
 * bandNum <= 2048 (one CTA-resident transform per frame); larger band counts are refused on stderr. */
void spectrogramObj_deconv(SpectrogramObj spectrogramObj, float *mDataArr1, float *mDataArr2, float *mDataArr3);
void spectrogramObj_free(SpectrogramObj spectrogramObj);                                    /* :3029-3169 */

#ifdef __cplusplus
}
#endif
#endif
