/* afb200_nsgt.h -- non-stationary Gabor transform of one 2^radix2Exp clip: per band a windowed slice of the clip's
 * spectrum, inverse-transformed to the band's own time grid (the "cells"), and a num x maxLen matrix that holds each
 * band's cells repeated on the common time grid of the widest band.
 * Replaces src/nsgt_algorithm.h:14-57 (src/nsgt_algorithm.c, src/filterbank/nsgt_filterBank.c).
 *
 * Differences from the reference, all on purpose:
 *   - nsgtObj_setMinLength rebuilds the time grids with the bank, so the object equals a fresh one built with that
 *     minLen.  The reference rebuilds the bank only (src/nsgt_algorithm.c:429-481) and maps its matrix columns with the
 *     old grids, reading past them when a length grows;
 *   - nsgtObj_new returns -2 with a message for radix2Exp > 20 (the longest forward FFT of the library) and for a band
 *     window longer than 16384 (the reference's dense inverse DFT would need 16 L^2 bytes, >= 4.3 GB, for that band);
 *   - each band's inverse transform runs in float32 (Bluestein FFT up to L = 4096, direct DFT above) where the
 *     reference multiplies by a dense float64 matrix (src/dsp/dft_algorithm.c:106-152). */
#ifndef AFB200_NSGT_H
#define AFB200_NSGT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

/* src/nsgt_algorithm.h:14-18 */
typedef enum { NSGTFilterBank_Efficient = 0, NSGTFilterBank_Standard } NSGTFilterBankType;

typedef struct OpaqueNSGT *NSGTObj;

/* src/nsgt_algorithm.c:72-251.  Defaults: samplate 32000, Octave, Hann, BandWidth, Efficient, minLen 3; Gammatone style
 * is taken as Hann and Area norm as BandWidth.  Returns -100 (radix2Exp outside 1..30), 1 (scaleType > Log), -1 (revised
 * highFre above Nyquist, num outside [2, fftLength/2+1]), -2 (see above) or 0.  Needs no GPU. */
int nsgtObj_new(NSGTObj *nsgtObj, int num, int radix2Exp,
                int *samplate, float *lowFre, float *highFre, int *binPerOctave,
                int *minLen,
                NSGTFilterBankType *nsgtFilterBankType,
                SpectralFilterBankScaleType *filterScaleType,
                SpectralFilterBankStyleType *filterStyleType,
                SpectralFilterBankNormalType *filterNormalType);

int nsgtObj_getMaxTimeLength(NSGTObj nsgtObj);      /* :614-617: the longest band window, columns of the matrix */
int nsgtObj_getTotalTimeLength(NSGTObj nsgtObj);    /* :619-622: sum of the band windows, length of the cells */
int *nsgtObj_getTimeLengthArr(NSGTObj nsgtObj);     /* :624-627: num band window lengths (owned by the object) */

float *nsgtObj_getFreBandArr(NSGTObj nsgtObj);      /* :629-632: num centre frequencies */
int *nsgtObj_getBinBandArr(NSGTObj nsgtObj);        /* :634-637: num centre bins */

/* :429-481: minLength >= 1, ignored otherwise; rebuilds the bank AND the time grids (see above) */
void nsgtObj_setMinLength(NSGTObj nsgtObj, int minLength);

/* :483-605: dataArr 2^radix2Exp samples -> mRealArr3 / mImageArr3 num x maxTimeLength.  On failure (no GPU, ...) the
 * outputs are left untouched and afb200_lastError() holds the message. */
void nsgtObj_nsgt(NSGTObj nsgtObj, float *dataArr, float *mRealArr3, float *mImageArr3);

/* :608-612: the cells (totalTimeLength each, band after band) of the last nsgtObj_nsgt call, owned by the object */
void nsgtObj_getCellData(NSGTObj nsgtObj, float **realArr3, float **imageArr3);

void nsgtObj_free(NSGTObj nsgtObj);                 /* :639-727 */

#ifdef __cplusplus
}
#endif
#endif
