/* afb200_swt.h -- stationary (undecimated) wavelet transform.  Replaces include/swt_algorithm.h (src/swt_algorithm.c).
 *
 * Level i = 0 .. num-1 of a signal of fftLength samples pads row i-1 of the approximation (the input at level 0)
 * periodically by upLength/2 samples on each side, upLength = decLength * 2^i, and keeps fftLength samples from offset
 * upLength of its full convolution with the filters dilated by 2^i (zeros inserted).  mDataArr1 (approximations) and
 * mDataArr2 (details) hold num x fftLength floats each.  Filters and refusals: afb200_dwt.h.
 *
 * Differences from the reference, on purpose: fftLength above 2^AFB200_WAVELET_MAX_EXP, and the refused filters,
 * return -2; num outside 0 .. 30 returns -1 (the reference shifts by it). */
#ifndef AFB200_SWT_H
#define AFB200_SWT_H
#include "afb200_dwt.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueSWT *SWTObj;

/* src :50-118: fftLength < 2^num or not a multiple of it: -1. */
int swtObj_new(SWTObj *swtObj, int num, int fftLength, WaveletDiscreteType *waveletType, int *t1, int *t2);

/* src :126-220 */
void swtObj_swt(SWTObj swtObj, float *dataArr, float *mDataArr1, float *mDataArr2);

void swtObj_free(SWTObj swtObj);

#ifdef __cplusplus
}
#endif
#endif
