/* afb200_xcorr.h -- cross-correlation and autocorrelation of real sequences.  Replaces include/dsp/xcorr_algorithm.h
 * (src/dsp/xcorr_algorithm.c).
 *
 * With n = length and M = the smallest power of two >= 2n (util_ceilPowerTwo(2n)), vArr3 gets the 2n-1 values
 *   vArr3[n-1+m] = sum_k a[k+m] b[k],  m = -(n-1) .. n-1,
 * i.e. numpy.correlate(a, b, 'full'), computed as IFFT_M(FFT_M(a) conj(FFT_M(b))) with the inverse divided by M, as the
 * reference computes it.  b = NULL gives the autocorrelation, from |FFT_M(a)|^2.
 *
 * Differences from the reference, on purpose (each refusal records a message in afb200_lastError() and leaves vArr3
 * and *maxValue untouched):
 *   - length < 1 returns -1 (the reference reads outside its arrays there);
 *   - length > AFB200_XCORR_MAX_LENGTH returns -2 (the long path runs transforms of up to 2^20 points);
 *   - every call is computed as on a fresh object.  The reference copies only `length` samples into buffers it keeps
 *     for the next call with the same M, so a shorter later call correlates samples left over from the earlier one. */
#ifndef AFB200_XCORR_H
#define AFB200_XCORR_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_XCORR_MAX_LENGTH (1 << 19)

/* include/dsp/xcorr_algorithm.h:14-18 */
typedef enum {
    XcorrNormal_None = 0,
    XcorrNormal_Coeff,
} XcorrNormalType;

typedef struct OpaqueXcorr *XcorrObj;

/* src :40-47.  Returns 0.  Needs no GPU. */
int xcorrObj_new(XcorrObj *xcorrObj);

/* src :49-115.  vArr1, vArr2 (NULL: autocorrelation): length floats; vArr3: 2*length-1 floats.  normType NULL means
 * XcorrNormal_Coeff, which divides every value by sqrtf(sum1 * sum2): each sum is the float of a double sum of the
 * float squares, the product is taken in float, and sum2 = sum1 for the autocorrelation.  A silent input with Coeff
 * gives NaN everywhere.  Returns the first index of the maximum of vArr3 (__vmax: a NaN vArr3[0] stays the maximum,
 * later NaNs are passed over) and stores that value in *maxValue when maxValue is not NULL.  vArr1 == NULL returns 0
 * and writes nothing; a refused call returns -1 / -2 (above), and -3 when the device work fails (no GPU, for one). */
int xcorrObj_xcorr(XcorrObj xcorrObj, float *vArr1, float *vArr2, int length,
                   XcorrNormalType *normType,
                   float *vArr3, float *maxValue);

void xcorrObj_free(XcorrObj xcorrObj);

#ifdef __cplusplus
}
#endif
#endif
