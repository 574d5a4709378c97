/* afb200_hpss.h -- harmonic-percussive source separation by median filtering.  Replaces include/mir/hpss_algorithm.h
 * (src/mir/hpss_algorithm.c).
 *
 * Per clip: the STFT (fftLength N = 2^radix2Exp, hop N/4, no padding) gives mag = |X| per frame and bin of the half
 * spectrum (W = N/2 + 1 bins); mH is the median of mag over hOrder frames of the same bin, mP the median over pOrder
 * bins of the same frame, both windows centred and zero beyond the clip's frames and the spectrum's bins.  With
 * h1 = mH^2, p1 = mP^2 and v = max(h1 + p1, 1e-16), the harmonic part keeps h1 / v * mag and the percussive part
 * p1 / v * mag, each with the phase of X, and each is taken back to the time domain by the inverse STFT (window-weighted
 * overlap-add divided by the sum of the squared window).  An order of 1 makes that median 0 (as in the reference, whose
 * filter does not run then): hOrder 1 gives H = 0, pOrder 1 gives P = 0.
 *
 * Differences from the reference, all on purpose (each refusal returns with a message in afb200_lastError() and leaves
 * the outputs untouched):
 *   - a dataLength shorter than one frame is refused (the reference crashes there);
 *   - radix2Exp outside 2 .. 20 is refused (no hop of N/4 below 2^2, no STFT above 2^20);
 *   - an order above AFB200_HPSS_MAX_ORDER is refused. */
#ifndef AFB200_HPSS_H
#define AFB200_HPSS_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueHPSS *HPSSObj;

/* largest hOrder / pOrder: the time window of the largest order and 32 frames of 128 bins fill the 227 KB of shared
 * memory an H100 CTA can hold */
#define AFB200_HPSS_MAX_ORDER 383

/* src :40-94.  windowType NULL: Hamm.  hOrder / pOrder are taken only when > 0 and odd, else 21 / 31.  slideLength is
 * ignored: the hop is always fftLength / 4.  Returns 0.  Needs no GPU. */
int hpssObj_new(HPSSObj *hpssObj,
                int radix2Exp, WindowType *windowType, int *slideLength,
                int *hOrder, int *pOrder);

/* src :96-111: (T - 1) * fftLength / 4 + fftLength with T = the STFT's frame count (0 below one frame: 3 fftLength / 4) */
int hpssObj_calDataLength(HPSSObj hpssObj, int dataLength);

/* src :118-345.  hArr / pArr hold hpssObj_calDataLength(dataLength) floats each; each result is ADDED to what the buffer
 * holds before the inverse STFT's division by the window sum, as in the reference.  A NULL output is skipped. */
void hpssObj_hpss(HPSSObj hpssObj, float *dataArr, int dataLength, float *hArr, float *pArr);

void hpssObj_free(HPSSObj hpssObj);
void hpssObj_debug(HPSSObj hpssObj);     /* no-op, as in the reference */

#ifdef __cplusplus
}
#endif
#endif
