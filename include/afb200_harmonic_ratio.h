/* afb200_harmonic_ratio.h -- harmonic ratio of framed audio.  Replaces include/mir/harmonicRatio_algorithm.h
 * (src/mir/harmonicRatio_algorithm.c).
 *
 * With W = 2^radix2Exp (the window) and N = 2W (the FFT), per frame t (samples t*slideLength .. +W-1, no padding):
 *   1. x = frame * Hamming(W) (window_calFFTWindow's periodic Hamming), zero-padded to N;
 *   2. r = IFFT_N(|FFT_N(x)|^2): the autocorrelation, divided by N as the reference's inverse FFT divides;
 *   3. E[j] = sum of x[m]^2 over m <= W-2-j;
 *   4. minIndex = (the first j in 2 .. maxLength where r[j] and r[j-1] have opposite signs, zeros included) - 1.  A
 *      frame without such a j keeps the minIndex of the last earlier frame of the same call that had one (0 when none);
 *   5. g[k] = r[j] / sqrtf(r[0] E[j] + 1e-16) for j = minIndex+1 .. maxLength-1 (the sum formed in double);
 *   6. the value is the first maximum of g, refined by the parabola through its neighbours unless it is the first or
 *      the last of g; 0 when g is empty.
 * Because r carries the 1/N of the inverse FFT, g is the normalised autocorrelation divided by sqrt(N).
 *
 * Differences from the reference, on purpose (each refusal records a message in afb200_lastError() and leaves
 * *harmonicRatioObj NULL):
 *   - radix2Exp above AFB200_HARMONIC_RATIO_MAX_EXP returns -2: one frame's transforms are held in shared memory;
 *   - a configuration with maxLength = 0 returns -3: radix2Exp = 0 (W = 1), or a samplate below 25 with the default
 *     lowFre.  The reference reads a power bin left over from the frame's spectrum there. */
#ifndef AFB200_HARMONIC_RATIO_H
#define AFB200_HARMONIC_RATIO_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_HARMONIC_RATIO_MAX_EXP 13

typedef struct OpaqueHarmonicRatio *HarmonicRatioObj;

/* src :52-155.  Each pointer may be NULL (its default).  samplate outside (0, 196000]: 32000; lowFre outside
 * (0, samplate/2), with the integer samplate/2: 25; radix2Exp outside 0 .. 29: the window of 2^11 samples; slideLength
 * <= 0: W/4.  maxLength = floorf(samplate / lowFre), at most W-1.  windowType is not read: the window is always Hamming,
 * as in the reference.  Returns 0, or -2 / -3 (above).  Needs no GPU. */
int harmonicRatioObj_new(HarmonicRatioObj *harmonicRatioObj,
                         int *samplate, float *lowFre,
                         int *radix2Exp, WindowType *windowType, int *slideLength);

/* src :157-170: 0 when dataLength < W, else (dataLength - W) / slideLength + 1 */
int harmonicRatioObj_calTimeLength(HarmonicRatioObj harmonicRatioObj, int dataLength);

/* src :172-287: valueArr holds harmonicRatioObj_calTimeLength(dataLength) floats; untouched when that is 0 */
void harmonicRatioObj_harmonicRatio(HarmonicRatioObj harmonicRatioObj, float *dataArr, int dataLength, float *valueArr);

void harmonicRatioObj_free(HarmonicRatioObj harmonicRatioObj);

#ifdef __cplusplus
}
#endif
#endif
