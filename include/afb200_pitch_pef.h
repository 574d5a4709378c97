/* afb200_pitch_pef.h -- pitch by the pitch estimation filter (PEF).  Replaces include/mir/_pitch_pef.h
 * (src/mir/_pitch_pef.c).
 *
 * With n = 2^radix2Exp (the frame), tables built once per object, in float as the reference builds them
 * (__pitchPEFObj_initData, :428-522, and __pitchPEFObj_calEstimateFilter, :696-785):
 *   - window = window_calFFTWindow(windowType, n);
 *   - lin = linspace(0, samplate/2, n+1), with the integer samplate/2;
 *   - fre1 = cutFre when samplate/2 > cutFre, else samplate/2 - 1 (integers); log = 10^linspace(1, log10f(fre1), 2n);
 *   - minIndex / maxIndex: the log points nearest to lowFre / highFre, by the reference's single loop over i = 1 ..
 *     2n-1: the first log[i] above highFre ends it (maxIndex = i, or i-1 when log[i-1] is at least as near), and until
 *     then the first log[i] above lowFre sets minIndex the same way.  minIndex stays -1 and maxIndex 0 when the loop
 *     never gets there;
 *   - bandWidth[j] = (log[j+1] - log[j-1]) / (4n), j = 1 .. 2n-2; both ends copy their neighbour;
 *   - q = 10^linspace(log10f(beta), log10f(alpha+beta), n), h = 1 / (gamma - cosf(2 pi q)); d = the widths of the
 *     intervals around each q (the midpoints, clamped to the ends); det = sum(d h) / sum(d) (double sums rounded to
 *     float); filter = h - det; filterPadNum P = #{q < 1}.  The reference correlates at xcorrFFTLength = 8n (P > 0) or
 *     4n (P = 0).
 * Per frame t (samples t*slideLength .. +n-1, no padding), :258-382 and __pitchPEFObj_dealResult, :384-426:
 *   1. x = frame * window, zero-padded to 2n; power[k] = |FFT_2n(x)[k]|^2, k = 0 .. n;
 *   2. s[P + i] = interp(power, lin -> log[i]) * bandWidth[i], i < 2n, with __vinterp_linear
 *      (src/vector/flux_vectorOp.c:580): y1 + (x - x1)(y2 - y1)/(x2 - x1) in float, power[n] beyond the last grid point;
 *      s[0 .. P-1] = 0;
 *   3. c = IFFT(FFT(s) conj(FFT(filter))): the circular cross-correlation c[k] = sum_j filter[j] s[j + k];
 *   4. len = maxIndex + 1 when maxIndex < 2n + P - 1, else 2n + P - 1; the reference stitches c[-len .. -1] and
 *      c[0 .. len] into one buffer b and takes util_peakPick's one peak over [minIndex, maxIndex] of b + maxIndex + 1
 *      (src/util/flux_util.c:783), which is __vmax's first maximum.  That is the lag k in minIndex .. maxIndex with
 *      the first maximum of c[k + maxIndex + 1 - len];
 *   5. freArr[t] = log[minIndex + that offset].
 * In the unclipped case (len = maxIndex + 1) step 4 is the first arg-max of c over the lags minIndex .. maxIndex.
 * The clipped case needs P = 0 and maxIndex = 2n - 1: the lags shift by one and the last one reads past the stitched
 * buffer, a value left over from earlier work; this library refuses it (below).
 *
 * Streaming (isContinue, :524-656): the samples that did not complete a hop are carried to the next call, and with
 * slideLength > n the carry is negative, a count of samples of the next call to skip; calTimeLength adds the carry.
 * This is the bookkeeping of the other streaming objects (STFT, CQT, Spectrogram), reproduced exactly.
 *
 * pitchPEFObj_setFilterParams (:685-694) recomputes the filter from the alpha, beta and gamma the object already holds
 * and never stores the new values, so it changes nothing; here it does nothing.
 *
 * Differences from the reference, on purpose (each refusal records a message in afb200_lastError() and leaves
 * *pitchPEFObj NULL):
 *   - radix2Exp above AFB200_PITCH_PEF_MAX_EXP returns -2: one frame's transforms are held in shared memory;
 *   - minIndex < 0 or maxIndex <= minIndex returns -3: the lag range is empty or starts before lag 0 (for example
 *     highFre >= fre1, or lowFre and highFre between the same two log points);
 *   - the clipped case of step 4 (P = 0, which needs beta >= 1, and maxIndex = 2n - 1) returns -4;
 *   - at radix2Exp 1 the default slideLength n/4 would be 0, where the reference divides by zero; this library uses 1. */
#ifndef AFB200_PITCH_PEF_H
#define AFB200_PITCH_PEF_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_PITCH_PEF_MAX_EXP 13

typedef struct OpaquePitchPEF *PitchPEFObj;

/* src :106-231.  Each pointer may be NULL (its default).  samplate outside (0, 196000]: 32000; lowFre below 27: 32;
 * highFre not in (lowFre, samplate/2), integer samplate/2: lowFre 32 and highFre 2000; cutFre below highFre: highFre
 * (default 4000); radix2Exp outside 1 .. 30: 12; windowType: Hamming; alpha <= 0: 10; beta <= 0: 0.5; gamma <= 1: 1.8;
 * slideLength <= 0: n/4; isContinue: 0.  Returns 0, or -2 / -3 / -4 (above).  Needs no GPU. */
int pitchPEFObj_new(PitchPEFObj *pitchPEFObj,
                    int *samplate, float *lowFre, float *highFre, float *cutFre,
                    int *radix2Exp, int *slideLength, WindowType *windowType,
                    float *alpha, float *beta, float *gamma,
                    int *isContinue);

/* src :658-683: with the streaming carry added when isContinue, 0 below n samples, else (length - n) / slideLength + 1 */
int pitchPEFObj_calTimeLength(PitchPEFObj pitchPEFObj, int dataLength);

/* src :685-694: changes nothing (above) */
void pitchPEFObj_setFilterParams(PitchPEFObj pitchPEFObj, float alpha, float beta, float gamma);

/* src :233-256: freArr holds pitchPEFObj_calTimeLength(dataLength) floats (taken before the call); untouched when that
 * is 0 */
void pitchPEFObj_pitch(PitchPEFObj pitchPEFObj, float *dataArr, int dataLength, float *freArr);

/* src :787-790: the reference only stores the flag; nothing here reads it */
void pitchPEFObj_enableDebug(PitchPEFObj pitchPEFObj, int isDebug);

void pitchPEFObj_free(PitchPEFObj pitchPEFObj);

#ifdef __cplusplus
}
#endif
#endif
