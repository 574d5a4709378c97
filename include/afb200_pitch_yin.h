/* afb200_pitch_yin.h -- pitch by YIN.  Replaces include/mir/_pitch_yin.h (src/mir/_pitch_yin.c).
 *
 * Parameters (pitchYINObj_new, :87-195), with n = 2^radix2Exp and A = autoLength:
 *   - diffLength = n - A; minIndex = floorf(samplate / highFre) and maxIndex = ceilf(samplate / lowFre), in float;
 *     maxIndex is clamped to diffLength - 1; yinLength = maxIndex - minIndex + 1; thresh = 0.1.
 * Per frame t (samples t*slideLength .. +n-1, no window, no padding), __pitchYINObj_calDiff (:350-453):
 *   1. c = IFFT_n(FFT_n(x) FFT_n(y)) (a plain complex product, __vcmul; the IFFT divides by n) with y[j] = x[A - j] for
 *      j <= A and 0 beyond; r[k] = c[A + k], set to 0 where fabs(r[k]) < 1e-6 (in double).  No product wraps for
 *      k <= n - 1 - A, so r[k] = sum_{m=0..A} x[m] x[m+k], A + 1 terms (:361-385);
 *   2. E = the float32 running sum of x^2 in sample order; e2[j] = E[A + j] - E[j] (A terms), set to 0 where
 *      fabs(e2[j]) < 1e-6 (:387-410);
 *   3. d[j] = e2[0] + e2[j] - 2 r[j] (:413-415);
 *   4. mean[k] = (float32 running sum of d[1 .. k+1]) / (k+1), a float division (:425-441);
 *      yin[k] = d[minIndex + k] / (mean[minIndex - 1 + k] + 1e-16), k < yinLength: 1e-16 is a double, so the division
 *      is done in double and rounded to float (:443-453);
 *   5. offset[j] = -num / (2 den + 1e-16) in double, num = (y[j+1] - y[j-1]) / 2 and den = (y[j-1] + y[j+1] - 2 y[j])
 *      / 2 in float, j = 1 .. yinLength-2, kept where |offset| <= 1 and 0 otherwise and at both ends
 *      (__pitchYINObj_calInterp, :462-503);
 *   6. a trough at j is j = 0 with y[0] < y[1] and y[0] < thresh, or y[j] <= y[j+1], y[j] < y[j-1] and y[j] < thresh,
 *      j < yinLength - 1.  For the first one, freArr[t] = samplate / (minIndex + j + offset[j]) in float and
 *      valueArr1[t] = y[j]; with no trough neither is written (the caller's values stay).  valueArr2[t] = __vmin of
 *      the whole row (its first minimum, `min > v`: a NaN first value stays the minimum), when valueArr2 is not NULL
 *      (__pitchYINObj_dealResult, :541-583);
 *   7. every trough of the frame, in order, goes into row t of mTroughArr (y[j]) and mFreArr (its frequency), rows of
 *      yinLength/2 + 1 floats, and their count into lenArr[t] (:585-625).
 *
 * Streaming (isContinue, __pitchYINObj_dealData, :791-938): the samples that did not complete a hop are carried to the
 * next call, and with slideLength > n the carry is negative, a count of samples of the next call to skip;
 * calTimeLength (:720-745) adds the carry.  This is the bookkeeping of the other streaming objects (STFT, CQT,
 * Spectrogram, PitchPEF), reproduced exactly.
 *
 * Differences from the reference, on purpose (each refusal records a message in afb200_lastError() and leaves
 * *pitchYINObj NULL):
 *   - radix2Exp above AFB200_PITCH_YIN_MAX_EXP returns -2: one frame's transform and running sums are held in shared
 *     memory;
 *   - minIndex < 1 returns -3: the reference reads mMeanArr[-1] (a heap read before its buffer, :445), for example at
 *     samplate 2000 with the default highFre;
 *   - yinLength < 1 returns -3: maxIndex clamped below minIndex, for example with autoLength near n;
 *   - at radix2Exp 1 the default slideLength n/4 would be 0, where the reference divides by zero; this library uses 1;
 *   - the trough rows past lenArr[t] are 0, where the reference leaves values of earlier calls;
 *   - enableDebug only stores the flag: the reference prints per-frame tables. */
#ifndef AFB200_PITCH_YIN_H
#define AFB200_PITCH_YIN_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_PITCH_YIN_MAX_EXP 14

typedef struct OpaquePitchYIN *PitchYINObj;

/* src :87-195.  Each pointer may be NULL (its default).  samplate outside (0, 196000]: 32000; lowFre below 27: 27;
 * highFre NULL: 2094; highFre not in (lowFre, samplate/2), integer samplate/2: lowFre 27 and highFre 2093; radix2Exp
 * outside 1 .. 30: 12; slideLength <= 0: n/4; autoLength outside [0, n): n/2; isContinue: 0.  Returns 0, or -2 / -3
 * (above).  Needs no GPU. */
int pitchYINObj_new(PitchYINObj *pitchYINObj,
                    int *samplate, float *lowFre, float *highFre,
                    int *radix2Exp, int *slideLength, int *autoLength,
                    int *isContinue);

/* src :217-226: any thresh > 0 is taken (default 0.1) */
void pitchYINObj_setThresh(PitchYINObj pitchYINObj, float thresh);

/* src :720-745: with the streaming carry added when isContinue, 0 below n samples, else (length - n) / slideLength + 1 */
int pitchYINObj_calTimeLength(PitchYINObj pitchYINObj, int dataLength);

/* src :228-244: freArr and, when not NULL, valueArr1 and valueArr2 hold pitchYINObj_calTimeLength(dataLength) floats
 * (taken before the call); untouched when that is 0, and freArr / valueArr1 untouched in frames without a trough */
void pitchYINObj_pitch(PitchYINObj pitchYINObj, float *dataArr, int dataLength,
                       float *freArr, float *valueArr1, float *valueArr2);

/* src :246-263: the trough rows of the last pitchYINObj_pitch call that computed frames (timeLength x mLen floats each,
 * and timeLength counts), valid until the next call or pitchYINObj_free; returns mLen = yinLength/2 + 1.  Each pointer
 * may be NULL; before the first such call the arrays are NULL. */
int pitchYINObj_getTroughData(PitchYINObj pitchYINObj, float **mFreArr, float **mTroughArr, int **lenArr);

/* src :747-750: the reference prints per-frame tables; here only the flag is stored */
void pitchYINObj_enableDebug(PitchYINObj pitchYINObj, int isDebug);

void pitchYINObj_free(PitchYINObj pitchYINObj);

#ifdef __cplusplus
}
#endif
#endif
