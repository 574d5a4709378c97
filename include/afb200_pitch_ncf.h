/* afb200_pitch_ncf.h -- pitch by the normalised correlation function.  Replaces include/mir/_pitch_ncf.h
 * (src/mir/_pitch_ncf.c).
 *
 * Parameters (pitchNCFObj_new, :77-164, and __pitchNCFObj_initData, :193-235), with n = 2^radix2Exp:
 *   - minIndex = roundf(samplate / highFre) and maxIndex = roundf(samplate / lowFre), float quotients (:217-218).
 * Per frame t (samples t*slideLength .. +n-1), __pitchNCFObj_calCorr (:380-467):
 *   1. the frame times the window (any windowType; Rect leaves it as it is), zero-padded to 2n samples;
 *   2. r = IFFT_2n(|FFT_2n(x)|^2), |X|^2 = re*re + im*im in float (__vcsquare); the IFFT divides by 2n
 *      (src/dsp/fft_algorithm.c:612-619), so r[k] = sum_m x[m] x[m+k];
 *   3. r times the float (float)(1.0/sqrtf(2n)) (:454); rms = sqrtf(r[0]); the lags minIndex .. maxIndex times the
 *      float (float)(1.0/rms) (:460-465).  Row slot j holds r[j+1]/rms for j = minIndex-1 .. maxIndex-1;
 *      slot maxIndex is never written and stays 0 (the row is calloc'd);
 *   4. util_peakPick (src/util/flux_util.c:783): __vmax's first maximum over slots minIndex .. maxIndex, so lags
 *      minIndex+1 .. maxIndex against a 0 at slot maxIndex, which wins when every correlation in range is negative;
 *      freArr[t] = samplate / (index + 1) (:490-493).  A NaN first slot stays the maximum: an all-zero frame
 *      (0/0) or a frame holding a NaN gives samplate / (minIndex + 1).
 *
 * Streaming (isContinue, __pitchNCFObj_dealData, :237-356): the samples that did not complete a hop are carried to the
 * next call, and with slideLength > n the carry is negative, a count of samples of the next call to skip;
 * calTimeLength (:166-191) adds the carry.  This is the bookkeeping of PitchPEF and PitchYIN, reproduced exactly.
 *
 * Differences from the reference, on purpose (each refusal records a message in afb200_lastError() and leaves
 * *pitchNCFObj NULL):
 *   - radix2Exp above AFB200_PITCH_NCF_MAX_EXP returns -2: one frame's 2n-point transform is held in shared memory;
 *   - maxIndex >= n returns -3: the reference copies 2 maxIndex + 1 floats into its 2n-float buffer (:456-457), a heap
 *     overflow, for example at samplate 32000 and lowFre 32 with radix2Exp 9;
 *   - minIndex < 1 returns -3: the reference passes a negative size to memset (:462), for example at samplate below
 *     1000 with the default highFre;
 *   - maxIndex < minIndex returns -3: an empty lag range, for example lowFre above the default highFre;
 *   - at radix2Exp 1 the default slideLength n/4 would be 0, where the reference divides by zero; this library uses 1;
 *   - slot maxIndex is 0 in every call.  The reference's peak pick writes NaN around the peak it found (:797) into
 *     rows that a later call with a similar frame count reuses, so there slot maxIndex can hold NaN left by an
 *     earlier call, and the reference then ignores it;
 *   - enableDebug only stores the flag. */
#ifndef AFB200_PITCH_NCF_H
#define AFB200_PITCH_NCF_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_PITCH_NCF_MAX_EXP 14

typedef struct OpaquePitchNCF *PitchNCFObj;

/* src :77-164.  Each pointer may be NULL (its default).  samplate outside (0, 196000]: 32000; lowFre below 27: 32;
 * highFre NULL: 2000; highFre not in (lowFre, samplate/2), integer samplate/2: lowFre 32 and highFre 2000; radix2Exp
 * outside 1 .. 30: 12; windowType: Rect; slideLength <= 0: n/4; isContinue: 0.  Returns 0, or -2 / -3 (above).
 * Needs no GPU. */
int pitchNCFObj_new(PitchNCFObj *pitchNCFObj,
                    int *samplate, float *lowFre, float *highFre,
                    int *radix2Exp, int *slideLength, WindowType *windowType,
                    int *isContinue);

/* src :166-191: with the streaming carry added when isContinue, 0 below n samples, else (length - n) / slideLength + 1 */
int pitchNCFObj_calTimeLength(PitchNCFObj pitchNCFObj, int dataLength);

/* src :358-378: freArr holds pitchNCFObj_calTimeLength(dataLength) floats (taken before the call); untouched when that
 * is 0 */
void pitchNCFObj_pitch(PitchNCFObj pitchNCFObj, float *dataArr, int dataLength,
                       float *freArr);

/* src :496-499: only the flag is stored */
void pitchNCFObj_enableDebug(PitchNCFObj pitchNCFObj, int isDebug);

void pitchNCFObj_free(PitchNCFObj pitchNCFObj);

#ifdef __cplusplus
}
#endif
#endif
