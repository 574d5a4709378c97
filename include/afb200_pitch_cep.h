/* afb200_pitch_cep.h -- pitch by the cepstrum.  Replaces include/mir/_pitch_cep.h (src/mir/_pitch_cep.c).
 *
 * Parameters (pitchCEPObj_new, :77-166, and __pitchCEPObj_initData, :195-237), with n = 2^radix2Exp:
 *   - minIndex = roundf(samplate / highFre) and maxIndex = roundf(samplate / lowFre), float quotients (:219-220);
 *   - windowType is taken only when windowType <= Window_Hamm (Rect, Hann, Hamm); any other keeps Hamm (:127-131).
 * Per frame t (samples t*slideLength .. +n-1), __pitchCEPObj_calCep (:381-447):
 *   1. the frame times the window, zero-padded to 2n samples;
 *   2. c = IFFT_2n(logf(|FFT_2n(x)|^2)) on all 2n bins, |X|^2 = re*re + im*im in float (__vcsquare, __vlog); the
 *      IFFT divides by 2n (src/dsp/fft_algorithm.c:612-619);
 *   3. util_peakPick (src/util/flux_util.c:783): __vmax's first maximum of c over minIndex .. maxIndex of the 2n-entry
 *      row; freArr[t] = samplate / (index + 1) (:470-473), the reference's own off-by-one.  A NaN first value stays
 *      the maximum: an all-zero frame (log 0 = -inf, then inf - inf) or a frame holding a NaN gives
 *      samplate / (minIndex + 1).
 *
 * Streaming (isContinue, __pitchCEPObj_dealData, :239-358): the samples that did not complete a hop are carried to the
 * next call, and with slideLength > n the carry is negative, a count of samples of the next call to skip;
 * calTimeLength (:168-193) adds the carry.  This is the bookkeeping of PitchPEF and PitchYIN, reproduced exactly.
 *
 * Differences from the reference, on purpose (each refusal records a message in afb200_lastError() and leaves
 * *pitchCEPObj NULL):
 *   - radix2Exp above AFB200_PITCH_CEP_MAX_EXP returns -2: one frame's 2n-point transform is held in shared memory;
 *   - maxIndex > 2n - 1 returns -3: the reference's peak search reads past the row (:471), for example at samplate
 *     32000 and lowFre 32 with radix2Exp 8;
 *   - maxIndex < minIndex returns -3: an empty lag range, for example lowFre above the default highFre;
 *   - at radix2Exp 1 the default slideLength n/4 would be 0, where the reference divides by zero; this library uses 1;
 *   - enableDebug only stores the flag. */
#ifndef AFB200_PITCH_CEP_H
#define AFB200_PITCH_CEP_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_PITCH_CEP_MAX_EXP 14

typedef struct OpaquePitchCEP *PitchCEPObj;

/* src :77-166.  Each pointer may be NULL (its default).  samplate outside (0, 196000]: 32000; lowFre below 27: 32;
 * highFre NULL: 2000; highFre not in (lowFre, samplate/2), integer samplate/2: lowFre 32 and highFre 2000; radix2Exp
 * outside 1 .. 30: 12; windowType above Window_Hamm: Hamm; slideLength <= 0: n/4; isContinue: 0.  Returns 0, or
 * -2 / -3 (above).  Needs no GPU. */
int pitchCEPObj_new(PitchCEPObj *pitchCEPObj,
                    int *samplate, float *lowFre, float *highFre,
                    int *radix2Exp, int *slideLength, WindowType *windowType,
                    int *isContinue);

/* src :168-193: with the streaming carry added when isContinue, 0 below n samples, else (length - n) / slideLength + 1 */
int pitchCEPObj_calTimeLength(PitchCEPObj pitchCEPObj, int dataLength);

/* src :360-379: freArr holds pitchCEPObj_calTimeLength(dataLength) floats (taken before the call); untouched when that
 * is 0 */
void pitchCEPObj_pitch(PitchCEPObj pitchCEPObj, float *dataArr, int dataLength,
                       float *freArr);

/* src :476-479: only the flag is stored */
void pitchCEPObj_enableDebug(PitchCEPObj pitchCEPObj, int isDebug);

void pitchCEPObj_free(PitchCEPObj pitchCEPObj);

#ifdef __cplusplus
}
#endif
#endif
