/* afb200_resample.h -- the resampler: band-limited sample-rate conversion by a windowed-sinc table interpolated at every
 * output position.  Replaces src/dsp/resample_algorithm.h (src/dsp/resample_algorithm.c).
 *
 * Per output i of a call: t = (float)(i / ratio) (the division in double), n = floorf(t); the left taps x[n], x[n-1], ...
 * take table phase min(1, ratio) * (t - n), the right taps x[n+1], x[n+2], ... the complementary phase, each weight read
 * from the table with linear interpolation between neighbouring entries.  The table is
 * rollOff * sinc(rollOff * x) on x = linspace(0, zeroNum, zeroNum * 2^nbit + 1) times the right half of a symmetric
 * window, scaled by the ratio when the ratio is below 1.
 *
 * Differences from the reference, all on purpose (each refusal returns 0 from resampleObj_resample with a message in
 * afb200_lastError() and leaves the output untouched):
 *   - resampleObj_newWithWindow returns -2 when zeroNum * 2^nbit + 1 exceeds AFB200_RESAMPLE_MAX_TABLE entries (the
 *     reference overflows int above 2^31 entries);
 *   - a window type above Tukey is refused by resampleObj_newWithWindow with -1 (the reference dereferences a NULL
 *     window);
 *   - resampleObj_resample refuses ratio * 2^nbit < 1 (the tap stride is 0: the reference divides by zero);
 *   - in continue mode it refuses a rate pair with q <= 1 (upsampling by an integer, equal rates, or any ratio set by
 *     resampleObj_setSamplateRatio) and lengths where sourceLength * p overflows int; in one-shot mode, output lengths
 *     of 2^31 or more;
 *   - where the reference would read past the end of the input (the float position of the last output can round up to
 *     the clip length above 2^24 samples), the missing sample is taken as 0. */
#ifndef AFB200_RESAMPLE_H
#define AFB200_RESAMPLE_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    ResampleAlg_Polyphase = 0,
    ResampleAlg_Bandlimited,      /* declared by the reference, implemented by neither library */
} ResampleAlgType;

typedef enum {
    ResampleQuality_Best = 0,     /* Kaiser, zeroNum 64, nbit 9, beta 14.7696565, rollOff 0.9475937 */
    ResampleQuality_Mid,          /* Kaiser, zeroNum 32, nbit 9, beta 11.6625806, rollOff 0.8987969 */
    ResampleQuality_Fast,         /* Kaiser, zeroNum 16, nbit 9, beta 8.5555046, rollOff 0.85 */
} ResampleQualityType;

typedef struct OpaqueResample *ResampleObj;

/* largest table: 2^22 + 1 floats (16 MB); every preset uses 2^15 + 1 or fewer */
#define AFB200_RESAMPLE_MAX_TABLE ((1 << 22) + 1)

/* src :59-97.  qualType NULL: Best.  isScale / isContinue NULL: 0.  Returns 0.  Needs no GPU. */
int resampleObj_new(ResampleObj *resampleObj, ResampleQualityType *qualType, int *isScale, int *isContinue);

/* src :107-211.  NULL or out-of-range arguments take their defaults: zeroNum <= 0 -> 64; nbit outside 1 .. 29 -> 9;
 * winType <= Rect -> Hann; value < 0 ignored, and a value of 0 becomes 5 for Kaiser and 2.5 for Gauss (Tukey takes it as
 * its taper, 0 = Rect); rollOff outside (0, 1] -> 0.945.  The object starts at 32000 -> 16000 (ratio 0.5, p 1, q 2).
 * Returns 0, -1 (window type above Tukey, or out of memory) or -2 (table longer than AFB200_RESAMPLE_MAX_TABLE). */
int resampleObj_newWithWindow(ResampleObj *resampleObj,
                              int *zeroNum, int *nbit,
                              WindowType *winType, float *value,
                              float *rollOff,
                              int *isScale,
                              int *isContinue);

/* src :219-251: one-shot floorf(dataLength * ratio) (float product); continue mode with q > 1: (dataLength - dataLength % q)
 * * p / q, else 0 */
int resampleObj_calDataLength(ResampleObj resampleObj, int dataLength);

/* src :253-301: p / q = targetRate / sourceRate reduced by their gcd, ratio = targetRate / (float)sourceRate.  When the
 * ratio changes and the old or the new ratio is below 1, the table is divided by the old ratio (when below 1) and then
 * multiplied by the new one (when below 1), in float, in place: its last bits carry the object's history.  Equal or
 * non-positive rates change nothing. */
void resampleObj_setSamplate(ResampleObj resampleObj, int sourceRate, int targetRate);
/* src :303-332: the same for an arbitrary ratio; p = q = 0.  A negative ratio is ignored. */
void resampleObj_setSamplateRatio(ResampleObj resampleObj, float ratio);
/* src :334-341 */
void resampleObj_enableContinue(ResampleObj resampleObj, int flag);

/* src :350-403.  dataArr2 holds resampleObj_calDataLength(dataLength1) floats; the result is ADDED to what it holds, and
 * with isScale the sums are then divided by sqrtf(ratio).  Continue mode drops the last dataLength1 % q samples of each
 * call, as the reference does (its tail carry only starts from a non-empty tail, which it never creates).  Returns the
 * number of outputs, 0 on a refusal. */
int resampleObj_resample(ResampleObj resampleObj, float *dataArr1, int dataLength1, float *dataArr2);

void resampleObj_free(ResampleObj resampleObj);
void resampleObj_debug(ResampleObj resampleObj);     /* no-op, as in the reference */

#ifdef __cplusplus
}
#endif
#endif
