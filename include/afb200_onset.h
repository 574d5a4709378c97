/* afb200_onset.h -- onset detection on a spectrogram.  Replaces include/mir/onset_algorithm.h (src/mir/onset_algorithm.c).
 *
 * Per clip of nLength frames x mLength bins (time-major):
 *   1. with filterOrder >= 2, a sliding max over bins of each frame, window [k - order/2, k - 1 + order - order/2]
 *      clipped to the frame;
 *   2. the novelty function of the object's type over the bins of indexArr (all bins when NULL), as the reference's
 *      spectral_* functions compute it (src/flux_spectral.c), on the filtered matrix; the phase types (PD, WPD, NWPD,
 *      CD, RCD) read the unfiltered phase mDataArr2.  The first `step` frames of FLUX / SD / SF are 0;
 *   3. evn -= min(evn), then evn /= max(evn) when that is > 0;
 *   4. peak picking: frame i is a point when evn[i] is the max of frames [i - preMax, i - 1 + postMax], evn[i] >=
 *      mean(frames [i - preAvg, i - 1 + postAvg]) + delta, and i is more than `wait` frames after the last point.
 *      The peak parameters come from the constructor (onsetObj_new below).
 * Of NoveltyParam only step, p, isPostive, isExp and type (FLUX / SD / SF / MKL) and threshold (BROADBAND) are read;
 * isNorm and gamma are accepted and unused, as in the reference.
 *
 * Differences from the reference, all on purpose (each refusal returns 0 points with a message in afb200_lastError()
 * and leaves the outputs untouched):
 *   - nLength or mLength below 1 is refused;
 *   - an indexArr entry outside [0, mLength), or an indexArr with indexLength < 1, is refused (the reference reads out
 *     of bounds);
 *   - a phase type without mDataArr2 is refused (the reference dereferences NULL);
 *   - a step above nLength is refused (the reference writes past evnArr);
 *   - frame 1 of PD / WPD / NWPD with step 1 is 0, and BROADBAND counts from 0: the reference keeps, or adds to, what
 *     evnArr held before the call.  With a zeroed evnArr (as the reference's Python binding passes) the results agree.
 * A filterOrder above mLength is accepted: the window is clipped to the frame, as in the reference. */
#ifndef AFB200_ONSET_H
#define AFB200_ONSET_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueOnset *OnsetObj;

/* src :58-133.  samplate NULL or <= 0: 32000; filterOrder NULL or <= 0: 1; type NULL: Novelty_Flux; slideLength < 1:
 * 512.  Peak parameters, each computed in double and floored as a float: preMax = 0.03 sr / slide, postMax = 1,
 * preAvg = 0.1 sr / slide, postAvg = 0.1 sr / slide + 1, wait = 0.03 sr / slide; delta = 0.07.  Returns 0.  Needs no
 * GPU. */
int onsetObj_new(OnsetObj *onsetObj, int nLength, int mLength, int slideLength,
                 int *samplate, int *filterOrder,
                 NoveltyType *type);

/* src :185-211.  mDataArr1 / mDataArr2: nLength x mLength; evnArr: nLength floats; pointArr: up to nLength ints, of
 * which the first (return value) are written.  param NULL: step 1, p 1, isPostive 1, the rest 0.  Returns the number of
 * points. */
int onsetObj_onset(OnsetObj onsetObj, float *mDataArr1, float *mDataArr2,
                   NoveltyParam *param, int *indexArr, int indexLength,
                   float *evnArr, int *pointArr);

void onsetObj_free(OnsetObj onsetObj);
/* src :405-415: the peak parameters and sizes, on stdout */
void onsetObj_debug(OnsetObj onsetObj);

#ifdef __cplusplus
}
#endif
#endif
