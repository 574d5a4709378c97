/* afb200_spectral.h -- spectral descriptors of a time-major spectrogram (centroid, flatness, rolloff, flux, ...).
 * Replaces src/feature/spectral_algorithm.h:16-81 (src/feature/spectral_algorithm.c, src/flux_spectral.c).
 *
 * Differences from the reference, all on purpose:
 *   - stateless: every call computes from its own input.  The reference caches the per-frame sum / centroid / spread /
 *     entropy / mean in the object and clears them only in setTimeLength / setEdge, so a second call on new data
 *     returned (or divided by) the first call's values;
 *   - step >= timeLength (flux / sd / sf / novelty) zeroes the timeLength frames; the reference's memset of `step`
 *     floats overruns the caller's array there;
 *   - spectralObj_new copies freBandArr (the reference borrows the pointer), and a frequency feature (rolloff, centroid,
 *     spread, skewness, kurtosis, slope, bandWidth, max, mean, var) fails with a message when it was NULL
 *     (the reference dereferences NULL). */
#ifndef AFB200_SPECTRAL_H
#define AFB200_SPECTRAL_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueSpectral *SpectralObj;

int spectralObj_new(SpectralObj *spectralObj, int num, float *freBandArr);   /* spectral_algorithm.c:57-92; -1 if num<2 */

/* :160-186: bins start..end; silently ignored unless 0 <= start < end <= num-1 */
void spectralObj_setEdge(SpectralObj spectralObj, int start, int end);
/* :188-218: takes ownership of the malloc'd / calloc'd indexArr (any order, repeats allowed); an index outside
 * 0..num-1 frees the array and leaves the edge unchanged, otherwise the previous list is freed */
void spectralObj_setEdgeArr(SpectralObj spectralObj, int *indexArr, int indexLength);
void spectralObj_setTimeLength(SpectralObj spectralObj, int timeLength);     /* :94-158 */

/* mDataArr / mSpecArr / mPhaseArr: timeLength x num; dataArr: timeLength.  Line numbers: src/flux_spectral.c. */
void spectralObj_flatness(SpectralObj spectralObj, float *mDataArr, float *dataArr);                  /* :21-55 */
/* :58-105; isExp default 0, type 0 sum | 1 mean (default 0) */
void spectralObj_flux(SpectralObj spectralObj, float *mDataArr, int step, float p, int isPostive, int *isExp, int *type,
                      float *dataArr);
void spectralObj_rolloff(SpectralObj spectralObj, float *mDataArr, float threshold, float *dataArr);   /* :107-146 */
void spectralObj_centroid(SpectralObj spectralObj, float *mDataArr, float *dataArr);                  /* :148-173 */
void spectralObj_spread(SpectralObj spectralObj, float *mDataArr, float *dataArr);                    /* :175-202 */
void spectralObj_skewness(SpectralObj spectralObj, float *mDataArr, float *dataArr);                  /* :204-231 */
void spectralObj_kurtosis(SpectralObj spectralObj, float *mDataArr, float *dataArr);                  /* :233-260 */
void spectralObj_entropy(SpectralObj spectralObj, float *mDataArr, int isNorm, float *dataArr);       /* :262-293 */
void spectralObj_crest(SpectralObj spectralObj, float *mDataArr, float *dataArr);                     /* :295-321 */
void spectralObj_slope(SpectralObj spectralObj, float *mDataArr, float *dataArr);                     /* :323-350 */
void spectralObj_decrease(SpectralObj spectralObj, float *mDataArr, float *dataArr);                  /* :352-376 */
void spectralObj_bandWidth(SpectralObj spectralObj, float *mDataArr, float p, float *dataArr);        /* :378-407 */
void spectralObj_rms(SpectralObj spectralObj, float *mDataArr, float *dataArr);                       /* :409-435 */
/* :794-823 with isPower = 0 (the input is squared); gamma <= 0 becomes 10 when isLog */
void spectralObj_energy(SpectralObj spectralObj, float *mDataArr, int isLog, float gamma, float *dataArr);
void spectralObj_hfc(SpectralObj spectralObj, float *mDataArr, float *dataArr);                       /* :439-458 */
void spectralObj_sd(SpectralObj spectralObj, float *mDataArr, int step, int isPostive, float *dataArr);   /* :461-492 */
void spectralObj_sf(SpectralObj spectralObj, float *mDataArr, int step, int isPostive, float *dataArr);   /* :495-526 */
void spectralObj_mkl(SpectralObj spectralObj, float *mDataArr, int type, float *dataArr);            /* :529-555 */
/* :557-629; frame 0 is 0 and frame 1 is left as the caller had it */
void spectralObj_pd(SpectralObj spectralObj, float *mSpecArr, float *mPhaseArr, float *dataArr);
void spectralObj_wpd(SpectralObj spectralObj, float *mSpecArr, float *mPhaseArr, float *dataArr);
void spectralObj_nwpd(SpectralObj spectralObj, float *mSpecArr, float *mPhaseArr, float *dataArr);
void spectralObj_cd(SpectralObj spectralObj, float *mSpecArr, float *mPhaseArr, float *dataArr);      /* :631-700 */
void spectralObj_rcd(SpectralObj spectralObj, float *mSpecArr, float *mPhaseArr, float *dataArr);
/* :703-720: ADDS the per-frame counts to dataArr[1..] (as the reference does); dataArr[0] = 0 */
void spectralObj_broadband(SpectralObj spectralObj, float *mDataArr, float threshold, float *dataArr);
/* :728-792; NULL methodType / dataType = Sub / Value */
void spectralObj_novelty(SpectralObj spectralObj, float *mDataArr, int step, float threshold,
                         SpectralNoveltyMethodType *methodType, SpectralNoveltyDataType *dataType, float *dataArr);
void spectralObj_eef(SpectralObj spectralObj, float *mDataArr, int isNorm, float *dataArr);   /* spectral_algorithm.c:781-815 */
void spectralObj_eer(SpectralObj spectralObj, float *mDataArr, int isNorm, float gamma, float *dataArr);   /* :818-852 */

/* statistics, spectral_algorithm.c:855-956: value and frequency per frame; var writes nothing with fewer than 2 bins */
void spectralObj_max(SpectralObj spectralObj, float *mDataArr, float *valueArr, float *freArr);
void spectralObj_mean(SpectralObj spectralObj, float *mDataArr, float *valueArr, float *freArr);
void spectralObj_var(SpectralObj spectralObj, float *mDataArr, float *valueArr, float *freArr);

void spectralObj_free(SpectralObj spectralObj);

#ifdef __cplusplus
}
#endif
#endif
