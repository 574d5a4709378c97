/* afb200_st.h -- the two Stockwell transforms of one 2^radix2Exp clip.
 *   ST:  per frequency bin i a Gaussian-windowed inverse FFT of the clip's spectrum, rows x N complex values.
 *   FST: the fast (dyadic) S-transform: the centred spectrum cut into a dyadic partition whose segments are
 *        inverse-transformed, then expanded to one N-column row per frequency.
 * Replaces src/st_algorithm.h:14-24 (src/st_algorithm.c) and src/fst_algorithm.h:14-20 (src/fst_algorithm.c).
 *
 * Differences from the reference, all on purpose:
 *   - no (N/2+1) x N table is built: ST evaluates its Gaussian in the kernel from one float per bin, FST maps each row to
 *     its partition segment in closed form (the reference tabulates 537 MB of floats / ints at 2^14);
 *   - stObj_new and fstObj_new return -2 with a message for radix2Exp > 14 (one clip's full-band output is 2.1 GB per
 *     plane at 2^15, and the reference's tables 2 GB); stObj_new returns -1 for radix2Exp < 1;
 *   - ST bin 0 writes an imaginary row of 0 where the reference leaves the caller's memory as it was (its Python
 *     binding passes zeros, so it sees the same result);
 *   - stObj_useBinArr accepts lists longer than N (the reference copies them into an N-int buffer and overruns it). */
#ifndef AFB200_ST_H
#define AFB200_ST_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueST *STObj;
typedef struct OpaqueFST *FSTObj;

/* src/st_algorithm.c:41-113.  Bins minIndex..maxIndex; min >= max, min < 0 or max > N/2 select 0..N/2.  factor / norm:
 * NULL or <= 0 means 1.  Returns 0, -1 (radix2Exp < 1) or -2 (radix2Exp > 14).  Needs no GPU. */
int stObj_new(STObj *stObj, int radix2Exp, int minIndex, int maxIndex, float *factor, float *norm);

/* :115-131: any order, repeats allowed; the whole list is ignored when one bin lies outside [0, N/2] */
void stObj_useBinArr(STObj stObj, int *binArr, int length);
/* :134-146: the Gaussian's factor and norm, taken as given */
void stObj_setValue(STObj stObj, float factor, float norm);

/* :152-208: dataArr N samples -> mRealArr / mImageArr binLength x N.  Bin 0: the clip's mean, imaginary row 0.  On
 * failure (no GPU, ...) the outputs are left untouched and afb200_lastError() holds the message. */
void stObj_st(STObj stObj, float *dataArr, float *mRealArr, float *mImageArr);

void stObj_free(STObj stObj);                 /* :258-297 */

/* src/fst_algorithm.c:49-106.  Returns 0, -1 (radix2Exp < 3) or -2 (radix2Exp > 14).  Needs no GPU. */
int fstObj_new(FSTObj *fstObj, int radix2Exp);

/* :113-280: dataArr N samples -> rows minIndex..maxIndex, each N columns.  minIndex < 0 becomes 0, maxIndex > N/2
 * becomes N/2; if then min > max, rows 0..N/2. */
void fstObj_fst(FSTObj fstObj, float *dataArr, int minIndex, int maxIndex, float *mRealArr, float *mImageArr);

void fstObj_free(FSTObj fstObj);              /* :412-468 */

#ifdef __cplusplus
}
#endif
#endif
