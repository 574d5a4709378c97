/* afb200_xxcc.h -- cepstral coefficients (rectify -> ortho DCT-II -> first ccNum).
 * Replaces src/feature/xxcc_algorithm.h:12-39 (src/feature/xxcc_algorithm.c). */
#ifndef AFB200_XXCC_H
#define AFB200_XXCC_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueXXCC *XXCCObj;

int xxccObj_new(XXCCObj *xxccObj, int num);                       /* xxcc_algorithm.c:32-62; -1 if num<2 */
void xxccObj_setTimeLength(XXCCObj xxccObj, int timeLength);      /* :64-89 */
/* :95-156.  mDataArr1: timeLength x num, mDataArr2: timeLength x mLength; silent return if mLength>num. */
void xxccObj_xxcc(XXCCObj xxccObj, float *mDataArr1, int mLength, CepstralRectifyType *rectifyType,
                  float *mDataArr2);
/* :168-296.  mDataArr1: timeLength x num; energyArr: timeLength (read unless energyType = Ignore);
 * mCoeArr / mDeltaArr1 / mDeltaArr2: timeLength x W, W = mLength (+1 when energyType = Append).
 * Defaults: deltaWindowLength 9 (odd >= 3), energyType Replace, rectifyType Log.  As in the reference the
 * delta FIR runs along the coefficient axis of each frame (util_delta, src/util/flux_util.c:803-815). */
void xxccObj_xxccStandard(XXCCObj xxccObj, float *mDataArr1, int mLength, float *energyArr,
                          int *deltaWindowLength, CepstralEnergyType *energyType,
                          CepstralRectifyType *rectifyType,
                          float *mCoeArr, float *mDeltaArr1, float *mDeltaArr2);
void xxccObj_free(XXCCObj xxccObj);

#ifdef __cplusplus
}
#endif
#endif
