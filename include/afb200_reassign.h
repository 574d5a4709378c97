/* afb200_reassign.h -- time-frequency reassignment object: drop-in for src/reassign_algorithm.h:26-55
 * (same names, argument meaning and defaults). */
#ifndef AFB200_REASSIGN_H
#define AFB200_REASSIGN_H

#include "afb200_types.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueReassign *ReassignObj;

/* reassign_algorithm.c:83-186.  Defaults: radix2Exp 12, samplate 32000, hann, slideLength fftLength/4, Reassign_All,
 * thresh 0.001, no padding.  `isContinue` is accepted and ignored, as in the reference (:100, :152). */
int reassignObj_new(ReassignObj *reassignObj, int radix2Exp, int *samplate, WindowType *windowType, int *slideLength,
                    ReassignType *reType, float *thresh, int *isPadding, int *isContinue);
int reassignObj_calTimeLength(ReassignObj reassignObj, int dataLength);          /* :188-191 */
void reassignObj_setResultType(ReassignObj reassignObj, int type);               /* :194-197  0 complex, 1 amplitude -> mRealArr1 */
void reassignObj_setOrder(ReassignObj reassignObj, int order);                    /* :200-203  >= 1 */
/* :212-262.  Planes [timeLength x (fftLength/2+1)].  Reassign_All / Fre / Time: the reassigned spectrum is ADDED to
 * mRealArr1 / mImageArr1 (callers pass zeros) and mRealArr2 / mImageArr2 (may be NULL) receive the plain half
 * spectrum S_h; Reassign_None: mRealArr1 / mImageArr1 = S_h. */
void reassignObj_reassign(ReassignObj reassignObj, float *dataArr, int dataLength, float *mRealArr1, float *mImageArr1,
                          float *mRealArr2, float *mImageArr2);
void reassignObj_free(ReassignObj reassignObj);

/* additive: `batch` clips of dataLength samples, planes [batch x T x (fftLength/2+1)]; memKind AFB200_MEM_HOST or
 * AFB200_MEM_DEVICE (asynchronous on `stream`).  Same accumulate-into semantics as above. */
int reassignObj_reassignBatch(ReassignObj reassignObj, const float *data, int dataLength, int batch, float *mRealArr1,
                              float *mImageArr1, float *mRealArr2, float *mImageArr2, int memKind, void *stream);

#ifdef __cplusplus
}
#endif
#endif
