/* afb200_wpt.h -- wavelet packet transform.  Replaces include/wpt_algorithm.h (src/wpt_algorithm.c).
 *
 * The step of DWTObj (afb200_dwt.h: periodic padding, valid convolution with loD / hiD, odd samples) splits every node
 * of the tree, level by level, (1 << num) - 1 splits with N = 2^radix2Exp.  Node i (breadth-first, the root is 0)
 * puts its low half in child 2i+1 and its high half in child 2i+2, swapped when i is even and non-zero.  coefArr
 * (N floats) is the last level, its 2^num nodes of N/2^num samples one after the other; mDataArr (2^num x N floats, may
 * be NULL) repeats node k of that level along time in row k.  Filters and refusals: afb200_dwt.h. */
#ifndef AFB200_WPT_H
#define AFB200_WPT_H
#include "afb200_dwt.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct OpaqueWPT *WPTObj;

/* src :54-135.  Same statuses as dwtObj_new. */
int wptObj_new(WPTObj *wptObj, int num, int radix2Exp, WaveletDiscreteType *waveletType, int *t1, int *t2);

/* src :144-274: coefArr N floats, mDataArr 2^num x N floats or NULL */
void wptObj_wpt(WPTObj wptObj, float *dataArr, float *coefArr, float *mDataArr);

void wptObj_free(WPTObj wptObj);

#ifdef __cplusplus
}
#endif
#endif
