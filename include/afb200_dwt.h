/* afb200_dwt.h -- discrete wavelet transform.  Replaces include/dwt_algorithm.h (src/dwt_algorithm.c).
 *
 * With N = 2^radix2Exp, each of the num levels pads the current approximation periodically by decLength/2 samples on
 * each side, convolves it with loD and hiD (valid part) and keeps the odd samples.  coefArr (N floats) holds the last
 * approximation at the front and the details of level num-1 .. 0 behind it: level i's detail at
 * [N/2^(i+1), N/2^i).  mDataArr (num x N floats, may be NULL) repeats coefArr[2^i .. 2^(i+1)-1] along time in row
 * i-1 (i = 1 .. num); those indices are the reference's, exact for num = radix2Exp-1 and kept as they are otherwise.
 *
 * Filters (waveletType, t1, t2): WaveletDiscrete_Haar; Db t1 = 2-10, 20, 30; Sym t1 = 2-6, 8, 9; Bior t1.t2 = 1.1,
 * 1.3, 1.5, 2.2, 2.4, 2.6, 2.8, 3.1, 3.3, 3.5, 3.7, 3.9, generated from their definitions (gen/gen_wavelets.py).  The
 * other combinations the reference lists (db40, sym7, sym10, sym20, sym30, coif1-5, fk4-22, bior4.4, 5.5, 6.8, dmey)
 * are refused with -2 and a message in afb200_lastError().  Any unlisted combination is sym4, as in the reference.
 *
 * Differences from the reference, on purpose: radix2Exp above AFB200_WAVELET_MAX_EXP, and the refused filters above,
 * return -2 and leave *dwtObj NULL. */
#ifndef AFB200_DWT_H
#define AFB200_DWT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_WAVELET_MAX_EXP 20

typedef enum { WaveletDiscrete_Haar = 0, WaveletDiscrete_Db, WaveletDiscrete_Sym, WaveletDiscrete_Coif,
               WaveletDiscrete_FK, WaveletDiscrete_Bior, WaveletDiscrete_DMey } WaveletDiscreteType;

typedef struct OpaqueDWT *DWTObj;

/* src :55-144.  waveletType / t1 / t2 may be NULL: Sym, 4, 4.  radix2Exp non-zero outside 1 .. 30: -100; num outside
 * 1 .. radix2Exp-1: -1.  Needs no GPU. */
int dwtObj_new(DWTObj *dwtObj, int num, int radix2Exp, WaveletDiscreteType *waveletType, int *t1, int *t2);

/* src :178-306: coefArr N floats, mDataArr num x N floats or NULL */
void dwtObj_dwt(DWTObj dwtObj, float *dataArr, float *coefArr, float *mDataArr);

void dwtObj_free(DWTObj dwtObj);

#ifdef __cplusplus
}
#endif
#endif
