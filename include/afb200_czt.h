/* afb200_czt.h -- chirp z-transform.  Replaces include/dsp/czt_algorithm.h (src/dsp/czt_algorithm.c).
 *
 * An object of radix2Exp makes the N = 2^radix2Exp point CZT
 *   X[k] = sum_{n<N} x[n] A^-n W^(nk),  A = e^(2 pi i lowW),  W = e^(-2 pi i (highW - lowW) / N),  k < N,
 * the zoom spectrum of N bins spread over [lowW, highW) of the normalised frequency, through M = 2N point transforms
 * (Bluestein).  The chirp tables are the reference's float32 tables, built on the host with the same float expressions
 * and the C library's cosf / sinf (src :114-161); they set the accuracy (at radix2Exp 12 about 6e-5 of the exact CZT
 * for the band (0.15, 0.25) and 6e-4 for (0, 1)).
 *
 * Differences from the reference, on purpose (each refusal records a message in afb200_lastError()):
 *   - radix2Exp < 0 returns -1 and radix2Exp > AFB200_CZT_MAX_EXP returns -2, leaving *cztObj NULL: the M-point
 *     transforms run in one CTA's shared memory;
 *   - cztObj_czt with both input planes NULL leaves the outputs untouched. */
#ifndef AFB200_CZT_H
#define AFB200_CZT_H
#include "afb200_types.h"
#ifdef __cplusplus
extern "C" {
#endif

#define AFB200_CZT_MAX_EXP 13

typedef struct OpaqueCZT *CZTObj;

/* src :50-80.  The tables start with the band (0, 1).  Returns 0, or -1 / -2 (above).  Needs no GPU. */
int cztObj_new(CZTObj *cztObj, int radix2Exp);

/* src :82-89, 163-257.  realArr1 / imageArr1: N samples each, either may be NULL (a real-only or imaginary-only input).
 * realArr3 / imageArr3 receive M = 2N values: [0, N) the CZT, [N, 2N) the inverse transform of the convolution at those
 * indices, not multiplied by the chirp (as the reference leaves them).  A valid band (0 <= lowW < highW <= 1) replaces
 * the object's tables; any other band keeps the tables of the last valid one. */
void cztObj_czt(CZTObj cztObj, float *realArr1, float *imageArr1,
                float lowW, float highW,
                float *realArr3, float *imageArr3);

void cztObj_free(CZTObj cztObj);

#ifdef __cplusplus
}
#endif
#endif
