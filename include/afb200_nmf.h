/* afb200_nmf.h -- non-negative matrix factorisation V ~ W H.  Replaces include/classic/nmf.h (src/classic/nmf.c).
 *
 * V is n x m, W n x k and H k x m, all row-major float.  W and H are in/out: the caller initialises them (the
 * reference's Python binding uses arange(1, ...) for both).  Before the loop and after every iteration W is divided
 * column by column by its column norm: the p-norm for norm 1 or 2, the column maximum for any other norm; a zero entry
 * stays zero and a zero norm is not guarded against.  One iteration, with D = W H and eps = 1e-16f:
 *   type 0 (KL):        D2 = V / (D + eps), D3 = 1;
 *   type 1 (IS):        D2 = V / (D^2 + eps), D3 = 1 / (D + eps), the divisions in double;
 *   other (Euclidean):  D2 = V, D3 = D;
 *   H <- H * (W^T D2) / (W^T D3 + eps), then W <- W * (D2 H^T) / (D3 H^T + eps) with the new H and the same D2, D3.
 * Every product is rounded to float, accumulated in double and stored as float.  The loop stops after the iteration
 * where both ||W - W_prev||_2 and ||H - H_prev||_2 are below thresh (W after its normalisation), or after maxIter
 * iterations; each norm is the reference's: the squares of the float differences summed in float in index order, then
 * sqrtf. */
#ifndef AFB200_NMF_H
#define AFB200_NMF_H
#ifdef __cplusplus
extern "C" {
#endif

/* src :19-280.  Each pointer argument among maxIter, type, thresh and norm may be NULL: 300, 1 (IS), 1e-3, 0 (column
 * max).  The reference's header comment numbers the types differently; the code, followed here, decides.  Any k >= 1
 * runs.  Nothing is written when n, m or k is below 1 or an array is NULL (afb200_lastError() then says why).  Needs a
 * GPU: the iterations run on the device. */
void nmf(float *mDataArr, int nLength, int mLength, int k,
         float *wArr, float *hArr,
         int *maxIter, int *type, float *thresh,
         int *norm);

#ifdef __cplusplus
}
#endif
#endif
