/* af_nmf.c -- nmf and nmfBatch of the C ABI (host C; compute = kernels/nmf.cu).  Interface spec:
 * include/classic/nmf.h, behaviour src/classic/nmf.c.  The matrices of a call flow through the shared staging path
 * (host pointers) or run in place (device pointers); the iterations of a chunk are queued without waiting. */
#include <string.h>
#include "../af_internal.h"

typedef struct { int n, m, k, maxIter, type, norm; float thresh; } NmfCall;

/* d[0] V nb x n x m, d[1] W nb x n x k, d[2] H nb x k x m, d[3] iters nb ints (or NULL) */
static int nmf_chunk(void *ctx, int nb, float *const *d, void *st) {
    const NmfCall *c = (const NmfCall *)ctx;
    AfNmfArgs a;
    memset(&a, 0, sizeof(a));
    a.V = d[0]; a.W = d[1]; a.H = d[2]; a.iters = (int *)d[3];
    a.n = c->n; a.m = c->m; a.k = c->k; a.batch = nb;
    a.maxIter = c->maxIter; a.type = c->type; a.norm = c->norm; a.thresh = c->thresh;
    return af_launch_nmf(&a, st);
}

int nmfBatch(const float *V, int batch, int n, int m, int k, float *W, float *H, const int *maxIter, const int *type,
             const float *thresh, const int *norm, int *iters, int memKind, void *stream) {
    af_clear_error();
    if (!V || !W || !H || batch < 1 || n < 1 || m < 1 || k < 1)
        return af_fail(-1, "nmfBatch: bad argument (V %p, W %p, H %p, batch %d, n %d, m %d, k %d)", (const void *)V,
                       (void *)W, (void *)H, batch, n, m, k);
    int rc = af_device_ready();
    if (rc) return rc;
    /* src :57-71; every type other than 0 (KL) and 1 (IS) is Euclidean (:208), and the kernels know it as 2 */
    const int tp = type ? *type : 1;
    NmfCall c = {n, m, k, maxIter ? *maxIter : 300, tp == 0 || tp == 1 ? tp : 2, norm ? *norm : 0,
                 thresh ? *thresh : 1e-3f};
    const AfPlane pl[4] = {{V, (size_t)n * m, AF_IN, 0}, {W, (size_t)n * k, AF_INOUT, 0}, {H, (size_t)k * m, AF_INOUT, 0},
                           {iters, 1, AF_OUT, 0}};
    AfPipe pipe;
    memset(&pipe, 0, sizeof(pipe));
    rc = af_run_batch(&pipe, memKind, stream, nmf_chunk, &c, pl, 4, batch, AF_PIPE_CHUNK_BYTES);
    af_pipe_free(&pipe);
    return rc;
}

void nmf(float *mDataArr, int nLength, int mLength, int k, float *wArr, float *hArr, int *maxIter, int *type,
         float *thresh, int *norm) {
    nmfBatch(mDataArr, 1, nLength, mLength, k, wArr, hArr, maxIter, type, thresh, norm, NULL, AFB200_MEM_HOST, NULL);
}
