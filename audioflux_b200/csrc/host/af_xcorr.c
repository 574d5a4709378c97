/* af_xcorr.c -- XcorrObj of the C ABI (host C; compute = kernels/xcorr.cu, one launch per staging chunk up to 8192
 * samples).  Interface spec: include/dsp/xcorr_algorithm.h, behaviour src/dsp/xcorr_algorithm.c.  The object holds the
 * staging pipeline and the long path's device workspace, no samples: every call is computed from its own inputs, as on
 * a fresh reference object. */
#include <stdlib.h>
#include "../af_internal.h"

struct OpaqueXcorr {
    AfPipe pipe;
    AfDevBuf work;        /* long path (more than 8192 samples): kept between calls */
    void *fence;          /* end of the last launch that used `work`, chained over every stream that used it */
};

int xcorrObj_new(XcorrObj *xcorrObj) {
    af_clear_error();
    if (!xcorrObj) return -1;
    *xcorrObj = (XcorrObj)calloc(1, sizeof(struct OpaqueXcorr));
    return *xcorrObj ? 0 : -1;
}

typedef struct { XcorrObj s; int n, coeff; } XcCall;

/* d[0] a, d[1] b (or NULL), d[2] out, d[3] maxValue (or NULL), d[4] maxIndex (or NULL) */
static int xc_chunk(void *ctx, int nb, float *const *d, void *st) {
    const XcCall *c = (const XcCall *)ctx;
    AfXcorrArgs a;
    a.a = d[0]; a.b = d[1]; a.out = d[2]; a.maxValue = d[3]; a.maxIndex = (int *)d[4];
    a.n = c->n; a.batch = nb; a.coeff = c->coeff; a.work = &c->s->work; a.fence = &c->s->fence;
    return af_launch_xcorr(&a, st);
}

int xcorrObj_xcorrBatch(XcorrObj s, const float *a, const float *b, int length, int batch, XcorrNormalType *normType,
                        float *out, float *maxValue, int *maxIndex, int memKind, void *stream) {
    af_clear_error();
    if (length < 1)
        return af_fail(-1, "xcorrObj_xcorr: length=%d; at least 1 is needed (the reference reads outside its arrays)",
                       length);
    if (length > AFB200_XCORR_MAX_LENGTH)
        return af_fail(-2, "xcorrObj_xcorr: length=%d; the largest supported is %d (transforms of up to 2^20 points)",
                       length, AFB200_XCORR_MAX_LENGTH);
    if (!s || !a || !out || batch < 0) return af_fail(-1, "xcorrObj_xcorrBatch: bad argument");
    int rc = af_device_ready();
    if (rc || batch == 0) return rc;
    XcCall c = {s, length, normType ? *normType == XcorrNormal_Coeff : 1};               /* :55-59 */
    const size_t n = (size_t)length;
    const AfPlane pl[5] = {{a, n, AF_IN, 0}, {b, n, AF_IN, 0}, {out, 2 * n - 1, AF_OUT, 0}, {maxValue, 1, AF_OUT, 0},
                           {maxIndex, 1, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, xc_chunk, &c, pl, 5, batch, AF_PIPE_CHUNK_BYTES);
}

/* :49-115 */
int xcorrObj_xcorr(XcorrObj s, float *vArr1, float *vArr2, int length, XcorrNormalType *normType, float *vArr3,
                   float *maxValue) {
    af_clear_error();
    if (!s || !vArr1) return 0;
    if (!vArr3 && length >= 1 && length <= AFB200_XCORR_MAX_LENGTH) return af_fail(-1, "xcorrObj_xcorr: no output array");
    int index = 0;
    const int rc = xcorrObj_xcorrBatch(s, vArr1, vArr2, length, 1, normType, vArr3, maxValue, &index, AFB200_MEM_HOST,
                                       NULL);
    if (rc) return rc < 0 ? rc : -3;
    return index;
}

void xcorrObj_free(XcorrObj s) {
    if (!s) return;
    af_fence_wait(s->fence);
    af_fence_free(s->fence);
    af_pipe_free(&s->pipe);
    af_devbuf_free(&s->work);
    free(s);
}
