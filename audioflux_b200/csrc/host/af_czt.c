/* af_czt.c -- CZTObj of the C ABI (host C; compute = kernels/czt.cu, one launch per staging chunk plus one per table
 * change).  Interface spec: include/dsp/czt_algorithm.h, behaviour src/dsp/czt_algorithm.c.
 *
 * The chirp tables are the reference's float32 tables (src :114-161), built here with the same float expressions and the
 * C library's cosf / sinf (this file is compiled with -ffp-contract=off, so every product is rounded as there).  The
 * reference compares the band with fields it never sets, so it rebuilds its tables on every valid band; the tables are a
 * function of the band, so rebuilding only when the band changes leaves the same tables.
 *
 * Every use of the device tables -- the upload with the filter transform, and each chunk's k_czt -- waits on the device
 * for the object's fence and records it again, on whatever stream it runs (the caller's, or the staging pipeline's
 * own).  So a launch never reads tables that are still being written, and a rebuild never overwrites tables a launch on
 * another stream still reads. */
#include <math.h>
#include <stdlib.h>
#include "../af_internal.h"

struct OpaqueCZT {
    int log2n, N, M;
    float lowW, highW;    /* band of the current tables */
    float *tables;        /* host, interleaved complex: pre-chirp (N), post-chirp (N), chirp filter h (M) */
    AfDevBuf dTables;     /* device: pre, post and H = FFT_M(h) in bit-reversed order */
    int stale;            /* the device tables are older than the host tables */
    void *fence;          /* end of the last use of the device tables, chained over every stream that used them */
    AfPipe pipe;
};

static size_t czt_table_floats(int N) { return (size_t)2 * (N + N + 2 * N); }

/* _cztObj_dealAW (:114-161) with nArr of cztObj_new (:68-74: -(N-1) .. N-1, and a last entry left at 0), then the
 * pre-chirp A^-n W^(n^2/2) of :212-213, the post-chirp of :255 and h of :243-248 */
static void czt_build(CZTObj s, float lowW, float highW) {
    const int N = s->N, M = s->M;
    float *pre = s->tables, *post = pre + 2 * N, *h = post + 2 * N;
    const float tA = 2 * M_PI * lowW;
    const float tW = -2 * M_PI * (highW - lowW) / N;
    for (int i = 0; i < M; i++) {
        const float n = i < M - 1 ? (float)(i - (N - 1)) : 0.0f;
        const float n1 = -n, n2 = n * n / 2;
        const float aR = cosf(n1 * tA), aI = sinf(n1 * tA);
        const float wR = cosf(n2 * tW), wI = sinf(n2 * tW);
        if (i >= N - 1 && i < M - 1) {
            const int k = i - (N - 1);
            pre[2 * k] = aR * wR - aI * wI;                                /* __complexMul */
            pre[2 * k + 1] = aI * wR + aR * wI;
            post[2 * k] = wR;
            post[2 * k + 1] = wI;
        }
        h[2 * i] = i < M - 1 ? wR : 0.0f;
        h[2 * i + 1] = i < M - 1 ? -wI : 0.0f;
    }
    s->lowW = lowW;
    s->highW = highW;
    s->stale = 1;
}

/* :127-131: an invalid band keeps the tables */
static void czt_band(CZTObj s, float lowW, float highW) {
    if (lowW >= highW || lowW < 0 || highW < 0 || highW > 1) return;
    if (lowW != s->lowW || highW != s->highW) czt_build(s, lowW, highW);
}

int cztObj_new(CZTObj *cztObj, int radix2Exp) {
    af_clear_error();
    if (!cztObj) return -1;
    *cztObj = NULL;
    if (radix2Exp < 0) return af_fail(-1, "cztObj_new: radix2Exp=%d; at least 0 is needed", radix2Exp);
    if (radix2Exp > AFB200_CZT_MAX_EXP)
        return af_fail(-2, "cztObj_new: radix2Exp=%d; the largest supported is %d (the 2N-point transforms run in one "
                       "CTA's shared memory)", radix2Exp, AFB200_CZT_MAX_EXP);
    CZTObj s = (CZTObj)calloc(1, sizeof(struct OpaqueCZT));
    if (!s) return -1;
    s->log2n = radix2Exp;
    s->N = 1 << radix2Exp;
    s->M = 2 * s->N;
    s->tables = (float *)malloc(sizeof(float) * czt_table_floats(s->N));
    if (!s->tables) { free(s); return -1; }
    czt_build(s, 0.0f, 1.0f);                                          /* :111 */
    *cztObj = s;
    return 0;
}

/* ctx: the object; d[0] re, d[1] im (either NULL), d[2] re3, d[3] im3 */
static int czt_chunk(void *ctx, int nb, float *const *d, void *st) {
    const CZTObj s = (CZTObj)ctx;
    float *dt = (float *)s->dTables.ptr;
    int rc = af_fence_order(s->fence, st);
    if (!rc && s->stale) {
        /* pageable source: the copy is staged before af_memcpy_h2d returns, so the next rebuild may overwrite it */
        if ((rc = af_memcpy_h2d(dt, s->tables, sizeof(float) * czt_table_floats(s->N), st)) ||
            (rc = af_launch_czt_filter(dt + 4 * s->N, s->log2n + 1, st)))
            return rc;
        s->stale = 0;
    }
    AfCztArgs a;
    a.re = d[0]; a.im = d[1]; a.re3 = d[2]; a.im3 = d[3]; a.tables = dt; a.log2n = s->log2n; a.batch = nb;
    if (rc || (rc = af_launch_czt(&a, st))) return rc;
    return af_fence_record(&s->fence, st);
}

int cztObj_cztBatch(CZTObj s, const float *re, const float *im, int batch, float lowW, float highW, float *re3,
                    float *im3, int memKind, void *stream) {
    af_clear_error();
    if (!s || (!re && !im) || !re3 || !im3 || batch < 0)
        return af_fail(-1, "cztObj_czt: bad argument (both input planes NULL, no output or a negative batch)");
    int rc = af_device_ready();
    if (rc) return rc;
    czt_band(s, lowW, highW);
    if ((rc = af_devbuf_reserve(&s->dTables, sizeof(float) * czt_table_floats(s->N)))) return rc;   /* once */
    if (batch == 0) return AF_OK;
    const size_t N = (size_t)s->N;
    const AfPlane pl[4] = {{re, N, AF_IN, 0}, {im, N, AF_IN, 0}, {re3, 2 * N, AF_OUT, 0}, {im3, 2 * N, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, czt_chunk, s, pl, 4, batch, AF_PIPE_CHUNK_BYTES);
}

/* :82-89 */
void cztObj_czt(CZTObj s, float *realArr1, float *imageArr1, float lowW, float highW, float *realArr3, float *imageArr3) {
    if (!s) return;
    cztObj_cztBatch(s, realArr1, imageArr1, 1, lowW, highW, realArr3, imageArr3, AFB200_MEM_HOST, NULL);
}

void cztObj_free(CZTObj s) {
    if (!s) return;
    af_fence_wait(s->fence);
    af_fence_free(s->fence);
    af_pipe_free(&s->pipe);
    af_devbuf_free(&s->dTables);
    free(s->tables);
    free(s);
}
