/* af_hpss.c -- HPSSObj of the C ABI (host C; compute = the STFT of kernels/stft_generic.cu, the masks of kernels/hpss.cu
 * and the inverse STFT of kernels/istft.cu, per group of clips).
 * Interface spec: include/mir/hpss_algorithm.h, behaviour src/mir/hpss_algorithm.c:40-371.  The object keeps its window
 * and a device workspace: the two half-spectrum planes of the STFT, the masked planes of H and P, and the inverse STFT's
 * frames, for one group of clips. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

#define HPSS_MIN_EXP 2      /* hop N/4 >= 1 */
#define HPSS_MAX_EXP 20     /* the longest STFT / inverse STFT */
#define HPSS_GROUP_CAP ((size_t)2 << 30)

struct OpaqueHPSS {
    int radix2Exp, fftLength, slideLength, hOrder, pOrder;
    WindowType windowType;
    float *window;        /* host, fftLength (af_window_fft, as the STFT object builds it); NULL outside 2 .. 20 */
    float *dWindow;       /* device copy; stays NULL for Rect (no multiply) */
    AfDevBuf dRe, dIm, dHRe, dHIm, dPRe, dPIm, dFrames;
    AfPipe pipe;
};

int hpssObj_new(HPSSObj *hpssObj, int radix2Exp, WindowType *windowType, int *slideLength, int *hOrder, int *pOrder) {
    af_clear_error();
    if (!hpssObj) return 0;
    *hpssObj = NULL;
    HPSSObj s = (HPSSObj)calloc(1, sizeof(struct OpaqueHPSS));
    if (!s) return 0;
    (void)slideLength;                                                 /* :81: the hop is always fftLength / 4 */
    s->radix2Exp = radix2Exp;
    s->fftLength = radix2Exp >= 0 && radix2Exp <= 30 ? 1 << radix2Exp : 0;
    s->slideLength = s->fftLength / 4;
    s->hOrder = hOrder && *hOrder > 0 && (*hOrder & 1) ? *hOrder : 21;        /* :65-75 */
    s->pOrder = pOrder && *pOrder > 0 && (*pOrder & 1) ? *pOrder : 31;
    s->windowType = windowType ? *windowType : Window_Hamm;
    if (radix2Exp >= HPSS_MIN_EXP && radix2Exp <= HPSS_MAX_EXP) {
        s->window = (float *)malloc(sizeof(float) * (size_t)s->fftLength);
        if (s->window) af_window_fft(s->windowType, s->fftLength, s->window);
    }
    *hpssObj = s;
    return 0;
}

static int hpss_time_length(HPSSObj s, int dataLength) {
    return dataLength < s->fftLength || s->slideLength <= 0 ? 0 : (dataLength - s->fftLength) / s->slideLength + 1;
}

int hpssObj_calDataLength(HPSSObj s, int dataLength) {
    if (!s) return 0;
    return (hpss_time_length(s, dataLength) - 1) * s->slideLength + s->fftLength;
}

void hpssObj_debug(HPSSObj s) { (void)s; }

/* the rules every compute call checks before any device work */
static int hpss_check(HPSSObj s, int dataLength, const char *who) {
    if (s->radix2Exp < HPSS_MIN_EXP || s->radix2Exp > HPSS_MAX_EXP)
        return af_fail(AF_ERR_UNSUPPORTED, "%s: radix2Exp=%d; %d .. %d are supported (a hop of fftLength/4 of at least one "
                       "sample, an STFT of at most 2^%d points)", who, s->radix2Exp, HPSS_MIN_EXP, HPSS_MAX_EXP, HPSS_MAX_EXP);
    if (!s->window) return af_fail(AF_ERR_NOMEM, "%s: no window", who);
    if (s->hOrder > AFB200_HPSS_MAX_ORDER || s->pOrder > AFB200_HPSS_MAX_ORDER)
        return af_fail(AF_ERR_UNSUPPORTED, "%s: hOrder=%d, pOrder=%d; orders up to %d are supported", who, s->hOrder,
                       s->pOrder, AFB200_HPSS_MAX_ORDER);
    if (dataLength < s->fftLength)
        return af_fail(AF_ERR_ARG, "%s: dataLength=%d is shorter than one frame (fftLength %d)", who, dataLength,
                       s->fftLength);
    return AF_OK;
}

static int hpss_device(HPSSObj s) {
    int rc = af_device_ready();
    if (rc || s->dWindow || s->windowType == Window_Rect) return rc;
    return af_dev_upload((void **)&s->dWindow, s->window, sizeof(float) * (size_t)s->fftLength);
}

typedef struct { HPSSObj s; int dataLength, timeLength, outLength, accumulate; } HpssCall;

/* d[0] data nb x dataLength, d[1] h / d[2] p nb x outLength (or NULL) */
static int hpss_chunk(void *ctx, int nb, float *const *d, void *st) {
    const HpssCall *c = (const HpssCall *)ctx;
    const HPSSObj s = c->s;
    const int T = c->timeLength, N = s->fftLength, W = N / 2 + 1;
    float *out[2] = {d[1], d[2]};
    const int nOut = (out[0] != NULL) + (out[1] != NULL);
    const size_t plane = sizeof(float) * (size_t)T * W;
    const int group = af_chunk_clips((2 + 2 * (size_t)nOut) * plane + sizeof(float) * (size_t)T * N, HPSS_GROUP_CAP, nb);
    int rc;
    if ((rc = af_devbuf_reserve(&s->dRe, plane * group)) || (rc = af_devbuf_reserve(&s->dIm, plane * group)) ||
        (out[0] && ((rc = af_devbuf_reserve(&s->dHRe, plane * group)) || (rc = af_devbuf_reserve(&s->dHIm, plane * group)))) ||
        (out[1] && ((rc = af_devbuf_reserve(&s->dPRe, plane * group)) || (rc = af_devbuf_reserve(&s->dPIm, plane * group)))) ||
        (rc = af_devbuf_reserve(&s->dFrames, sizeof(float) * (size_t)group * T * N)))
        return rc;
    float *re = (float *)s->dRe.ptr, *im = (float *)s->dIm.ptr;
    float *mRe[2] = {(float *)s->dHRe.ptr, (float *)s->dPRe.ptr}, *mIm[2] = {(float *)s->dHIm.ptr, (float *)s->dPIm.ptr};
    for (int c0 = 0; c0 < nb; c0 += group) {
        const int g = nb - c0 < group ? nb - c0 : group;
        AfFrameSrc src;
        memset(&src, 0, sizeof(src));
        src.fftLength = N; src.slideLength = s->slideLength; src.dataLength = c->dataLength;
        src.timeLength = T; src.batch = g; src.validLength = c->dataLength; src.window = s->dWindow;
        src.data = d[0] + (size_t)c0 * c->dataLength;
        if ((rc = af_launch_stft(&src, AF_STFT_HALF, 1.0f, re, im, st))) return rc;
        AfHpssArgs a;
        memset(&a, 0, sizeof(a));
        a.re = re; a.im = im;
        if (out[0]) { a.hRe = mRe[0]; a.hIm = mIm[0]; }
        if (out[1]) { a.pRe = mRe[1]; a.pIm = mIm[1]; }
        a.clips = g; a.timeLength = T; a.width = W; a.hOrder = s->hOrder; a.pOrder = s->pOrder;
        if ((rc = af_launch_hpss_mask(&a, st))) return rc;
        for (int k = 0; k < 2; k++) {
            if (!out[k]) continue;
            float *y = out[k] + (size_t)c0 * c->outLength;
            if (!c->accumulate && (rc = af_memset_d(y, 0, sizeof(float) * (size_t)g * c->outLength, st))) return rc;
            if ((rc = af_launch_istft(mRe[k], mIm[k], W, N, s->slideLength, T, g, s->dWindow, 0, (float *)s->dFrames.ptr, y,
                                      st)))
                return rc;
        }
    }
    return AF_OK;
}

static int hpss_run(HPSSObj s, const float *data, int dataLength, int batch, float *h, float *p, int accumulate,
                    int memKind, void *stream, const char *who) {
    int rc = hpss_check(s, dataLength, who);
    if (rc || (rc = hpss_device(s)) || batch == 0) return rc;
    HpssCall c = {s, dataLength, hpss_time_length(s, dataLength), hpssObj_calDataLength(s, dataLength), accumulate};
    const int dir = accumulate ? AF_INOUT : AF_OUT;
    const AfPlane pl[3] = {{data, (size_t)dataLength, AF_IN, 0}, {h, (size_t)c.outLength, dir, 0},
                           {p, (size_t)c.outLength, dir, 0}};
    return af_run_batch(&s->pipe, memKind, stream, hpss_chunk, &c, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

int hpssObj_hpssBatch(HPSSObj s, const float *data, int dataLength, int batch, float *h, float *p, int memKind,
                      void *stream) {
    if (!s || !data || dataLength <= 0 || batch < 0 || (!h && !p))
        return af_fail(AF_ERR_ARG, "hpssObj_hpssBatch: bad argument");
    af_clear_error();
    return hpss_run(s, data, dataLength, batch, h, p, 0, memKind, stream, "hpssObj_hpssBatch");
}

/* :118-345.  Both outputs NULL: nothing to do, as in the reference. */
void hpssObj_hpss(HPSSObj s, float *dataArr, int dataLength, float *hArr, float *pArr) {
    if (!s || (!hArr && !pArr)) return;
    af_clear_error();
    if (!dataArr) { af_fail(AF_ERR_ARG, "hpssObj_hpss: no input"); return; }
    hpss_run(s, dataArr, dataLength, 1, hArr, pArr, 1, AFB200_MEM_HOST, NULL, "hpssObj_hpss");
}

void hpssObj_free(HPSSObj s) {
    if (!s) return;
    af_pipe_free(&s->pipe);
    af_devbuf_free(&s->dRe); af_devbuf_free(&s->dIm);
    af_devbuf_free(&s->dHRe); af_devbuf_free(&s->dHIm);
    af_devbuf_free(&s->dPRe); af_devbuf_free(&s->dPIm);
    af_devbuf_free(&s->dFrames);
    af_dev_free(s->dWindow);
    free(s->window);
    free(s);
}
