/* af_reassign.c -- ReassignObj of the C ABI (host C; compute = kernels/stft_generic.cu x 3 + kernels/reassign.cu).
 * Interface spec: src/reassign_algorithm.h:26-55; behaviour src/reassign_algorithm.c:83-451, 587-822.
 * Three STFTs of the clip -- window h, its wrapped central difference dh and the ramp-weighted t.h -- give per cell the
 * reassigned frequency f - Im(S_dh / S_h) sr / 2 pi and time t + Re(S_th / S_h) / sr; cells are rounded to the grid and
 * the sign-alternated S_h is scatter-added.  Cell indices are integer outcomes of float32 divides: a cell within an ulp
 * of a rounding boundary may land one bin apart from the reference, so parity of the reassigned planes is stated
 * statistically (tests/test_gpu_reassign.py), while S_h itself meets the usual 1e-4. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"
#include "../../../include/afb200_stft.h"
#include "../../../include/afb200_reassign.h"

struct OpaqueReassign {
    STFTObj stft[3];                 /* windows h, dh, t.h */
    int radix2Exp, fftLength, slideLength, samplate, isPadding;
    ReassignType reType;
    float thresh;
    int resultType, order;
    void *stream;
    AfDevBuf dIn, dS[6], dIdx[2], dMax, dAcc[2], dOut[2];
};

int reassignObj_new(ReassignObj *out, int radix2Exp, int *samplate, WindowType *windowType, int *slideLength,
                    ReassignType *reType, float *thresh, int *isPadding, int *isContinue) {
    (void)isContinue;                /* read by nobody in the reference either (reassign_algorithm.c:100, 152) */
    if (!out) return -1;
    *out = NULL;
    ReassignObj r = (ReassignObj)calloc(1, sizeof(struct OpaqueReassign));
    if (!r) return -1;
    r->reType = reType ? *reType : Reassign_All;
    r->samplate = (samplate && *samplate > 0) ? *samplate : 32000;
    r->isPadding = isPadding ? *isPadding : 0;
    r->radix2Exp = (radix2Exp > 1 && radix2Exp < 31) ? radix2Exp : 12;
    WindowType wt = windowType ? *windowType : Window_Hann;
    r->fftLength = 1 << r->radix2Exp;
    r->slideLength = (slideLength && *slideLength > 0) ? *slideLength : r->fftLength / 4;
    r->thresh = (thresh && *thresh >= 0) ? *thresh : 0.001f;
    r->order = 1;
    const int n = r->fftLength;
    int zero = 0, status = 0;
    for (int k = 0; k < 3 && !status; k++) {
        status = stftObj_new(&r->stft[k], r->radix2Exp, &wt, &r->slideLength, &zero);
        if (!status) stftObj_enablePadding(r->stft[k], r->isPadding);
    }
    float *dh = (float *)malloc(sizeof(float) * (size_t)n), *th = (float *)malloc(sizeof(float) * (size_t)n);
    if (status || !dh || !th) {
        free(dh); free(th);
        reassignObj_free(r);
        return status ? status : -1;
    }
    /* _reassignObj_initWindowData (:417-451): dh = __vgradient of [w[n-1], w[0..n-1], w[0]] at entries 1..n,
     * th[i] = (i - n/2) * w[i] */
    const float *w = stftObj_getWindowDataArr(r->stft[0]);
    for (int i = 0; i < n; i++) {
        const float next = w[i + 1 < n ? i + 1 : 0], prev = w[i > 0 ? i - 1 : n - 1];
        dh[i] = (next - prev) / 2;
        th[i] = (float)(i - n / 2) * w[i];
    }
    stftObj_useWindowDataArr(r->stft[1], dh);
    stftObj_useWindowDataArr(r->stft[2], th);
    free(dh); free(th);
    *out = r;
    return 0;
}

int reassignObj_calTimeLength(ReassignObj r, int dataLength) { return r ? stftObj_calTimeLength(r->stft[0], dataLength) : 0; }
void reassignObj_setResultType(ReassignObj r, int type) { if (r) r->resultType = type; }
void reassignObj_setOrder(ReassignObj r, int order) { if (r) r->order = order; }

/* device planes; out4 planes are accumulated into */
static int reassign_device(ReassignObj r, const float *dData, int dataLength, int batch, float *dRe4, float *dIm4,
                           float *dRe5, float *dIm5, void *st) {
    const int T = reassignObj_calTimeLength(r, dataLength), W = r->fftLength / 2 + 1;
    if (T <= 0) return AF_OK;
    const size_t cells = (size_t)batch * T * W, plane = sizeof(float) * cells;
    int rc;
    const int none = r->reType == Reassign_None;
    const int needF = r->reType == Reassign_All || r->reType == Reassign_Fre;
    const int needT = r->reType == Reassign_All || r->reType == Reassign_Time;
    /* S_h goes straight into the caller's second pair of planes when there is one (Reassign_None: into the first) */
    float *s1r = none ? dRe4 : dRe5, *s1i = none ? dIm4 : dIm5;
    if (!s1r || !s1i) {
        if ((rc = af_devbuf_reserve(&r->dS[0], plane)) || (rc = af_devbuf_reserve(&r->dS[1], plane))) return rc;
        s1r = (float *)r->dS[0].ptr; s1i = (float *)r->dS[1].ptr;
    }
    if ((rc = stftObj_stftBatch(r->stft[0], dData, dataLength, batch, s1r, s1i, AFB200_MEM_DEVICE, st))) return rc;
    if (none) return AF_OK;
    for (int k = 2; k < 6; k++) {
        const int used = k < 4 ? needF : needT;
        if (used && (rc = af_devbuf_reserve(&r->dS[k], plane))) return rc;
    }
    if (needF && (rc = stftObj_stftBatch(r->stft[1], dData, dataLength, batch, (float *)r->dS[2].ptr, (float *)r->dS[3].ptr, AFB200_MEM_DEVICE, st))) return rc;
    if (needT && (rc = stftObj_stftBatch(r->stft[2], dData, dataLength, batch, (float *)r->dS[4].ptr, (float *)r->dS[5].ptr, AFB200_MEM_DEVICE, st))) return rc;
    if ((rc = af_devbuf_reserve(&r->dIdx[0], sizeof(int) * cells)) || (rc = af_devbuf_reserve(&r->dIdx[1], sizeof(int) * cells)) ||
        (rc = af_devbuf_reserve(&r->dMax, sizeof(unsigned) * (size_t)batch)) ||
        (rc = af_devbuf_reserve(&r->dAcc[0], sizeof(unsigned long long) * cells)) ||
        (rc = af_devbuf_reserve(&r->dAcc[1], sizeof(unsigned long long) * cells))) return rc;
    AfReassignArgs a;
    a.fftLength = r->fftLength; a.slideLength = r->slideLength; a.samplate = r->samplate; a.timeLength = T; a.batch = batch;
    a.reType = (int)r->reType; a.order = r->order; a.resultType = r->resultType; a.thresh = r->thresh;
    return af_launch_reassign(&a, s1r, s1i, (const float *)r->dS[2].ptr, (const float *)r->dS[3].ptr,
                              (const float *)r->dS[4].ptr, (const float *)r->dS[5].ptr, (int *)r->dIdx[0].ptr, (int *)r->dIdx[1].ptr,
                              (unsigned *)r->dMax.ptr, (unsigned long long *)r->dAcc[0].ptr, (unsigned long long *)r->dAcc[1].ptr,
                              dRe4, dIm4, st);
}

int reassignObj_reassignBatch(ReassignObj r, const float *data, int dataLength, int batch, float *re4, float *im4,
                              float *re5, float *im5, int memKind, void *stream) {
    if (!r || !data || !re4 || !im4 || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "reassignObj_reassignBatch: bad argument");
    af_clear_error();
    int rc = af_device_ready();
    if (rc) return rc;
    if (memKind == AFB200_MEM_DEVICE) return reassign_device(r, data, dataLength, batch, re4, im4, re5, im5, stream);
    if (!r->stream && (rc = af_stream_create(&r->stream))) return rc;
    void *st = stream ? stream : r->stream;
    const int T = reassignObj_calTimeLength(r, dataLength), W = r->fftLength / 2 + 1;
    if (T <= 0) return AF_OK;
    const size_t plane = sizeof(float) * (size_t)batch * T * W, inB = sizeof(float) * (size_t)batch * dataLength;
    if ((rc = af_devbuf_reserve(&r->dIn, inB)) || (rc = af_devbuf_reserve(&r->dOut[0], plane)) || (rc = af_devbuf_reserve(&r->dOut[1], plane)) ||
        (rc = af_devbuf_reserve(&r->dS[0], plane)) || (rc = af_devbuf_reserve(&r->dS[1], plane))) return rc;
    if ((rc = af_memcpy_h2d(r->dIn.ptr, data, inB, st))) return rc;
    const int none = r->reType == Reassign_None;
    if (!none && ((rc = af_memcpy_h2d(r->dOut[0].ptr, re4, plane, st)) || (rc = af_memcpy_h2d(r->dOut[1].ptr, im4, plane, st)))) return rc;
    if ((rc = reassign_device(r, (const float *)r->dIn.ptr, dataLength, batch, (float *)r->dOut[0].ptr, (float *)r->dOut[1].ptr,
                              none ? NULL : (float *)r->dS[0].ptr, none ? NULL : (float *)r->dS[1].ptr, st))) return rc;
    if ((rc = af_memcpy_d2h(re4, r->dOut[0].ptr, plane, st))) return rc;
    if ((none || r->resultType == 0) && (rc = af_memcpy_d2h(im4, r->dOut[1].ptr, plane, st))) return rc;
    if (!none && re5 && (rc = af_memcpy_d2h(re5, r->dS[0].ptr, plane, st))) return rc;
    if (!none && im5 && (rc = af_memcpy_d2h(im5, r->dS[1].ptr, plane, st))) return rc;
    return af_stream_sync(st);
}

void reassignObj_reassign(ReassignObj r, float *dataArr, int dataLength, float *mRealArr4, float *mImageArr4,
                          float *mRealArr5, float *mImageArr5) {
    if (!r || !dataArr || !mRealArr4 || !mImageArr4 || dataLength <= 0) return;
    reassignObj_reassignBatch(r, dataArr, dataLength, 1, mRealArr4, mImageArr4, mRealArr5, mImageArr5, AFB200_MEM_HOST, NULL);
}

void reassignObj_free(ReassignObj r) {
    if (!r) return;
    for (int k = 0; k < 3; k++) stftObj_free(r->stft[k]);
    af_devbuf_free(&r->dIn); af_devbuf_free(&r->dMax);
    for (int k = 0; k < 6; k++) af_devbuf_free(&r->dS[k]);
    for (int k = 0; k < 2; k++) { af_devbuf_free(&r->dIdx[k]); af_devbuf_free(&r->dAcc[k]); af_devbuf_free(&r->dOut[k]); }
    af_stream_destroy(r->stream);
    free(r);
}
