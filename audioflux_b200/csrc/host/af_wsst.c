/* af_wsst.c -- synchrosqueezing objects of the C ABI: WSSTObj (wavelet synchrosqueezed transform) and SynsqObj
 * (phase-difference synchrosqueezing of any time-frequency matrix).
 * Interface spec: src/wsst_algorithm.h:12-49, src/synsq_algorithm.h:12-33; behaviour
 * src/wsst_algorithm.c:64-352 and src/synsq_algorithm.c:38-300.  Compute = the CWT core (kernels/cwt.cu: W and the
 * derivative transform W' from one forward spectrum) + kernels/squeeze.cu (frequency index, row scatter).
 * Row indices are integer outcomes of float32 transcendental math (log2f / atan2f): cells whose value sits within a
 * few ulp of a rounding boundary may land one row apart from the reference -- parity for these rows is therefore
 * stated statistically (tests/test_gpu_squeeze.py: share of identical cells, Frobenius error). */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"
#include "../../../include/afb200_cwt.h"
#include "../../../include/afb200_wsst.h"

struct OpaqueWSST {
    CWTObj cwt;
    int num, fftLength, samplate, order;
    float thresh;
    SpectralFilterBankScaleType scaleType;
    void *stream;
    float *dNorm;                     /* freArr / samplate (mel / bark / erb index) */
    AfDevBuf dIn, dW[4], dOut[2], dIdx;
};

static int upload_norm(const float *fre, int num, int samplate, float **dNorm) {
    float *v = (float *)malloc(sizeof(float) * (size_t)num);
    if (!v) return AF_ERR_NOMEM;
    for (int i = 0; i < num; i++) v[i] = fre[i] / (float)samplate;
    int rc = af_dev_upload((void **)dNorm, v, sizeof(float) * (size_t)num);
    free(v);
    return rc;
}

int wsstObj_new(WSSTObj *out, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre, int *binPerOctave,
                WaveletContinueType *waveletType, SpectralFilterBankScaleType *scaleType, float *gamma, float *beta,
                float *thresh, int *isPadding) {
    if (!out) return -1;
    *out = NULL;
    float th = 0.001f;
    if (thresh && *thresh >= 0) th = *thresh;
    int sr = 32000;
    if (samplate && *samplate > 0 && *samplate <= 196000) sr = *samplate;
    WaveletContinueType wt = waveletType ? *waveletType : WaveletContinue_Morlet;
    SpectralFilterBankScaleType sc = scaleType ? *scaleType : SpectralFilterBankScale_Octave;
    if (sc > SpectralFilterBankScale_Log) { printf("scaleType is error!\n"); return 1; }
    WSSTObj w = (WSSTObj)calloc(1, sizeof(struct OpaqueWSST));
    if (!w) return -1;
    int status = cwtObj_new(&w->cwt, num, radix2Exp, samplate, lowFre, highFre, binPerOctave, &wt, &sc, gamma, beta, isPadding);
    if (status != 0 || !w->cwt) { free(w); return status ? status : -1; }
    cwtObj_enableDet(w->cwt, 1);
    w->num = num; w->fftLength = 1 << radix2Exp; w->samplate = sr; w->thresh = th; w->scaleType = sc; w->order = 0;
    *out = w;
    return 0;
}

float *wsstObj_getFreBandArr(WSSTObj w) { return w ? cwtObj_getFreBandArr(w->cwt) : NULL; }
int *wsstObj_getBinBandArr(WSSTObj w) { return w ? cwtObj_getBinBandArr(w->cwt) : NULL; }

void wsstObj_setOrder(WSSTObj w, int order) {
    if (!w) return;
    if (order > 1) {
        /* the reference's order > 1 branch writes through a scratch pointer it never allocates (wsst_algorithm.c:45, :299) */
        af_fail(AF_ERR_UNSUPPORTED, "wsstObj_setOrder(%d): only order 1 is supported (the reference crashes for order > 1)", order);
        return;
    }
    w->order = order;
}

/* planes [num x N]: out4 / out5 accumulate-into semantics of the reference (out4 += squeezed, out5 = plain CWT) */
int wsstObj_wsstDevice(WSSTObj w, const float *dData, float *dOutRe, float *dOutIm, float *dCwtRe, float *dCwtIm, void *st) {
    const int num = w->num, n = w->fftLength;
    const size_t plane = sizeof(float) * (size_t)num * n;
    int rc;
    for (int i = 0; i < 4; i++) if ((rc = af_devbuf_reserve(&w->dW[i], plane))) return rc;
    if ((rc = af_devbuf_reserve(&w->dIdx, sizeof(int) * (size_t)num * n))) return rc;
    float *wr = dCwtRe ? dCwtRe : (float *)w->dW[0].ptr, *wi = dCwtIm ? dCwtIm : (float *)w->dW[1].ptr;
    float *dr = (float *)w->dW[2].ptr, *di = (float *)w->dW[3].ptr;
    if ((rc = cwtObj_cwtBatch(w->cwt, dData, 1, wr, wi, AFB200_MEM_DEVICE, st))) return rc;
    if ((rc = cwtObj_cwtDetBatch(w->cwt, NULL, 1, dr, di, AFB200_MEM_DEVICE, st))) return rc;      /* reuses the spectrum */
    const float *fre = cwtObj_getFreBandArr(w->cwt);
    if (!w->dNorm && (rc = upload_norm(fre, num, w->samplate, &w->dNorm))) return rc;
    if ((rc = af_launch_wsst_index(wr, wi, dr, di, num, n, (int)w->scaleType, fre[0], fre[num - 1], w->samplate, w->dNorm,
                                   (int *)w->dIdx.ptr, st))) return rc;
    return af_launch_squeeze_scatter(wr, wi, (const int *)w->dIdx.ptr, num, n, w->thresh, dOutRe, dOutIm, st);
}

void wsstObj_wsst(WSSTObj w, float *dataArr, float *mRealArr4, float *mImageArr4, float *mRealArr5, float *mImageArr5) {
    if (!w || !dataArr || !mRealArr4 || !mImageArr4) return;
    af_clear_error();
    if (af_device_ready()) return;
    if (!w->stream && af_stream_create(&w->stream)) return;
    void *st = w->stream;
    const int num = w->num, n = w->fftLength;
    const size_t plane = sizeof(float) * (size_t)num * n;
    if (af_devbuf_reserve(&w->dIn, sizeof(float) * (size_t)n) || af_devbuf_reserve(&w->dOut[0], plane) || af_devbuf_reserve(&w->dOut[1], plane)) return;
    for (int i = 0; i < 2; i++) if (af_devbuf_reserve(&w->dW[i], plane)) return;
    if (af_memcpy_h2d(w->dIn.ptr, dataArr, sizeof(float) * (size_t)n, st)) return;
    /* the reference ADDS into the caller's planes */
    if (af_memcpy_h2d(w->dOut[0].ptr, mRealArr4, plane, st) || af_memcpy_h2d(w->dOut[1].ptr, mImageArr4, plane, st)) return;
    if (wsstObj_wsstDevice(w, (const float *)w->dIn.ptr, (float *)w->dOut[0].ptr, (float *)w->dOut[1].ptr,
                           (float *)w->dW[0].ptr, (float *)w->dW[1].ptr, st)) return;
    if (af_memcpy_d2h(mRealArr4, w->dOut[0].ptr, plane, st) || af_memcpy_d2h(mImageArr4, w->dOut[1].ptr, plane, st)) return;
    if (mRealArr5 && af_memcpy_d2h(mRealArr5, w->dW[0].ptr, plane, st)) return;
    if (mImageArr5 && af_memcpy_d2h(mImageArr5, w->dW[1].ptr, plane, st)) return;
    af_stream_sync(st);
}

void wsstObj_free(WSSTObj w) {
    if (!w) return;
    cwtObj_free(w->cwt);
    af_devbuf_free(&w->dIn); af_devbuf_free(&w->dIdx);
    for (int i = 0; i < 4; i++) af_devbuf_free(&w->dW[i]);
    for (int i = 0; i < 2; i++) af_devbuf_free(&w->dOut[i]);
    af_dev_free(w->dNorm);
    af_stream_destroy(w->stream);
    free(w);
}

/* ---------------------------------------------------------------- SynsqObj ---------------------------------------- */
struct OpaqueSynsq {
    int num, fftLength, samplate, order;
    float thresh;
    void *stream;
    AfDevBuf dIn[2], dOut[2], dIdx, dNorm;
};

int synsqObj_new(SynsqObj *out, int num, int radix2Exp, int *samplate, int *order, float *thresh) {
    if (!out) return -1;
    *out = NULL;
    if (num < 1 || radix2Exp < 1 || radix2Exp > 30) return -1;
    SynsqObj s = (SynsqObj)calloc(1, sizeof(struct OpaqueSynsq));
    if (!s) return -1;
    s->num = num; s->fftLength = 1 << radix2Exp;
    s->samplate = 32000;
    if (samplate && *samplate > 0 && *samplate < 196000) s->samplate = *samplate;
    s->order = 1;
    if (order && *order > 1) {
        af_fail(AF_ERR_UNSUPPORTED, "synsqObj_new: order %d > 1 is not supported", *order);
        free(s);
        return -2;
    }
    s->thresh = 0.001f;
    if (thresh && *thresh > 1) s->thresh = *thresh;            /* (sic) synsq_algorithm.c:71-75 only accepts thresh > 1 */
    *out = s;
    return 0;
}

int synsqObj_synsqDevice(SynsqObj s, const float *freArr /* host, num */, int scaleType, const float *dRe, const float *dIm,
                         float *dOutRe, float *dOutIm, void *st) {
    const int num = s->num, n = s->fftLength;
    int rc;
    if ((rc = af_devbuf_reserve(&s->dIdx, sizeof(int) * (size_t)num * n)) || (rc = af_devbuf_reserve(&s->dNorm, sizeof(float) * (size_t)num))) return rc;
    float *v = (float *)malloc(sizeof(float) * (size_t)num);
    if (!v) return AF_ERR_NOMEM;
    for (int i = 0; i < num; i++) v[i] = freArr[i] / (float)s->samplate;
    rc = af_memcpy_h2d(s->dNorm.ptr, v, sizeof(float) * (size_t)num, st);
    if (!rc) rc = af_stream_sync(st);
    free(v);
    if (rc) return rc;
    if ((rc = af_launch_synsq_index(dRe, dIm, num, n, scaleType, freArr[0], freArr[num - 1], s->samplate, (const float *)s->dNorm.ptr,
                                    (int *)s->dIdx.ptr, st))) return rc;
    return af_launch_squeeze_scatter(dRe, dIm, (const int *)s->dIdx.ptr, num, n, s->thresh, dOutRe, dOutIm, st);
}

void synsqObj_synsq(SynsqObj s, float *freArr, SpectralFilterBankScaleType scaleType, float *mRealArr1, float *mImageArr1,
                    float *mRealArr2, float *mImageArr2) {
    if (!s || !freArr || !mRealArr1 || !mImageArr1 || !mRealArr2 || !mImageArr2) return;
    if (scaleType > SpectralFilterBankScale_Log) { printf("scaleType is error!\n"); return; }
    af_clear_error();
    if (af_device_ready()) return;
    if (!s->stream && af_stream_create(&s->stream)) return;
    void *st = s->stream;
    const size_t plane = sizeof(float) * (size_t)s->num * s->fftLength;
    for (int i = 0; i < 2; i++) if (af_devbuf_reserve(&s->dIn[i], plane) || af_devbuf_reserve(&s->dOut[i], plane)) return;
    if (af_memcpy_h2d(s->dIn[0].ptr, mRealArr1, plane, st) || af_memcpy_h2d(s->dIn[1].ptr, mImageArr1, plane, st)) return;
    if (af_memcpy_h2d(s->dOut[0].ptr, mRealArr2, plane, st) || af_memcpy_h2d(s->dOut[1].ptr, mImageArr2, plane, st)) return;
    if (synsqObj_synsqDevice(s, freArr, (int)scaleType, (const float *)s->dIn[0].ptr, (const float *)s->dIn[1].ptr,
                             (float *)s->dOut[0].ptr, (float *)s->dOut[1].ptr, st)) return;
    if (af_memcpy_d2h(mRealArr2, s->dOut[0].ptr, plane, st) || af_memcpy_d2h(mImageArr2, s->dOut[1].ptr, plane, st)) return;
    af_stream_sync(st);
}

void synsqObj_free(SynsqObj s) {
    if (!s) return;
    for (int i = 0; i < 2; i++) { af_devbuf_free(&s->dIn[i]); af_devbuf_free(&s->dOut[i]); }
    af_devbuf_free(&s->dIdx); af_devbuf_free(&s->dNorm);
    af_stream_destroy(s->stream);
    free(s);
}
