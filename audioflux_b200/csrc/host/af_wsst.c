/* af_wsst.c -- synchrosqueezing objects of the C ABI: WSSTObj (wavelet synchrosqueezed transform) and SynsqObj
 * (phase-difference synchrosqueezing of any time-frequency matrix).
 * Interface spec: src/wsst_algorithm.h:12-49, src/synsq_algorithm.h:12-33; behaviour
 * src/wsst_algorithm.c:64-352 and src/synsq_algorithm.c:38-300.  Compute = the CWT core (kernels/cwt.cu: W and the
 * derivative transform W' from one forward spectrum) + kernels/squeeze.cu (frequency index, row scatter).
 * Row indices are integer outcomes of float32 math on the transform's planes: a cell within a few ulp of a rounding
 * boundary may land one row apart between two pipelines whose planes differ in the last bits, so parity with the
 * reference's output is stated statistically (tests/test_gpu_squeeze.py).  On the GPU's own planes the index and the
 * scatter are checked cell by cell (tests/test_gpu_scatter_cells.py): bit for bit on the Linear, Linspace, Mel, Bark
 * and Erb scales; on Octave / Log (log2f) and for synsq (atan2f) within the CUDA Math API's ulp bounds. */
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
    float *dNorm;                     /* freArr / samplate (mel / bark / erb index) */
    AfDevBuf dW[4], dIdx;             /* W (when the caller does not take it) and W', row indices */
    AfPipe pipe;
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
    af_clear_error();
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

static int wsst_chunk(void *p, int nb, float *const *d, void *st) {
    (void)nb;                                            /* one clip */
    return wsstObj_wsstDevice((WSSTObj)p, d[0], d[1], d[2], d[3], d[4], st);
}

void wsstObj_wsst(WSSTObj w, float *dataArr, float *mRealArr4, float *mImageArr4, float *mRealArr5, float *mImageArr5) {
    if (!w || !dataArr || !mRealArr4 || !mImageArr4) return;
    af_clear_error();
    if (af_device_ready()) return;
    /* the reference ADDS into the caller's planes */
    const size_t plane = (size_t)w->num * w->fftLength;
    const AfPlane pl[5] = {{dataArr, (size_t)w->fftLength, AF_IN, 0}, {mRealArr4, plane, AF_INOUT, 0}, {mImageArr4, plane, AF_INOUT, 0},
                           {mRealArr5, plane, AF_OUT, 0}, {mImageArr5, plane, AF_OUT, 0}};
    af_run_batch(&w->pipe, AFB200_MEM_HOST, NULL, wsst_chunk, w, pl, 5, 1, AF_PIPE_CHUNK_BYTES);
}

void wsstObj_free(WSSTObj w) {
    if (!w) return;
    cwtObj_free(w->cwt);
    af_devbuf_free(&w->dIdx);
    for (int i = 0; i < 4; i++) af_devbuf_free(&w->dW[i]);
    af_dev_free(w->dNorm);
    af_pipe_free(&w->pipe);
    free(w);
}

/* ---------------------------------------------------------------- SynsqObj ---------------------------------------- */
struct OpaqueSynsq {
    int num, fftLength, samplate, order;
    float thresh;
    AfDevBuf dIdx, dNorm;
    AfPipe pipe;
};

int synsqObj_new(SynsqObj *out, int num, int radix2Exp, int *samplate, int *order, float *thresh) {
    af_clear_error();
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

typedef struct { SynsqObj s; const float *freArr; int scaleType; } SynsqCall;

static int synsq_chunk(void *p, int nb, float *const *d, void *st) {
    const SynsqCall *a = (const SynsqCall *)p;
    (void)nb;                                            /* one matrix */
    return synsqObj_synsqDevice(a->s, a->freArr, a->scaleType, d[0], d[1], d[2], d[3], st);
}

void synsqObj_synsq(SynsqObj s, float *freArr, SpectralFilterBankScaleType scaleType, float *mRealArr1, float *mImageArr1,
                    float *mRealArr2, float *mImageArr2) {
    if (!s || !freArr || !mRealArr1 || !mImageArr1 || !mRealArr2 || !mImageArr2) return;
    if (scaleType > SpectralFilterBankScale_Log) { printf("scaleType is error!\n"); return; }
    af_clear_error();
    if (af_device_ready()) return;
    SynsqCall a = {s, freArr, (int)scaleType};
    const size_t plane = (size_t)s->num * s->fftLength;
    const AfPlane pl[4] = {{mRealArr1, plane, AF_IN, 0}, {mImageArr1, plane, AF_IN, 0},
                           {mRealArr2, plane, AF_INOUT, 0}, {mImageArr2, plane, AF_INOUT, 0}};
    af_run_batch(&s->pipe, AFB200_MEM_HOST, NULL, synsq_chunk, &a, pl, 4, 1, AF_PIPE_CHUNK_BYTES);
}

void synsqObj_free(SynsqObj s) {
    if (!s) return;
    af_devbuf_free(&s->dIdx); af_devbuf_free(&s->dNorm);
    af_pipe_free(&s->pipe);
    free(s);
}
