/* af_cepstrogram.c -- CepstrogramObj of the C ABI (host C; compute = kernels/cepstrogram.cu, one launch per call).
 * Interface spec: include/cepstrogram_algorithm.h:14-39, behaviour src/cepstrogram_algorithm.c:55-305.  The object keeps
 * its window only (the reference keeps ten T x N float planes); the window goes to the device at the first compute
 * call. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueCepstrogram {
    int radix2Exp, fftLength, slideLength;
    WindowType windowType;
    float *window;        /* host, fftLength (af_window_fft, as the STFT object builds it) */
    float *dWindow;       /* device copy; stays NULL for Rect (no multiply) */
    AfPipe pipe;
};

int cepstrogramObj_new(CepstrogramObj *cepstrogramObj, int radix2Exp, WindowType *windowType, int *slideLength) {
    af_clear_error();
    if (!cepstrogramObj) return -1;
    *cepstrogramObj = NULL;
    if (radix2Exp < 1 || radix2Exp > 30) {                          /* :68-72 */
        af_fail(-100, "cepstrogramObj_new: radix2Exp=%d; 1 .. 30 are legal", radix2Exp);
        return -100;
    }
    if (radix2Exp > AF_CEPS_MAX_EXP) {
        af_fail(-2, "cepstrogramObj_new: radix2Exp=%d; the largest supported is %d (one frame's transforms are held in "
                "shared memory)", radix2Exp, AF_CEPS_MAX_EXP);
        return -2;
    }
    CepstrogramObj s = (CepstrogramObj)calloc(1, sizeof(struct OpaqueCepstrogram));
    if (!s) return -1;
    s->radix2Exp = radix2Exp;
    s->fftLength = 1 << radix2Exp;
    s->windowType = windowType ? *windowType : Window_Rect;        /* :76-78 */
    /* :80-85; N/4 is 0 at N = 2, where the reference divides by zero in calTimeLength: 1 here */
    s->slideLength = slideLength && *slideLength > 0 ? *slideLength : s->fftLength >= 4 ? s->fftLength / 4 : 1;
    s->window = (float *)malloc(sizeof(float) * (size_t)s->fftLength);
    if (!s->window || af_window_fft(s->windowType, s->fftLength, s->window)) { cepstrogramObj_free(s); return -1; }
    *cepstrogramObj = s;
    return 0;
}

/* :104-109: stftObj_calTimeLength of an STFT object without padding or streaming */
int cepstrogramObj_calTimeLength(CepstrogramObj s, int dataLength) {
    if (!s || dataLength < s->fftLength) return 0;
    return (dataLength - s->fftLength) / s->slideLength + 1;
}

void cepstrogramObj_enableDebug(CepstrogramObj s, int flag) { (void)s; (void)flag; }

static int ceps_check(CepstrogramObj s, int cepNum, const char *who) {
    if (cepNum < 1 || cepNum > s->fftLength / 2)
        return af_fail(AF_ERR_ARG, "%s: cepNum=%d; 1 .. %d (fftLength/2) are supported", who, cepNum, s->fftLength / 2);
    return AF_OK;
}

static int ceps_device(CepstrogramObj s) {
    int rc = af_device_ready();
    if (rc || s->dWindow || s->windowType == Window_Rect) return rc;
    return af_dev_upload((void **)&s->dWindow, s->window, sizeof(float) * (size_t)s->fftLength);
}

typedef struct { CepstrogramObj s; int cepNum, dataLength, timeLength, specWidth; } CepsCall;

static void ceps_args(const CepsCall *c, float *const *d, AfCepsArgs *a) {
    memset(a, 0, sizeof(*a));
    a->log2n = c->s->radix2Exp; a->cepNum = c->cepNum;
    a->cep = d[2]; a->env = d[3]; a->det = d[4];
}

static int ceps_chunk(void *p, int nb, float *const *d, void *st) {
    const CepsCall *c = (const CepsCall *)p;
    AfCepsArgs a;
    ceps_args(c, d, &a);
    a.data = d[0]; a.window = c->s->dWindow;
    a.dataLength = c->dataLength; a.hop = c->s->slideLength; a.timeLength = c->timeLength; a.batch = nb;
    return af_launch_cepstrogram(&a, st);
}

static int ceps2_chunk(void *p, int nb, float *const *d, void *st) {
    const CepsCall *c = (const CepsCall *)p;
    AfCepsArgs a;
    ceps_args(c, d, &a);
    a.specRe = d[0]; a.specIm = d[1]; a.rows = nb; a.specWidth = c->specWidth;
    return af_launch_cepstrogram(&a, st);
}

int cepstrogramObj_cepstrogramBatch(CepstrogramObj s, int cepNum, const float *data, int dataLength, int batch,
                                    float *cep, float *env, float *det, int memKind, void *stream) {
    if (!s || !data || dataLength <= 0 || batch < 0 || (!cep && !env && !det))
        return af_fail(AF_ERR_ARG, "cepstrogramObj_cepstrogramBatch: bad argument");
    af_clear_error();
    int rc = ceps_check(s, cepNum, "cepstrogramObj_cepstrogramBatch");
    if (rc || (rc = ceps_device(s))) return rc;
    const int T = cepstrogramObj_calTimeLength(s, dataLength);
    if (batch == 0 || T == 0) return AF_OK;
    CepsCall c = {s, cepNum, dataLength, T, 0};
    const size_t outPer = (size_t)T * (s->fftLength / 2 + 1);
    const AfPlane pl[5] = {{data, (size_t)dataLength, AF_IN, 0}, {NULL, 0, AF_IN, 0}, {cep, outPer, AF_OUT, 0},
                           {env, outPer, AF_OUT, 0}, {det, outPer, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, ceps_chunk, &c, pl, 5, batch, AF_PIPE_CHUNK_BYTES);
}

int cepstrogramObj_cepstrogram2Batch(CepstrogramObj s, int cepNum, const float *mReal, const float *mImag, int rows,
                                     int specWidth, float *cep, float *env, float *det, int memKind, void *stream) {
    if (!s || !mReal || !mImag || rows < 0 || (!cep && !env && !det))
        return af_fail(AF_ERR_ARG, "cepstrogramObj_cepstrogram2Batch: bad argument");
    if (specWidth != s->fftLength && specWidth != s->fftLength / 2 + 1)
        return af_fail(AF_ERR_ARG, "cepstrogramObj_cepstrogram2Batch: specWidth=%d must be fftLength or fftLength/2+1",
                       specWidth);
    af_clear_error();
    int rc = ceps_check(s, cepNum, "cepstrogramObj_cepstrogram2Batch");
    if (rc || (rc = af_device_ready())) return rc;
    if (rows == 0) return AF_OK;
    CepsCall c = {s, cepNum, 0, 0, specWidth};
    const size_t outPer = (size_t)(s->fftLength / 2 + 1);
    const AfPlane pl[5] = {{mReal, (size_t)specWidth, AF_IN, 0}, {mImag, (size_t)specWidth, AF_IN, 0},
                           {cep, outPer, AF_OUT, 0}, {env, outPer, AF_OUT, 0}, {det, outPer, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, ceps2_chunk, &c, pl, 5, rows, AF_PIPE_CHUNK_BYTES);
}

/* :111-117.  All three outputs NULL: nothing to compute (the reference computes and drops the result). */
void cepstrogramObj_cepstrogram(CepstrogramObj s, int cepNum, float *dataArr, int dataLength,
                                float *mDataArr1, float *mDataArr2, float *mDataArr3) {
    if (!s) return;
    af_clear_error();
    if (ceps_check(s, cepNum, "cepstrogramObj_cepstrogram") || !dataArr || dataLength <= 0 ||
        (!mDataArr1 && !mDataArr2 && !mDataArr3))
        return;
    cepstrogramObj_cepstrogramBatch(s, cepNum, dataArr, dataLength, 1, mDataArr1, mDataArr2, mDataArr3,
                                    AFB200_MEM_HOST, NULL);
}

/* :119-125, with the caller's planes as the input (see include/afb200_cepstrogram.h) */
void cepstrogramObj_cepstrogram2(CepstrogramObj s, int cepNum, float *mRealArr, float *mImageArr, int nLength,
                                 float *mDataArr1, float *mDataArr2, float *mDataArr3) {
    if (!s) return;
    af_clear_error();
    if (ceps_check(s, cepNum, "cepstrogramObj_cepstrogram2") || !mRealArr || !mImageArr || nLength <= 0 ||
        (!mDataArr1 && !mDataArr2 && !mDataArr3))
        return;
    cepstrogramObj_cepstrogram2Batch(s, cepNum, mRealArr, mImageArr, nLength, s->fftLength, mDataArr1, mDataArr2,
                                     mDataArr3, AFB200_MEM_HOST, NULL);
}

void cepstrogramObj_free(CepstrogramObj s) {
    if (!s) return;
    af_pipe_free(&s->pipe);
    af_dev_free(s->dWindow);
    free(s->window);
    free(s);
}
