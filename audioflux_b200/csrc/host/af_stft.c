/* af_stft.c -- STFT object of the C ABI (host C; compute = kernels/stft_generic.cu).
 * Interface spec: src/stft_algorithm.h:14-40, behaviour src/stft_algorithm.c. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueSTFT {
    int radix2Exp, fftLength, slideLength;
    WindowType windowType;
    int useWindow;                 /* window multiply needed (non-rect or user window) */
    float *window;                 /* host, fftLength */
    int isPad;
    PaddingPositionType position;
    PaddingModeType mode;
    float padValue1, padValue2;
    /* device side (lazy) */
    int windowDirty;
    float *dWindow;
    AfDevBuf dFrames;              /* inverse: frames before the overlap-add */
    AfPipe pipe;
    /* streaming (isContinue, stft_algorithm.c:474-599) */
    int isContinue;
    AfTail tail;
    int timeLength;                /* frames of the last stftObj_stft call */
};

int stftObj_new(STFTObj *out, int radix2Exp, WindowType *windowType, int *slideLength, int *isContinue) {
    af_clear_error();
    if (!out) return -1;
    *out = NULL;
    if (radix2Exp < 1 || radix2Exp > 30) return -100;
    STFTObj s = (STFTObj)calloc(1, sizeof(struct OpaqueSTFT));
    if (!s) return -1;
    s->isContinue = isContinue ? *isContinue != 0 : 0;
    s->radix2Exp = radix2Exp;
    s->fftLength = 1 << radix2Exp;
    s->windowType = windowType ? *windowType : Window_Rect;
    s->slideLength = s->fftLength / 4;
    if (slideLength && *slideLength > 0) s->slideLength = *slideLength;
    s->window = (float *)malloc(sizeof(float) * (size_t)s->fftLength);
    if (!s->window) { free(s); return -1; }
    af_window_fft(s->windowType, s->fftLength, s->window);
    s->useWindow = s->windowType != Window_Rect;
    s->position = PaddingPosition_Center;
    s->mode = PaddingMode_Constant;
    s->windowDirty = 1;
    *out = s;
    return 0;
}

void stftObj_setSlideLength(STFTObj s, int slideLength) { if (s && slideLength > 0) s->slideLength = slideLength; }
void stftObj_enablePadding(STFTObj s, int flag) { if (s) s->isPad = flag; }
void stftObj_enableContinue(STFTObj s, int flag) { if (s) { s->isContinue = flag != 0; } }
void stftObj_setPadding(STFTObj s, PaddingPositionType *position, PaddingModeType *mode, float *v1, float *v2) {
    if (!s || !s->isPad) return;          /* like the reference: only honoured once padding is enabled */
    if (position) s->position = *position;
    if (mode) s->mode = *mode;
    if (v1) s->padValue1 = *v1;
    if (v2) s->padValue2 = *v2;
}
void stftObj_useWindowDataArr(STFTObj s, float *w) {
    if (!s || !w) return;
    memcpy(s->window, w, sizeof(float) * (size_t)s->fftLength);
    s->useWindow = 1; s->windowDirty = 1;
}
float *stftObj_getWindowDataArr(STFTObj s) { return s ? s->window : NULL; }

static int time_length(const struct OpaqueSTFT *s, int dataLength) {
    if (!s->isPad) return dataLength < s->fftLength ? 0 : (dataLength - s->fftLength) / s->slideLength + 1;
    return dataLength <= 0 ? 0 : dataLength / s->slideLength + 1;
}
int stftObj_calTimeLength(STFTObj s, int dataLength) {
    if (!s) return 0;
    if (!s->isPad && s->isContinue) dataLength += s->tail.length;         /* stft_algorithm.c:242-245 */
    return time_length(s, dataLength);
}
int stftObj_calDataLength(STFTObj s, int timeLength) { return s ? (timeLength - 1) * s->slideLength + s->fftLength : 0; }
void stftObj_debug(STFTObj s) {
    if (s) printf("stft params is: fftLength=%d, slideLength=%d\n", s->fftLength, s->slideLength);
}

static int stft_device(STFTObj s) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (s->windowDirty) {
        af_dev_free(s->dWindow); s->dWindow = NULL;
        if ((rc = af_dev_upload((void **)&s->dWindow, s->window, sizeof(float) * (size_t)s->fftLength))) return rc;
        s->windowDirty = 0;
    }
    return AF_OK;
}

static int stft_frame_src(STFTObj s, int dataLength, int batch, AfFrameSrc *src) {
    memset(src, 0, sizeof(*src));
    src->fftLength = s->fftLength; src->slideLength = s->slideLength;
    src->dataLength = dataLength; src->batch = batch;
    src->timeLength = time_length(s, dataLength);
    src->validLength = dataLength;
    src->window = s->useWindow ? s->dWindow : NULL;
    if (s->isPad) {
        /* the tail that does not fill a hop is dropped when more than one frame exists (stft_algorithm.c:813-826);
         * then fftLength samples are added: n/2 + n/2 (Center), n left (Left) or n right (Right), holding a constant,
         * the mirror image or the periodic extension of the kept samples (__stftObj_dealPadData, :583-694) */
        if (src->timeLength > 1) src->validLength = dataLength - dataLength % s->slideLength;
        src->padLeft = s->position == PaddingPosition_Center ? s->fftLength / 2
                     : s->position == PaddingPosition_Left ? s->fftLength : 0;
        src->padMode = s->mode;
        if (s->position == PaddingPosition_Center) { src->padValue1 = s->padValue1; src->padValue2 = s->padValue2; }
        else src->padValue1 = src->padValue2 = (float)(int)s->padValue1;   /* __vpad_left1/right1 take an int (:641-652) */
    }
    return AF_OK;
}

/* streaming bookkeeping of __stftObj_dealData (stft_algorithm.c:474-599, non-padding mode) */
int af_tail_assemble(AfTail *t, int n, int hop, const float *data, int dataLength, const float **cur, int *curLength) {
    if (!t->buf) {
        t->buf = (float *)calloc((size_t)n + (size_t)hop + 1, sizeof(float));
        if (!t->buf) return 0;
    }
    const int total = t->length + dataLength;
    if (total < n) {                                          /* not a frame yet: keep everything */
        if (t->length >= 0) memcpy(t->buf + t->length, data, sizeof(float) * (size_t)dataLength);
        else if (dataLength + t->length > 0) memcpy(t->buf, data - t->length, sizeof(float) * (size_t)(dataLength + t->length));
        t->length = total;
        return 0;
    }
    const int tailLen = (total - n) % hop + (n - hop);      /* __calTimeAndTailLen */
    if ((size_t)total + (size_t)n > t->curCap) {
        free(t->cur);
        t->curCap = (size_t)total + (size_t)n;
        t->cur = (float *)malloc(sizeof(float) * t->curCap);
        if (!t->cur) { t->curCap = 0; return 0; }
    }
    int len = 0;
    if (t->length < 0) {
        len = dataLength + t->length;
        memcpy(t->cur, data - t->length, sizeof(float) * (size_t)len);
    } else {
        if (t->length > 0) memcpy(t->cur, t->buf, sizeof(float) * (size_t)t->length);
        memcpy(t->cur + t->length, data, sizeof(float) * (size_t)dataLength);
        len = t->length + dataLength;
    }
    if (tailLen > 0) memcpy(t->buf, t->cur + (len - tailLen), sizeof(float) * (size_t)tailLen);
    t->length = tailLen;
    *cur = t->cur; *curLength = len;
    return 1;
}

void af_tail_free(AfTail *t) { free(t->buf); free(t->cur); memset(t, 0, sizeof(*t)); }

typedef struct { STFTObj s; int dataLength, mode; } StftCall;

static int stft_chunk(void *p, int nb, float *const *d, void *st) {
    const StftCall *c = (const StftCall *)p;
    AfFrameSrc src;
    int rc = stft_frame_src(c->s, c->dataLength, nb, &src);
    if (rc) return rc;
    src.data = d[0];
    return af_launch_stft(&src, c->mode, 1.0f, d[1], d[2], st);
}

/* mode AF_STFT_HALF (planes batch x T x (n/2+1)) or AF_STFT_FULL (mirrored, batch x T x n) */
static int stft_run(STFTObj s, const float *data, int dataLength, int batch, int mode, float *re, float *im,
                    int memKind, void *stream) {
    const size_t outPer = (size_t)time_length(s, dataLength) * (mode == AF_STFT_FULL ? s->fftLength : s->fftLength / 2 + 1);
    StftCall c = {s, dataLength, mode};
    const AfPlane pl[3] = {{data, (size_t)dataLength, AF_IN, 0}, {re, outPer, AF_OUT, 0}, {im, outPer, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, stft_chunk, &c, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

void stftObj_stft(STFTObj s, float *dataArr, int dataLength, float *mRealArr, float *mImageArr) {
    if (!s || !dataArr || dataLength <= 0 || !mRealArr || !mImageArr) return;
    const float *x = dataArr;
    int len = dataLength;
    if (s->isContinue && !s->isPad && !af_tail_assemble(&s->tail, s->fftLength, s->slideLength, dataArr, dataLength, &x, &len)) {
        s->timeLength = 0;
        return;
    }
    af_clear_error();
    if (stft_device(s)) return;
    s->timeLength = time_length(s, len);
    if (s->timeLength <= 0) return;
    stft_run(s, x, len, 1, AF_STFT_FULL, mRealArr, mImageArr, AFB200_MEM_HOST, NULL);
}

int stftObj_stftBatch(STFTObj s, const float *data, int dataLength, int batch, float *mReal, float *mImag,
                      int memKind, void *stream) {
    if (!s || !data || !mReal || !mImag || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "stftObj_stftBatch: bad argument");
    af_clear_error();
    int rc = stft_device(s);
    if (rc) return rc;
    if (time_length(s, dataLength) <= 0) return AF_OK;
    return stft_run(s, data, dataLength, batch, AF_STFT_HALF, mReal, mImag, memKind, stream);
}

/* ---- inverse: planes [batch x T x width] -> data [batch x ((T-1)*hop + n)]  (stft_algorithm.c:304-409) ----
 * width = fftLength (full mirrored planes, the reference layout) or fftLength/2+1 (what stftObj_stftBatch produces).
 * As in the reference the frames are ADDED to what `data` holds before the division by the window sum, so the
 * caller passes a zeroed buffer. */
typedef struct { STFTObj s; int timeLength, specWidth, methodType; } IstftCall;

static int istft_chunk(void *p, int nb, float *const *d, void *st) {
    const IstftCall *c = (const IstftCall *)p;
    STFTObj s = c->s;
    int rc = af_devbuf_reserve(&s->dFrames, sizeof(float) * (size_t)nb * c->timeLength * s->fftLength);
    if (rc) return rc;
    return af_launch_istft(d[0], d[1], c->specWidth, s->fftLength, s->slideLength, c->timeLength, nb,
                           s->useWindow ? s->dWindow : NULL, c->methodType, (float *)s->dFrames.ptr, d[2], st);
}

int stftObj_istftBatch(STFTObj s, const float *mReal, const float *mImag, int timeLength, int batch, int specWidth,
                       int methodType, float *data, int memKind, void *stream) {
    if (!s || !mReal || !mImag || !data || timeLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "stftObj_istftBatch: bad argument");
    if (specWidth != s->fftLength && specWidth != s->fftLength / 2 + 1)
        return af_fail(AF_ERR_ARG, "stftObj_istftBatch: specWidth=%d must be fftLength or fftLength/2+1", specWidth);
    af_clear_error();
    int rc = stft_device(s);
    if (rc) return rc;
    IstftCall c = {s, timeLength, specWidth, methodType};
    const size_t plane = (size_t)timeLength * specWidth;
    const AfPlane pl[3] = {{mReal, plane, AF_IN, 0}, {mImag, plane, AF_IN, 0},
                           {data, (size_t)(timeLength - 1) * s->slideLength + s->fftLength, AF_INOUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, istft_chunk, &c, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

void stftObj_istft(STFTObj s, float *mRealArr, float *mImageArr, int timeLength, int methodType, float *dataArr) {
    if (!s || !mRealArr || !mImageArr || !dataArr || timeLength <= 0) return;
    stftObj_istftBatch(s, mRealArr, mImageArr, timeLength, 1, s->fftLength, methodType, dataArr, AFB200_MEM_HOST, NULL);
}

void stftObj_free(STFTObj s) {
    if (!s) return;
    af_devbuf_free(&s->dFrames);
    af_pipe_free(&s->pipe);
    af_dev_free(s->dWindow);
    free(s->window);
    af_tail_free(&s->tail);
    free(s);
}
