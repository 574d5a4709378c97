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
    int devReady, windowDirty;
    void *stream;
    float *dWindow;
    AfDevBuf dIn, dRe, dIm, dFrames;
    AfPipe pipe;                   /* host-pointer batches: chunked copy-in / transform / copy-out */
    int pipeLength;
    /* streaming (isContinue, stft_algorithm.c:474-599): the samples that did not complete a hop are carried to the next call */
    int isContinue;
    float *tail;                   /* host, fftLength + slideLength floats */
    int tailLength;                /* may be negative when slideLength > fftLength: samples of the next call to skip */
    float *cur; size_t curCap;     /* host staging: tail + new samples */
    int timeLength;                /* frames of the last stftObj_stft call */
};

int stftObj_new(STFTObj *out, int radix2Exp, WindowType *windowType, int *slideLength, int *isContinue) {
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
    if (!s->isPad && s->isContinue) dataLength += s->tailLength;         /* stft_algorithm.c:242-245 */
    return time_length(s, dataLength);
}
int stftObj_calDataLength(STFTObj s, int timeLength) { return s ? (timeLength - 1) * s->slideLength + s->fftLength : 0; }
void stftObj_debug(STFTObj s) {
    if (s) printf("stft params is: fftLength=%d, slideLength=%d\n", s->fftLength, s->slideLength);
}

static int stft_device(STFTObj s) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (!s->devReady) {
        if ((rc = af_stream_create(&s->stream))) return rc;
        s->devReady = 1;
    }
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

/* streaming bookkeeping of __stftObj_dealData (stft_algorithm.c:474-599, non-padding mode): returns the samples to
 * transform (tail of the previous calls + the new ones) in *cur / *curLength, or 0 when they do not fill a frame yet */
static int stft_continue_assemble(STFTObj s, const float *data, int dataLength, const float **cur, int *curLength) {
    const int n = s->fftLength, hop = s->slideLength;
    if (!s->tail) {
        s->tail = (float *)calloc((size_t)n + (size_t)hop + 1, sizeof(float));
        if (!s->tail) return 0;
    }
    const int total = s->tailLength + dataLength;
    if (total < n) {                                          /* not a frame yet: keep everything */
        if (s->tailLength >= 0) memcpy(s->tail + s->tailLength, data, sizeof(float) * (size_t)dataLength);
        else if (dataLength + s->tailLength > 0) memcpy(s->tail, data - s->tailLength, sizeof(float) * (size_t)(dataLength + s->tailLength));
        s->tailLength = total;
        s->timeLength = 0;
        return 0;
    }
    const int tailLen = (total - n) % hop + (n - hop);      /* __calTimeAndTailLen */
    if ((size_t)total + (size_t)n > s->curCap) {
        free(s->cur);
        s->curCap = (size_t)total + (size_t)n;
        s->cur = (float *)malloc(sizeof(float) * s->curCap);
        if (!s->cur) { s->curCap = 0; return 0; }
    }
    int len = 0;
    if (s->tailLength < 0) {
        len = dataLength + s->tailLength;
        memcpy(s->cur, data - s->tailLength, sizeof(float) * (size_t)len);
    } else {
        if (s->tailLength > 0) memcpy(s->cur, s->tail, sizeof(float) * (size_t)s->tailLength);
        memcpy(s->cur + s->tailLength, data, sizeof(float) * (size_t)dataLength);
        len = s->tailLength + dataLength;
    }
    if (tailLen > 0) memcpy(s->tail, s->cur + (len - tailLen), sizeof(float) * (size_t)tailLen);
    s->tailLength = tailLen;
    *cur = s->cur; *curLength = len;
    return 1;
}

/* the same bookkeeping for objects that frame through an STFT object of their own (SpectrogramObj streaming) */
int af_stft_continue_assemble(STFTObj s, const float *data, int dataLength, const float **cur, int *curLength) {
    if (!s || !data || dataLength <= 0) return 0;
    return stft_continue_assemble(s, data, dataLength, cur, curLength);
}

void stftObj_stft(STFTObj s, float *dataArr, int dataLength, float *mRealArr, float *mImageArr) {
    if (!s || !dataArr || dataLength <= 0 || !mRealArr || !mImageArr) return;
    af_clear_error();
    const float *x = dataArr;
    int len = dataLength;
    if (s->isContinue && !s->isPad) {
        if (!stft_continue_assemble(s, dataArr, dataLength, &x, &len)) return;
    }
    if (stft_device(s)) return;
    AfFrameSrc src;
    if (stft_frame_src(s, len, 1, &src)) return;
    s->timeLength = src.timeLength;
    if (src.timeLength <= 0) return;
    size_t plane = sizeof(float) * (size_t)src.timeLength * s->fftLength;
    if (af_devbuf_reserve(&s->dIn, sizeof(float) * (size_t)len) || af_devbuf_reserve(&s->dRe, plane) ||
        af_devbuf_reserve(&s->dIm, plane)) return;
    if (af_memcpy_h2d(s->dIn.ptr, x, sizeof(float) * (size_t)len, s->stream)) return;
    src.data = (const float *)s->dIn.ptr;
    if (af_launch_stft(&src, AF_STFT_FULL, 1.0f, (float *)s->dRe.ptr, (float *)s->dIm.ptr, s->stream)) return;
    if (af_memcpy_d2h(mRealArr, s->dRe.ptr, plane, s->stream) || af_memcpy_d2h(mImageArr, s->dIm.ptr, plane, s->stream)) return;
    af_stream_sync(s->stream);
}

static int stft_chunk(void *obj, const float *dIn, int nb, float *dOut0, float *dOut1, void *st) {
    STFTObj s = (STFTObj)obj;
    AfFrameSrc src;
    int rc = stft_frame_src(s, s->pipeLength, nb, &src);
    if (rc) return rc;
    src.data = dIn;
    return af_launch_stft(&src, AF_STFT_HALF, 1.0f, dOut0, dOut1, st);
}

int stftObj_stftBatch(STFTObj s, const float *data, int dataLength, int batch, float *mReal, float *mImag,
                      int memKind, void *stream) {
    if (!s || !data || !mReal || !mImag || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "stftObj_stftBatch: bad argument");
    af_clear_error();
    int rc = stft_device(s);
    if (rc) return rc;
    AfFrameSrc src;
    if ((rc = stft_frame_src(s, dataLength, batch, &src))) return rc;
    if (src.timeLength <= 0) return AF_OK;
    void *st = stream ? stream : s->stream;
    if (memKind == AFB200_MEM_DEVICE) {
        st = stream;                      /* NULL = the CUDA default stream */
        src.data = data;
        if ((rc = af_launch_stft(&src, AF_STFT_HALF, 1.0f, mReal, mImag, st))) return rc;
        return AF_OK;                       /* asynchronous on the caller's stream */
    }
    s->pipeLength = dataLength;
    return af_pipe_run(&s->pipe, stft_chunk, s, data, (size_t)dataLength, batch, mReal, mImag,
                       (size_t)src.timeLength * (s->fftLength / 2 + 1), st);
}

/* ---- inverse: planes [batch x T x width] -> data [batch x ((T-1)*hop + n)]  (stft_algorithm.c:304-409) ----
 * width = fftLength (full mirrored planes, the reference layout) or fftLength/2+1 (what stftObj_stftBatch produces).
 * As in the reference the frames are ADDED to what `data` holds before the division by the window sum, so the
 * caller passes a zeroed buffer. */
int stftObj_istftBatch(STFTObj s, const float *mReal, const float *mImag, int timeLength, int batch, int specWidth,
                       int methodType, float *data, int memKind, void *stream) {
    if (!s || !mReal || !mImag || !data || timeLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "stftObj_istftBatch: bad argument");
    if (specWidth != s->fftLength && specWidth != s->fftLength / 2 + 1)
        return af_fail(AF_ERR_ARG, "stftObj_istftBatch: specWidth=%d must be fftLength or fftLength/2+1", specWidth);
    af_clear_error();
    int rc = stft_device(s);
    if (rc) return rc;
    const int n = s->fftLength, dataLength = (timeLength - 1) * s->slideLength + n;
    const size_t plane = sizeof(float) * (size_t)batch * timeLength * specWidth;
    const size_t frameB = sizeof(float) * (size_t)batch * timeLength * n, dataB = sizeof(float) * (size_t)batch * dataLength;
    if ((rc = af_devbuf_reserve(&s->dFrames, frameB))) return rc;
    const float *win = s->useWindow ? s->dWindow : NULL;
    if (memKind == AFB200_MEM_DEVICE)
        return af_launch_istft(mReal, mImag, specWidth, n, s->slideLength, timeLength, batch, win, methodType,
                               (float *)s->dFrames.ptr, data, stream);
    void *st = stream ? stream : s->stream;
    if ((rc = af_devbuf_reserve(&s->dRe, plane)) || (rc = af_devbuf_reserve(&s->dIm, plane)) || (rc = af_devbuf_reserve(&s->dIn, dataB))) return rc;
    if ((rc = af_memcpy_h2d(s->dRe.ptr, mReal, plane, st)) || (rc = af_memcpy_h2d(s->dIm.ptr, mImag, plane, st)) ||
        (rc = af_memcpy_h2d(s->dIn.ptr, data, dataB, st))) return rc;
    if ((rc = af_launch_istft((const float *)s->dRe.ptr, (const float *)s->dIm.ptr, specWidth, n, s->slideLength, timeLength,
                              batch, win, methodType, (float *)s->dFrames.ptr, (float *)s->dIn.ptr, st))) return rc;
    if ((rc = af_memcpy_d2h(data, s->dIn.ptr, dataB, st))) return rc;
    return af_stream_sync(st);
}

void stftObj_istft(STFTObj s, float *mRealArr, float *mImageArr, int timeLength, int methodType, float *dataArr) {
    if (!s || !mRealArr || !mImageArr || !dataArr || timeLength <= 0) return;
    stftObj_istftBatch(s, mRealArr, mImageArr, timeLength, 1, s->fftLength, methodType, dataArr, AFB200_MEM_HOST, NULL);
}

void stftObj_free(STFTObj s) {
    if (!s) return;
    af_devbuf_free(&s->dIn); af_devbuf_free(&s->dRe); af_devbuf_free(&s->dIm); af_devbuf_free(&s->dFrames);
    af_pipe_free(&s->pipe);
    af_dev_free(s->dWindow);
    af_stream_destroy(s->stream);
    free(s->window); free(s->tail); free(s->cur);
    free(s);
}
