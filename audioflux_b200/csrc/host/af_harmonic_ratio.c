/* af_harmonic_ratio.c -- HarmonicRatioObj of the C ABI (host C; compute = kernels/harmonic_ratio.cu, two launches per
 * staging chunk).  Interface spec: include/mir/harmonicRatio_algorithm.h, behaviour src/mir/harmonicRatio_algorithm.c.
 * The object keeps its window (uploaded at the first compute call) and the device workspace of one crossing index per
 * frame of a chunk; the reference keeps an FFT object and seven N-float buffers. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueHarmonicRatio {
    int samplate, log2w, windowLength, slideLength, maxLength;
    float *window;        /* host, W (af_window_fft(Window_Hamm)) */
    float *dWindow;
    AfDevBuf dMinIdx;     /* one int per frame of the current chunk */
    AfPipe pipe;
};

int harmonicRatioObj_new(HarmonicRatioObj *harmonicRatioObj, int *samplate, float *lowFre, int *radix2Exp,
                         WindowType *windowType, int *slideLength) {
    af_clear_error();
    (void)windowType;                                              /* never read: the window is Hamming (:119) */
    if (!harmonicRatioObj) return -1;
    *harmonicRatioObj = NULL;
    const int sr = samplate && *samplate > 0 && *samplate <= 196000 ? *samplate : 32000;     /* :85-89 */
    const float lf = lowFre && *lowFre > 0 && *lowFre < sr / 2 ? *lowFre : 25.f;              /* :91-95 */
    const int log2w = radix2Exp && *radix2Exp + 1 >= 1 && *radix2Exp + 1 <= 30 ? *radix2Exp : 11;   /* :97-101 */
    if (log2w > AFB200_HARMONIC_RATIO_MAX_EXP) {
        af_fail(-2, "harmonicRatioObj_new: radix2Exp=%d; the largest supported is %d (one frame's transforms are held "
                "in shared memory)", log2w, AFB200_HARMONIC_RATIO_MAX_EXP);
        return -2;
    }
    const int W = 1 << log2w;
    const float q = floorf(sr / lf);                               /* :112-115, capped before the conversion */
    const int maxLength = q > (float)(W - 1) ? W - 1 : (int)q;
    if (maxLength < 1) {
        af_fail(-3, "harmonicRatioObj_new: maxLength=%d (samplate=%d, lowFre=%g, window %d); at least 1 is needed (the "
                "reference reads a stale power bin there)", maxLength, sr, (double)lf, W);
        return -3;
    }
    HarmonicRatioObj s = (HarmonicRatioObj)calloc(1, sizeof(struct OpaqueHarmonicRatio));
    if (!s) return -1;
    s->samplate = sr;
    s->log2w = log2w;
    s->windowLength = W;
    s->slideLength = slideLength && *slideLength > 0 ? *slideLength : W / 4;                   /* :105-110 */
    if (s->slideLength < 1) s->slideLength = 1;                    /* W / 4 at W = 2: the reference divides by zero */
    s->maxLength = maxLength;
    s->window = (float *)malloc(sizeof(float) * (size_t)W);
    if (!s->window || af_window_fft(Window_Hamm, W, s->window)) { harmonicRatioObj_free(s); return -1; }
    *harmonicRatioObj = s;
    return 0;
}

int harmonicRatioObj_calTimeLength(HarmonicRatioObj s, int dataLength) {
    if (!s || dataLength < s->windowLength) return 0;
    return (dataLength - s->windowLength) / s->slideLength + 1;
}

typedef struct { HarmonicRatioObj s; int dataLength, timeLength; } HrCall;

/* d[0] clips nb x dataLength, d[1] values nb x T */
static int hr_chunk(void *ctx, int nb, float *const *d, void *st) {
    const HrCall *c = (const HrCall *)ctx;
    const HarmonicRatioObj s = c->s;
    int rc = af_devbuf_reserve(&s->dMinIdx, sizeof(int) * (size_t)nb * c->timeLength);
    if (rc) return rc;
    AfHarmonicRatioArgs a;
    a.data = d[0]; a.window = s->dWindow; a.value = d[1]; a.minIdx = (int *)s->dMinIdx.ptr;
    a.log2w = s->log2w; a.maxLength = s->maxLength; a.dataLength = c->dataLength; a.hop = s->slideLength;
    a.timeLength = c->timeLength; a.batch = nb;
    return af_launch_harmonic_ratio(&a, st);
}

int harmonicRatioObj_harmonicRatioBatch(HarmonicRatioObj s, const float *data, int dataLength, int batch, float *value,
                                        int memKind, void *stream) {
    const int T = harmonicRatioObj_calTimeLength(s, dataLength);
    if (!s || !data || (!value && T > 0 && batch > 0) || dataLength <= 0 || batch < 0)   /* value may be NULL when empty */
        return af_fail(AF_ERR_ARG, "harmonicRatioObj_harmonicRatioBatch: bad argument");
    af_clear_error();
    int rc = af_device_ready();
    if (rc || (!s->dWindow && (rc = af_dev_upload((void **)&s->dWindow, s->window, sizeof(float) * (size_t)s->windowLength))))
        return rc;
    if (batch == 0 || T == 0) return AF_OK;
    HrCall c = {s, dataLength, T};
    const AfPlane pl[2] = {{data, (size_t)dataLength, AF_IN, 0}, {value, (size_t)T, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, hr_chunk, &c, pl, 2, batch, AF_PIPE_CHUNK_BYTES);
}

/* :172-287 */
void harmonicRatioObj_harmonicRatio(HarmonicRatioObj s, float *dataArr, int dataLength, float *valueArr) {
    if (!s) return;
    af_clear_error();
    if (!dataArr || !valueArr || harmonicRatioObj_calTimeLength(s, dataLength) == 0) return;
    harmonicRatioObj_harmonicRatioBatch(s, dataArr, dataLength, 1, valueArr, AFB200_MEM_HOST, NULL);
}

void harmonicRatioObj_free(HarmonicRatioObj s) {
    if (!s) return;
    af_pipe_free(&s->pipe);
    af_devbuf_free(&s->dMinIdx);
    af_dev_free(s->dWindow);
    free(s->window);
    free(s);
}
