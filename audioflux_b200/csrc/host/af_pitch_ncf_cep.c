/* af_pitch_ncf_cep.c -- PitchNCFObj and PitchCEPObj of the C ABI (host C; compute = kernels/pitch_ncf_cep.cu, one launch
 * per staging chunk).  Interface spec: include/mir/_pitch_{ncf,cep}.h, behaviour src/mir/_pitch_{ncf,cep}.c (restated in
 * include/afb200_pitch_{ncf,cep}.h).  The two objects share one core: the parameter rules, the window, the streaming
 * carry and the staging pipe; they differ in the window rule, the refusals and the kernel's mode.  The reference keeps
 * an FFT object, five 2n-float buffers and a timeLength x 2n matrix per object. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

typedef struct {
    int mode, samplate, log2n, n, slideLength, isContinue, isDebug;
    int minIndex, maxIndex;
    float *window, *dWindow;      /* host n floats, and its device copy from the first compute call */
    AfTail tail;
    AfPipe pipe;
} PitchLag;

struct OpaquePitchNCF { PitchLag c; };
struct OpaquePitchCEP { PitchLag c; };

static void lag_free(PitchLag *c) {
    if (!c) return;
    af_pipe_free(&c->pipe);
    af_tail_free(&c->tail);
    af_dev_free(c->dWindow);
    free(c->window);
    free(c);
}

/* pitchNCFObj_new :77-164 / pitchCEPObj_new :77-166 and their initData; the window rule is the caller's */
static int lag_new(PitchLag **out, int mode, const char *who, int *samplate, float *lowFre, float *highFre,
                   int *radix2Exp, int *slideLength, int winType, int *isContinue) {
    af_clear_error();
    *out = NULL;
    /* in the reference's order: highFre is checked against the lowFre already taken, and against the integer
     * samplate/2; a rejected highFre resets both ends to 32 / 2000 */
    const int sr = samplate && *samplate > 0 && *samplate <= 196000 ? *samplate : 32000;
    float lf = lowFre && *lowFre >= 27 ? *lowFre : 32, hf = 2000;
    if (highFre) {
        if (*highFre > lf && *highFre < sr / 2) hf = *highFre;
        else { lf = 32; hf = 2000; }
    }
    const int log2n = radix2Exp && *radix2Exp >= 1 && *radix2Exp <= 30 ? *radix2Exp : 12;
    const int maxExp = mode == AF_PITCH_NCF ? AFB200_PITCH_NCF_MAX_EXP : AFB200_PITCH_CEP_MAX_EXP;
    if (log2n > maxExp) {
        af_fail(-2, "%s: radix2Exp=%d; the largest supported is %d (one frame's 2n-point transform is held in shared "
                "memory)", who, log2n, maxExp);
        return -2;
    }
    const int n = 1 << log2n;
    /* initData: float quotients, rounded by roundf */
    const int minIndex = (int)roundf(sr / hf), maxIndex = (int)roundf(sr / lf);
    if (mode == AF_PITCH_NCF && maxIndex >= n) {
        af_fail(-3, "%s: maxIndex=%d (samplate=%d, lowFre=%g) is not below n=%d; the reference copies 2 maxIndex + 1 "
                "floats into its 2n-float buffer", who, maxIndex, sr, (double)lf, n);
        return -3;
    }
    if (mode == AF_PITCH_CEP && maxIndex > 2 * n - 1) {
        af_fail(-3, "%s: maxIndex=%d (samplate=%d, lowFre=%g) is past the 2n=%d-entry cepstrum; the reference's peak "
                "search reads past its row", who, maxIndex, sr, (double)lf, 2 * n);
        return -3;
    }
    if (mode == AF_PITCH_NCF && minIndex < 1) {
        af_fail(-3, "%s: minIndex=%d (samplate=%d, highFre=%g); the reference clears a negative count of floats", who,
                minIndex, sr, (double)hf);
        return -3;
    }
    if (maxIndex < minIndex) {
        af_fail(-3, "%s: the lag range minIndex=%d .. maxIndex=%d is empty (samplate=%d, lowFre=%g, highFre=%g)", who,
                minIndex, maxIndex, sr, (double)lf, (double)hf);
        return -3;
    }
    PitchLag *c = (PitchLag *)calloc(1, sizeof(PitchLag));
    if (c) c->window = (float *)malloc(sizeof(float) * (size_t)n);
    if (!c || !c->window || af_window_fft(winType, n, c->window)) { lag_free(c); return -1; }
    c->mode = mode;
    c->samplate = sr;
    c->log2n = log2n;
    c->n = n;
    c->slideLength = slideLength && *slideLength > 0 ? *slideLength : n / 4;
    if (c->slideLength < 1) c->slideLength = 1;                 /* n/4 at n = 2: the reference divides by zero */
    c->isContinue = isContinue ? *isContinue : 0;
    c->minIndex = minIndex;
    c->maxIndex = maxIndex;
    *out = c;
    return 0;
}

static int frames(const PitchLag *c, int dataLength) {
    return dataLength < c->n ? 0 : (dataLength - c->n) / c->slideLength + 1;
}

static int lag_time_length(const PitchLag *c, int dataLength) {
    if (!c) return 0;
    return frames(c, c->isContinue ? dataLength + c->tail.length : dataLength);
}

typedef struct { const PitchLag *c; int dataLength, timeLength; } LagCall;

/* d[0] clips nb x dataLength, d[1] frequencies nb x T */
static int lag_chunk(void *ctx, int nb, float *const *d, void *st) {
    const LagCall *k = (const LagCall *)ctx;
    const PitchLag *c = k->c;
    AfPitchLagArgs a;
    a.data = d[0]; a.window = c->dWindow; a.fre = d[1];
    a.mode = c->mode; a.log2n = c->log2n; a.minIndex = c->minIndex; a.maxIndex = c->maxIndex; a.samplate = c->samplate;
    a.dataLength = k->dataLength; a.hop = c->slideLength; a.timeLength = k->timeLength; a.batch = nb;
    return af_launch_pitch_ncf_cep(&a, st);
}

static int lag_batch(PitchLag *c, const char *who, const float *data, int dataLength, int batch, float *freArr,
                     int memKind, void *stream) {
    const int T = c && dataLength > 0 ? frames(c, dataLength) : 0;
    if (!c || !data || (!freArr && T > 0 && batch > 0) || dataLength <= 0 || batch < 0)   /* freArr may be NULL when empty */
        return af_fail(AF_ERR_ARG, "%s: bad argument", who);
    af_clear_error();
    int rc = af_device_ready();
    if (rc || (!c->dWindow && (rc = af_dev_upload((void **)&c->dWindow, c->window, sizeof(float) * (size_t)c->n))))
        return rc;
    if (batch == 0 || T == 0) return AF_OK;
    LagCall k = {c, dataLength, T};
    const AfPlane pl[2] = {{data, (size_t)dataLength, AF_IN, 0}, {freArr, (size_t)T, AF_OUT, 0}};
    return af_run_batch(&c->pipe, memKind, stream, lag_chunk, &k, pl, 2, batch, AF_PIPE_CHUNK_BYTES);
}

/* pitchNCFObj_pitch :358-378 / pitchCEPObj_pitch :360-379 */
static void lag_pitch(PitchLag *c, const char *who, float *dataArr, int dataLength, float *freArr) {
    if (!c) return;
    af_clear_error();
    if (!dataArr || dataLength <= 0) return;
    const float *x = dataArr;
    if (c->isContinue && !af_tail_assemble(&c->tail, c->n, c->slideLength, dataArr, dataLength, &x, &dataLength)) return;
    if (!freArr || frames(c, dataLength) == 0) return;
    lag_batch(c, who, x, dataLength, 1, freArr, AFB200_MEM_HOST, NULL);
}

/* ---- PitchNCFObj: any window, Rect by default ---- */

int pitchNCFObj_new(PitchNCFObj *pitchNCFObj, int *samplate, float *lowFre, float *highFre, int *radix2Exp,
                    int *slideLength, WindowType *windowType, int *isContinue) {
    if (!pitchNCFObj) return -1;
    PitchLag *c;
    const int rc = lag_new(&c, AF_PITCH_NCF, "pitchNCFObj_new", samplate, lowFre, highFre, radix2Exp, slideLength,
                           windowType ? (int)*windowType : Window_Rect, isContinue);
    *pitchNCFObj = (PitchNCFObj)c;
    return rc;
}

int pitchNCFObj_calTimeLength(PitchNCFObj s, int dataLength) { return lag_time_length(s ? &s->c : NULL, dataLength); }

void pitchNCFObj_enableDebug(PitchNCFObj s, int isDebug) {
    if (s) s->c.isDebug = isDebug;
}

int pitchNCFObj_pitchBatch(PitchNCFObj s, const float *data, int dataLength, int batch, float *freArr, int memKind,
                           void *stream) {
    return lag_batch(s ? &s->c : NULL, "pitchNCFObj_pitchBatch", data, dataLength, batch, freArr, memKind, stream);
}

void pitchNCFObj_pitch(PitchNCFObj s, float *dataArr, int dataLength, float *freArr) {
    lag_pitch(s ? &s->c : NULL, "pitchNCFObj_pitch", dataArr, dataLength, freArr);
}

void pitchNCFObj_free(PitchNCFObj s) { lag_free(s ? &s->c : NULL); }

/* ---- PitchCEPObj: Rect, Hann or Hamm (:127-131), Hamm otherwise ---- */

int pitchCEPObj_new(PitchCEPObj *pitchCEPObj, int *samplate, float *lowFre, float *highFre, int *radix2Exp,
                    int *slideLength, WindowType *windowType, int *isContinue) {
    if (!pitchCEPObj) return -1;
    PitchLag *c;
    const int rc = lag_new(&c, AF_PITCH_CEP, "pitchCEPObj_new", samplate, lowFre, highFre, radix2Exp, slideLength,
                           windowType && *windowType <= Window_Hamm ? (int)*windowType : Window_Hamm, isContinue);
    *pitchCEPObj = (PitchCEPObj)c;
    return rc;
}

int pitchCEPObj_calTimeLength(PitchCEPObj s, int dataLength) { return lag_time_length(s ? &s->c : NULL, dataLength); }

void pitchCEPObj_enableDebug(PitchCEPObj s, int isDebug) {
    if (s) s->c.isDebug = isDebug;
}

int pitchCEPObj_pitchBatch(PitchCEPObj s, const float *data, int dataLength, int batch, float *freArr, int memKind,
                           void *stream) {
    return lag_batch(s ? &s->c : NULL, "pitchCEPObj_pitchBatch", data, dataLength, batch, freArr, memKind, stream);
}

void pitchCEPObj_pitch(PitchCEPObj s, float *dataArr, int dataLength, float *freArr) {
    lag_pitch(s ? &s->c : NULL, "pitchCEPObj_pitch", dataArr, dataLength, freArr);
}

void pitchCEPObj_free(PitchCEPObj s) { lag_free(s ? &s->c : NULL); }
