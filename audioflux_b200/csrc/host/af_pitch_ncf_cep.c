/* af_pitch_ncf_cep.c -- PitchNCFObj and PitchCEPObj of the C ABI (host C; compute = kernels/pitch_ncf_cep.cu, one launch
 * per staging chunk).  Interface spec: include/mir/_pitch_{ncf,cep}.h, behaviour src/mir/_pitch_{ncf,cep}.c (restated in
 * include/afb200_pitch_{ncf,cep}.h).  The parameter rules, the frame count, the streaming carry and the staging pipe are
 * the pitch trackers' common core (af_pitch_frames.c); the two objects add the window, uploaded at the first compute
 * call, and differ in the window rule, the refusals and the kernel's mode.  The reference keeps an FFT object, five
 * 2n-float buffers and a timeLength x 2n matrix per object. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

typedef struct {
    AfPitchFrames f;
    int mode, minIndex, maxIndex;
    float *window, *dWindow;      /* host n floats, and its device copy from the first compute call */
} PitchLag;

struct OpaquePitchNCF { PitchLag c; };
struct OpaquePitchCEP { PitchLag c; };

static void lag_free(PitchLag *c) {
    if (!c) return;
    af_pitch_frames_free(&c->f);
    af_dev_free(c->dWindow);
    free(c->window);
    free(c);
}

/* pitchNCFObj_new :77-164 / pitchCEPObj_new :77-166 and their initData; the window rule is the caller's */
static int lag_new(PitchLag **out, int mode, int *samplate, float *lowFre, float *highFre, int *radix2Exp,
                   int *slideLength, int winType, int *isContinue) {
    af_clear_error();
    *out = NULL;
    static const AfPitchRules rules[2] = {
        {"pitchNCFObj_new", AFB200_PITCH_NCF_MAX_EXP, "one frame's 2n-point transform is held in shared memory", 32,
         2000, 2000},
        {"pitchCEPObj_new", AFB200_PITCH_CEP_MAX_EXP, "one frame's 2n-point transform is held in shared memory", 32,
         2000, 2000}};
    const char *who = rules[mode].who;
    AfPitchFrames f;
    float lf, hf;
    if (af_pitch_frames_init(&f, &lf, &hf, &rules[mode], samplate, lowFre, highFre, radix2Exp, slideLength, isContinue))
        return -2;
    const int sr = f.samplate, n = f.n;
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
    c->f = f;
    c->mode = mode;
    c->minIndex = minIndex;
    c->maxIndex = maxIndex;
    *out = c;
    return 0;
}

typedef struct { const PitchLag *c; int dataLength, timeLength; } LagCall;

/* d[0] clips nb x dataLength, d[1] frequencies nb x T */
static int lag_chunk(void *ctx, int nb, float *const *d, void *st) {
    const LagCall *k = (const LagCall *)ctx;
    const PitchLag *c = k->c;
    AfPitchLagArgs a;
    a.data = d[0]; a.window = c->dWindow; a.fre = d[1];
    a.mode = c->mode; a.log2n = c->f.log2n; a.minIndex = c->minIndex; a.maxIndex = c->maxIndex;
    a.samplate = c->f.samplate;
    a.dataLength = k->dataLength; a.hop = c->f.slideLength; a.timeLength = k->timeLength; a.batch = nb;
    return af_launch_pitch_ncf_cep(&a, st);
}

static int lag_batch(PitchLag *c, const char *who, const float *data, int dataLength, int batch, float *freArr,
                     int memKind, void *stream) {
    int T, rc = af_pitch_batch_begin(c ? &c->f : NULL, who, data, dataLength, batch, freArr, &T);
    if (rc || !T || (!c->dWindow && (rc = af_dev_upload((void **)&c->dWindow, c->window,
                                                        sizeof(float) * (size_t)c->f.n))))
        return rc;
    LagCall k = {c, dataLength, T};
    const AfPlane pl[2] = {{data, (size_t)dataLength, AF_IN, 0}, {freArr, (size_t)T, AF_OUT, 0}};
    return af_run_batch(&c->f.pipe, memKind, stream, lag_chunk, &k, pl, 2, batch, AF_PIPE_CHUNK_BYTES);
}

/* pitchNCFObj_pitch :358-378 / pitchCEPObj_pitch :360-379 */
static void lag_pitch(PitchLag *c, const char *who, float *dataArr, int dataLength, float *freArr) {
    const float *x;
    int len;
    if (af_pitch_legacy_input(c ? &c->f : NULL, dataArr, dataLength, &x, &len) && freArr)
        lag_batch(c, who, x, len, 1, freArr, AFB200_MEM_HOST, NULL);
}

/* ---- PitchNCFObj: any window, Rect by default ---- */

int pitchNCFObj_new(PitchNCFObj *pitchNCFObj, int *samplate, float *lowFre, float *highFre, int *radix2Exp,
                    int *slideLength, WindowType *windowType, int *isContinue) {
    if (!pitchNCFObj) return -1;
    PitchLag *c;
    const int rc = lag_new(&c, AF_PITCH_NCF, samplate, lowFre, highFre, radix2Exp, slideLength,
                           windowType ? (int)*windowType : Window_Rect, isContinue);
    *pitchNCFObj = (PitchNCFObj)c;
    return rc;
}

int pitchNCFObj_calTimeLength(PitchNCFObj s, int dataLength) {
    return af_pitch_time_length(s ? &s->c.f : NULL, dataLength);
}

void pitchNCFObj_enableDebug(PitchNCFObj s, int isDebug) { (void)s; (void)isDebug; }

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
    const int rc = lag_new(&c, AF_PITCH_CEP, samplate, lowFre, highFre, radix2Exp, slideLength,
                           windowType && *windowType <= Window_Hamm ? (int)*windowType : Window_Hamm, isContinue);
    *pitchCEPObj = (PitchCEPObj)c;
    return rc;
}

int pitchCEPObj_calTimeLength(PitchCEPObj s, int dataLength) {
    return af_pitch_time_length(s ? &s->c.f : NULL, dataLength);
}

void pitchCEPObj_enableDebug(PitchCEPObj s, int isDebug) { (void)s; (void)isDebug; }

int pitchCEPObj_pitchBatch(PitchCEPObj s, const float *data, int dataLength, int batch, float *freArr, int memKind,
                           void *stream) {
    return lag_batch(s ? &s->c : NULL, "pitchCEPObj_pitchBatch", data, dataLength, batch, freArr, memKind, stream);
}

void pitchCEPObj_pitch(PitchCEPObj s, float *dataArr, int dataLength, float *freArr) {
    lag_pitch(s ? &s->c : NULL, "pitchCEPObj_pitch", dataArr, dataLength, freArr);
}

void pitchCEPObj_free(PitchCEPObj s) { lag_free(s ? &s->c : NULL); }
