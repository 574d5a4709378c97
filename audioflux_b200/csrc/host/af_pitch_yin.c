/* af_pitch_yin.c -- PitchYINObj of the C ABI (host C; compute = kernels/pitch_yin.cu, one launch per staging chunk).
 * Interface spec: include/mir/_pitch_yin.h, behaviour src/mir/_pitch_yin.c (restated in include/afb200_pitch_yin.h).
 * The object holds only its parameters, the streaming carry and the trough rows of the last legacy call; the reference
 * keeps three FFT buffer pairs and nine timeLength-sized matrices.  The parameter rules, the frame count, the carry and
 * the staging pipe are the pitch trackers' common core (af_pitch_frames.c). */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaquePitchYIN {
    AfPitchFrames f;
    int autoLength, minIndex, maxIndex, yinLength;
    float thresh;
    float *mFre, *mTrough;    /* host, cap x (yinLength/2 + 1): the trough rows of the last legacy call */
    int *lens;
    int cap;
};

static const AfPitchRules RULES = {"pitchYINObj_new", AFB200_PITCH_YIN_MAX_EXP,
                                   "one frame's transform and running sums are held in shared memory", 27, 2094, 2093};

int pitchYINObj_new(PitchYINObj *pitchYINObj, int *samplate, float *lowFre, float *highFre, int *radix2Exp,
                    int *slideLength, int *autoLength, int *isContinue) {
    af_clear_error();
    if (!pitchYINObj) return -1;
    *pitchYINObj = NULL;
    /* :115-170 */
    AfPitchFrames f;
    float lf, hf;
    if (af_pitch_frames_init(&f, &lf, &hf, &RULES, samplate, lowFre, highFre, radix2Exp, slideLength, isContinue))
        return -2;
    const int sr = f.samplate, n = f.n;
    const int A = autoLength && *autoLength >= 0 && *autoLength < n ? *autoLength : n / 2;
    /* :164-170: float quotients, as the reference computes them */
    const int minIndex = (int)floorf(sr / hf);
    int maxIndex = (int)ceilf(sr / lf);
    if (maxIndex > n - A - 1) maxIndex = n - A - 1;
    if (minIndex < 1) {
        af_fail(-3, "pitchYINObj_new: minIndex=%d (samplate=%d, highFre=%g); the reference reads the mean before its "
                "first lag", minIndex, sr, (double)hf);
        return -3;
    }
    if (maxIndex < minIndex) {
        af_fail(-3, "pitchYINObj_new: yinLength=%d is empty: maxIndex=%d (clamped to n - autoLength - 1 = %d) is below "
                "minIndex=%d", maxIndex - minIndex + 1, maxIndex, n - A - 1, minIndex);
        return -3;
    }
    PitchYINObj s = (PitchYINObj)calloc(1, sizeof(struct OpaquePitchYIN));
    if (!s) return -1;
    s->f = f;
    s->autoLength = A;
    s->minIndex = minIndex;
    s->maxIndex = maxIndex;
    s->yinLength = maxIndex - minIndex + 1;
    s->thresh = 0.1f;
    *pitchYINObj = s;
    return 0;
}

void pitchYINObj_setThresh(PitchYINObj s, float thresh) {
    if (s && thresh > 0) s->thresh = thresh;
}

int pitchYINObj_calTimeLength(PitchYINObj s, int dataLength) {
    return af_pitch_time_length(s ? &s->f : NULL, dataLength);
}

void pitchYINObj_enableDebug(PitchYINObj s, int isDebug) { (void)s; (void)isDebug; }

int pitchYINObj_getTroughData(PitchYINObj s, float **mFreArr, float **mTroughArr, int **lenArr) {
    if (!s) return 0;
    if (mFreArr) *mFreArr = s->mFre;
    if (mTroughArr) *mTroughArr = s->mTrough;
    if (lenArr) *lenArr = s->lens;
    return s->yinLength / 2 + 1;
}

typedef struct { PitchYINObj s; int dataLength, timeLength; } YinCall;

/* d: clips, fre, value1, value2, mFre, mTrough, lens (NULL when not requested) */
static int yin_chunk(void *ctx, int nb, float *const *d, void *st) {
    const YinCall *c = (const YinCall *)ctx;
    const PitchYINObj s = c->s;
    AfPitchYinArgs a;
    a.data = d[0]; a.fre = d[1]; a.value1 = d[2]; a.value2 = d[3]; a.mFre = d[4]; a.mTrough = d[5];
    a.lens = (int *)d[6];
    a.log2n = s->f.log2n; a.autoLength = s->autoLength; a.minIndex = s->minIndex; a.maxIndex = s->maxIndex;
    a.samplate = s->f.samplate; a.thresh = s->thresh;
    a.dataLength = c->dataLength; a.hop = s->f.slideLength; a.timeLength = c->timeLength; a.batch = nb;
    return af_launch_pitch_yin(&a, st);
}

int pitchYINObj_pitchBatch(PitchYINObj s, const float *data, int dataLength, int batch, float *freArr, float *valueArr1,
                           float *valueArr2, float *mFreArr, float *mTroughArr, int *lenArr, int memKind, void *stream) {
    int T, rc = af_pitch_batch_begin(s ? &s->f : NULL, "pitchYINObj_pitchBatch", data, dataLength, batch, freArr, &T);
    if (rc || !T) return rc;
    YinCall c = {s, dataLength, T};
    const size_t mLen = (size_t)(s->yinLength / 2 + 1);
    /* fre and value1 are in-out: frames without a trough keep the caller's values, through host staging as well */
    const AfPlane pl[7] = {{data, (size_t)dataLength, AF_IN, 0},  {freArr, (size_t)T, AF_INOUT, 0},
                           {valueArr1, (size_t)T, AF_INOUT, 0},   {valueArr2, (size_t)T, AF_OUT, 0},
                           {mFreArr, (size_t)T * mLen, AF_OUT, 0}, {mTroughArr, (size_t)T * mLen, AF_OUT, 0},
                           {lenArr, (size_t)T, AF_OUT, 0}};
    return af_run_batch(&s->f.pipe, memKind, stream, yin_chunk, &c, pl, 7, batch, AF_PIPE_CHUNK_BYTES);
}

/* :228-244; the trough rows go to the object's arrays for pitchYINObj_getTroughData */
void pitchYINObj_pitch(PitchYINObj s, float *dataArr, int dataLength, float *freArr, float *valueArr1,
                       float *valueArr2) {
    const float *x;
    int len;
    const int T = af_pitch_legacy_input(s ? &s->f : NULL, dataArr, dataLength, &x, &len);
    if (!freArr || T == 0) return;
    const size_t mLen = (size_t)(s->yinLength / 2 + 1);
    if (T > s->cap) {
        float *f = (float *)realloc(s->mFre, sizeof(float) * (size_t)T * mLen);
        if (f) s->mFre = f;
        float *v = f ? (float *)realloc(s->mTrough, sizeof(float) * (size_t)T * mLen) : NULL;
        if (v) s->mTrough = v;
        int *l = v ? (int *)realloc(s->lens, sizeof(int) * (size_t)T) : NULL;
        if (l) s->lens = l;
        if (!l) { af_fail(AF_ERR_NOMEM, "pitchYINObj_pitch: %d trough rows", T); return; }
        s->cap = T;
    }
    pitchYINObj_pitchBatch(s, x, len, 1, freArr, valueArr1, valueArr2, s->mFre, s->mTrough, s->lens,
                           AFB200_MEM_HOST, NULL);
}

void pitchYINObj_free(PitchYINObj s) {
    if (!s) return;
    af_pitch_frames_free(&s->f);
    free(s->mFre);
    free(s->mTrough);
    free(s->lens);
    free(s);
}
