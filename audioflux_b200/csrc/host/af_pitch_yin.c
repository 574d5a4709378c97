/* af_pitch_yin.c -- PitchYINObj of the C ABI (host C; compute = kernels/pitch_yin.cu, one launch per staging chunk).
 * Interface spec: include/mir/_pitch_yin.h, behaviour src/mir/_pitch_yin.c (restated in include/afb200_pitch_yin.h).
 * The object holds only its parameters, the streaming carry and the trough rows of the last legacy call; the reference
 * keeps three FFT buffer pairs and nine timeLength-sized matrices. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaquePitchYIN {
    int samplate, log2n, n, slideLength, autoLength, isContinue, isDebug;
    int minIndex, maxIndex, yinLength;
    float thresh;
    float *mFre, *mTrough;    /* host, cap x (yinLength/2 + 1): the trough rows of the last legacy call */
    int *lens;
    int cap;
    AfTail tail;
    AfPipe pipe;
};

int pitchYINObj_new(PitchYINObj *pitchYINObj, int *samplate, float *lowFre, float *highFre, int *radix2Exp,
                    int *slideLength, int *autoLength, int *isContinue) {
    af_clear_error();
    if (!pitchYINObj) return -1;
    *pitchYINObj = NULL;
    /* :115-170, in the reference's order: highFre is checked against the lowFre already taken, and against the integer
     * samplate/2; a NULL highFre keeps 2094, a rejected one resets both ends to 27 / 2093 */
    const int sr = samplate && *samplate > 0 && *samplate <= 196000 ? *samplate : 32000;
    float lf = lowFre && *lowFre >= 27 ? *lowFre : 27, hf = 2094;
    if (highFre) {
        if (*highFre > lf && *highFre < sr / 2) hf = *highFre;
        else { lf = 27; hf = 2093; }
    }
    const int log2n = radix2Exp && *radix2Exp >= 1 && *radix2Exp <= 30 ? *radix2Exp : 12;
    if (log2n > AFB200_PITCH_YIN_MAX_EXP) {
        af_fail(-2, "pitchYINObj_new: radix2Exp=%d; the largest supported is %d (one frame's transform and running sums "
                "are held in shared memory)", log2n, AFB200_PITCH_YIN_MAX_EXP);
        return -2;
    }
    const int n = 1 << log2n;
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
    s->samplate = sr;
    s->log2n = log2n;
    s->n = n;
    s->slideLength = slideLength && *slideLength > 0 ? *slideLength : n / 4;
    if (s->slideLength < 1) s->slideLength = 1;                 /* n/4 at n = 2: the reference divides by zero */
    s->autoLength = A;
    s->isContinue = isContinue ? *isContinue : 0;
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

static int frames(PitchYINObj s, int dataLength) {
    return dataLength < s->n ? 0 : (dataLength - s->n) / s->slideLength + 1;
}

int pitchYINObj_calTimeLength(PitchYINObj s, int dataLength) {
    if (!s) return 0;
    return frames(s, s->isContinue ? dataLength + s->tail.length : dataLength);
}

void pitchYINObj_enableDebug(PitchYINObj s, int isDebug) {
    if (s) s->isDebug = isDebug;
}

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
    a.log2n = s->log2n; a.autoLength = s->autoLength; a.minIndex = s->minIndex; a.maxIndex = s->maxIndex;
    a.samplate = s->samplate; a.thresh = s->thresh;
    a.dataLength = c->dataLength; a.hop = s->slideLength; a.timeLength = c->timeLength; a.batch = nb;
    return af_launch_pitch_yin(&a, st);
}

int pitchYINObj_pitchBatch(PitchYINObj s, const float *data, int dataLength, int batch, float *freArr, float *valueArr1,
                           float *valueArr2, float *mFreArr, float *mTroughArr, int *lenArr, int memKind, void *stream) {
    const int T = s && dataLength > 0 ? frames(s, dataLength) : 0;
    if (!s || !data || (!freArr && T > 0 && batch > 0) || dataLength <= 0 || batch < 0)   /* freArr may be NULL when empty */
        return af_fail(AF_ERR_ARG, "pitchYINObj_pitchBatch: bad argument");
    af_clear_error();
    int rc = af_device_ready();
    if (rc) return rc;
    if (batch == 0 || T == 0) return AF_OK;
    YinCall c = {s, dataLength, T};
    const size_t mLen = (size_t)(s->yinLength / 2 + 1);
    /* fre and value1 are in-out: frames without a trough keep the caller's values, through host staging as well */
    const AfPlane pl[7] = {{data, (size_t)dataLength, AF_IN, 0},  {freArr, (size_t)T, AF_INOUT, 0},
                           {valueArr1, (size_t)T, AF_INOUT, 0},   {valueArr2, (size_t)T, AF_OUT, 0},
                           {mFreArr, (size_t)T * mLen, AF_OUT, 0}, {mTroughArr, (size_t)T * mLen, AF_OUT, 0},
                           {lenArr, (size_t)T, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, yin_chunk, &c, pl, 7, batch, AF_PIPE_CHUNK_BYTES);
}

/* :228-244; the trough rows go to the object's arrays for pitchYINObj_getTroughData */
void pitchYINObj_pitch(PitchYINObj s, float *dataArr, int dataLength, float *freArr, float *valueArr1,
                       float *valueArr2) {
    if (!s) return;
    af_clear_error();
    if (!dataArr || dataLength <= 0) return;
    const float *x = dataArr;
    if (s->isContinue && !af_tail_assemble(&s->tail, s->n, s->slideLength, dataArr, dataLength, &x, &dataLength)) return;
    const int T = frames(s, dataLength);
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
    pitchYINObj_pitchBatch(s, x, dataLength, 1, freArr, valueArr1, valueArr2, s->mFre, s->mTrough, s->lens,
                           AFB200_MEM_HOST, NULL);
}

void pitchYINObj_free(PitchYINObj s) {
    if (!s) return;
    af_pipe_free(&s->pipe);
    af_tail_free(&s->tail);
    free(s->mFre);
    free(s->mTrough);
    free(s->lens);
    free(s);
}
