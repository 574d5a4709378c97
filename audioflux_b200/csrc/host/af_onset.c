/* af_onset.c -- OnsetObj of the C ABI (host C; compute = k_onset_maxfilter and k_onset_pick of kernels/onset.cu around
 * the novelty function of kernels/spectral.cu, per group of clips).
 * Interface spec: include/mir/onset_algorithm.h, behaviour src/mir/onset_algorithm.c and src/flux_spectral.c.  The
 * object keeps its peak parameters, the device copy of the last bin list and a device workspace for the max-filtered
 * spectrogram of one group of clips. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

#define ONSET_GROUP_CAP ((size_t)1 << 30)

struct OpaqueOnset {
    int type, nLength, mLength, order;
    int preMax, postMax, preAvg, postAvg, wait;
    float delta;
    int step;                 /* of the last call, for onsetObj_debug */
    int *idx, idxLen;         /* host copy of the bin list on the device */
    int *dIdx;
    void *fence;              /* end of the last launch that read dIdx */
    AfDevBuf dFilt;
    AfPipe pipe;
};

int onsetObj_new(OnsetObj *onsetObj, int nLength, int mLength, int slideLength, int *samplate, int *filterOrder,
                 NoveltyType *type) {
    af_clear_error();
    if (!onsetObj) return 0;
    *onsetObj = NULL;
    OnsetObj s = (OnsetObj)calloc(1, sizeof(struct OpaqueOnset));
    if (!s) return 0;
    const int sr = samplate && *samplate > 0 ? *samplate : 32000;          /* :76-94 */
    if (slideLength < 1) slideLength = 512;
    s->type = type ? (int)*type : Novelty_Flux;
    s->order = filterOrder && *filterOrder > 0 ? *filterOrder : 1;
    s->nLength = nLength;
    s->mLength = mLength;
    /* :123-133, in double and then floored as a float */
    s->preMax = (int)floorf((float)(0.03 * sr / slideLength));
    s->postMax = (int)floorf((float)(0.0 * sr / slideLength + 1));
    s->preAvg = (int)floorf((float)(0.1 * sr / slideLength));
    s->postAvg = (int)floorf((float)(0.1 * sr / slideLength + 1));
    s->wait = (int)floorf((float)(0.03 * sr / slideLength));
    s->delta = 0.07f;
    *onsetObj = s;
    return 0;
}

void onsetObj_debug(OnsetObj s) {
    if (!s) return;
    printf("onsetObj is :\n");
    printf("preMax=%d,postMax=%d, preAvg=%d,postAvg=%d, wait=%d,delta=%f\n", s->preMax, s->postMax, s->preAvg, s->postAvg,
           s->wait, s->delta);
    printf("timeLength=%d,freNum=%d, step=%d,order=%d\n", s->nLength, s->mLength, s->step, s->order);
    printf("\n");
    fflush(stdout);
}

static int is_phase_type(int t) { return t >= Novelty_PD && t <= Novelty_RCD; }

/* the spectral feature id of a novelty type; any other value is FLUX, as in the reference's else branch (:372-377) */
static int feature_of(int t) {
    switch (t) {
    case Novelty_HFC: return AFB200_SPECTRAL_HFC;
    case Novelty_SD: return AFB200_SPECTRAL_SD;
    case Novelty_SF: return AFB200_SPECTRAL_SF;
    case Novelty_MKL: return AFB200_SPECTRAL_MKL;
    case Novelty_PD: return AFB200_SPECTRAL_PD;
    case Novelty_WPD: return AFB200_SPECTRAL_WPD;
    case Novelty_NWPD: return AFB200_SPECTRAL_NWPD;
    case Novelty_CD: return AFB200_SPECTRAL_CD;
    case Novelty_RCD: return AFB200_SPECTRAL_RCD;
    case Novelty_Broadband: return AFB200_SPECTRAL_BROADBAND;
    default: return AFB200_SPECTRAL_FLUX;
    }
}

/* the rules every compute call checks before any device work; fills the novelty request (:135-179 for the defaults) */
static int onset_check(OnsetObj s, int hasPhase, const NoveltyParam *param, const int *indexArr, int indexLength,
                       AfSpectralArgs *a, const char *who) {
    if (s->nLength < 1 || s->mLength < 1)
        return af_fail(AF_ERR_ARG, "%s: nLength=%d, mLength=%d; both must be at least 1", who, s->nLength, s->mLength);
    if (indexArr) {
        if (indexLength < 1) return af_fail(AF_ERR_ARG, "%s: indexLength=%d with an indexArr", who, indexLength);
        for (int i = 0; i < indexLength; i++)
            if (indexArr[i] < 0 || indexArr[i] >= s->mLength)
                return af_fail(AF_ERR_ARG, "%s: indexArr[%d]=%d outside [0, %d)", who, i, indexArr[i], s->mLength);
    }
    if (is_phase_type(s->type) && !hasPhase)
        return af_fail(AF_ERR_ARG, "%s: novelty type %d needs the phase matrix mDataArr2", who, s->type);
    int step = 1, isPos = 1, isExp = 0, type = 0;
    float p = 1.f, threshold = 0.f;
    if (param) {
        if (param->step > 0) step = param->step;
        if (param->p != 0.f) p = param->p;
        isPos = param->isPostive; isExp = param->isExp; type = param->type; threshold = param->threshold;
    }
    if (step > s->nLength)
        return af_fail(AF_ERR_ARG, "%s: step=%d is above nLength=%d", who, step, s->nLength);
    memset(a, 0, sizeof(*a));
    const int f = feature_of(s->type);
    a->req[0] = f;
    a->nReq = 1;
    a->par[0] = (float)step;
    a->par[1] = p;
    a->par[2] = threshold;
    a->par[3] = (float)((isPos ? 1 : 0) | (isExp ? 2 : 0) | (type ? 4 : 0));
    a->fresh = 1;
    a->num = s->mLength;
    a->T = s->nLength;
    a->nb = indexArr ? indexLength : s->mLength;
    s->step = step;
    return AF_OK;
}

/* the bin list on the device; a changed list waits for the kernels that may still read the old one */
static int onset_device(OnsetObj s, const int *indexArr, int indexLength) {
    int rc = af_device_ready();
    if (rc || !indexArr) return rc;
    if (s->dIdx && s->idxLen == indexLength && !memcmp(s->idx, indexArr, sizeof(int) * (size_t)indexLength)) return AF_OK;
    if ((rc = af_fence_wait(s->fence))) return rc;
    int *h = (int *)realloc(s->idx, sizeof(int) * (size_t)indexLength);
    if (!h) return af_fail(AF_ERR_NOMEM, "onset: out of host memory");
    s->idx = h;
    memcpy(s->idx, indexArr, sizeof(int) * (size_t)indexLength);
    s->idxLen = 0;
    if ((rc = af_dev_upload((void **)&s->dIdx, s->idx, sizeof(int) * (size_t)indexLength))) return rc;
    s->idxLen = indexLength;
    return AF_OK;
}

typedef struct { OnsetObj s; AfSpectralArgs a; } OnsetCall;

/* d[0] spec, d[1] phase (or NULL) nb x T x M; d[2] evn, d[3] points nb x T; d[4] counts nb */
static int onset_chunk(void *ctx, int nb, float *const *d, void *st) {
    const OnsetCall *c = (const OnsetCall *)ctx;
    const OnsetObj s = c->s;
    const int T = s->nLength, M = s->mLength, filt = s->order >= 2;
    const size_t clip = (size_t)T * M;
    int group = nb, rc;
    if (filt) {
        group = af_chunk_clips(sizeof(float) * clip, ONSET_GROUP_CAP, nb);
        if ((rc = af_devbuf_reserve(&s->dFilt, sizeof(float) * clip * group))) return rc;
    }
    for (int c0 = 0; c0 < nb; c0 += group) {
        const int g = nb - c0 < group ? nb - c0 : group;
        const float *spec = d[0] + c0 * clip;
        if (filt) {
            if ((rc = af_launch_onset_maxfilter(spec, (long long)g * T, M, s->order, (float *)s->dFilt.ptr, st))) return rc;
            spec = (const float *)s->dFilt.ptr;
        }
        AfSpectralArgs a = c->a;
        a.spec = spec;
        a.phase = d[1] ? d[1] + c0 * clip : NULL;
        a.out = d[2] + (size_t)c0 * T;
        a.batch = g;
        if ((rc = af_launch_spectral(&a, st))) return rc;
        AfOnsetPickArgs p;
        p.evn = d[2] + (size_t)c0 * T;
        p.points = (int *)d[3] + (size_t)c0 * T;
        p.counts = (int *)d[4] + c0;
        p.clips = g; p.T = T;
        p.preMax = s->preMax; p.postMax = s->postMax; p.preAvg = s->preAvg; p.postAvg = s->postAvg; p.wait = s->wait;
        p.delta = s->delta;
        if ((rc = af_launch_onset_pick(&p, st))) return rc;
    }
    return c->a.idx ? af_fence_record(&s->fence, st) : AF_OK;
}

int onsetObj_onsetBatch(OnsetObj s, const float *spec, const float *phase, int batch, const NoveltyParam *param,
                        const int *indexArr, int indexLength, float *evn, int *points, int *counts, int memKind,
                        void *stream) {
    if (!s || !spec || !evn || !points || !counts || batch < 0)
        return af_fail(AF_ERR_ARG, "onsetObj_onsetBatch: bad argument");
    af_clear_error();
    OnsetCall c;
    c.s = s;
    int rc = onset_check(s, phase != NULL, param, indexArr, indexLength, &c.a, "onsetObj_onsetBatch");
    if (rc || (rc = onset_device(s, indexArr, indexLength)) || batch == 0) return rc;
    c.a.idx = indexArr ? s->dIdx : NULL;
    const size_t in = (size_t)s->nLength * s->mLength;
    const AfPlane pl[5] = {{spec, in, AF_IN, 0}, {is_phase_type(s->type) ? phase : NULL, in, AF_IN, 0},
                           {evn, (size_t)s->nLength, AF_OUT, 0}, {points, (size_t)s->nLength, AF_OUT, 0},
                           {counts, 1, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, onset_chunk, &c, pl, 5, batch, AF_PIPE_CHUNK_BYTES);
}

/* :185-211.  The points after the count are left as the caller's array held them, as in the reference. */
int onsetObj_onset(OnsetObj s, float *mDataArr1, float *mDataArr2, NoveltyParam *param, int *indexArr, int indexLength,
                   float *evnArr, int *pointArr) {
    if (!s) return 0;
    af_clear_error();
    if (!mDataArr1 || !evnArr || !pointArr) { af_fail(AF_ERR_ARG, "onsetObj_onset: bad argument"); return 0; }
    if (s->nLength < 1) { af_fail(AF_ERR_ARG, "onsetObj_onset: nLength=%d; it must be at least 1", s->nLength); return 0; }
    int *pts = (int *)malloc(sizeof(int) * (size_t)s->nLength);
    if (!pts) { af_fail(AF_ERR_NOMEM, "onsetObj_onset: out of host memory"); return 0; }
    int count = 0;
    if (onsetObj_onsetBatch(s, mDataArr1, mDataArr2, 1, param, indexArr, indexLength, evnArr, pts, &count,
                            AFB200_MEM_HOST, NULL) != AF_OK)
        count = 0;
    else
        memcpy(pointArr, pts, sizeof(int) * (size_t)count);
    free(pts);
    return count;
}

void onsetObj_free(OnsetObj s) {
    if (!s) return;
    af_fence_wait(s->fence);
    af_fence_free(s->fence);
    af_pipe_free(&s->pipe);
    af_devbuf_free(&s->dFilt);
    af_dev_free(s->dIdx);
    free(s->idx);
    free(s);
}
