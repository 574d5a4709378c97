/* af_resample.c -- ResampleObj of the C ABI (host C; compute = kernels/resample.cu, one launch per staging chunk).
 * Interface spec: src/dsp/resample_algorithm.h, behaviour src/dsp/resample_algorithm.c:59-634.  The object keeps the
 * float32 table on the host with the reference's in-place scaling history, and a device copy that is refreshed at the
 * first compute call after the table changed.  The reference's second table (the differences of neighbouring entries)
 * is recomputed by the kernel from the first, bit for bit. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueResample {
    int isContinue, isScale;
    WindowType winType;
    float value, rollOff;
    int zeroNum, bitLength, interpLength;
    float *interpArr;     /* host table, scaled in place by the ratio while the ratio is below 1; one spare entry */
    float ratio;          /* targetRate / sourceRate */
    int p, q;             /* up / down factors; 0 after setSamplateRatio */
    int sourceRate, targetRate;
    float *dTable;        /* device copy of interpArr */
    int dStale;           /* interpArr changed since the last upload */
    void *fence;          /* end of the last launch that reads dTable */
    AfPipe pipe;
};

int resampleObj_new(ResampleObj *resampleObj, ResampleQualityType *qualType, int *isScale, int *isContinue) {
    int zeroNum = 64, nbit = 9;                                        /* :62-87 */
    WindowType winType = Window_Kaiser;
    float value = 14.7696565f, rollOff = 0.9475937f;
    const ResampleQualityType q = qualType ? *qualType : ResampleQuality_Best;
    if (q == ResampleQuality_Mid) { zeroNum = 32; value = 11.6625806f; rollOff = 0.8987969f; }
    else if (q == ResampleQuality_Fast) { zeroNum = 16; value = 8.5555046f; rollOff = 0.85f; }
    return resampleObj_newWithWindow(resampleObj, &zeroNum, &nbit, &winType, &value, &rollOff, isScale, isContinue);
}

/* :546-634: rollOff * sinc(rollOff * x) on x = linspace(0, zeroNum, interpLength), times the right half of the symmetric
 * window of length 2 * (interpLength - 1) + 1, in the reference's float order */
static int rs_table(ResampleObj s) {
    const int L = s->interpLength, order = 2 * (L - 1);
    float *a = (float *)malloc(sizeof(float) * ((size_t)L + 1));     /* + the copy of the last entry the kernel reads */
    double *win = (double *)malloc(sizeof(double) * ((size_t)order + 1));
    if (!a || !win) { free(a); free(win); return AF_ERR_NOMEM; }
    af_window_symmetric(s->winType, order + 1, &s->value, win);
    const float step = (float)s->zeroNum / (float)(L - 1);            /* __vlinspace, flux_vector.c:2145-2162 */
    for (int i = 0; i < L; i++) {
        const float x = (float)i * step * s->rollOff;
        const float v = (float)(x * M_PI);                             /* __vsinc, flux_vectorOp.c:378-400 */
        const float sinc = fabsf(v) < 1e-9 ? 1.0f : sinf(v) / v;
        a[i] = sinc * s->rollOff * (float)win[L - 1 + i];
    }
    free(win);
    s->interpArr = a;
    return AF_OK;
}

/* :281-293 / :314-326 and :536-540: undo the old scaling, apply the new one */
static void rs_set_ratio(ResampleObj s, float ratio) {
    if (ratio != s->ratio && (s->ratio < 1 || ratio < 1)) {
        if (s->ratio < 1)
            for (int i = 0; i < s->interpLength; i++) s->interpArr[i] /= s->ratio;
        if (ratio < 1)
            for (int i = 0; i < s->interpLength; i++) s->interpArr[i] *= ratio;
        s->dStale = 1;
    }
    s->ratio = ratio;
}

int resampleObj_newWithWindow(ResampleObj *resampleObj, int *zeroNum, int *nbit, WindowType *winType, float *value,
                              float *rollOff, int *isScale, int *isContinue) {
    af_clear_error();
    if (!resampleObj) return -1;
    *resampleObj = NULL;
    int z = 64, nb = 9;                                                /* :115-175 */
    WindowType w = Window_Hann;
    float v = 0, r = 0.945f;
    if (zeroNum && *zeroNum > 0) z = *zeroNum;
    if (nbit && *nbit > 0 && *nbit < 30) nb = *nbit;
    if (winType && *winType > Window_Rect) w = *winType;
    if (value) {
        if (*value >= 0) v = *value;
        if (v == 0) v = w == Window_Kaiser ? 5.0f : w == Window_Gauss ? 2.5f : v;
    }
    if (rollOff && *rollOff > 0 && *rollOff <= 1) r = *rollOff;
    if (w > Window_Tukey) {
        af_fail(-1, "resampleObj_newWithWindow: winType=%d; Hann .. Tukey (1 .. %d) are supported", (int)w, Window_Tukey);
        return -1;
    }
    const long long length = (long long)z * (1LL << nb) + 1;
    if (length > AFB200_RESAMPLE_MAX_TABLE) {
        af_fail(-2, "resampleObj_newWithWindow: zeroNum * 2^nbit + 1 = %lld table entries; at most %d are supported",
                length, AFB200_RESAMPLE_MAX_TABLE);
        return -2;
    }
    ResampleObj s = (ResampleObj)calloc(1, sizeof(struct OpaqueResample));
    if (!s) return -1;
    s->isContinue = isContinue ? *isContinue : 0;
    s->isScale = isScale ? *isScale : 0;
    s->winType = w; s->value = v; s->rollOff = r;
    s->zeroNum = z; s->bitLength = 1 << nb; s->interpLength = (int)length;
    s->sourceRate = 32000; s->targetRate = 16000;                      /* :194-201 */
    s->p = 1; s->q = 2;
    s->ratio = 1;
    if (rs_table(s)) { free(s); return -1; }
    rs_set_ratio(s, 0.5f);
    *resampleObj = s;
    return 0;
}

/* :219-251.  Returns 0, or -1 when the output length does not fit an int. */
static int rs_lengths(ResampleObj s, int dataLength, int *src, int *tgt) {
    *src = *tgt = 0;
    if (!s->isContinue) {
        const float f = floorf((float)dataLength * s->ratio);
        if (!(f < 2147483648.0f)) return -1;
        *src = dataLength;
        *tgt = (int)f;
    } else if (s->q > 1) {
        *src = dataLength - dataLength % s->q;
        const long long t = (long long)*src * s->p;
        if (t > 2147483647LL) return -1;
        *tgt = (int)t / s->q;
    }
    return 0;
}

int resampleObj_calDataLength(ResampleObj s, int dataLength) {
    int src, tgt;
    if (!s || rs_lengths(s, dataLength, &src, &tgt)) return 0;
    return tgt;
}

static int gcd(int a, int b) { while (b) { const int c = a % b; a = b; b = c; } return a; }

void resampleObj_setSamplate(ResampleObj s, int sourceRate, int targetRate) {
    if (!s || sourceRate == targetRate || sourceRate <= 0 || targetRate <= 0) return;   /* :263-266 */
    const int g = gcd(sourceRate, targetRate);
    rs_set_ratio(s, targetRate / (float)sourceRate);
    s->sourceRate = sourceRate; s->targetRate = targetRate;
    s->p = targetRate / g; s->q = sourceRate / g;
}

void resampleObj_setSamplateRatio(ResampleObj s, float ratio) {
    if (!s || ratio < 0) return;                                       /* :307-309 */
    rs_set_ratio(s, ratio);
    s->p = s->q = 0;
}

void resampleObj_enableContinue(ResampleObj s, int flag) {
    if (s) s->isContinue = flag;
}

void resampleObj_debug(ResampleObj s) { (void)s; }

/* the rules every compute call checks before any device work; fills the lengths and the tap stride */
static int rs_check(ResampleObj s, int dataLength, int *src, int *tgt, int *step, const char *who) {
    if (s->isContinue && s->q <= 1)
        return af_fail(AF_ERR_UNSUPPORTED, "%s: continue mode needs a rate pair p/q with q > 1 (q=%d)", who, s->q);
    if (rs_lengths(s, dataLength, src, tgt))
        return af_fail(AF_ERR_ARG, "%s: the output length of %d samples at ratio %g does not fit an int", who, dataLength,
                       (double)s->ratio);
    const float scale = 1.0 > s->ratio ? s->ratio : 1.0f;             /* :455-456 */
    *step = (int)floorf(scale * (float)s->bitLength);
    if (*step <= 0)
        return af_fail(AF_ERR_UNSUPPORTED, "%s: ratio %g times 2^nbit (%d) is below 1: the table has no tap stride", who,
                       (double)s->ratio, s->bitLength);
    return AF_OK;
}

static int rs_device(ResampleObj s) {
    int rc = af_device_ready();
    if (rc || (s->dTable && !s->dStale)) return rc;
    /* kernels queued earlier may still read the old table: the rebuild waits for the last of them */
    if ((rc = af_fence_wait(s->fence))) return rc;
    s->interpArr[s->interpLength] = s->interpArr[s->interpLength - 1];     /* its difference to the last entry is 0 */
    if ((rc = af_dev_upload((void **)&s->dTable, s->interpArr, sizeof(float) * ((size_t)s->interpLength + 1)))) return rc;
    s->dStale = 0;
    return AF_OK;
}

typedef struct { ResampleObj s; int inLen, srcLen, outLen, step, accumulate; } RsCall;

static int rs_chunk(void *p, int nb, float *const *d, void *st) {
    const RsCall *c = (const RsCall *)p;
    const ResampleObj s = c->s;
    AfResampleArgs a;
    memset(&a, 0, sizeof(a));
    a.data = d[0]; a.out = d[1]; a.table = s->dTable;
    a.inLen = c->inLen; a.srcLen = c->srcLen; a.outLen = c->outLen; a.batch = nb;
    a.tableLength = s->interpLength; a.bitLength = s->bitLength; a.step = c->step;
    a.ratio = s->ratio;
    a.scale = 1.0 > s->ratio ? s->ratio : 1.0f;
    a.scaleDiv = s->isScale ? sqrtf(s->ratio) : 0.0f;                 /* :387-396 */
    a.accumulate = c->accumulate;
    int rc = af_launch_resample(&a, st);
    return rc ? rc : af_fence_record(&s->fence, st);
}

static int rs_run(ResampleObj s, const float *data, int dataLength, int batch, float *out, int accumulate, int memKind,
                  void *stream, const char *who) {
    int src = 0, tgt = 0, step = 0;
    int rc = rs_check(s, dataLength, &src, &tgt, &step, who);
    if (rc || batch == 0 || tgt <= 0) return rc;
    if (!out) return af_fail(AF_ERR_ARG, "%s: no output buffer", who);
    if ((rc = rs_device(s))) return rc;
    RsCall c = {s, dataLength, src, tgt, step, accumulate};
    const AfPlane pl[2] = {{data, (size_t)dataLength, AF_IN, 0}, {out, (size_t)tgt, accumulate ? AF_INOUT : AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, rs_chunk, &c, pl, 2, batch, AF_PIPE_CHUNK_BYTES);
}

int resampleObj_resampleBatch(ResampleObj s, const float *data, int dataLength, int batch, float *out, int memKind,
                              void *stream) {
    if (!s || !data || dataLength <= 0 || batch < 0)
        return af_fail(AF_ERR_ARG, "resampleObj_resampleBatch: bad argument");
    af_clear_error();
    if (s->isContinue)
        return af_fail(AF_ERR_ARG, "resampleObj_resampleBatch: the object is in continue mode; feed a stream through "
                       "resampleObj_resample");
    return rs_run(s, data, dataLength, batch, out, 0, memKind, stream, "resampleObj_resampleBatch");
}

/* :350-403.  The reference's continue-mode tail (:377-384) is only written when a tail already exists, and none ever
 * does: each call resamples the first dataLength1 - dataLength1 % q samples and drops the rest, as here. */
int resampleObj_resample(ResampleObj s, float *dataArr1, int dataLength1, float *dataArr2) {
    if (!s) return 0;
    af_clear_error();
    if (!dataArr1 || !dataArr2 || dataLength1 <= 0) return 0;
    int src, tgt;
    if (rs_run(s, dataArr1, dataLength1, 1, dataArr2, 1, AFB200_MEM_HOST, NULL, "resampleObj_resample") ||
        rs_lengths(s, dataLength1, &src, &tgt))
        return 0;
    return tgt;
}

void resampleObj_free(ResampleObj s) {
    if (!s) return;
    af_pipe_free(&s->pipe);
    af_fence_wait(s->fence);
    af_fence_free(s->fence);
    af_dev_free(s->dTable);
    free(s->interpArr);
    free(s);
}
