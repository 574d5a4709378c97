/* af_pitch_pef.c -- PitchPEFObj of the C ABI (host C; compute = kernels/pitch_pef.cu, one launch per staging chunk).
 * Interface spec: include/mir/_pitch_pef.h, behaviour src/mir/_pitch_pef.c (restated in include/afb200_pitch_pef.h).
 * The object builds its tables in float as the reference does, and the filter's spectrum at the kernel's transform
 * length in double, once; they are uploaded at the first compute call.  The parameter rules, the frame count, the
 * streaming carry and the staging pipe are the pitch trackers' common core (af_pitch_frames.c).  The reference keeps
 * two FFT objects and timeLength x 8n-float matrices. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaquePitchPEF {
    AfPitchFrames f;
    int minIndex, maxIndex, padNum, log2L;
    float *tables;        /* host, AF_PEF_TABLE_FLOATS(n, L) (af_internal.h) */
    float *dTables;
};

static const AfPitchRules RULES = {"pitchPEFObj_new", AFB200_PITCH_PEF_MAX_EXP,
                                   "one frame's transforms are held in shared memory", 32, 2000, 2000};

/* __vlinspace (src/vector/flux_vector.c:2145), type 0 */
static void linspace_ref(float start, float stop, int length, float *out) {
    const float step = (stop - start) / (length - 1 > 0 ? length - 1 : 1);
    for (int i = 0; i < length; i++) out[i] = start + i * step;
}

/* __vlogspace (:2164) */
static void logspace_ref(float start, float stop, int length, float *out) {
    linspace_ref(start, stop, length, out);
    for (int i = 0; i < length; i++) out[i] = powf(10, out[i]);
}

static double dsum(const float *v, int n) {                   /* __vsum: a double accumulator */
    double s = 0;
    for (int i = 0; i < n; i++) s += v[i];
    return s;
}

/* __pitchPEFObj_initData (:428-522) and __pitchPEFObj_calEstimateFilter (:696-785); filter gets n floats */
static int build_tables(PitchPEFObj s, int winType, float lowFre, float highFre, float cutFre, float alpha, float beta,
                        float gamma, float *filter) {
    const int n = s->f.n, sr2 = s->f.samplate / 2;
    float *win = s->tables, *lin = s->tables + AF_PEF_LIN(n), *lg = s->tables + AF_PEF_LOG(n);
    float *bw = s->tables + AF_PEF_BW(n);
    int *idx = (int *)(s->tables + AF_PEF_IDX(n));
    if (af_window_fft(winType, n, win)) return -1;
    linspace_ref(0, sr2, n + 1, lin);
    const float fre1 = sr2 > cutFre ? cutFre : sr2 - 1;
    logspace_ref(1, log10f(fre1), 2 * n, lg);
    int minIndex = -1, maxIndex = 0;
    for (int i = 1; i < 2 * n; i++) {
        if (highFre < lg[i]) {
            maxIndex = lg[i] - highFre < highFre - lg[i - 1] ? i : i - 1;
            break;
        }
        if (minIndex != -1) continue;
        if (lowFre < lg[i]) minIndex = lg[i] - lowFre < lowFre - lg[i - 1] ? i : i - 1;
    }
    for (int i = 2, j = 1; i < 2 * n; i++, j++) bw[j] = (lg[i] - lg[i - 2]) / (2 * n * 2);
    bw[0] = bw[1];
    bw[2 * n - 1] = bw[2 * n - 2];
    /* __vinterp_linear's segment for each log point: its index only moves forward */
    for (int i = 0, j = 0; i < 2 * n; i++) {
        while (j < n && lg[i] > lin[j + 1]) j++;
        idx[i] = j;
    }

    float *q = (float *)malloc(sizeof(float) * 3 * ((size_t)n + 1));
    if (!q) return -1;
    float *h = q + n + 1, *d = h + n + 1;
    logspace_ref(log10f(beta), log10f(alpha + beta), n, q);
    int pad = 0;
    for (int i = 0; i < n; i++) {
        if (q[i] < 1) pad++;
        h[i] = 1 / (gamma - cosf(2 * M_PI * q[i]));
    }
    d[0] = q[0];
    for (int i = 1; i < n; i++) d[i] = (q[i - 1] + q[i]) / 2;
    d[n] = q[n - 1];
    for (int i = 1; i < n + 1; i++) d[i - 1] = d[i] - d[i - 1];
    const float v1 = (float)dsum(d, n);
    for (int i = 0; i < n; i++) d[i] = d[i] * h[i];
    const float v2 = (float)dsum(d, n);
    const float det = v2 / v1;
    for (int i = 0; i < n; i++) filter[i] = h[i] - det;
    free(q);
    s->minIndex = minIndex;
    s->maxIndex = maxIndex;
    s->padNum = pad;
    return 0;
}

/* the L-point spectrum of the filter (n floats, zero-padded), bins 0 .. L/2, in double rounded to float pairs */
static int filter_spectrum(const float *filter, int n, int L, float *out) {
    double *re = (double *)calloc(2 * (size_t)L, sizeof(double));
    if (!re) return -1;
    double *im = re + L;
    for (int i = 0; i < n; i++) re[i] = filter[i];
    af_fft_double(re, im, L);
    for (int k = 0; k <= L / 2; k++) { out[2 * k] = (float)re[k]; out[2 * k + 1] = (float)im[k]; }
    free(re);
    return 0;
}

int pitchPEFObj_new(PitchPEFObj *pitchPEFObj, int *samplate, float *lowFre, float *highFre, float *cutFre,
                    int *radix2Exp, int *slideLength, WindowType *windowType, float *alpha, float *beta, float *gamma,
                    int *isContinue) {
    af_clear_error();
    if (!pitchPEFObj) return -1;
    *pitchPEFObj = NULL;
    /* :135-204 */
    AfPitchFrames f;
    float lf, hf;
    if (af_pitch_frames_init(&f, &lf, &hf, &RULES, samplate, lowFre, highFre, radix2Exp, slideLength, isContinue))
        return -2;
    const int sr = f.samplate, log2n = f.log2n, n = f.n;
    const float cf = !cutFre ? 4000 : *cutFre >= hf ? *cutFre : hf;
    const int wt = windowType ? (int)*windowType : Window_Hamm;
    const float al = alpha && *alpha > 0 ? *alpha : 10, be = beta && *beta > 0 ? *beta : 0.5f,
                ga = gamma && *gamma > 1 ? *gamma : 1.8f;
    PitchPEFObj s = (PitchPEFObj)calloc(1, sizeof(struct OpaquePitchPEF));
    float *filter = (float *)malloc(sizeof(float) * (size_t)n);
    /* the largest table: L = 4n */
    if (s) s->tables = (float *)calloc(AF_PEF_TABLE_FLOATS(n, 4 * n), sizeof(float));
    if (!s || !filter || !s->tables) { free(filter); pitchPEFObj_free(s); return -1; }
    s->f = f;
    if (build_tables(s, wt, lf, hf, cf, al, be, ga, filter)) { free(filter); pitchPEFObj_free(s); return -1; }
    int rc = 0;
    if (s->minIndex < 0 || s->maxIndex <= s->minIndex) {
        af_fail(-3, "pitchPEFObj_new: lag range minIndex=%d .. maxIndex=%d is empty (samplate=%d, lowFre=%g, "
                "highFre=%g, cutFre=%g)", s->minIndex, s->maxIndex, sr, (double)lf, (double)hf, (double)cf);
        rc = -3;
    } else if (s->padNum == 0 && s->maxIndex >= 2 * n - 1) {
        af_fail(-4, "pitchPEFObj_new: maxIndex=%d with no filter padding (beta=%g): the reference's peak search reads "
                "past its correlation buffer", s->maxIndex, (double)be);
        rc = -4;
    }
    if (!rc) {
        /* the kernel's transform: s (P + 2n values) fits, and no product filter[j] s[j + k], k <= maxIndex, wraps */
        const int need = s->padNum + 2 * n > n + s->maxIndex + 1 ? s->padNum + 2 * n : n + s->maxIndex + 1;
        int log2L = log2n + 1;
        while ((1 << log2L) < need) log2L++;
        s->log2L = log2L;
        if (filter_spectrum(filter, n, 1 << log2L, s->tables + AF_PEF_SPEC(n))) rc = -1;
    }
    free(filter);
    if (rc) { pitchPEFObj_free(s); return rc; }
    *pitchPEFObj = s;
    return 0;
}

int pitchPEFObj_calTimeLength(PitchPEFObj s, int dataLength) {
    return af_pitch_time_length(s ? &s->f : NULL, dataLength);
}

void pitchPEFObj_setFilterParams(PitchPEFObj s, float alpha, float beta, float gamma) {
    (void)s; (void)alpha; (void)beta; (void)gamma;              /* the reference rebuilds the same filter (:685-694) */
}

void pitchPEFObj_enableDebug(PitchPEFObj s, int isDebug) { (void)s; (void)isDebug; }

typedef struct { PitchPEFObj s; int dataLength, timeLength; } PefCall;

/* d[0] clips nb x dataLength, d[1] frequencies nb x T */
static int pef_chunk(void *ctx, int nb, float *const *d, void *st) {
    const PefCall *c = (const PefCall *)ctx;
    const PitchPEFObj s = c->s;
    AfPitchPefArgs a;
    a.data = d[0]; a.tables = s->dTables; a.fre = d[1];
    a.log2n = s->f.log2n; a.log2L = s->log2L; a.padNum = s->padNum; a.minIndex = s->minIndex; a.maxIndex = s->maxIndex;
    a.dataLength = c->dataLength; a.hop = s->f.slideLength; a.timeLength = c->timeLength; a.batch = nb;
    return af_launch_pitch_pef(&a, st);
}

int pitchPEFObj_pitchBatch(PitchPEFObj s, const float *data, int dataLength, int batch, float *freArr, int memKind,
                           void *stream) {
    int T, rc = af_pitch_batch_begin(s ? &s->f : NULL, "pitchPEFObj_pitchBatch", data, dataLength, batch, freArr, &T);
    if (rc || !T || (!s->dTables && (rc = af_dev_upload((void **)&s->dTables, s->tables,
                                                        sizeof(float) * AF_PEF_TABLE_FLOATS(s->f.n, 1 << s->log2L)))))
        return rc;
    PefCall c = {s, dataLength, T};
    const AfPlane pl[2] = {{data, (size_t)dataLength, AF_IN, 0}, {freArr, (size_t)T, AF_OUT, 0}};
    return af_run_batch(&s->f.pipe, memKind, stream, pef_chunk, &c, pl, 2, batch, AF_PIPE_CHUNK_BYTES);
}

/* :233-256 */
void pitchPEFObj_pitch(PitchPEFObj s, float *dataArr, int dataLength, float *freArr) {
    const float *x;
    int len;
    if (af_pitch_legacy_input(s ? &s->f : NULL, dataArr, dataLength, &x, &len) && freArr)
        pitchPEFObj_pitchBatch(s, x, len, 1, freArr, AFB200_MEM_HOST, NULL);
}

void pitchPEFObj_free(PitchPEFObj s) {
    if (!s) return;
    af_pitch_frames_free(&s->f);
    af_dev_free(s->dTables);
    free(s->tables);
    free(s);
}
