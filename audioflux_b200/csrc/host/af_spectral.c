/* af_spectral.c -- SpectralObj of the C ABI (host C; compute = kernels/spectral.cu `k_spectral`).
 * Interface spec: src/feature/spectral_algorithm.h:16-81, behaviour src/feature/spectral_algorithm.c and
 * src/flux_spectral.c.  Stateless: no per-frame sums are cached between calls (the reference's caches go stale when
 * an object is reused on new data, see include/afb200_spectral.h). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueSpectral {
    int num, timeLength;
    float *fre;                 /* host copy of freBandArr (NULL when none was given) */
    int contig, start, nb;      /* contig: bins start .. start+nb-1, else the owned list idx */
    int *idx;
    int idxDirty;
    float *dFre;
    int *dIdx;
    AfPipe pipe;
};

static int needs_fre(int f) {
    return f == AFB200_SPECTRAL_ROLLOFF || f == AFB200_SPECTRAL_CENTROID || f == AFB200_SPECTRAL_SPREAD ||
           f == AFB200_SPECTRAL_SKEWNESS || f == AFB200_SPECTRAL_KURTOSIS || f == AFB200_SPECTRAL_SLOPE ||
           f == AFB200_SPECTRAL_BANDWIDTH || f == AFB200_SPECTRAL_MAX || f == AFB200_SPECTRAL_MEAN ||
           f == AFB200_SPECTRAL_VAR;
}
static int needs_phase(int f) { return f >= AFB200_SPECTRAL_PD && f <= AFB200_SPECTRAL_RCD; }
/* features that leave frames as they were (pd frame 1, var with < 2 bins) or add into them (broadband) */
static int reads_out(int f) {
    return f == AFB200_SPECTRAL_BROADBAND || f == AFB200_SPECTRAL_PD || f == AFB200_SPECTRAL_WPD ||
           f == AFB200_SPECTRAL_NWPD || f == AFB200_SPECTRAL_VAR;
}
static int planes_of(int f) { return f == AFB200_SPECTRAL_MAX || f == AFB200_SPECTRAL_MEAN || f == AFB200_SPECTRAL_VAR ? 2 : 1; }

int spectralObj_new(SpectralObj *out, int num, float *freBandArr) {
    af_clear_error();
    if (!out) return -1;
    *out = NULL;
    if (num < 2) { printf("num is error!!!\n"); return -1; }
    SpectralObj s = (SpectralObj)calloc(1, sizeof(struct OpaqueSpectral));
    if (!s) return -1;
    s->num = num;
    s->contig = 1; s->start = 0; s->nb = num;
    if (freBandArr) {                 /* copied: the reference keeps the caller's pointer */
        s->fre = (float *)malloc(sizeof(float) * (size_t)num);
        if (!s->fre) { free(s); return -1; }
        memcpy(s->fre, freBandArr, sizeof(float) * (size_t)num);
    }
    *out = s;
    return 0;
}

void spectralObj_setTimeLength(SpectralObj s, int timeLength) { if (s) s->timeLength = timeLength; }

void spectralObj_setEdge(SpectralObj s, int start, int end) {
    if (!s) return;
    if (start >= 0 && end <= s->num - 1 && end > start) {     /* spectral_algorithm.c:164 */
        free(s->idx);
        s->idx = NULL;
        s->contig = 1; s->start = start; s->nb = end - start + 1;
    }
}

void spectralObj_setEdgeArr(SpectralObj s, int *indexArr, int indexLength) {
    if (!s || !indexArr) return;
    int ok = indexLength >= 1;
    for (int i = 0; ok && i < indexLength; i++)
        if (indexArr[i] < 0 || indexArr[i] > s->num - 1) ok = 0;
    if (!ok) { free(indexArr); return; }                    /* :193-199 */
    free(s->idx);
    s->idx = indexArr;
    s->contig = 0; s->nb = indexLength;
    s->idxDirty = 1;
}

static int spectral_device(SpectralObj s, int wantFre) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (wantFre && !s->dFre && (rc = af_dev_upload((void **)&s->dFre, s->fre, sizeof(float) * (size_t)s->num))) return rc;
    if (!s->contig && (s->idxDirty || !s->dIdx)) {
        if ((rc = af_dev_upload((void **)&s->dIdx, s->idx, sizeof(int) * (size_t)s->nb))) return rc;
        s->idxDirty = 0;
    }
    return AF_OK;
}

static int spectral_chunk(void *p, int nb, float *const *d, void *st) {
    AfSpectralArgs a = *(const AfSpectralArgs *)p;
    a.spec = d[0]; a.phase = d[1]; a.out = d[2]; a.batch = nb;
    return af_launch_spectral(&a, st);
}

int spectralObj_spectralBatch(SpectralObj s, const float *spec, const float *phase, int timeLength, int batch,
                              int nReq, const int *req, const float *par, float *out, int memKind, void *stream) {
    if (!s || !spec || !out || !req || !par || timeLength < 1 || batch < 0)
        return af_fail(AF_ERR_ARG, "spectralObj_spectralBatch: bad argument");
    if (nReq < 1 || nReq > AFB200_SPECTRAL_MAX_REQ)
        return af_fail(AF_ERR_ARG, "spectralObj_spectralBatch: nReq=%d outside [1, %d]", nReq, AFB200_SPECTRAL_MAX_REQ);
    AfSpectralArgs a;
    memset(&a, 0, sizeof(a));
    int wantFre = 0, wantPh = 0, readOut = 0, planes = 0;
    for (int i = 0; i < nReq; i++) {
        const int f = req[i];
        if (f < 0 || f >= AFB200_SPECTRAL_COUNT) return af_fail(AF_ERR_ARG, "spectralObj_spectralBatch: feature id %d", f);
        wantFre |= needs_fre(f);
        wantPh |= needs_phase(f);
        readOut |= reads_out(f);
        a.req[i] = f;
        a.plane[i] = planes;
        planes += planes_of(f);
        for (int k = 0; k < 4; k++) a.par[4 * i + k] = par[4 * i + k];
    }
    if (wantFre && !s->fre)
        return af_fail(AF_ERR_ARG, "spectralObj_spectralBatch: a frequency feature needs the freBandArr of spectralObj_new");
    if (wantPh && !phase) return af_fail(AF_ERR_ARG, "spectralObj_spectralBatch: a phase feature needs the phase planes");
    af_clear_error();
    int rc = spectral_device(s, wantFre);
    if (rc) return rc;

    a.num = s->num; a.T = timeLength; a.batch = batch; a.nReq = nReq;
    a.start = s->contig ? s->start : 0;
    a.nb = s->nb;
    a.idx = s->contig ? NULL : s->dIdx;
    a.fre = wantFre ? s->dFre : NULL;
    if (s->fre) {                   /* spectral_algorithm.c:1124-1130 on a fresh object: float, list order */
        float m = 0.f;
        for (int j = 0; j < s->nb; j++) m += s->fre[s->contig ? s->start + j : s->idx[j]];
        a.meanFre = m / (float)s->nb;
    }
    if (batch == 0) return AF_OK;
    /* clips as items; `out` holds `planes` planes of batch x T, so it moves as one layered plane */
    const size_t in = (size_t)timeLength * s->num;
    const AfPlane pl[3] = {{spec, in, AF_IN, 0}, {wantPh ? phase : NULL, in, AF_IN, 0},
                           {out, (size_t)timeLength, readOut ? AF_INOUT : AF_OUT, planes}};
    return af_run_batch(&s->pipe, memKind, stream, spectral_chunk, &a, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

/* ---- the reference's per-feature entry points: one clip of timeLength frames, host pointers ---- */
static void one(SpectralObj s, int f, const float *spec, const float *phase, float step, float p, float thr, int flags,
                float *out) {
    if (!s || !spec || !out || s->timeLength < 1) return;
    const float par[4] = {step, p, thr, (float)flags};
    spectralObj_spectralBatch(s, spec, phase, s->timeLength, 1, 1, &f, par, out, AFB200_MEM_HOST, NULL);
}

static void two(SpectralObj s, int f, const float *spec, float *valueArr, float *freArr) {
    if (!s || !spec || !valueArr || !freArr || s->timeLength < 1) return;
    const size_t T = (size_t)s->timeLength;
    float *buf = (float *)malloc(sizeof(float) * 2 * T);
    if (!buf) { af_fail(AF_ERR_NOMEM, "spectral: out of host memory"); return; }
    const float par[4] = {0, 0, 0, 0};
    if (spectralObj_spectralBatch(s, spec, NULL, s->timeLength, 1, 1, &f, par, buf, AFB200_MEM_HOST, NULL) == AF_OK) {
        memcpy(valueArr, buf, sizeof(float) * T);
        memcpy(freArr, buf + T, sizeof(float) * T);
    }
    free(buf);
}

void spectralObj_flatness(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_FLATNESS, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_flux(SpectralObj s, float *m, int step, float p, int isPostive, int *isExp, int *type, float *d) {
    one(s, AFB200_SPECTRAL_FLUX, m, NULL, (float)step, p, 0,
        (isPostive ? 1 : 0) | (isExp && *isExp ? 2 : 0) | (type && *type ? 4 : 0), d);
}
void spectralObj_rolloff(SpectralObj s, float *m, float threshold, float *d) { one(s, AFB200_SPECTRAL_ROLLOFF, m, NULL, 0, 0, threshold, 0, d); }
void spectralObj_centroid(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_CENTROID, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_spread(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_SPREAD, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_skewness(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_SKEWNESS, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_kurtosis(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_KURTOSIS, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_entropy(SpectralObj s, float *m, int isNorm, float *d) { one(s, AFB200_SPECTRAL_ENTROPY, m, NULL, 0, 0, 0, isNorm ? 1 : 0, d); }
void spectralObj_crest(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_CREST, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_slope(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_SLOPE, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_decrease(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_DECREASE, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_bandWidth(SpectralObj s, float *m, float p, float *d) { one(s, AFB200_SPECTRAL_BANDWIDTH, m, NULL, 0, p, 0, 0, d); }
void spectralObj_rms(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_RMS, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_energy(SpectralObj s, float *m, int isLog, float gamma, float *d) { one(s, AFB200_SPECTRAL_ENERGY, m, NULL, 0, gamma, 0, isLog ? 1 : 0, d); }
void spectralObj_hfc(SpectralObj s, float *m, float *d) { one(s, AFB200_SPECTRAL_HFC, m, NULL, 0, 0, 0, 0, d); }
void spectralObj_sd(SpectralObj s, float *m, int step, int isPostive, float *d) { one(s, AFB200_SPECTRAL_SD, m, NULL, (float)step, 0, 0, isPostive ? 1 : 0, d); }
void spectralObj_sf(SpectralObj s, float *m, int step, int isPostive, float *d) { one(s, AFB200_SPECTRAL_SF, m, NULL, (float)step, 0, 0, isPostive ? 1 : 0, d); }
void spectralObj_mkl(SpectralObj s, float *m, int type, float *d) { one(s, AFB200_SPECTRAL_MKL, m, NULL, 0, 0, 0, type ? 4 : 0, d); }
void spectralObj_pd(SpectralObj s, float *m, float *ph, float *d) { if (ph) one(s, AFB200_SPECTRAL_PD, m, ph, 0, 0, 0, 0, d); }
void spectralObj_wpd(SpectralObj s, float *m, float *ph, float *d) { if (ph) one(s, AFB200_SPECTRAL_WPD, m, ph, 0, 0, 0, 0, d); }
void spectralObj_nwpd(SpectralObj s, float *m, float *ph, float *d) { if (ph) one(s, AFB200_SPECTRAL_NWPD, m, ph, 0, 0, 0, 0, d); }
void spectralObj_cd(SpectralObj s, float *m, float *ph, float *d) { if (ph) one(s, AFB200_SPECTRAL_CD, m, ph, 0, 0, 0, 0, d); }
void spectralObj_rcd(SpectralObj s, float *m, float *ph, float *d) { if (ph) one(s, AFB200_SPECTRAL_RCD, m, ph, 0, 0, 0, 0, d); }
void spectralObj_broadband(SpectralObj s, float *m, float threshold, float *d) { one(s, AFB200_SPECTRAL_BROADBAND, m, NULL, 0, 0, threshold, 0, d); }
void spectralObj_novelty(SpectralObj s, float *m, int step, float threshold, SpectralNoveltyMethodType *methodType,
                         SpectralNoveltyDataType *dataType, float *d) {
    const int mt = methodType ? (int)*methodType : SpectralNoveltyMethod_Sub;
    const int dt = dataType ? (int)*dataType : SpectralNoveltyData_Value;
    one(s, AFB200_SPECTRAL_NOVELTY, m, NULL, (float)step, 0, threshold, (mt & 3) | (dt == SpectralNoveltyData_Value ? 0 : 4), d);
}
void spectralObj_eef(SpectralObj s, float *m, int isNorm, float *d) { one(s, AFB200_SPECTRAL_EEF, m, NULL, 0, 0, 0, isNorm ? 1 : 0, d); }
void spectralObj_eer(SpectralObj s, float *m, int isNorm, float gamma, float *d) { one(s, AFB200_SPECTRAL_EER, m, NULL, 0, gamma, 0, isNorm ? 1 : 0, d); }
void spectralObj_max(SpectralObj s, float *m, float *v, float *f) { two(s, AFB200_SPECTRAL_MAX, m, v, f); }
void spectralObj_mean(SpectralObj s, float *m, float *v, float *f) { two(s, AFB200_SPECTRAL_MEAN, m, v, f); }
void spectralObj_var(SpectralObj s, float *m, float *v, float *f) {
    if (s && s->nb < 2) return;                  /* spectral_algorithm.c:929-931 */
    two(s, AFB200_SPECTRAL_VAR, m, v, f);
}

void spectralObj_free(SpectralObj s) {
    if (!s) return;
    af_pipe_free(&s->pipe);
    af_dev_free(s->dFre); af_dev_free(s->dIdx);
    free(s->fre); free(s->idx);
    free(s);
}
