/* af_st.c -- STObj and FSTObj of the C ABI (host C; compute = the forward FFT of af_launch_stft, then kernels/st.cu).
 * Interface spec: src/st_algorithm.h:14-24 and src/fst_algorithm.h:14-20; behaviour src/st_algorithm.c:41-297 and
 * src/fst_algorithm.c:49-362.  Neither object builds an N x N table: ST keeps its bin list and one float per bin (the
 * Gaussian's exponent scale), FST one int per frequency row (its partition segment).  Both go to the device at the first
 * compute call after a change. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueST {
    int radix2Exp, fftLength;
    float factor, norm;
    int *bins;            /* binLength */
    float *v;             /* binLength: -factor 2 pi^2 / i^(2 norm) as the reference rounds it (v of bin 0 unused) */
    int binLength;
    int dirty;            /* bins / v changed since the last upload */
    void *dBins, *dV;
    AfDevBuf spec;        /* FULL spectrum planes of the clips */
    AfPipe pipe;
};

struct OpaqueFST {
    int radix2Exp, fftLength;
    int *seg;             /* N/2+1: (partition offset << 5) | log2 of the segment length of frequency row f */
    void *dSeg;
    AfDevBuf spec, part;  /* HALF spectrum planes, right half of the partition (N/2+1 complex per clip) */
    AfPipe pipe;
};

static int too_long(const char *who, int radix2Exp) {
    const long long n = 1LL << radix2Exp;
    return af_fail(-2, "%s: radix2Exp=%d; the largest supported is %d (one clip's full-band output would be %lld MB per "
                   "plane)", who, radix2Exp, AF_ST_MAX_EXP, (n / 2 + 1) * n * 4 / (1 << 20));
}

/* ---------------- ST (st_algorithm.c) ---------------- */

/* _stObj_initWinData (:235): evaluated in double from the float factor and powf, stored as a float */
static float st_v(int i, float factor, float norm) {
    float value = 0;
    if (i != 0) value = -factor * 2 * M_PI * M_PI / (powf(i, 2 * norm));
    return value;
}

static void st_fill_v(STObj s) {
    for (int r = 0; r < s->binLength; r++) s->v[r] = st_v(s->bins[r], s->factor, s->norm);
    s->dirty = 1;
}

int stObj_new(STObj *stObj, int radix2Exp, int minIndex, int maxIndex, float *factor, float *norm) {
    af_clear_error();
    if (!stObj) return -1;
    if (radix2Exp < 1) { af_fail(-1, "stObj_new: radix2Exp=%d; at least 1 is needed", radix2Exp); return -1; }
    if (radix2Exp > AF_ST_MAX_EXP) { too_long("stObj_new", radix2Exp); return -2; }
    const int N = 1 << radix2Exp;
    STObj s = (STObj)calloc(1, sizeof(struct OpaqueST));
    if (!s) return -1;
    s->radix2Exp = radix2Exp; s->fftLength = N;
    s->factor = factor && *factor > 0 ? *factor : 1;               /* :64-74 */
    s->norm = norm && *norm > 0 ? *norm : 1;
    if (minIndex >= maxIndex || minIndex < 0 || maxIndex > N / 2) { minIndex = 0; maxIndex = N / 2; }   /* :90-93 */
    s->binLength = maxIndex - minIndex + 1;
    s->bins = (int *)malloc(sizeof(int) * (size_t)s->binLength);
    s->v = (float *)malloc(sizeof(float) * (size_t)s->binLength);
    if (!s->bins || !s->v) { stObj_free(s); return -1; }
    for (int r = 0; r < s->binLength; r++) s->bins[r] = minIndex + r;
    st_fill_v(s);
    *stObj = s;
    return 0;
}

void stObj_useBinArr(STObj s, int *binArr, int length) {
    if (!s || length < 0 || (!binArr && length > 0)) return;
    for (int i = 0; i < length; i++)
        if (binArr[i] > s->fftLength / 2 || binArr[i] < 0) return;   /* :120-125: the whole list is ignored */
    int *bins = (int *)malloc(sizeof(int) * (size_t)(length ? length : 1));
    float *v = (float *)malloc(sizeof(float) * (size_t)(length ? length : 1));
    if (!bins || !v) { free(bins); free(v); af_fail(AF_ERR_NOMEM, "stObj_useBinArr: out of host memory"); return; }
    if (length) memcpy(bins, binArr, sizeof(int) * (size_t)length);
    free(s->bins); free(s->v);
    s->bins = bins; s->v = v; s->binLength = length;
    st_fill_v(s);
}

void stObj_setValue(STObj s, float factor, float norm) {
    if (!s || (s->factor == factor && s->norm == norm)) return;     /* :137-139 */
    s->factor = factor; s->norm = norm;
    st_fill_v(s);
}

int stObj_getBinLength(STObj s) { return s ? s->binLength : 0; }

static int st_device(STObj s) {
    int rc = af_device_ready();
    if (rc || !s->dirty) return rc;
    af_dev_free(s->dBins); af_dev_free(s->dV);
    s->dBins = s->dV = NULL;
    const size_t n = (size_t)(s->binLength ? s->binLength : 1);
    if ((rc = af_dev_upload(&s->dBins, s->bins, sizeof(int) * n)) || (rc = af_dev_upload(&s->dV, s->v, sizeof(float) * n)))
        return rc;
    s->dirty = 0;
    return AF_OK;
}

static int st_chunk(void *p, int nb, float *const *d, void *st) {
    STObj s = (STObj)p;
    const int N = s->fftLength;
    int rc;
    if ((rc = af_devbuf_reserve(&s->spec, sizeof(float) * 2 * (size_t)nb * N))) return rc;
    float *specRe = (float *)s->spec.ptr, *specIm = specRe + (size_t)nb * N;
    AfFrameSrc src;
    memset(&src, 0, sizeof(src));
    src.fftLength = N; src.slideLength = N; src.dataLength = N; src.timeLength = 1; src.batch = nb;
    src.validLength = N; src.padMode = PaddingMode_Constant; src.data = d[0];
    if ((rc = af_launch_stft(&src, AF_STFT_FULL, 1.0f, specRe, specIm, st))) return rc;
    return af_launch_st(d[0], specRe, specIm, (const int *)s->dBins, (const float *)s->dV, s->binLength, s->radix2Exp, nb,
                        d[1], d[2], st);
}

int stObj_stBatch(STObj s, const float *data, int batch, float *mReal, float *mImag, int memKind, void *stream) {
    if (!s || !data || !mReal || !mImag || batch < 0) return af_fail(AF_ERR_ARG, "stObj_stBatch: bad argument");
    af_clear_error();
    int rc = st_device(s);
    if (rc) return rc;
    if (batch == 0 || s->binLength == 0) return AF_OK;
    const size_t outPer = (size_t)s->binLength * s->fftLength;
    const AfPlane pl[3] = {{data, (size_t)s->fftLength, AF_IN, 0}, {mReal, outPer, AF_OUT, 0}, {mImag, outPer, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, st_chunk, s, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

void stObj_st(STObj s, float *dataArr, float *mRealArr, float *mImageArr) {
    if (!s || !dataArr || !mRealArr || !mImageArr) return;
    stObj_stBatch(s, dataArr, 1, mRealArr, mImageArr, AFB200_MEM_HOST, NULL);
}

void stObj_free(STObj s) {
    if (!s) return;
    af_dev_free(s->dBins); af_dev_free(s->dV);
    af_devbuf_free(&s->spec);
    af_pipe_free(&s->pipe);
    free(s->bins); free(s->v);
    free(s);
}

/* ---------------- FST (fst_algorithm.c) ---------------- */

int fstObj_new(FSTObj *fstObj, int radix2Exp) {
    af_clear_error();
    if (!fstObj) return -1;
    if (radix2Exp < 3) return -1;                                   /* :67-69 */
    if (radix2Exp > AF_ST_MAX_EXP) { too_long("fstObj_new", radix2Exp); return -2; }
    const int N = 1 << radix2Exp, length = 2 * radix2Exp;
    FSTObj s = (FSTObj)calloc(1, sizeof(struct OpaqueFST));
    int *lenArr = (int *)calloc((size_t)length, sizeof(int));
    if (s) s->seg = (int *)calloc((size_t)N / 2 + 1, sizeof(int));
    if (!s || !lenArr || !s->seg) { free(lenArr); fstObj_free(s); return -1; }
    s->radix2Exp = radix2Exp; s->fftLength = N;
    /* _fstObj_initPartition (:293-317): 1, N/4 .. 2, 1, 1, 1, 2 .. N/4 */
    lenArr[0] = lenArr[length / 2 - 1] = lenArr[length / 2] = 1;
    for (int i = 1; i < length / 2 - 1; i++) lenArr[i] = 1 << (length / 2 - 1 - i);
    for (int i = length / 2 + 1, j = 0; i < length; i++, j++) lenArr[i] = 1 << j;
    /* _fstObj_initReassign (:319-362): segment i (first element `start`) fills index rows N - start - len .. N - start - 1,
     * and fstObj_fst reads row N/2 - f for frequency f; column l holds element start + l / (N / len).  Only rows 0 .. N/2
     * are read, so every frequency lands in the right half of the partition, from position N/2 - 1 on. */
    for (int i = 0, start = 0; i < length; start += lenArr[i], i++) {
        int lg = 0;
        while ((1 << lg) < lenArr[i]) lg++;
        for (int k = N - start - lenArr[i]; k < N - start; k++) {
            if (k < 0 || k > N / 2) continue;
            s->seg[N / 2 - k] = ((start - (N / 2 - 1)) << 5) | lg;
        }
    }
    free(lenArr);
    *fstObj = s;
    return 0;
}

static int fst_device(FSTObj s) {
    int rc = af_device_ready();
    if (rc || s->dSeg) return rc;
    return af_dev_upload(&s->dSeg, s->seg, sizeof(int) * ((size_t)s->fftLength / 2 + 1));
}

typedef struct { FSTObj s; int minIndex, rows; } FstCall;

static int fst_chunk(void *p, int nb, float *const *d, void *st) {
    const FstCall *c = (const FstCall *)p;
    FSTObj s = c->s;
    const int N = s->fftLength, width = N / 2 + 1;
    int rc;
    if ((rc = af_devbuf_reserve(&s->spec, sizeof(float) * 2 * (size_t)nb * width)) ||
        (rc = af_devbuf_reserve(&s->part, sizeof(float) * 2 * (size_t)nb * width)))
        return rc;
    float *specRe = (float *)s->spec.ptr, *specIm = specRe + (size_t)nb * width;
    AfFrameSrc src;
    memset(&src, 0, sizeof(src));
    src.fftLength = N; src.slideLength = N; src.dataLength = N; src.timeLength = 1; src.batch = nb;
    src.validLength = N; src.padMode = PaddingMode_Constant; src.data = d[0];
    if ((rc = af_launch_stft(&src, AF_STFT_HALF, 1.0f, specRe, specIm, st))) return rc;
    return af_launch_fst(specRe, specIm, (float *)s->part.ptr, (const int *)s->dSeg, c->minIndex, c->rows, s->radix2Exp, nb,
                         d[1], d[2], st);
}

int fstObj_fstBatch(FSTObj s, const float *data, int batch, int minIndex, int maxIndex, float *mReal, float *mImag,
                    int memKind, void *stream) {
    if (!s || !data || !mReal || !mImag || batch < 0) return af_fail(AF_ERR_ARG, "fstObj_fstBatch: bad argument");
    af_clear_error();
    const int N = s->fftLength;
    if (minIndex < 0) minIndex = 0;                                 /* :160-171 */
    if (maxIndex > N / 2) maxIndex = N / 2;
    if (minIndex > maxIndex) { minIndex = 0; maxIndex = N / 2; }
    int rc = fst_device(s);
    if (rc) return rc;
    if (batch == 0) return AF_OK;
    FstCall c = {s, minIndex, maxIndex - minIndex + 1};
    const size_t outPer = (size_t)c.rows * N;
    const AfPlane pl[3] = {{data, (size_t)N, AF_IN, 0}, {mReal, outPer, AF_OUT, 0}, {mImag, outPer, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, fst_chunk, &c, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

void fstObj_fst(FSTObj s, float *dataArr, int minIndex, int maxIndex, float *mRealArr, float *mImageArr) {
    if (!s || !dataArr || !mRealArr || !mImageArr) return;
    fstObj_fstBatch(s, dataArr, 1, minIndex, maxIndex, mRealArr, mImageArr, AFB200_MEM_HOST, NULL);
}

void fstObj_free(FSTObj s) {
    if (!s) return;
    af_dev_free(s->dSeg);
    af_devbuf_free(&s->spec);
    af_devbuf_free(&s->part);
    af_pipe_free(&s->pipe);
    free(s->seg);
    free(s);
}
