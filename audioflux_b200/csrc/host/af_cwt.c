/* af_cwt.c -- CWT object of the C ABI (host C; compute = kernels/cwt.cu).
 * Interface spec: src/cwt_algorithm.h:14-45; behaviour src/cwt_algorithm.c:73-334
 * (parameters), :361-483 (compute). */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"
#include "../../../include/afb200_pwt.h"

struct OpaqueCWT {
    int num, radix2Exp, dataLength, padLength, fftLength, log2fft, samplate, binPerOctave;
    float lowFre, highFre;
    SpectralFilterBankScaleType scaleType;
    AfWavelet wavelet;
    float *freBandArr, *scaleArr;
    int *binBandArr;
    /* device (lazy) */
    int devReady;
    void *stream;
    float *dScale;
    AfDevBuf dIn, dWork, dOutRe, dOutIm;
    float *bankHost, *dBank;       /* PWT: auditory bank num x (fftLength/2+1) instead of a wavelet family */
    int bankWidth;
    int detEnabled;                /* cwtObj_enableDet */
    int haveSpec;                  /* dWork starts with the spectrum of the last single-clip call */
    AfDevBuf dSupport;             /* fast path: per bank row the bins above 2^-28 of its peak (filled by the launcher) */
    int supportReady;
};

int cwtObj_new(CWTObj *out, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre,
               int *binPerOctave, WaveletContinueType *waveletType, SpectralFilterBankScaleType *scaleType,
               float *gamma, float *beta, int *isPad) {
    if (!out) return -1;
    *out = NULL;
    if (radix2Exp < 1 || radix2Exp > 30) { printf("radix2Exp is error!\n"); return -100; }
    int sr = 32000;
    if (samplate && *samplate > 0 && *samplate <= 196000) sr = *samplate;
    SpectralFilterBankScaleType scale = scaleType ? *scaleType : SpectralFilterBankScale_Octave;
    if (scale > SpectralFilterBankScale_Log) { printf("scaleType is error!\n"); return 1; }
    int bpo = 12;
    if (binPerOctave && *binPerOctave >= 4 && *binPerOctave <= 48) bpo = *binPerOctave;
    const int N = 1 << radix2Exp;
    AfRange range;
    if (af_revise_range(num, N, sr, lowFre, highFre, scale, bpo, &range)) {
        printf(scale == SpectralFilterBankScale_Linear ? "scale linear: lowFre and num is large, overflow error\n"
                                                        : "scale log: lowFre and num is large, overflow error!\n");
        return -1;
    }
    if (num < 2 || num > N / 2 + 1) { printf("num is error!\n"); return -1; }
    AfWavelet w;
    if (af_wavelet_setup(&w, waveletType ? (int)*waveletType : WaveletContinue_Morse, gamma, beta)) return -1;
    if (w.waveletType == WaveletContinue_Bump && w.beta > w.gamma) {
        /* psi_hat(s w) = e^{1 - 1/(1 - ((s w - gamma)/beta)^2)} on |s w - gamma| < beta: with beta > gamma that interval
         * reaches w <= 0, and the reference (which evaluates the bump on its negative-frequency bins too,
         * cwt_filterBank.c:428-462) keeps those bins.  Every kernel of this library is one-sided. */
        af_fail(AF_ERR_UNSUPPORTED, "cwtObj_new: bump wavelet with beta %g > gamma %g has support on negative frequencies", w.beta, w.gamma);
        return -2;
    }
    int pad = 0;
    if (isPad && *isPad) pad = N <= 1e5 ? N / 2 : (int)ceilf(log2f((float)N));
    const int fftLength = N + 2 * pad;
    if (fftLength & (fftLength - 1)) {
        af_fail(AF_ERR_UNSUPPORTED, "cwtObj_new: isPad with 2^%d samples gives a non power-of-two length %d "
                "(the reference falls back to an O(N^2) dense DFT there); use isPad=0", radix2Exp, fftLength);
        return -2;
    }
    CWTObj c = (CWTObj)calloc(1, sizeof(struct OpaqueCWT));
    if (!c) return -1;
    c->num = num; c->radix2Exp = radix2Exp; c->dataLength = N; c->padLength = pad; c->fftLength = fftLength;
    c->log2fft = radix2Exp + (pad ? 1 : 0);
    c->samplate = sr; c->binPerOctave = bpo; c->lowFre = range.low; c->highFre = range.high; c->scaleType = scale;
    c->wavelet = w;
    c->freBandArr = (float *)calloc((size_t)num + 2, sizeof(float));
    c->binBandArr = (int *)calloc((size_t)num + 2, sizeof(int));
    c->scaleArr = (float *)calloc((size_t)num, sizeof(float));
    if (!c->freBandArr || !c->binBandArr || !c->scaleArr) { cwtObj_free(c); return -1; }
    af_cwt_scales(num, N, sr, c->lowFre, c->highFre, scale, bpo, w.cf, c->freBandArr, c->binBandArr, c->scaleArr);
    *out = c;
    return 0;
}

float *cwtObj_getFreBandArr(CWTObj c) { return c ? c->freBandArr : NULL; }
int *cwtObj_getBinBandArr(CWTObj c) { return c ? c->binBandArr : NULL; }

static int cwt_device(CWTObj c) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (c->devReady) return AF_OK;
    if ((rc = af_stream_create(&c->stream))) return rc;
    if ((rc = af_dev_upload((void **)&c->dScale, c->scaleArr, sizeof(float) * (size_t)c->num))) return rc;
    if (c->bankHost && (rc = af_dev_upload((void **)&c->dBank, c->bankHost, sizeof(float) * (size_t)c->num * c->bankWidth))) return rc;
    if ((rc = af_devbuf_reserve(&c->dSupport, sizeof(int) * 3 * (size_t)c->num))) return rc;
    c->devReady = 1;
    return AF_OK;
}

static void cwt_args(CWTObj c, int batch, int det, AfCwtArgs *a) {
    memset(a, 0, sizeof(*a));
    a->det = det;
    a->log2n = c->log2fft; a->num = c->num; a->batch = batch; a->padLength = c->padLength;
    a->dataLength = c->dataLength; a->wavelet = c->wavelet; a->scaleArr = c->dScale;
    a->bankTable = c->dBank; a->bankWidth = c->bankWidth;
    a->support = (int *)c->dSupport.ptr; a->supportReady = &c->supportReady;
}

/* dData [batch x N] -> planes [batch x num x N]; the batch is cut into chunks that fit the workspace */
static int cwt_compute(CWTObj c, const float *dData, int batch, int det, float *dRe, float *dIm, void *st) {
    AfCwtArgs a;
    size_t budget = af_dev_free_bytes() / 3 + c->dWork.bytes;
    if (budget > ((size_t)24 << 30)) budget = (size_t)24 << 30;
    /* largest chunk whose workspace (spectra + inter-leg buffer, or the fused path's fixed ring) fits the budget */
    int chunk = batch;
    const char *force = getenv("AFB200_CWT_CHUNK");       /* test hook: clips per workspace chunk */
    if (force && atoi(force) > 0 && atoi(force) < chunk) chunk = atoi(force);
    for (;;) {
        cwt_args(c, chunk, det, &a);
        if (af_cwt_workspace_bytes(&a) <= budget || chunk == 1) break;
        chunk = (chunk + 1) / 2;
    }
    while ((long long)chunk * c->num > 0x7fffffffLL / 2) chunk /= 2;
    cwt_args(c, chunk, det, &a);
    int rc = af_devbuf_reserve(&c->dWork, af_cwt_workspace_bytes(&a));
    if (rc) return rc;
    const size_t outClip = (size_t)c->num * c->dataLength;
    for (int c0 = 0; c0 < batch; c0 += chunk) {
        const int nb = batch - c0 < chunk ? batch - c0 : chunk;
        cwt_args(c, nb, det, &a);
        if ((rc = af_launch_cwt(&a, dData ? dData + (size_t)c0 * c->dataLength : NULL, c->dWork.ptr, dRe + (size_t)c0 * outClip,
                                dIm + (size_t)c0 * outClip, st))) return rc;
    }
    c->haveSpec = batch == 1;       /* the workspace now starts with this clip's spectrum (cwtObj_cwtDet(NULL) reuses it) */
    return AF_OK;
}

static int cwt_batch(CWTObj c, const float *data, int batch, int det, float *mReal4, float *mImag4, int memKind,
                     void *stream, const char *who) {
    if (!c || !mReal4 || !mImag4 || batch <= 0) return af_fail(AF_ERR_ARG, "%s: bad argument", who);
    af_clear_error();
    int rc = cwt_device(c);
    if (rc) return rc;
    void *st = stream ? stream : c->stream;
    if (!data) {                        /* cwtObj_cwtDet(obj, NULL, ...): the spectrum of the last single-clip call */
        if (batch != 1 || !c->haveSpec) return af_fail(AF_ERR_ARG, "%s: no data and no spectrum of a previous single-clip call", who);
        if (memKind == AFB200_MEM_DEVICE) return cwt_compute(c, NULL, 1, det, mReal4, mImag4, stream);
        const size_t outB = sizeof(float) * (size_t)c->num * c->dataLength;
        if ((rc = af_devbuf_reserve(&c->dOutRe, outB)) || (rc = af_devbuf_reserve(&c->dOutIm, outB))) return rc;
        if ((rc = cwt_compute(c, NULL, 1, det, (float *)c->dOutRe.ptr, (float *)c->dOutIm.ptr, st))) return rc;
        if ((rc = af_memcpy_d2h(mReal4, c->dOutRe.ptr, outB, st)) || (rc = af_memcpy_d2h(mImag4, c->dOutIm.ptr, outB, st))) return rc;
        return af_stream_sync(st);
    }
    if (memKind == AFB200_MEM_DEVICE) {
        st = stream;
        return cwt_compute(c, data, batch, det, mReal4, mImag4, st);
    }
    /* host pointers: chunks of clips whose planes fit a bounded staging buffer (<= 512 MB per plane, at least one clip):
     * one copy in, one launch sequence over chunk x num items, two copies out per chunk.  Long transforms (2^19 points:
     * 176 MB per plane and clip) go two clips at a time, the short windows of CWT.ccwt (2^12 points) hundreds at a time
     * instead of one latency-bound round trip per window. */
    const size_t inB = sizeof(float) * (size_t)c->dataLength, outB = sizeof(float) * (size_t)c->num * c->dataLength;
    size_t chunk = ((size_t)512 << 20) / outB;
    if (chunk < 1) chunk = 1;
    if (chunk > (size_t)batch) chunk = (size_t)batch;
    if ((rc = af_devbuf_reserve(&c->dIn, chunk * inB)) || (rc = af_devbuf_reserve(&c->dOutRe, chunk * outB)) ||
        (rc = af_devbuf_reserve(&c->dOutIm, chunk * outB))) return rc;
    for (int b = 0; b < batch; b += (int)chunk) {
        const size_t nb = (size_t)(batch - b) < chunk ? (size_t)(batch - b) : chunk;
        if ((rc = af_memcpy_h2d(c->dIn.ptr, data + (size_t)b * c->dataLength, nb * inB, st))) return rc;
        if ((rc = cwt_compute(c, (const float *)c->dIn.ptr, (int)nb, det, (float *)c->dOutRe.ptr, (float *)c->dOutIm.ptr, st))) return rc;
        if ((rc = af_memcpy_d2h(mReal4 + (size_t)b * c->num * c->dataLength, c->dOutRe.ptr, nb * outB, st)) ||
            (rc = af_memcpy_d2h(mImag4 + (size_t)b * c->num * c->dataLength, c->dOutIm.ptr, nb * outB, st))) return rc;
        if ((rc = af_stream_sync(st))) return rc;
    }
    if (batch > 1) c->haveSpec = 0;      /* cwtObj_cwtDet(NULL) continues a SINGLE-clip call only */
    return AF_OK;
}

int cwtObj_cwtBatch(CWTObj c, const float *data, int batch, float *mReal4, float *mImag4, int memKind, void *stream) {
    if (!data) return af_fail(AF_ERR_ARG, "cwtObj_cwtBatch: bad argument");
    return cwt_batch(c, data, batch, 0, mReal4, mImag4, memKind, stream, "cwtObj_cwtBatch");
}

void cwtObj_cwt(CWTObj c, float *dataArr, float *mRealArr4, float *mImageArr4) {
    if (!c || !dataArr) return;
    cwtObj_cwtBatch(c, dataArr, 1, mRealArr4, mImageArr4, AFB200_MEM_HOST, NULL);
}

/* ---- derivative transform: bank * j*omega (cwt_algorithm.c:352-358, 485-528); feeds synchrosqueezing ---- */
void cwtObj_enableDet(CWTObj c, int flag) { if (c && flag) c->detEnabled = 1; }   /* never switched off again, as :494-496 */

int cwtObj_cwtDetBatch(CWTObj c, const float *data, int batch, float *mReal4, float *mImag4, int memKind, void *stream) {
    if (c && !c->detEnabled) return af_fail(AF_ERR_ARG, "cwtObj_cwtDetBatch: call cwtObj_enableDet(obj, 1) first");
    return cwt_batch(c, data, batch, 1, mReal4, mImag4, memKind, stream, "cwtObj_cwtDetBatch");
}

void cwtObj_cwtDet(CWTObj c, float *dataArr, float *mRealArr4, float *mImageArr4) {
    if (!c || !c->detEnabled) return;                 /* silent without enableDet, like :355 */
    cwtObj_cwtDetBatch(c, dataArr, 1, mRealArr4, mImageArr4, AFB200_MEM_HOST, NULL);
}

int cwtObj_getFilterBankArr(CWTObj c, float *bank) {
    if (!c || !bank) return af_fail(AF_ERR_ARG, "cwtObj_getFilterBankArr: bad argument");
    /* host evaluation of the same closed form the device uses (row 0 = highest band) */
    const int n = c->fftLength;
    for (int i = 0; i < c->num; i++)
        for (int k = 0; k < n; k++) {
            float v = 0.0f;
            if (c->bankHost) { bank[(size_t)i * n + k] = k < c->bankWidth ? c->bankHost[(size_t)i * c->bankWidth + k] : 0.0f; continue; }
            if (k <= n / 2) { float omega = (float)((double)k * 2.0 * M_PI / (double)n); v = af_wavelet_eval(&c->wavelet, c->scaleArr[i] * omega); }
            bank[(size_t)i * n + k] = v;
        }
    return AF_OK;
}

void cwtObj_free(CWTObj c) {
    if (!c) return;
    af_devbuf_free(&c->dIn); af_devbuf_free(&c->dWork); af_devbuf_free(&c->dOutRe); af_devbuf_free(&c->dOutIm);
    af_dev_free(c->dScale); af_dev_free(c->dBank);
    af_devbuf_free(&c->dSupport);
    free(c->bankHost);
    af_stream_destroy(c->stream);
    free(c->freBandArr); free(c->binBandArr); free(c->scaleArr);
    free(c);
}

/* ================= PWT: pseudo wavelet transform (src/pwt_algorithm.h:16-31, src/pwt_algorithm.c:63-348) =================
 * Same FFT -> bank x spectrum -> IFFT structure as the CWT with the auditory filter bank of the BFT path
 * (auditory_filterBank with isPseudo = 1: rows of fftLength entries, zero above fftLength/2) instead of an analytic
 * wavelet, so the object is a CWT core whose kernels read the bank from a table. */
struct OpaquePWT { struct OpaqueCWT c; };

int pwtObj_new(PWTObj *out, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre, int *binPerOctave,
               SpectralFilterBankScaleType *scaleType, SpectralFilterBankStyleType *styleType,
               SpectralFilterBankNormalType *normalType, int *isPadding) {
    if (!out) return -1;
    *out = NULL;
    if (radix2Exp < 1 || radix2Exp > 30) { printf("radix2Exp is error!\n"); return -100; }
    int sr = 32000;
    if (samplate && *samplate > 0 && *samplate <= 196000) sr = *samplate;
    SpectralFilterBankScaleType scale = scaleType ? *scaleType : SpectralFilterBankScale_Octave;
    if (scale > SpectralFilterBankScale_Log) { printf("scaleType is error!\n"); return 1; }
    int bpo = 12;
    if (binPerOctave && *binPerOctave >= 4 && *binPerOctave <= 48) bpo = *binPerOctave;
    const int N = 1 << radix2Exp;
    AfRange range;
    if (af_revise_range(num, N, sr, lowFre, highFre, scale, bpo, &range)) {
        printf(scale == SpectralFilterBankScale_Linear ? "scale linear: lowFre and num is large, overflow error\n"
                                                        : "scale log: lowFre and num is large, overflow error!\n");
        return -1;
    }
    if (num < 2 || num > N / 2 + 1) { printf("num is error!\n"); return -1; }
    int pad = 0;
    if (isPadding && *isPadding) pad = N <= 1e5 ? N / 2 : (int)ceilf(log2f((float)N));
    const int fftLength = N + 2 * pad;
    if (fftLength & (fftLength - 1)) {
        af_fail(AF_ERR_UNSUPPORTED, "pwtObj_new: isPadding with 2^%d samples gives a non power-of-two length %d "
                "(the reference falls back to an O(N^2) dense DFT there); use isPadding=0", radix2Exp, fftLength);
        return -2;
    }
    PWTObj p = (PWTObj)calloc(1, sizeof(struct OpaquePWT));
    if (!p) return -1;
    CWTObj c = &p->c;
    c->num = num; c->radix2Exp = radix2Exp; c->dataLength = N; c->padLength = pad; c->fftLength = fftLength;
    c->log2fft = radix2Exp + (pad ? 1 : 0);
    c->samplate = sr; c->binPerOctave = bpo; c->lowFre = range.low; c->highFre = range.high; c->scaleType = scale;
    c->bankWidth = fftLength / 2 + 1;
    c->bankHost = (float *)calloc((size_t)num * c->bankWidth, sizeof(float));
    c->freBandArr = (float *)calloc((size_t)num + 2, sizeof(float));
    c->binBandArr = (int *)calloc((size_t)num + 2, sizeof(int));
    c->scaleArr = (float *)calloc((size_t)num, sizeof(float));
    if (!c->bankHost || !c->freBandArr || !c->binBandArr || !c->scaleArr) { pwtObj_free(p); return -1; }
    const int style = styleType ? (int)*styleType : SpectralFilterBankStyle_Slaney;
    if (style == SpectralFilterBankStyle_Gammatone) {
        /* the reference writes the gammatone rows of its pseudo bank fftLength/2+1 apart into rows that are fftLength long
         * (auditory_filterBank.c:541-549 with isPseudo = 1): the rows it then transforms with overlap one another */
        af_fail(AF_ERR_UNSUPPORTED, "pwtObj_new: the Gammatone style is not supported (the reference's pseudo bank rows overlap)");
        pwtObj_free(p); return -2;
    }
    if (af_auditory_filterbank(num, fftLength, sr, scale, style,
                               normalType ? (int)*normalType : SpectralFilterBankNormal_None, c->lowFre, c->highFre, bpo,
                               c->bankHost, c->freBandArr, c->binBandArr)) { pwtObj_free(p); return -2; }
    if (af_filterbank_clipped()) {
        /* band edges beyond samplate / 2 (Log / Linspace scales with highFre at Nyquist): the reference's pseudo bank keeps
         * those weights on the negative-frequency bins; this library's transform is one-sided */
        af_fail(AF_ERR_UNSUPPORTED, "pwtObj_new: %d filter weights fall above the Nyquist bin (band edges beyond samplate/2); "
                "lower highFre", af_filterbank_clipped());
        pwtObj_free(p); return -2;
    }
    *out = p;
    return 0;
}

float *pwtObj_getFreBandArr(PWTObj p) { return p ? p->c.freBandArr : NULL; }
int *pwtObj_getBinBandArr(PWTObj p) { return p ? p->c.binBandArr : NULL; }
void pwtObj_enableDet(PWTObj p, int flag) { if (p) cwtObj_enableDet(&p->c, flag); }
int pwtObj_pwtBatch(PWTObj p, const float *data, int batch, float *mReal3, float *mImag3, int memKind, void *stream) {
    if (!p || !data) return af_fail(AF_ERR_ARG, "pwtObj_pwtBatch: bad argument");
    return cwt_batch(&p->c, data, batch, 0, mReal3, mImag3, memKind, stream, "pwtObj_pwtBatch");
}
int pwtObj_pwtDetBatch(PWTObj p, const float *data, int batch, float *mReal3, float *mImag3, int memKind, void *stream) {
    if (!p) return af_fail(AF_ERR_ARG, "pwtObj_pwtDetBatch: bad argument");
    if (!p->c.detEnabled) return af_fail(AF_ERR_ARG, "pwtObj_pwtDetBatch: call pwtObj_enableDet(obj, 1) first");
    return cwt_batch(&p->c, data, batch, 1, mReal3, mImag3, memKind, stream, "pwtObj_pwtDetBatch");
}
void pwtObj_pwt(PWTObj p, float *dataArr, float *mRealArr3, float *mImageArr3) {
    if (!p || !dataArr) return;
    pwtObj_pwtBatch(p, dataArr, 1, mRealArr3, mImageArr3, AFB200_MEM_HOST, NULL);
}
void pwtObj_pwtDet(PWTObj p, float *dataArr, float *mRealArr3, float *mImageArr3) {
    if (!p || !p->c.detEnabled) return;
    pwtObj_pwtDetBatch(p, dataArr, 1, mRealArr3, mImageArr3, AFB200_MEM_HOST, NULL);
}
int pwtObj_getFilterBankArr(PWTObj p, float *bank) { return p ? cwtObj_getFilterBankArr(&p->c, bank) : af_fail(AF_ERR_ARG, "pwtObj_getFilterBankArr: bad argument"); }
void pwtObj_free(PWTObj p) {
    if (!p) return;
    CWTObj c = &p->c;
    af_devbuf_free(&c->dIn); af_devbuf_free(&c->dWork); af_devbuf_free(&c->dOutRe); af_devbuf_free(&c->dOutIm);
    af_dev_free(c->dScale); af_dev_free(c->dBank);
    af_devbuf_free(&c->dSupport);
    af_stream_destroy(c->stream);
    free(c->bankHost); free(c->freBandArr); free(c->binBandArr); free(c->scaleArr);
    free(p);
}
