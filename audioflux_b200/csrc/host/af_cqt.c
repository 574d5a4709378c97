/* af_cqt.c -- CQT object of the C ABI (host C; compute = kernels/cqt.cu).
 * Interface spec: src/cqt_algorithm.h:14-62; behaviour src/cqt_algorithm.c:110-247
 * (parameters), :266-299 (time length), :845-1061 (octave recursion). */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueCQT {
    int num, samplate, binPerOctave, octaveNum, fftLength, slideLength, isScale;
    float minFre;
    AfCqtBank bank;
    float *kappa2;                 /* host: interleaved (re, im) [bpo][fftLength] */
    float left32[32], right31[32];
    /* device (lazy) */
    int devReady;
    void *stream;
    float *dBfrag;                               /* tensor-core octave kernel: pre-split kernel fragments */
    unsigned char *dBimg;                        /* wgmma octave kernel: pre-swizzled shared-memory images of the kernels */
    float *dKappa2, *dLeft, *dRight, *dScale;    /* dScale: octaveNum x bpo, rebuilt when isScale flips */
    int scaleDirty;
    AfDevBuf dIn, dSigA, dSigB, dOutRe, dOutIm;
    /* post-processing of the last transform (chroma / cqcc) */
    int timeLength;                /* frames of the last cqtObj_cqt call (cqt_algorithm.c:463-478) */
    int chromaNum;
    float *dChromaBank, *dDctT;
    AfDevBuf dPostA, dPostB, dPostOut;
    AfPipe pipe;                   /* host-pointer batches: chunked copy-in / transform / copy-out */
    int pipeLength;
    /* streaming (isContinue, cqt_algorithm.c:346-456): full-rate samples that did not complete a hop wait for the next call */
    int isContinue;
    float *tail; int tailLength;   /* host; tailLength < 0: samples of the next call to skip (slide > fftLength) */
    float *cur; size_t curCap;
};

int cqtObj_newWith(CQTObj *out, int num, int *samplate, float *minFre, int *binPerOctave, float *factor,
                   float *beta, float *thresh, WindowType *windowType, int *slideLength, int *isContinue,
                   SpectralFilterBankNormalType *normalType, int *isScale) {
    if (!out) return -1;
    *out = NULL;
    int bpo = 12;
    if (binPerOctave && *binPerOctave > 0) bpo = *binPerOctave;
    if (bpo % 12 != 0) { printf("binPerOctave is error\n"); return -1; }
    if (num < bpo || num % bpo != 0) { printf("num is error\n"); return -1; }
    int sr = 32000; float fmin = 32.703196f, fac = 1, bet = 0, thr = 0.01f;
    if (samplate && *samplate > 0) sr = *samplate;
    if (minFre && *minFre > 0) fmin = *minFre;
    if (factor && *factor > 0) fac = *factor;
    if (beta && *beta > 0) bet = *beta;
    if (thresh && *thresh > 0) thr = *thresh;
    CQTObj c = (CQTObj)calloc(1, sizeof(struct OpaqueCQT));
    if (!c) return -1;
    c->num = num; c->samplate = sr; c->binPerOctave = bpo; c->octaveNum = num / bpo; c->minFre = fmin;
    c->isScale = isScale ? *isScale : 1;
    c->isContinue = isContinue ? *isContinue != 0 : 0;
    if (af_cqt_bank_build(&c->bank, num, sr, fmin, bpo, fac, bet, thr, windowType ? (int)*windowType : Window_Hann,
                          normalType ? (int)*normalType : SpectralFilterBankNormal_None)) { cqtObj_free(c); return -1; }
    c->fftLength = c->bank.fftLength;
    c->slideLength = (slideLength && *slideLength > 0) ? *slideLength : c->fftLength / 4;
    if ((c->slideLength >> (c->octaveNum - 1)) < 1) {
        af_fail(AF_ERR_ARG, "cqtObj_newWith: slideLength %d cannot be halved %d times", c->slideLength, c->octaveNum - 1);
        cqtObj_free(c); return -1;
    }
    const int n = c->fftLength;
    const size_t rows = (size_t)c->bank.rows;                     /* bpo, or num when beta != 0 (one kernel set per octave) */
    float *kr = (float *)malloc(sizeof(float) * rows * n), *ki = (float *)malloc(sizeof(float) * rows * n);
    c->kappa2 = (float *)malloc(sizeof(float) * 2 * rows * n);
    if (!kr || !ki || !c->kappa2 || af_cqt_time_kernels(&c->bank, kr, ki)) { free(kr); free(ki); cqtObj_free(c); return -1; }
    for (size_t i = 0; i < rows * n; i++) { c->kappa2[2 * i] = kr[i]; c->kappa2[2 * i + 1] = ki[i]; }
    free(kr); free(ki);
    af_decimator_taps(c->left32, c->right31);
    c->scaleDirty = 1;
    *out = c;
    return 0;
}

int cqtObj_new(CQTObj *out, int num, int samplate, float minFre, int *isContinue) {
    return cqtObj_newWith(out, num, &samplate, &minFre, NULL, NULL, NULL, NULL, NULL, NULL, isContinue, NULL, NULL);
}

/* cqt_algorithm.c:266-299: centre-padded frames, or -- streaming -- whole frames of (carried samples + new samples) */
static int cqt_time_length(const struct OpaqueCQT *c, int dataLength, int isContinue) {
    if (dataLength <= 0) return 0;
    if (!isContinue) return dataLength / c->slideLength + 1;
    return dataLength < c->fftLength ? 0 : (dataLength - c->fftLength) / c->slideLength + 1;
}
int cqtObj_calTimeLength(CQTObj c, int dataLength) {
    if (!c) return 0;
    if (c->isContinue) return dataLength + c->tailLength <= 0 ? 0 : cqt_time_length(c, dataLength + c->tailLength, 1);
    return cqt_time_length(c, dataLength, 0);
}
int cqtObj_getFFTLength(CQTObj c) { return c ? c->fftLength : 0; }
float *cqtObj_getFreBandArr(CQTObj c) { return c ? c->bank.freBandArr : NULL; }
void cqtObj_setScale(CQTObj c, int flag) { if (c && c->isScale != flag) { c->isScale = flag; c->scaleDirty = 1; } }

int cqtObj_getKernelBank(CQTObj c, float *kr, float *ki) {
    if (!c || !kr || !ki) return af_fail(AF_ERR_ARG, "cqtObj_getKernelBank: bad argument");
    size_t n = (size_t)c->bank.rows * (c->fftLength / 2 + 1);
    memcpy(kr, c->bank.kr, sizeof(float) * n); memcpy(ki, c->bank.ki, sizeof(float) * n);
    return AF_OK;
}

static int cqt_device(CQTObj c) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (!c->devReady) {
        if ((rc = af_stream_create(&c->stream))) return rc;
        /* kernel sets: one (the top octave's, shared) or -- VQT -- one per octave, set o at offset o * bpo rows */
        const int sets = c->bank.vqt ? c->octaveNum : 1;
        const size_t setFloats = 2 * (size_t)c->binPerOctave * c->fftLength;
        if ((rc = af_dev_upload((void **)&c->dKappa2, c->kappa2, sizeof(float) * setFloats * sets))) return rc;
        if (c->binPerOctave == 12 && c->fftLength % 64 == 0) {
            const size_t nf = (size_t)(c->fftLength / 8) * 96 * 4;
            float *bf = (float *)malloc(sizeof(float) * nf * sets);
            if (!bf) return AF_ERR_NOMEM;
            for (int s = 0; s < sets; s++) af_cqt_tc_fragments(c->kappa2 + setFloats * s, c->fftLength, bf + nf * s);
            rc = af_dev_upload((void **)&c->dBfrag, bf, sizeof(float) * nf * sets);
            free(bf);
            if (rc) return rc;
        }
        if (c->binPerOctave == 12 && c->fftLength % 128 == 0 && c->fftLength >= 256) {
            const size_t nb = (size_t)(c->fftLength / 128) * 32768;
            unsigned char *img = (unsigned char *)malloc(nb * sets);
            if (!img) return AF_ERR_NOMEM;
            for (int s = 0; s < sets; s++) af_cqt_wgmma_bimage(c->kappa2 + setFloats * s, c->fftLength, img + nb * s);
            rc = af_dev_upload((void **)&c->dBimg, img, nb * sets);
            free(img);
            if (rc) return rc;
        }
        if ((rc = af_dev_upload((void **)&c->dLeft, c->left32, sizeof(float) * 32))) return rc;
        if ((rc = af_dev_upload((void **)&c->dRight, c->right31, sizeof(float) * 32))) return rc;
        c->devReady = 1;
    }
    if (c->scaleDirty) {
        /* per (octave step k, bin j): sqrt(2^k) [/ sqrt(len)]  (cqt_algorithm.c:972-989, 1029-1036) */
        const int bpo = c->binPerOctave, octs = c->octaveNum;
        float *s = (float *)malloc(sizeof(float) * (size_t)octs * bpo);
        if (!s) return AF_ERR_NOMEM;
        for (int k = 0; k < octs; k++) {
            const int o = octs - 1 - k;
            const float d = k == 0 ? 1.0f : sqrtf((float)(1 << k));
            for (int j = 0; j < bpo; j++) {
                float v = d;
                if (c->isScale) v = v / c->bank.sLenArr[o * bpo + j];
                s[k * bpo + j] = v;
            }
        }
        af_dev_free(c->dScale); c->dScale = NULL;
        rc = af_dev_upload((void **)&c->dScale, s, sizeof(float) * (size_t)octs * bpo);
        free(s);
        if (rc) return rc;
        c->scaleDirty = 0;
    }
    return AF_OK;
}

/* dData [batch x dataLength] -> planes [batch x T x num] */
static int cqt_compute_ex(CQTObj c, const float *dData, int dataLength, int batch, int T, int padLeft, float *dRe, float *dIm, void *st) {
    if (T <= 0) return AF_OK;
    int rc;
    const size_t half = sizeof(float) * (size_t)batch * (dataLength / 2 + 1);
    if (c->octaveNum > 1 && ((rc = af_devbuf_reserve(&c->dSigA, half)) || (rc = af_devbuf_reserve(&c->dSigB, half)))) return rc;
    const float *sig = dData;
    int len = dataLength, stride = dataLength, hop = c->slideLength;
    for (int k = 0; k < c->octaveNum; k++) {
        const int o = c->octaveNum - 1 - k;
        if (k > 0) {
            float *dst = (float *)((k & 1) ? c->dSigA.ptr : c->dSigB.ptr);
            const int outStride = len / 2;
            if ((rc = af_launch_decimate2(sig, len, stride, batch, c->dLeft, c->dRight, dst, outStride, st))) return rc;
            sig = dst; len = len / 2; stride = outStride; hop /= 2;
        }
        if (len <= 0 || hop < 1) break;
        /* padded STFT semantics: drop the tail that does not fill a hop when more than one frame exists */
        const int frames = len / hop + 1;
        const int valid = frames > 1 ? len - len % hop : len;
        const char *kq = getenv("AFB200_CQT_KERNEL");
        /* kernel set of this octave: the shared top-octave set, or -- VQT -- the octave's own */
        const size_t set = c->bank.vqt ? (size_t)o : 0;
        const unsigned char *bimg = c->dBimg ? c->dBimg + set * (size_t)(c->fftLength / 128) * 32768 : NULL;
        const float *bfrag = c->dBfrag ? c->dBfrag + set * (size_t)(c->fftLength / 8) * 96 * 4 : NULL;
        const float *kappa = c->dKappa2 + set * 2 * (size_t)c->binPerOctave * c->fftLength;
        /* wgmma (default where the hop allows it) > mma.sync 3xTF32 > FP32 loop; AFB200_CQT_KERNEL = mma | fp32 forces the older ones */
        if (c->dBimg && af_cqt_wgmma_supported(c->fftLength, hop, c->binPerOctave) && !kq) {
            if ((rc = af_launch_cqt_octave_wgmma(sig, stride, batch, valid, c->fftLength, hop, padLeft, T, bimg,
                                                c->dScale + (size_t)k * c->binPerOctave, c->num, o * c->binPerOctave, dRe, dIm, st))) return rc;
            continue;
        }
        if (c->dBfrag && af_cqt_tc_supported(c->fftLength, hop, c->binPerOctave) && !(kq && !strcmp(kq, "fp32"))) {
            if ((rc = af_launch_cqt_octave_tc(sig, stride, batch, valid, c->fftLength, hop, padLeft, T, bfrag,
                                              c->dScale + (size_t)k * c->binPerOctave, c->num, o * c->binPerOctave, dRe, dIm, st))) return rc;
            continue;
        }
        if ((rc = af_launch_cqt_octave(sig, len, stride, batch, valid, c->fftLength, hop, padLeft, T, c->binPerOctave,
                                       kappa, c->dScale + (size_t)k * c->binPerOctave, c->num,
                                       o * c->binPerOctave, dRe, dIm, st))) return rc;
    }
    return AF_OK;
}

/* batched / device entry points are stateless: centre padding, every clip on its own */
static int cqt_compute(CQTObj c, const float *dData, int dataLength, int batch, float *dRe, float *dIm, void *st) {
    return cqt_compute_ex(c, dData, dataLength, batch, cqt_time_length(c, dataLength, 0), c->fftLength / 2, dRe, dIm, st);
}

static int cqt_chunk(void *obj, const float *dIn, int nb, float *dOut0, float *dOut1, void *st) {
    CQTObj c = (CQTObj)obj;
    return cqt_compute(c, dIn, c->pipeLength, nb, dOut0, dOut1, st);
}

int cqtObj_cqtBatch(CQTObj c, const float *data, int dataLength, int batch, float *mReal3, float *mImag3,
                    int memKind, void *stream) {
    if (!c || !data || !mReal3 || !mImag3 || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "cqtObj_cqtBatch: bad argument");
    af_clear_error();
    int rc = cqt_device(c);
    if (rc) return rc;
    const int T = cqt_time_length(c, dataLength, 0);
    void *st = stream ? stream : c->stream;
    if (memKind == AFB200_MEM_DEVICE) {
        st = stream;
        return cqt_compute(c, data, dataLength, batch, mReal3, mImag3, st);
    }
    c->pipeLength = dataLength;
    return af_pipe_run(&c->pipe, cqt_chunk, c, data, (size_t)dataLength, batch, mReal3, mImag3, (size_t)T * c->num, st);
}

/* streaming bookkeeping of _cqtObj_dealData (cqt_algorithm.c:346-456): 1 = *cur / *curLength hold tail + new samples */
static int cqt_continue_assemble(CQTObj c, const float *data, int dataLength, const float **cur, int *curLength) {
    const int n = c->fftLength, hop = c->slideLength;
    if (!c->tail) {
        c->tail = (float *)calloc((size_t)n + (size_t)hop + 1, sizeof(float));
        if (!c->tail) return 0;
    }
    const int total = c->tailLength + dataLength;
    if (total < n) {
        if (c->tailLength >= 0) memcpy(c->tail + c->tailLength, data, sizeof(float) * (size_t)dataLength);
        else if (dataLength + c->tailLength > 0) memcpy(c->tail, data - c->tailLength, sizeof(float) * (size_t)(dataLength + c->tailLength));
        c->tailLength = total;
        c->timeLength = 0;
        return 0;
    }
    const int tailLen = (total - n) % hop + (n - hop);
    if ((size_t)total + (size_t)n > c->curCap) {
        free(c->cur);
        c->curCap = (size_t)total + (size_t)n;
        c->cur = (float *)malloc(sizeof(float) * c->curCap);
        if (!c->cur) { c->curCap = 0; return 0; }
    }
    int len;
    if (c->tailLength < 0) {
        len = dataLength + c->tailLength;
        memcpy(c->cur, data - c->tailLength, sizeof(float) * (size_t)len);
    } else {
        if (c->tailLength > 0) memcpy(c->cur, c->tail, sizeof(float) * (size_t)c->tailLength);
        memcpy(c->cur + c->tailLength, data, sizeof(float) * (size_t)dataLength);
        len = c->tailLength + dataLength;
    }
    if (tailLen > 0) memcpy(c->tail, c->cur + (len - tailLen), sizeof(float) * (size_t)tailLen);
    c->tailLength = tailLen;
    *cur = c->cur; *curLength = len;
    return 1;
}

void cqtObj_cqt(CQTObj c, float *dataArr, int dataLength, float *mRealArr3, float *mImageArr3) {
    if (!c || !dataArr || dataLength <= 0) return;
    if (!c->isContinue) {
        c->timeLength = cqt_time_length(c, dataLength, 0);
        cqtObj_cqtBatch(c, dataArr, dataLength, 1, mRealArr3, mImageArr3, AFB200_MEM_HOST, NULL);
        return;
    }
    /* streaming: carried samples + new samples, frames start at t * slide (right zero padding, cqt_algorithm.c:1317-1319) */
    const float *x = NULL;
    int len = 0;
    if (!mRealArr3 || !mImageArr3) return;
    if (!cqt_continue_assemble(c, dataArr, dataLength, &x, &len)) return;
    af_clear_error();
    if (cqt_device(c)) return;
    const int T = cqt_time_length(c, len, 1);
    c->timeLength = T;
    if (T <= 0) return;
    const size_t inB = sizeof(float) * (size_t)len, outB = sizeof(float) * (size_t)T * c->num;
    void *st = c->stream;
    if (af_devbuf_reserve(&c->dIn, inB) || af_devbuf_reserve(&c->dOutRe, outB) || af_devbuf_reserve(&c->dOutIm, outB)) return;
    if (af_memcpy_h2d(c->dIn.ptr, x, inB, st)) return;
    if (cqt_compute_ex(c, (const float *)c->dIn.ptr, len, 1, T, 0, (float *)c->dOutRe.ptr, (float *)c->dOutIm.ptr, st)) return;
    if (af_memcpy_d2h(mRealArr3, c->dOutRe.ptr, outB, st) || af_memcpy_d2h(mImageArr3, c->dOutIm.ptr, outB, st)) return;
    af_stream_sync(st);
}

/* ---- chroma: rows x num CQT planes -> rows x chromaNum (cqt_algorithm.c:484-600) ---- */
int cqtObj_chromaBatch(CQTObj c, const float *mReal, const float *mImag, int rows, int chromaNum, int dataType,
                       int normType, float *out, int memKind, void *stream) {
    if (!c || !mReal || !mImag || !out || rows < 0) return af_fail(AF_ERR_ARG, "cqtObj_chromaBatch: bad argument");
    if (chromaNum < 1 || chromaNum > c->binPerOctave || c->binPerOctave % chromaNum != 0)
        return af_fail(AF_ERR_ARG, "cqtObj_chromaBatch: chromaNum=%d does not divide binPerOctave=%d", chromaNum, c->binPerOctave);
    if (normType < ChromaDataNormal_None || normType > ChromaDataNormal_P1) return af_fail(AF_ERR_ARG, "cqtObj_chromaBatch: normType=%d", normType);
    af_clear_error();
    int rc = cqt_device(c);
    if (rc) return rc;
    if (chromaNum != c->chromaNum) {
        float *bank = (float *)malloc(sizeof(float) * (size_t)chromaNum * c->num);
        if (!bank) return AF_ERR_NOMEM;
        af_chroma_cqt_bank(chromaNum, c->num, c->binPerOctave, c->minFre, bank);
        af_dev_free(c->dChromaBank); c->dChromaBank = NULL;
        rc = af_dev_upload((void **)&c->dChromaBank, bank, sizeof(float) * (size_t)chromaNum * c->num);
        free(bank);
        if (rc) return rc;
        c->chromaNum = chromaNum;
    }
    const int isMag = dataType == SpectralData_Mag;
    if (memKind == AFB200_MEM_DEVICE)
        return af_launch_chroma(mReal, mImag, rows, c->num, chromaNum, isMag, normType, c->dChromaBank, out, stream);
    void *st = stream ? stream : c->stream;
    const size_t inB = sizeof(float) * (size_t)rows * c->num, outB = sizeof(float) * (size_t)rows * chromaNum;
    if ((rc = af_devbuf_reserve(&c->dPostA, inB)) || (rc = af_devbuf_reserve(&c->dPostB, inB)) || (rc = af_devbuf_reserve(&c->dPostOut, outB))) return rc;
    if ((rc = af_memcpy_h2d(c->dPostA.ptr, mReal, inB, st)) || (rc = af_memcpy_h2d(c->dPostB.ptr, mImag, inB, st))) return rc;
    if ((rc = af_launch_chroma((const float *)c->dPostA.ptr, (const float *)c->dPostB.ptr, rows, c->num, chromaNum, isMag,
                               normType, c->dChromaBank, (float *)c->dPostOut.ptr, st))) return rc;
    if ((rc = af_memcpy_d2h(out, c->dPostOut.ptr, outB, st))) return rc;
    return af_stream_sync(st);
}

void cqtObj_chroma(CQTObj c, int *chromaNum, SpectralDataType *dataType, ChromaDataNormalType *normType,
                   float *mRealArr1, float *mImageArr1, float *mDataArr3) {
    if (!c || !mRealArr1 || !mImageArr1 || !mDataArr3) return;
    const int cn = chromaNum ? *chromaNum : 12;
    if (cn < 1 || cn > c->binPerOctave || c->binPerOctave % cn != 0) {
        printf("chromaNum and binPerOctave not map!!!");      /* cqt_algorithm.c:524-527 */
        return;
    }
    if (c->timeLength <= 0) return;
    cqtObj_chromaBatch(c, mRealArr1, mImageArr1, c->timeLength, cn, dataType ? (int)*dataType : SpectralData_Power,
                       normType ? (int)*normType : ChromaDataNormal_Max, mDataArr3, AFB200_MEM_HOST, NULL);
}

/* ---- cqcc: rows x num (power or magnitude) -> rectify -> ortho DCT-II -> first ccNum (cqt_algorithm.c:602-660) ---- */
int cqtObj_cqccBatch(CQTObj c, const float *in, int rows, int ccNum, int rectifyType, float *out, int memKind, void *stream) {
    if (!c || !in || !out || rows < 0) return af_fail(AF_ERR_ARG, "cqtObj_cqccBatch: bad argument");
    if (ccNum < 1 || ccNum > c->num) return af_fail(AF_ERR_ARG, "cqtObj_cqccBatch: ccNum=%d outside [1, %d]", ccNum, c->num);
    af_clear_error();
    int rc = cqt_device(c);
    if (rc) return rc;
    if (!c->dDctT) {
        const int n = c->num;
        float *d = (float *)malloc(sizeof(float) * (size_t)n * n), *t = (float *)malloc(sizeof(float) * (size_t)n * n);
        if (!d || !t) { free(d); free(t); return AF_ERR_NOMEM; }
        af_dct2_matrix(n, n, d);
        for (int k = 0; k < n; k++) for (int j = 0; j < n; j++) t[(size_t)j * n + k] = d[(size_t)k * n + j];
        rc = af_dev_upload((void **)&c->dDctT, t, sizeof(float) * (size_t)n * n);
        free(d); free(t);
        if (rc) return rc;
    }
    if (memKind == AFB200_MEM_DEVICE) return af_launch_xxcc(in, rows, c->num, ccNum, rectifyType, c->dDctT, out, stream);
    void *st = stream ? stream : c->stream;
    const size_t inB = sizeof(float) * (size_t)rows * c->num, outB = sizeof(float) * (size_t)rows * ccNum;
    if ((rc = af_devbuf_reserve(&c->dPostA, inB)) || (rc = af_devbuf_reserve(&c->dPostOut, outB))) return rc;
    if ((rc = af_memcpy_h2d(c->dPostA.ptr, in, inB, st))) return rc;
    if ((rc = af_launch_xxcc((const float *)c->dPostA.ptr, rows, c->num, ccNum, rectifyType, c->dDctT, (float *)c->dPostOut.ptr, st))) return rc;
    if ((rc = af_memcpy_d2h(out, c->dPostOut.ptr, outB, st))) return rc;
    return af_stream_sync(st);
}

void cqtObj_cqcc(CQTObj c, float *mDataArr1, int ccNum, CepstralRectifyType *rectifyType, float *mDataArr2) {
    if (!c || !mDataArr1 || !mDataArr2) return;
    if (ccNum > c->num || ccNum < 1 || c->timeLength <= 0) return;     /* silent, like cqt_algorithm.c:625-627 */
    cqtObj_cqccBatch(c, mDataArr1, c->timeLength, ccNum, rectifyType ? (int)*rectifyType : CepstralRectify_Log,
                     mDataArr2, AFB200_MEM_HOST, NULL);
}

/* ---- cqhc / deconv: rows x num magnitudes (or powers) -> harmonic-index picks of the timbre sequence / timbre + pitch
 * (cqt_algorithm.c:662-781).  mode 0: out0 [rows x hcNum]; mode 1: out0 = timbre, out1 = pitch [rows x num] ---- */
static int cqt_deconv_batch(CQTObj c, const float *in, int rows, int mode, int hcNum, float *out0, float *out1, int memKind, void *stream) {
    af_clear_error();
    int rc = cqt_device(c);
    if (rc) return rc;
    if (rows <= 0) return AF_OK;
    if (memKind == AFB200_MEM_DEVICE) return af_launch_cq_deconv(in, rows, c->num, mode, hcNum, c->binPerOctave, out0, out1, stream);
    void *st = stream ? stream : c->stream;
    const size_t inB = sizeof(float) * (size_t)rows * c->num, outB = sizeof(float) * (size_t)rows * (mode ? c->num : hcNum);
    if ((rc = af_devbuf_reserve(&c->dPostA, inB)) || (rc = af_devbuf_reserve(&c->dPostOut, outB)) ||
        (mode && (rc = af_devbuf_reserve(&c->dPostB, outB)))) return rc;
    if ((rc = af_memcpy_h2d(c->dPostA.ptr, in, inB, st))) return rc;
    if ((rc = af_launch_cq_deconv((const float *)c->dPostA.ptr, rows, c->num, mode, hcNum, c->binPerOctave, (float *)c->dPostOut.ptr,
                                  mode ? (float *)c->dPostB.ptr : NULL, st))) return rc;
    if ((rc = af_memcpy_d2h(out0, c->dPostOut.ptr, outB, st))) return rc;
    if (mode && (rc = af_memcpy_d2h(out1, c->dPostB.ptr, outB, st))) return rc;
    return af_stream_sync(st);
}

int cqtObj_cqhcBatch(CQTObj c, const float *in, int rows, int hcNum, float *out, int memKind, void *stream) {
    if (!c || !in || !out || rows < 0 || hcNum < 1) return af_fail(AF_ERR_ARG, "cqtObj_cqhcBatch: bad argument");
    return cqt_deconv_batch(c, in, rows, 0, hcNum, out, NULL, memKind, stream);
}
int cqtObj_deconvBatch(CQTObj c, const float *in, int rows, float *timbre, float *pitch, int memKind, void *stream) {
    if (!c || !in || !timbre || !pitch || rows < 0) return af_fail(AF_ERR_ARG, "cqtObj_deconvBatch: bad argument");
    return cqt_deconv_batch(c, in, rows, 1, 0, timbre, pitch, memKind, stream);
}

void cqtObj_cqhc(CQTObj c, float *mDataArr1, int hcNum, float *mDataArr2) {
    if (!c || !mDataArr1 || !mDataArr2 || hcNum < 1 || c->timeLength <= 0) return;
    cqtObj_cqhcBatch(c, mDataArr1, c->timeLength, hcNum, mDataArr2, AFB200_MEM_HOST, NULL);
}
void cqtObj_deconv(CQTObj c, float *mDataArr1, float *mDataArr2, float *mDataArr3) {
    if (!c || !mDataArr1 || !mDataArr2 || !mDataArr3 || c->timeLength <= 0) return;
    cqtObj_deconvBatch(c, mDataArr1, c->timeLength, mDataArr2, mDataArr3, AFB200_MEM_HOST, NULL);
}

void cqtObj_free(CQTObj c) {
    if (!c) return;
    af_devbuf_free(&c->dIn); af_devbuf_free(&c->dSigA); af_devbuf_free(&c->dSigB);
    af_devbuf_free(&c->dOutRe); af_devbuf_free(&c->dOutIm);
    af_devbuf_free(&c->dPostA); af_devbuf_free(&c->dPostB); af_devbuf_free(&c->dPostOut);
    af_pipe_free(&c->pipe);
    af_dev_free(c->dChromaBank); af_dev_free(c->dDctT);
    af_dev_free(c->dBfrag); af_dev_free(c->dBimg);
    af_dev_free(c->dKappa2); af_dev_free(c->dLeft); af_dev_free(c->dRight); af_dev_free(c->dScale);
    af_stream_destroy(c->stream);
    af_cqt_bank_free(&c->bank);
    free(c->kappa2); free(c->tail); free(c->cur);
    free(c);
}
