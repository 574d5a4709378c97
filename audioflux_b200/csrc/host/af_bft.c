/* af_bft.c -- BFT object of the C ABI: STFT -> power / magnitude -> filter bank (-> fused MFCC).
 * Interface spec: src/bft_algorithm.h:14-57; behaviour src/bft_algorithm.c:87-276
 * (parameter rules), :397-540 (compute).  Compute = kernels/stft_generic.cu + kernels/bank_xxcc.cu,
 * or kernels/mfcc_fused.cu for the fftLength=2048 MFCC path. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"
#include "../../../include/afb200_reassign.h"

struct OpaqueBFT {
    int num, radix2Exp, fftLength, slideLength, samplate, binPerOctave;
    float lowFre, highFre;
    int lowIndex, highIndex;
    WindowType windowType;
    SpectralDataType dataType;
    SpectralFilterBankScaleType scaleType;
    SpectralFilterBankStyleType styleType;
    SpectralFilterBankNormalType normalType;
    float normValue;
    int resultType;
    /* host tables */
    float *window, *bank, *freBandArr;
    int *binBandArr;
    AfBands bands;
    /* device (lazy) */
    int devReady;
    void *stream;
    float *dWindow, *dBank, *dPacked;
    int *dStart, *dLen, *dOff;
    AfBankDev bankDev;
    AfDevBuf dIn, dSpecRe, dSpecIm, dOutRe, dOutIm;
    /* fused MFCC plan cache */
    void *mfccPlan;
    int mfccPlanCc;
    void *melPlan;                       /* same fused kernel stopped after the bank (real-mode bftObj_bft at n = 2048) */
    void *mfccPlan2, *melPlan2;          /* second-generation fused kernel (kernels/mfcc_fused2.cu), preferred when the bank qualifies */
    int mfccPlan2Cc, v2State;            /* v2State: 0 unknown, 1 usable, -1 not (bank structure / AFB200_MFCC_KERNEL=v1) */
    float *dDctT; int dctReady;          /* general path: transposed DCT [num][num] */
    AfPipe pipe;                         /* host-pointer batches: chunked copy-in / transform / copy-out */
    int pipeLength, pipeCc, pipeRectify; /* arguments of the call the pipe is currently serving */
    int isTemporal;                      /* bft_algorithm.c:376, 532-534: energy / rms / zcr of the frames of the last bftObj_bft call */
    float *tempHost; int tempLength;     /* host: [energy | rms | zcr], tempLength frames each */
    AfDevBuf dTemp;
    ReassignObj reassign;                /* isReassign = 1 (bft_algorithm.c:332-341): the bank is applied to the reassigned spectrum */
};

static int bft_chunk(void *obj, const float *dIn, int nb, float *dOut0, float *dOut1, void *st);
static int mfcc_chunk(void *obj, const float *dIn, int nb, float *dOut0, float *dOut1, void *st);

int bftObj_new(BFTObj *out, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre,
               int *binPerOctave, WindowType *windowType, int *slideLength,
               SpectralFilterBankScaleType *scaleType, SpectralFilterBankStyleType *styleType,
               SpectralFilterBankNormalType *normalType, SpectralDataType *dataType,
               int *isReassign, int *isTemporal) {
    if (!out) return -1;
    *out = NULL;
    int r = radix2Exp ? radix2Exp : 12;
    if (r < 1 || r > 30) { printf("radix2Exp is error!\n"); return -100; }
    const int n = 1 << r;
    int sr = 32000;
    if (samplate && *samplate > 0 && *samplate <= 196000) sr = *samplate;
    SpectralFilterBankScaleType scale = scaleType ? *scaleType : SpectralFilterBankScale_Linear;
    if (scale > SpectralFilterBankScale_Log) { printf("scaleType is error!\n"); return 1; }
    int bpo = 12;
    if (binPerOctave && *binPerOctave >= 4 && *binPerOctave <= 48) bpo = *binPerOctave;
    AfRange range;
    if (af_revise_range(num, n, sr, lowFre, highFre, scale, bpo, &range)) {
        printf(scale == SpectralFilterBankScale_Linear ? "scale linear: lowFre and num is large, overflow error\n"
                                                        : "scale log: lowFre and num is large, overflow error!\n");
        return -1;
    }
    if (num < 2 || num > n / 2 + 1) { printf("num is error!\n"); return -1; }
    AfBftSpec spec;
    spec.num = num; spec.radix2Exp = r; spec.samplate = sr; spec.binPerOctave = bpo;
    spec.lowFre = range.low; spec.highFre = range.high; spec.lowIndex = range.lowIndex; spec.highIndex = range.highIndex;
    spec.windowType = windowType ? (int)*windowType : Window_Hann;
    spec.slideLength = (slideLength && *slideLength > 0) ? *slideLength : n / 4;
    spec.dataType = dataType ? (int)*dataType : SpectralData_Power;
    spec.scaleType = scale;
    spec.styleType = styleType ? (int)*styleType : SpectralFilterBankStyle_Slaney;
    spec.normalType = normalType ? (int)*normalType : SpectralFilterBankNormal_None;
    int status = af_bft_create(&spec, out);
    if (!status && isReassign && *isReassign) {
        /* bft_algorithm.c:332-341: Reassign_All with the reassign object's own defaults (thresh 0.001, no padding) */
        ReassignType reType = Reassign_All;
        WindowType wt = (WindowType)spec.windowType;
        status = reassignObj_new(&(*out)->reassign, r, &sr, &wt, &spec.slideLength, &reType, NULL, NULL, NULL);
        if (status) { bftObj_free(*out); *out = NULL; }
    }
    if (!status && isTemporal && *isTemporal) (*out)->isTemporal = 1;
    return status;
}

/* tables of a BFT object from fully resolved parameters (shared with spectrogramObj_new, host/af_spectrogram.c) */
int af_bft_create(const AfBftSpec *p, BFTObj *out) {
    const int num = p->num, r = p->radix2Exp, n = 1 << r, sr = p->samplate, scale = p->scaleType;
    *out = NULL;
    if (r > 20) { af_fail(AF_ERR_UNSUPPORTED, "radix2Exp > 20 is not supported"); return -2; }
    BFTObj b = (BFTObj)calloc(1, sizeof(struct OpaqueBFT));
    if (!b) return -1;
    b->num = num; b->radix2Exp = r; b->fftLength = n; b->samplate = sr; b->binPerOctave = p->binPerOctave;
    b->lowFre = p->lowFre; b->highFre = p->highFre; b->lowIndex = p->lowIndex; b->highIndex = p->highIndex;
    b->windowType = (WindowType)p->windowType;
    b->slideLength = p->slideLength;
    b->dataType = (SpectralDataType)p->dataType;
    b->scaleType = (SpectralFilterBankScaleType)scale;
    b->styleType = (SpectralFilterBankStyleType)p->styleType;
    b->normalType = (SpectralFilterBankNormalType)p->normalType;
    b->normValue = 1.0f;

    const int width = n / 2 + 1;
    b->window = (float *)malloc(sizeof(float) * (size_t)n);
    b->bank = (float *)calloc((size_t)num * width, sizeof(float));
    b->freBandArr = (float *)calloc((size_t)num + 2, sizeof(float));
    b->binBandArr = (int *)calloc((size_t)num + 2, sizeof(int));
    if (!b->window || !b->bank || !b->freBandArr || !b->binBandArr) { bftObj_free(b); return -1; }
    af_window_fft(b->windowType, n, b->window);
    if (scale == SpectralFilterBankScale_Linear) {
        const float det = sr / (float)n;
        for (int i = b->lowIndex, j = 0; i <= b->highIndex && j < num; i++, j++) {
            b->freBandArr[j] = i * det; b->binBandArr[j] = i;
            if (i < width) b->bank[(size_t)j * width + i] = 1.0f;
        }
    } else if (af_auditory_filterbank(num, n, sr, scale, b->styleType, b->normalType, b->lowFre, b->highFre,
                                      p->binPerOctave, b->bank, b->freBandArr, b->binBandArr)) {
        bftObj_free(b);
        return -2;
    }
    if (af_bands_build(b->bank, num, width, &b->bands)) { bftObj_free(b); return -1; }
    *out = b;
    return 0;
}

int bftObj_calTimeLength(BFTObj b, int dataLength) {
    if (!b || dataLength < b->fftLength) return 0;
    return (dataLength - b->fftLength) / b->slideLength + 1;
}
float *bftObj_getFreBandArr(BFTObj b) { return b ? b->freBandArr : NULL; }
int *bftObj_getBinBandArr(BFTObj b) { return b ? b->binBandArr : NULL; }
void bftObj_setResultType(BFTObj b, int type) { if (b) b->resultType = type; }
void bftObj_setDataNormValue(BFTObj b, float v) { if (b && v > 0) b->normValue = v; }
/* bft_algorithm.c:541-547: arrays [timeLength of the last bftObj_bft call], owned by the object; nothing without isTemporal */
void bftObj_getTemporalData(BFTObj b, float **e, float **r, float **z) {
    if (!b || !b->isTemporal || !b->tempHost) return;
    if (e) *e = b->tempHost;
    if (r) *r = b->tempHost + b->tempLength;
    if (z) *z = b->tempHost + 2 * (size_t)b->tempLength;
}
int bftObj_mfccPlanMode(BFTObj b) { return b ? af_mfcc_plan_mode(b->mfccPlan) : -1; }
int bftObj_getFilterBankArr(BFTObj b, float *bank) {
    if (!b || !bank) return af_fail(AF_ERR_ARG, "bftObj_getFilterBankArr: bad argument");
    memcpy(bank, b->bank, sizeof(float) * (size_t)b->num * (b->fftLength / 2 + 1));
    return AF_OK;
}

/* the v2 fused kernel needs fftLength 2048 and a bank whose bins are covered by at most two consecutive filters */
static int bft_v2_usable(BFTObj b, int ccNum) {
    if (b->v2State == 0) {
        const char *k = getenv("AFB200_MFCC_KERNEL");
        b->v2State = (k && !strcmp(k, "v1")) ? -1 : (af_mfcc2_supported(b->fftLength, b->num, 1, b->bank) ? 1 : -1);
    }
    return b->v2State > 0 && ccNum >= 1 && ccNum <= 64;
}

static int bft_device(BFTObj b) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (b->devReady) return AF_OK;
    if ((rc = af_stream_create(&b->stream))) return rc;
    const int width = b->fftLength / 2 + 1, num = b->num;
    if ((rc = af_dev_upload((void **)&b->dWindow, b->window, sizeof(float) * (size_t)b->fftLength))) return rc;
    /* banded representation when the support is sparse, dense matrix otherwise */
    int banded = (long long)b->bands.nnz * 4 <= (long long)num * width;
    b->bankDev.num = num; b->bankDev.width = width; b->bankDev.banded = banded; b->bankDev.maxLen = b->bands.maxLen;
    if (banded) {
        int *off = (int *)malloc(sizeof(int) * (size_t)num);
        float *packed = (float *)malloc(sizeof(float) * (size_t)(b->bands.nnz > 0 ? b->bands.nnz : 1));
        if (!off || !packed) { free(off); free(packed); return AF_ERR_NOMEM; }
        int o = 0;
        for (int m = 0; m < num; m++) {
            off[m] = o;
            memcpy(packed + o, b->bank + (size_t)m * width + b->bands.start[m], sizeof(float) * (size_t)b->bands.len[m]);
            o += b->bands.len[m];
        }
        rc = af_dev_upload((void **)&b->dPacked, packed, sizeof(float) * (size_t)(o > 0 ? o : 1));
        if (!rc) rc = af_dev_upload((void **)&b->dOff, off, sizeof(int) * (size_t)num);
        if (!rc) rc = af_dev_upload((void **)&b->dStart, b->bands.start, sizeof(int) * (size_t)num);
        if (!rc) rc = af_dev_upload((void **)&b->dLen, b->bands.len, sizeof(int) * (size_t)num);
        free(off); free(packed);
        if (rc) return rc;
        b->bankDev.packed = b->dPacked; b->bankDev.packedOff = b->dOff; b->bankDev.start = b->dStart; b->bankDev.len = b->dLen;
    } else {
        if ((rc = af_dev_upload((void **)&b->dBank, b->bank, sizeof(float) * (size_t)num * width))) return rc;
        b->bankDev.dense = b->dBank;
    }
    b->devReady = 1;
    return AF_OK;
}

/* device-resident compute: dData [batch x dataLength] -> dRe (and dIm) [batch x T x num] */
static int bft_compute(BFTObj b, const float *dData, int dataLength, int batch, float *dRe, float *dIm, void *st) {
    const int T = bftObj_calTimeLength(b, dataLength);
    const int width = b->fftLength / 2 + 1;
    if (T <= 0) return AF_OK;
    /* real mode at fftLength 2048 with a banded bank: the fused TMA-fed kernel of the MFCC path, stopped after the
     * filter bank (one launch, no spectrum round trip through HBM: 3.3x the general composition below) */
    if (!b->reassign && b->resultType && b->normValue == 1.0f && b->scaleType != SpectralFilterBankScale_Linear && b->bankDev.banded &&
        af_mfcc_fused_supported(b->fftLength, b->num, 1, &b->bands) && b->slideLength % 4 == 0 && dataLength % 4 == 0 &&
        ((size_t)dData & 15) == 0 && !getenv("AFB200_BFT_GENERAL")) {
        int rc = AF_OK;
        if (bft_v2_usable(b, 1)) {
            if (!b->melPlan2) {
                float *dct = (float *)calloc((size_t)b->num, sizeof(float));      /* unused by this mode */
                if (!dct) return AF_ERR_NOMEM;
                rc = af_mfcc2_plan_build(&b->melPlan2, b->fftLength, b->num, 1, b->window, b->bank, dct, b->dataType);
                free(dct);
                if (rc) return rc;
            }
            return af_launch_mel2(b->melPlan2, dData, dataLength, batch, T, b->slideLength, dRe, st);
        }
        if (!b->melPlan) {
            float *dct = (float *)calloc((size_t)b->num, sizeof(float));      /* unused by this mode */
            if (!dct) return AF_ERR_NOMEM;
            rc = af_mfcc_plan_build(&b->melPlan, b->fftLength, b->num, 1, b->window, b->bank, &b->bands, dct, b->dataType, NULL);
            free(dct);
            if (rc) return rc;
        }
        if (af_mfcc_plan_mode(b->melPlan) == 0)
            return af_launch_mel_fused(b->melPlan, dData, dataLength, batch, T, b->slideLength, dRe, st);
    }
    const int linear = b->scaleType == SpectralFilterBankScale_Linear;
    const int count = b->highIndex - b->lowIndex + 1 < b->num ? b->highIndex - b->lowIndex + 1 : b->num;
    /* the spectrum workspace is bounded: process the batch in chunks of clips */
    const size_t perClip = sizeof(float) * (size_t)T * width;
    size_t budget = af_dev_free_bytes() / 4;
    if (budget < perClip) budget = perClip;
    if (budget > ((size_t)3 << 30)) budget = (size_t)3 << 30;
    int chunk = (int)(budget / perClip);
    if (chunk < 1) chunk = 1;
    if (chunk > batch) chunk = batch;
    int rc;
    if ((rc = af_devbuf_reserve(&b->dSpecRe, perClip * chunk))) return rc;
    if (!b->resultType && (rc = af_devbuf_reserve(&b->dSpecIm, perClip * chunk))) return rc;
    for (int c0 = 0; c0 < batch; c0 += chunk) {
        const int nb = batch - c0 < chunk ? batch - c0 : chunk;
        AfFrameSrc src;
        memset(&src, 0, sizeof(src));
        src.fftLength = b->fftLength; src.slideLength = b->slideLength; src.dataLength = dataLength;
        src.timeLength = T; src.batch = nb; src.validLength = dataLength; src.window = b->dWindow;
        src.data = dData + (size_t)c0 * dataLength;
        const int rows = nb * T;
        float *oRe = dRe + (size_t)c0 * T * b->num;
        float *oIm = dIm ? dIm + (size_t)c0 * T * b->num : NULL;
        float *sRe = (float *)b->dSpecRe.ptr, *sIm = (float *)b->dSpecIm.ptr;
        if (b->reassign) {
            /* reassigned half spectrum (added into zeroed planes), then the same square / power / magnitude step */
            if ((rc = af_devbuf_reserve(&b->dSpecIm, perClip * chunk))) return rc;
            sIm = (float *)b->dSpecIm.ptr;
            if ((rc = af_memset_d(sRe, 0, perClip * nb, st)) || (rc = af_memset_d(sIm, 0, perClip * nb, st))) return rc;
            if ((rc = reassignObj_reassignBatch(b->reassign, src.data, dataLength, nb, sRe, sIm, NULL, NULL, AFB200_MEM_DEVICE, st))) return rc;
            const int mode = b->resultType ? (b->dataType == SpectralData_Mag ? AF_STFT_MAG : AF_STFT_POWER)
                                           : (b->dataType == SpectralData_Power ? AF_STFT_SQUARE : AF_STFT_HALF);
            if ((rc = af_launch_spec_post(sRe, sIm, (long long)rows * width, mode, b->normValue, st))) return rc;
        }
        if (b->resultType) {                                  /* real: sum_k w |z|^2 (or |z|) */
            const int mode = b->dataType == SpectralData_Mag ? AF_STFT_MAG : AF_STFT_POWER;
            if (!b->reassign && (rc = af_launch_stft(&src, mode, b->normValue, sRe, NULL, st))) return rc;
            const float post = (b->dataType == SpectralData_Mag) ? b->normValue : 1.0f;
            if (linear && post == 1.0f) {
                if ((rc = af_launch_copy_cols(sRe, rows, width, b->lowIndex, count, oRe, st))) return rc;
            } else {                                          /* (Linear + Mag + norm: the 0/1 bank, then ^norm) */
                if ((rc = af_launch_bank(&b->bankDev, sRe, rows, post, oRe, st))) return rc;
            }
        } else {                                              /* complex: sum_k w z^2 (or z) */
            const int mode = b->dataType == SpectralData_Power ? AF_STFT_SQUARE : AF_STFT_HALF;
            if (!b->reassign && (rc = af_launch_stft(&src, mode, 1.0f, sRe, sIm, st))) return rc;
            if (linear) {
                if ((rc = af_launch_copy_cols(sRe, rows, width, b->lowIndex, count, oRe, st))) return rc;
                if (oIm && (rc = af_launch_copy_cols(sIm, rows, width, b->lowIndex, count, oIm, st))) return rc;
            } else {
                if ((rc = af_launch_bank(&b->bankDev, sRe, rows, 1.0f, oRe, st))) return rc;
                if (oIm && (rc = af_launch_bank(&b->bankDev, sIm, rows, 1.0f, oIm, st))) return rc;
            }
        }
    }
    return AF_OK;
}

int bftObj_bftBatch(BFTObj b, const float *data, int dataLength, int batch, float *mReal3, float *mImag3,
                    int memKind, void *stream) {
    if (!b || !data || !mReal3 || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "bftObj_bftBatch: bad argument");
    af_clear_error();
    int rc = bft_device(b);
    if (rc) return rc;
    const int T = bftObj_calTimeLength(b, dataLength);
    if (T <= 0) return AF_OK;
    void *st = stream ? stream : b->stream;
    const int needIm = !b->resultType && mImag3;
    if (memKind == AFB200_MEM_DEVICE) {
        st = stream;                      /* NULL = the CUDA default stream */
        if ((rc = bft_compute(b, data, dataLength, batch, mReal3, needIm ? mImag3 : NULL, st))) return rc;
        return AF_OK;                       /* asynchronous on the caller's stream */
    }
    b->pipeLength = dataLength;
    return af_pipe_run(&b->pipe, bft_chunk, b, data, (size_t)dataLength, batch, mReal3, needIm ? mImag3 : NULL,
                       (size_t)T * b->num, st);
}

/* temporal descriptors of the clip's frames (isTemporal): one more small kernel on the object's stream */
static int bft_temporal(BFTObj b, const float *dataArr, int dataLength) {
    const int T = bftObj_calTimeLength(b, dataLength);
    if (T <= 0) return AF_OK;
    int rc;
    if (T != b->tempLength) {
        free(b->tempHost);
        b->tempHost = (float *)calloc((size_t)3 * T, sizeof(float));
        if (!b->tempHost) { b->tempLength = 0; return AF_ERR_NOMEM; }
        b->tempLength = T;
    }
    if ((rc = af_devbuf_reserve(&b->dIn, sizeof(float) * (size_t)dataLength)) || (rc = af_devbuf_reserve(&b->dTemp, sizeof(float) * 3 * (size_t)T))) return rc;
    float *d = (float *)b->dTemp.ptr;
    if ((rc = af_memcpy_h2d(b->dIn.ptr, dataArr, sizeof(float) * (size_t)dataLength, b->stream))) return rc;
    if ((rc = af_launch_temporal((const float *)b->dIn.ptr, b->fftLength, b->slideLength, T, b->dWindow, d, d + T, d + 2 * (size_t)T, b->stream))) return rc;
    if ((rc = af_memcpy_d2h(b->tempHost, d, sizeof(float) * 3 * (size_t)T, b->stream))) return rc;
    return af_stream_sync(b->stream);
}

void bftObj_bft(BFTObj b, float *dataArr, int dataLength, float *mRealArr3, float *mImageArr3) {
    if (!b || !dataArr || !mRealArr3) return;
    if (bftObj_bftBatch(b, dataArr, dataLength, 1, mRealArr3, mImageArr3, AFB200_MEM_HOST, NULL)) return;
    if (b->isTemporal) bft_temporal(b, dataArr, dataLength);
}

/* phase of the STFT bins lowIndex..highIndex as spectrogramObj_spectrogram reports it for the Linear scale
 * (src/spectrogram_algorithm.c:1040-1056): atan2f(im, re < 1e-16 ? 1e-16 : re).  phase: batch x T x count. */
int af_bft_phase(BFTObj b, const float *data, int dataLength, int batch, int lowIndex, int count, float *phase,
                 int memKind, void *stream) {
    if (!b || !data || !phase || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "spectrogram phase: bad argument");
    int rc = bft_device(b);
    if (rc) return rc;
    const int T = bftObj_calTimeLength(b, dataLength), width = b->fftLength / 2 + 1;
    if (T <= 0) return AF_OK;
    void *st = memKind == AFB200_MEM_DEVICE ? stream : (stream ? stream : b->stream);
    const float *dData = data;
    float *dPhase = phase;
    const size_t inB = sizeof(float) * (size_t)batch * dataLength, outB = sizeof(float) * (size_t)batch * T * count;
    if (memKind != AFB200_MEM_DEVICE) {
        if ((rc = af_devbuf_reserve(&b->dIn, inB)) || (rc = af_devbuf_reserve(&b->dOutRe, outB))) return rc;
        if ((rc = af_memcpy_h2d(b->dIn.ptr, data, inB, st))) return rc;
        dData = (const float *)b->dIn.ptr; dPhase = (float *)b->dOutRe.ptr;
    }
    const size_t perClip = sizeof(float) * (size_t)T * width;
    size_t budget = af_dev_free_bytes() / 4;
    if (budget < perClip) budget = perClip;
    if (budget > ((size_t)2 << 30)) budget = (size_t)2 << 30;
    int chunk = (int)(budget / perClip);
    if (chunk < 1) chunk = 1;
    if (chunk > batch) chunk = batch;
    if ((rc = af_devbuf_reserve(&b->dSpecRe, perClip * chunk)) || (rc = af_devbuf_reserve(&b->dSpecIm, perClip * chunk))) return rc;
    for (int c0 = 0; c0 < batch; c0 += chunk) {
        const int nb = batch - c0 < chunk ? batch - c0 : chunk;
        AfFrameSrc src;
        memset(&src, 0, sizeof(src));
        src.fftLength = b->fftLength; src.slideLength = b->slideLength; src.dataLength = dataLength;
        src.timeLength = T; src.batch = nb; src.validLength = dataLength; src.window = b->dWindow;
        src.data = dData + (size_t)c0 * dataLength;
        if ((rc = af_launch_stft(&src, AF_STFT_HALF, 1.0f, (float *)b->dSpecRe.ptr, (float *)b->dSpecIm.ptr, st))) return rc;
        if ((rc = af_launch_phase((const float *)b->dSpecRe.ptr, (const float *)b->dSpecIm.ptr, nb * T, width, lowIndex, count,
                                  dPhase + (size_t)c0 * T * count, st))) return rc;
    }
    if (memKind == AFB200_MEM_DEVICE) return AF_OK;
    if ((rc = af_memcpy_d2h(phase, b->dOutRe.ptr, outB, st))) return rc;
    return af_stream_sync(st);
}

/* ---- fused / composed MFCC: bft(real mode) -> rectify -> ortho DCT-II -> first ccNum ---- */
static int mfcc_compute(BFTObj b, const float *dData, int dataLength, int batch, int ccNum, int rectifyType,
                        float *dOut, int nPeer, float *const *peerOut, void *st) {
    const int T = bftObj_calTimeLength(b, dataLength);
    int rc;
    const int fusable = !b->reassign && b->normValue == 1.0f && b->scaleType != SpectralFilterBankScale_Linear &&
                        b->bankDev.banded && af_mfcc_fused_supported(b->fftLength, b->num, ccNum, &b->bands) &&
                        b->slideLength % 4 == 0 && dataLength % 4 == 0 && ((size_t)dData & 15) == 0;
    if (fusable && bft_v2_usable(b, ccNum)) {
        if (!b->mfccPlan2 || b->mfccPlan2Cc != ccNum) {
            af_mfcc2_plan_free(b->mfccPlan2); b->mfccPlan2 = NULL;
            float *dct = (float *)malloc(sizeof(float) * (size_t)ccNum * b->num);
            if (!dct) return AF_ERR_NOMEM;
            af_dct2_matrix(b->num, ccNum, dct);
            rc = af_mfcc2_plan_build(&b->mfccPlan2, b->fftLength, b->num, ccNum, b->window, b->bank, dct, b->dataType);
            free(dct);
            if (rc) return rc;
            b->mfccPlan2Cc = ccNum;
        }
        return af_launch_mfcc2(b->mfccPlan2, dData, dataLength, batch, T, b->slideLength, rectifyType, dOut, nPeer, peerOut, st);
    }
    if (fusable) {
        if (!b->mfccPlan || b->mfccPlanCc != ccNum) {
            af_mfcc_plan_free(b->mfccPlan); b->mfccPlan = NULL;
            float *dct = (float *)malloc(sizeof(float) * (size_t)ccNum * b->num);
            if (!dct) return AF_ERR_NOMEM;
            af_dct2_matrix(b->num, ccNum, dct);
            /* per-filter gain of the bank normalisation (row peak over the un-normalised row peak): lets the kernel
             * use the interval form of triangular banks; a bank without that structure is detected and ignored */
            float *gain = NULL;
            if (b->normalType != SpectralFilterBankNormal_None) {
                const int width = b->fftLength / 2 + 1;
                float *unit = (float *)calloc((size_t)b->num * width, sizeof(float));
                float *fre = (float *)calloc((size_t)b->num + 2, sizeof(float));
                int *bin = (int *)calloc((size_t)b->num + 2, sizeof(int));
                gain = (float *)malloc(sizeof(float) * (size_t)b->num);
                if (unit && fre && bin && gain &&
                    !af_auditory_filterbank(b->num, b->fftLength, b->samplate, b->scaleType, b->styleType,
                                            SpectralFilterBankNormal_None, b->lowFre, b->highFre, b->binPerOctave, unit, fre, bin)) {
                    for (int m = 0; m < b->num; m++) {
                        float pn = 0, pu = 0;
                        for (int k = 0; k < width; k++) {
                            if (b->bank[(size_t)m * width + k] > pn) pn = b->bank[(size_t)m * width + k];
                            if (unit[(size_t)m * width + k] > pu) pu = unit[(size_t)m * width + k];
                        }
                        gain[m] = pu > 0 ? pn / pu : 0.0f;
                    }
                } else { free(gain); gain = NULL; }
                free(unit); free(fre); free(bin);
                if (!gain) { free(dct); return AF_ERR_NOMEM; }
            }
            rc = af_mfcc_plan_build(&b->mfccPlan, b->fftLength, b->num, ccNum, b->window, b->bank, &b->bands, dct, b->dataType, gain);
            free(gain);
            free(dct);
            if (rc) return rc;
            b->mfccPlanCc = ccNum;
        }
        return af_launch_mfcc_fused(b->mfccPlan, dData, dataLength, batch, T, b->slideLength, rectifyType, dOut, nPeer, peerOut, st);
    }
    if (nPeer > 0) return af_fail(AF_ERR_UNSUPPORTED, "bftObj_mfccBatchScatter: only the fused fftLength=2048 path can store to peers");
    /* general composition (any fftLength / bank / alignment), still entirely on the device */
    if (!b->dctReady) {
        const int n = b->num;
        float *d = (float *)malloc(sizeof(float) * (size_t)n * n), *t = (float *)malloc(sizeof(float) * (size_t)n * n);
        if (!d || !t) { free(d); free(t); return AF_ERR_NOMEM; }
        af_dct2_matrix(n, n, d);
        for (int k = 0; k < n; k++) for (int j = 0; j < n; j++) t[(size_t)j * n + k] = d[(size_t)k * n + j];
        rc = af_dev_upload((void **)&b->dDctT, t, sizeof(float) * (size_t)n * n);
        free(d); free(t);
        if (rc) return rc;
        b->dctReady = 1;
    }
    const int savedType = b->resultType;
    b->resultType = 1;
    const size_t melB = sizeof(float) * (size_t)batch * T * b->num;
    rc = af_devbuf_reserve(&b->dOutIm, melB);          /* reuse as mel scratch */
    if (!rc) rc = bft_compute(b, dData, dataLength, batch, (float *)b->dOutIm.ptr, NULL, st);
    b->resultType = savedType;
    if (rc) return rc;
    return af_launch_xxcc((const float *)b->dOutIm.ptr, batch * T, b->num, ccNum, rectifyType, b->dDctT, dOut, st);
}

static int mfcc_chunk(void *obj, const float *dIn, int nb, float *dOut0, float *dOut1, void *st) {
    BFTObj b = (BFTObj)obj;
    (void)dOut1;
    return mfcc_compute(b, dIn, b->pipeLength, nb, b->pipeCc, b->pipeRectify, dOut0, 0, NULL, st);
}
static int bft_chunk(void *obj, const float *dIn, int nb, float *dOut0, float *dOut1, void *st) {
    BFTObj b = (BFTObj)obj;
    return bft_compute(b, dIn, b->pipeLength, nb, dOut0, dOut1, st);
}

int bftObj_mfccBatch(BFTObj b, const float *data, int dataLength, int batch, int ccNum, int rectifyType,
                     float *out, int memKind, void *stream) {
    if (!b || !data || !out || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "bftObj_mfccBatch: bad argument");
    if (ccNum < 1 || ccNum > b->num) return af_fail(AF_ERR_ARG, "bftObj_mfccBatch: ccNum=%d outside [1, %d]", ccNum, b->num);
    af_clear_error();
    int rc = bft_device(b);
    if (rc) return rc;
    const int T = bftObj_calTimeLength(b, dataLength);
    if (T <= 0) return AF_OK;
    void *st = stream ? stream : b->stream;
    if (memKind == AFB200_MEM_DEVICE) {
        st = stream;                      /* NULL = the CUDA default stream */
        if ((rc = mfcc_compute(b, data, dataLength, batch, ccNum, rectifyType, out, 0, NULL, st))) return rc;
        return AF_OK;                       /* asynchronous on the caller's stream */
    }
    b->pipeLength = dataLength; b->pipeCc = ccNum; b->pipeRectify = rectifyType;
    return af_pipe_run(&b->pipe, mfcc_chunk, b, data, (size_t)dataLength, batch, out, NULL, (size_t)T * ccNum, st);
}

/* MFCC + all-gather in one kernel: device pointers only.  `out` is this GPU's destination, peerOut[0..nPeer) are
 * the same logical location inside other GPUs' buffers (mapped with afb200_ipcOpenHandle); every finished tile is
 * stored to all of them from the kernel epilogue.  Asynchronous on `stream`; the caller fences across ranks. */
int bftObj_mfccBatchScatter(BFTObj b, const float *data, int dataLength, int batch, int ccNum, int rectifyType,
                            float *out, int nPeer, void **peerOut, void *stream) {
    if (!b || !data || !out || dataLength <= 0 || batch <= 0 || nPeer < 0 || (nPeer > 0 && !peerOut))
        return af_fail(AF_ERR_ARG, "bftObj_mfccBatchScatter: bad argument");
    if (ccNum < 1 || ccNum > b->num) return af_fail(AF_ERR_ARG, "bftObj_mfccBatchScatter: ccNum=%d outside [1, %d]", ccNum, b->num);
    af_clear_error();
    int rc = bft_device(b);
    if (rc) return rc;
    if (bftObj_calTimeLength(b, dataLength) <= 0) return AF_OK;
    return mfcc_compute(b, data, dataLength, batch, ccNum, rectifyType, out, nPeer, (float *const *)peerOut, stream);
}

void bftObj_free(BFTObj b) {
    if (!b) return;
    af_mfcc_plan_free(b->mfccPlan); af_mfcc_plan_free(b->melPlan);
    af_mfcc2_plan_free(b->mfccPlan2); af_mfcc2_plan_free(b->melPlan2);
    reassignObj_free(b->reassign);
    free(b->tempHost); af_devbuf_free(&b->dTemp);
    af_devbuf_free(&b->dIn); af_devbuf_free(&b->dSpecRe); af_devbuf_free(&b->dSpecIm);
    af_devbuf_free(&b->dOutRe); af_devbuf_free(&b->dOutIm);
    af_dev_free(b->dWindow); af_dev_free(b->dBank); af_dev_free(b->dPacked);
    af_dev_free(b->dStart); af_dev_free(b->dLen); af_dev_free(b->dOff); af_dev_free(b->dDctT);
    af_stream_destroy(b->stream);
    af_pipe_free(&b->pipe);
    af_bands_free(&b->bands);
    free(b->window); free(b->bank); free(b->freBandArr); free(b->binBandArr);
    free(b);
}
