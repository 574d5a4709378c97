/* af_bft.c -- BFT object of the C ABI: STFT -> power / magnitude -> filter bank (-> fused MFCC).
 * Interface spec: src/bft_algorithm.h:14-57; behaviour src/bft_algorithm.c:87-276
 * (parameter rules), :397-540 (compute).  Compute = kernels/stft_generic.cu + kernels/bank_xxcc.cu,
 * or one of the fused kernels at fftLength 2048 (af_mfcc_route: kernels/mfcc_fused.cu, kernels/mfcc_fused2.cu). */
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
    float *dWindow, *dBank, *dPacked;
    int *dStart, *dLen, *dOff;
    AfBankDev bankDev;
    AfDevBuf dSpecRe, dSpecIm, dMel;     /* spectrum planes; mel planes of the general MFCC path */
    /* fused plans: the bank-only one (real-mode bftObj_bft) and the MFCC one for mfccCc coefficients */
    AfMfccPlan *bankPlan, *mfccPlan;
    int mfccCc;
    int mfccRoute;                       /* AF_MFCC_* that served the last MFCC call (bftObj_mfccPlanMode) */
    int v2Bank;                          /* v2's verdict on the bank (AfMfccCall) */
    float *dDctT;                        /* general path: transposed DCT [num][num] */
    AfPipe pipe;
    int isTemporal;                      /* bft_algorithm.c:376, 532-534: energy / rms / zcr of the frames of the last bftObj_bft call */
    float *tempHost; int tempLength;     /* host: [energy | rms | zcr], tempLength frames each */
    ReassignObj reassign;                /* isReassign = 1 (bft_algorithm.c:332-341): the bank is applied to the reassigned spectrum */
};

int bftObj_new(BFTObj *out, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre,
               int *binPerOctave, WindowType *windowType, int *slideLength,
               SpectralFilterBankScaleType *scaleType, SpectralFilterBankStyleType *styleType,
               SpectralFilterBankNormalType *normalType, SpectralDataType *dataType,
               int *isReassign, int *isTemporal) {
    af_clear_error();
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
    b->mfccRoute = AF_MFCC_COMPOSED;

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
int bftObj_mfccPlanMode(BFTObj b) { return b ? b->mfccRoute : AF_MFCC_COMPOSED; }
int bftObj_getFilterBankArr(BFTObj b, float *bank) {
    if (!b || !bank) return af_fail(AF_ERR_ARG, "bftObj_getFilterBankArr: bad argument");
    memcpy(bank, b->bank, sizeof(float) * (size_t)b->num * (b->fftLength / 2 + 1));
    return AF_OK;
}

int af_bft_device(BFTObj b) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (b->devReady) return AF_OK;
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

/* the kernel that serves a fused call on these clips: ccNum 0 = the bank output (real or complex mode) */
static int bft_route(BFTObj b, const float *dData, int dataLength, int ccNum, int realMode) {
    const AfMfccCall c = {ccNum == 0, realMode, ccNum, b->reassign != NULL, b->scaleType == SpectralFilterBankScale_Linear,
                          b->bankDev.banded, b->normValue, b->fftLength, b->num, b->slideLength, dataLength, dData, b->bank,
                          &b->bands, &b->v2Bank};
    return af_mfcc_route(&c);
}

/* the object's cached plan in *slot, rebuilt when it was made for another kernel (or another ccNum) */
static int bft_plan(BFTObj b, AfMfccPlan **slot, int kernel, int ccNum) {
    const int bankOnly = slot == &b->bankPlan;
    if (*slot && af_mfcc_plan_kind(*slot) == kernel && (bankOnly || b->mfccCc == ccNum)) return AF_OK;
    af_mfcc_plan_free(*slot);
    *slot = NULL;
    const int rc = af_mfcc_plan_build(slot, kernel, bankOnly, b->fftLength, b->num, ccNum, b->window, b->bank, &b->bands, b->dataType);
    if (!rc && !bankOnly) b->mfccCc = ccNum;
    return rc;
}

/* device-resident compute: dData [batch x dataLength] -> dRe (and, complex mode, dIm) [batch x T x num] */
static int bft_compute(BFTObj b, const float *dData, int dataLength, int batch, float *dRe, float *dIm, int realMode, void *st) {
    const int T = bftObj_calTimeLength(b, dataLength);
    const int width = b->fftLength / 2 + 1;
    if (T <= 0) return AF_OK;
    /* real mode at fftLength 2048 with a banded bank: a fused kernel stopped after the filter bank (one launch, no
     * spectrum round trip through HBM: 3.3x the general composition below) */
    const int route = bft_route(b, dData, dataLength, 0, realMode);
    int rc;
    if (route != AF_MFCC_COMPOSED) {
        if ((rc = bft_plan(b, &b->bankPlan, route, 1))) return rc;
        return af_launch_mfcc(b->bankPlan, dData, dataLength, batch, T, b->slideLength, 0, dRe, 0, NULL, st);
    }
    const int linear = b->scaleType == SpectralFilterBankScale_Linear;
    const int count = b->highIndex - b->lowIndex + 1 < b->num ? b->highIndex - b->lowIndex + 1 : b->num;
    /* the spectrum workspace is bounded: process the batch in chunks of clips */
    const size_t perClip = sizeof(float) * (size_t)T * width;
    const int chunk = af_chunk_clips(perClip, (size_t)3 << 30, batch);
    if ((rc = af_devbuf_reserve(&b->dSpecRe, perClip * chunk))) return rc;
    if (!realMode && (rc = af_devbuf_reserve(&b->dSpecIm, perClip * chunk))) return rc;
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
            const int mode = realMode ? (b->dataType == SpectralData_Mag ? AF_STFT_MAG : AF_STFT_POWER)
                                           : (b->dataType == SpectralData_Power ? AF_STFT_SQUARE : AF_STFT_HALF);
            if ((rc = af_launch_spec_post(sRe, sIm, (long long)rows * width, mode, b->normValue, st))) return rc;
        }
        if (realMode) {                                       /* real: sum_k w |z|^2 (or |z|) */
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

/* one argument block for every chunk function of this file */
typedef struct { BFTObj b; int dataLength, ccNum, rectifyType; } BftCall;

static int bft_chunk(void *p, int nb, float *const *d, void *st) {
    const BftCall *a = (const BftCall *)p;
    return bft_compute(a->b, d[0], a->dataLength, nb, d[1], d[2], a->b->resultType, st);
}

int bftObj_bftBatch(BFTObj b, const float *data, int dataLength, int batch, float *mReal3, float *mImag3,
                    int memKind, void *stream) {
    if (!b || !data || !mReal3 || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "bftObj_bftBatch: bad argument");
    af_clear_error();
    int rc = af_bft_device(b);
    if (rc) return rc;
    const int T = bftObj_calTimeLength(b, dataLength);
    if (T <= 0) return AF_OK;
    BftCall a = {b, dataLength, 0, 0};
    const size_t outPer = (size_t)T * b->num;
    const AfPlane pl[3] = {{data, (size_t)dataLength, AF_IN, 0}, {mReal3, outPer, AF_OUT, 0},
                           {!b->resultType ? mImag3 : NULL, outPer, AF_OUT, 0}};
    return af_run_batch(&b->pipe, memKind, stream, bft_chunk, &a, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

static int temporal_chunk(void *p, int nb, float *const *d, void *st) {
    const BftCall *a = (const BftCall *)p;
    const int T = bftObj_calTimeLength(a->b, a->dataLength);
    (void)nb;                                         /* one clip */
    return af_launch_temporal(d[0], a->b->fftLength, a->b->slideLength, T, a->b->dWindow, d[1], d[1] + T, d[1] + 2 * (size_t)T, st);
}

/* temporal descriptors of the clip's frames (isTemporal): one more small kernel */
static int bft_temporal(BFTObj b, const float *dataArr, int dataLength) {
    const int T = bftObj_calTimeLength(b, dataLength);
    if (T <= 0) return AF_OK;
    if (T != b->tempLength) {
        free(b->tempHost);
        b->tempHost = (float *)calloc((size_t)3 * T, sizeof(float));
        if (!b->tempHost) { b->tempLength = 0; return AF_ERR_NOMEM; }
        b->tempLength = T;
    }
    BftCall a = {b, dataLength, 0, 0};
    const AfPlane pl[2] = {{dataArr, (size_t)dataLength, AF_IN, 0}, {b->tempHost, 3 * (size_t)T, AF_OUT, 0}};
    return af_run_batch(&b->pipe, AFB200_MEM_HOST, NULL, temporal_chunk, &a, pl, 2, 1, AF_PIPE_CHUNK_BYTES);
}

void bftObj_bft(BFTObj b, float *dataArr, int dataLength, float *mRealArr3, float *mImageArr3) {
    if (!b || !dataArr || !mRealArr3) return;
    if (bftObj_bftBatch(b, dataArr, dataLength, 1, mRealArr3, mImageArr3, AFB200_MEM_HOST, NULL)) return;
    if (b->isTemporal) bft_temporal(b, dataArr, dataLength);
}

/* real-mode bank of the clips, then -- with dPhase -- the phase of the STFT bins lowIndex..lowIndex+count-1 as
 * spectrogramObj_spectrogram reports it for the Linear scale (src/spectrogram_algorithm.c:1040-1056):
 * atan2f(im, re < 1e-16 ? 1e-16 : re).  phase: batch x T x count. */
int af_bft_spectrogram(BFTObj b, const float *dData, int dataLength, int batch, float *dSpect, int lowIndex, int count,
                       float *dPhase, void *st) {
    int rc = bft_compute(b, dData, dataLength, batch, dSpect, NULL, b->resultType, st);
    if (rc || !dPhase) return rc;
    const int T = bftObj_calTimeLength(b, dataLength), width = b->fftLength / 2 + 1;
    const size_t perClip = sizeof(float) * (size_t)T * width;
    const int chunk = af_chunk_clips(perClip, (size_t)2 << 30, batch);
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
    return AF_OK;
}

/* ---- fused / composed MFCC: bft(real mode) -> rectify -> ortho DCT-II -> first ccNum ---- */
static int mfcc_compute(BFTObj b, const float *dData, int dataLength, int batch, int ccNum, int rectifyType,
                        float *dOut, int nPeer, float *const *peerOut, void *st) {
    const int T = bftObj_calTimeLength(b, dataLength);
    int rc;
    b->mfccRoute = bft_route(b, dData, dataLength, ccNum, 1);
    if (b->mfccRoute != AF_MFCC_COMPOSED) {
        if ((rc = bft_plan(b, &b->mfccPlan, b->mfccRoute, ccNum))) return rc;
        return af_launch_mfcc(b->mfccPlan, dData, dataLength, batch, T, b->slideLength, rectifyType, dOut, nPeer, peerOut, st);
    }
    if (nPeer > 0) return af_fail(AF_ERR_UNSUPPORTED, "bftObj_mfccBatchScatter: only the fused fftLength=2048 path can store to peers");
    /* general composition (any fftLength / bank / alignment), still entirely on the device */
    if (!b->dDctT && (rc = af_dct2_upload_transposed(&b->dDctT, b->num))) return rc;
    if ((rc = af_devbuf_reserve(&b->dMel, sizeof(float) * (size_t)batch * T * b->num)) ||
        (rc = bft_compute(b, dData, dataLength, batch, (float *)b->dMel.ptr, NULL, 1, st))) return rc;
    return af_launch_xxcc((const float *)b->dMel.ptr, batch * T, b->num, ccNum, rectifyType, b->dDctT, dOut, st);
}

static int mfcc_chunk(void *p, int nb, float *const *d, void *st) {
    const BftCall *a = (const BftCall *)p;
    return mfcc_compute(a->b, d[0], a->dataLength, nb, a->ccNum, a->rectifyType, d[1], 0, NULL, st);
}

int bftObj_mfccBatch(BFTObj b, const float *data, int dataLength, int batch, int ccNum, int rectifyType,
                     float *out, int memKind, void *stream) {
    if (!b || !data || !out || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "bftObj_mfccBatch: bad argument");
    if (ccNum < 1 || ccNum > b->num) return af_fail(AF_ERR_ARG, "bftObj_mfccBatch: ccNum=%d outside [1, %d]", ccNum, b->num);
    af_clear_error();
    int rc = af_bft_device(b);
    if (rc) return rc;
    const int T = bftObj_calTimeLength(b, dataLength);
    if (T <= 0) return AF_OK;
    BftCall a = {b, dataLength, ccNum, rectifyType};
    const AfPlane pl[2] = {{data, (size_t)dataLength, AF_IN, 0}, {out, (size_t)T * ccNum, AF_OUT, 0}};
    return af_run_batch(&b->pipe, memKind, stream, mfcc_chunk, &a, pl, 2, batch, AF_PIPE_CHUNK_BYTES);
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
    int rc = af_bft_device(b);
    if (rc) return rc;
    if (bftObj_calTimeLength(b, dataLength) <= 0) return AF_OK;
    return mfcc_compute(b, data, dataLength, batch, ccNum, rectifyType, out, nPeer, (float *const *)peerOut, stream);
}

void bftObj_free(BFTObj b) {
    if (!b) return;
    af_mfcc_plan_free(b->mfccPlan); af_mfcc_plan_free(b->bankPlan);
    reassignObj_free(b->reassign);
    free(b->tempHost);
    af_devbuf_free(&b->dSpecRe); af_devbuf_free(&b->dSpecIm); af_devbuf_free(&b->dMel);
    af_dev_free(b->dWindow); af_dev_free(b->dBank); af_dev_free(b->dPacked);
    af_dev_free(b->dStart); af_dev_free(b->dLen); af_dev_free(b->dOff); af_dev_free(b->dDctT);
    af_pipe_free(&b->pipe);
    af_bands_free(&b->bands);
    free(b->window); free(b->bank); free(b->freBandArr); free(b->binBandArr);
    free(b);
}
