/* af_spectrogram.c -- SpectrogramObj front door of the C ABI (host C).
 * Interface spec: src/spectrogram_algorithm.h:40-119; behaviour
 * src/spectrogram_algorithm.c:326-583 (parameters), :584-791 (tables), :864-1395 (spectrogram), :1409-1525 (xxcc).
 * For the scale types on the time-frequency path the spectrogram is mathematically bftObj_bft in real mode, so
 * the object owns a BFT core (same kernels, including the fused MFCC kernel) and only restates the reference's
 * own parameter rules, which differ from bftObj_new's (Linear band count, binPerOctave, band arrays). */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"
#include "../../../include/afb200_spectrogram.h"

struct OpaqueSpectrogram {
    BFTObj core;
    XXCCObj cc;
    int num, fftLength, samplate, lowIndex, highIndex, timeLength;
    SpectralFilterBankScaleType scaleType;
    SpectralFilterBankStyleType styleType;
    float *freBandArr;      /* Linear: own arrays (grid of __vlinspace); else borrowed from the core */
    int *binBandArr;
    int ownBands;
    void *cuStream;         /* deconv with host pointers: staging buffers and the stream they are filled on */
    AfDevBuf dPostA, dPostB, dPostOut;
    STFTObj stream;         /* isContinue = 1: an STFT object that only keeps the tail between calls (stft_algorithm.c:474-599) */
};

int spectrogramObj_new(SpectrogramObj *out, int num, int *samplate, float *lowFre, float *highFre, int *binPerOctave,
                       int *radix2Exp, WindowType *windowType, int *slideLength, int *isContinue,
                       SpectralDataType *dataType, SpectralFilterBankScaleType *filterScaleType,
                       SpectralFilterBankStyleType *filterStyleType, SpectralFilterBankNormalType *filterNormalType) {
    if (!out) return -1;
    *out = NULL;
    int r = 12;
    if (radix2Exp) {
        r = *radix2Exp;
        if (r < 1 || r > 30) { printf("radix2Exp is error!\n"); return -100; }
    }
    const int n = 1 << r;
    int sr = 32000;
    if (samplate && *samplate > 0 && *samplate <= 196000) sr = *samplate;
    const SpectralFilterBankScaleType scale = filterScaleType ? *filterScaleType : SpectralFilterBankScale_Linear;
    if (scale > SpectralFilterBankScale_Log || scale < SpectralFilterBankScale_Linear) {
        af_fail(AF_ERR_UNSUPPORTED, "spectrogramObj_new: scale type %d (Chroma / Deep family) is not supported", (int)scale);
        return -2;
    }
    const int streaming = isContinue && *isContinue;
    int bpo = 12;
    if (binPerOctave && *binPerOctave > 0) bpo = *binPerOctave;
    if (bpo % 12 != 0) bpo = 12;

    AfBftSpec spec;
    memset(&spec, 0, sizeof(spec));
    if (scale == SpectralFilterBankScale_Linear) {
        /* :395-443, 470-472: band count from the rounded edge bins, edges themselves are not snapped */
        float lo = 0, hi = sr / 2.0;
        if (lowFre && *lowFre >= 0 && *lowFre < sr / 2.0) lo = *lowFre;
        if (highFre && *highFre > 0 && *highFre <= sr / 2.0) hi = *highFre;
        if (hi < lo) { lo = 0; hi = sr / 2.0; }
        const float det = sr / (float)n;
        spec.lowIndex = roundf(lo / det);
        spec.highIndex = roundf(hi / det);
        spec.lowFre = lo; spec.highFre = hi;
        num = spec.highIndex - spec.lowIndex + 1;
    } else {
        AfRange range;
        if (af_revise_range(num, n, sr, lowFre, highFre, scale, bpo, &range)) {
            printf("scale log: lowFre and num is large, overflow error!\n");
            return -1;
        }
        spec.lowFre = range.low; spec.highFre = range.high;
    }
    if (num < 2 || num > n / 2 + 1) { printf("num is error!\n"); return -1; }
    spec.num = num; spec.radix2Exp = r; spec.samplate = sr; spec.binPerOctave = bpo;
    spec.windowType = windowType ? (int)*windowType : Window_Hann;
    spec.slideLength = (slideLength && *slideLength > 0) ? *slideLength : n / 4;
    spec.dataType = dataType ? (int)*dataType : SpectralData_Power;
    spec.scaleType = scale;
    spec.styleType = filterStyleType ? (int)*filterStyleType : SpectralFilterBankStyle_Slaney;
    spec.normalType = filterNormalType ? (int)*filterNormalType : SpectralFilterBankNormal_None;

    SpectrogramObj s = (SpectrogramObj)calloc(1, sizeof(struct OpaqueSpectrogram));
    if (!s) return -1;
    int rc = af_bft_create(&spec, &s->core);
    if (rc) { free(s); return rc; }
    bftObj_setResultType(s->core, 1);
    if (xxccObj_new(&s->cc, num)) { spectrogramObj_free(s); return -1; }
    if (streaming) {
        /* the reference hands isContinue to its STFT object (spectrogram_algorithm.c:655-664): samples that did not
         * complete a frame wait for the next call.  Same bookkeeping here, in front of the fused / general kernels. */
        WindowType wt = (WindowType)spec.windowType;
        int one = 1;
        if (stftObj_new(&s->stream, r, &wt, &spec.slideLength, &one)) { spectrogramObj_free(s); return -1; }
    }
    s->num = num; s->fftLength = n; s->samplate = sr; s->lowIndex = spec.lowIndex; s->highIndex = spec.highIndex;
    s->scaleType = scale; s->styleType = (SpectralFilterBankStyleType)spec.styleType;
    if (scale == SpectralFilterBankScale_Linear) {
        /* :1909-1941: slices of linspace(0, sr/2, n/2+1) and arange(n/2+1) starting at lowIndex */
        s->freBandArr = (float *)calloc((size_t)num + 2, sizeof(float));
        s->binBandArr = (int *)calloc((size_t)num + 2, sizeof(int));
        if (!s->freBandArr || !s->binBandArr) { s->ownBands = 1; spectrogramObj_free(s); return -1; }
        s->ownBands = 1;
        const float stop = sr / 2.0, step = (stop - 0.0f) / (n / 2 > 0 ? n / 2 : 1);
        for (int j = 0; j < num; j++) {
            s->freBandArr[j] = 0.0f + (s->lowIndex + j) * step;
            s->binBandArr[j] = s->lowIndex + j;
        }
    } else {
        s->freBandArr = bftObj_getFreBandArr(s->core);
        s->binBandArr = bftObj_getBinBandArr(s->core);
    }
    *out = s;
    return 0;
}

static int new_scale(SpectrogramObj *out, int num, int samplate, int radix2Exp, int *isContinue,
                     SpectralFilterBankScaleType scale) {
    return spectrogramObj_new(out, num, &samplate, NULL, NULL, NULL, &radix2Exp, NULL, NULL, isContinue, NULL, &scale, NULL, NULL);
}
int spectrogramObj_newLinear(SpectrogramObj *o, int samplate, int radix2Exp, int *isContinue) {
    return new_scale(o, 2, samplate, radix2Exp, isContinue, SpectralFilterBankScale_Linear);
}
int spectrogramObj_newMel(SpectrogramObj *o, int num, int samplate, int radix2Exp, int *isContinue) {
    return new_scale(o, num, samplate, radix2Exp, isContinue, SpectralFilterBankScale_Mel);
}
int spectrogramObj_newBark(SpectrogramObj *o, int num, int samplate, int radix2Exp, int *isContinue) {
    return new_scale(o, num, samplate, radix2Exp, isContinue, SpectralFilterBankScale_Bark);
}
int spectrogramObj_newErb(SpectrogramObj *o, int num, int samplate, int radix2Exp, int *isContinue) {
    return new_scale(o, num, samplate, radix2Exp, isContinue, SpectralFilterBankScale_Erb);
}

/* constructors of the scale families outside the path: exported so that a caller resolving them gets a loud refusal
 * (status -2 + afb200_lastError) instead of a missing symbol */
static int refuse_family(SpectrogramObj *o, const char *what) {
    if (o) *o = NULL;
    af_fail(AF_ERR_UNSUPPORTED, "%s: the Chroma / Deep spectrogram families are not part of libaudioflux_b200", what);
    return -2;
}
int spectrogramObj_newChroma(SpectrogramObj *o, int samplate, int radix2Exp, int *isContinue) {
    (void)samplate; (void)radix2Exp; (void)isContinue;
    return refuse_family(o, "spectrogramObj_newChroma");
}
int spectrogramObj_newDeep(SpectrogramObj *o, int num, int samplate, int radix2Exp, int *isContinue) {
    (void)num; (void)samplate; (void)radix2Exp; (void)isContinue;
    return refuse_family(o, "spectrogramObj_newDeep");
}
int spectrogramObj_newDeepChroma(SpectrogramObj *o, int samplate, int radix2Exp, int *isContinue) {
    (void)samplate; (void)radix2Exp; (void)isContinue;
    return refuse_family(o, "spectrogramObj_newDeepChroma");
}
void spectrogramObj_enableDebug(SpectrogramObj s, int flag) { (void)s; (void)flag; }   /* the reference only prints */

void spectrogramObj_setDataNormValue(SpectrogramObj s, float v) { if (s) bftObj_setDataNormValue(s->core, v); }
int spectrogramObj_calTimeLength(SpectrogramObj s, int dataLength) {
    if (!s) return 0;
    return s->stream ? stftObj_calTimeLength(s->stream, dataLength) : bftObj_calTimeLength(s->core, dataLength);   /* :848-853 */
}
float *spectrogramObj_getFreBandArr(SpectrogramObj s) { return s ? s->freBandArr : NULL; }
int *spectrogramObj_getBinBandArr(SpectrogramObj s) { return s ? s->binBandArr : NULL; }
int spectrogramObj_getBandNum(SpectrogramObj s) { return s ? s->num : 0; }
int spectrogramObj_getBinBandLength(SpectrogramObj s) { return s ? s->num : 0; }

/* batch x dataLength -> spect: batch x T x bandNum (and phase, Linear scale only, may be NULL) */
int spectrogramObj_spectrogramBatch(SpectrogramObj s, const float *data, int dataLength, int batch, float *spect,
                                    float *phase, int memKind, void *stream) {
    if (!s || !data || !spect || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "spectrogramObj_spectrogramBatch: bad argument");
    int rc = bftObj_bftBatch(s->core, data, dataLength, batch, spect, NULL, memKind, stream);
    if (rc) return rc;
    if (phase && s->scaleType == SpectralFilterBankScale_Linear)
        rc = af_bft_phase(s->core, data, dataLength, batch, s->lowIndex, s->num, phase, memKind, stream);
    return rc;
}

/* the fused path of the headline metric behind this front door: batch x dataLength -> batch x T x ccNum */
int spectrogramObj_mfccBatch(SpectrogramObj s, const float *data, int dataLength, int batch, int ccNum, int rectifyType,
                             float *out, int memKind, void *stream) {
    if (!s) return af_fail(AF_ERR_ARG, "spectrogramObj_mfccBatch: bad argument");
    return bftObj_mfccBatch(s->core, data, dataLength, batch, ccNum, rectifyType, out, memKind, stream);
}

void spectrogramObj_spectrogram(SpectrogramObj s, float *dataArr, int dataLength, float *mSpectArr, float *mPhaseArr) {
    if (!s || !dataArr || dataLength <= 0 || !mSpectArr) return;      /* :966-978: nothing to do without data */
    const float *x = dataArr;
    if (s->stream) {                                                  /* streaming: tail of the earlier calls ++ dataArr */
        s->timeLength = 0;
        if (!af_stft_continue_assemble(s->stream, dataArr, dataLength, &x, &dataLength)) return;
    }
    s->timeLength = bftObj_calTimeLength(s->core, dataLength);
    spectrogramObj_spectrogramBatch(s, x, dataLength, 1, mSpectArr, mPhaseArr, AFB200_MEM_HOST, NULL);
}

void spectrogramObj_xxcc(SpectrogramObj s, float *mDataArr1, int ccNum, CepstralRectifyType *rectifyType, float *mDataArr2) {
    if (!s || !mDataArr1 || !mDataArr2) return;
    if (ccNum > s->num) return;                     /* silent, :1430-1432 */
    xxccObj_setTimeLength(s->cc, s->timeLength);
    xxccObj_xxcc(s->cc, mDataArr1, ccNum, rectifyType, mDataArr2);
}
void spectrogramObj_mfcc(SpectrogramObj s, float *a, int ccNum, float *b) {
    if (s && s->scaleType == SpectralFilterBankScale_Mel) spectrogramObj_xxcc(s, a, ccNum, NULL, b);
}
void spectrogramObj_bfcc(SpectrogramObj s, float *a, int ccNum, float *b) {
    if (s && s->scaleType == SpectralFilterBankScale_Bark) spectrogramObj_xxcc(s, a, ccNum, NULL, b);
}
void spectrogramObj_gtcc(SpectrogramObj s, float *a, int ccNum, float *b) {
    if (s && s->styleType == SpectralFilterBankStyle_Gammatone) spectrogramObj_xxcc(s, a, ccNum, NULL, b);
}
void spectrogramObj_lfcc(SpectrogramObj s, float *a, int ccNum, float *b) {
    if (s && s->scaleType == SpectralFilterBankScale_Linear) spectrogramObj_xxcc(s, a, ccNum, NULL, b);
}
void spectrogramObj_mfccStandard(SpectrogramObj s, float *a, int *d, CepstralEnergyType *e, CepstralRectifyType *r, float *b) {
    (void)s; (void)a; (void)d; (void)e; (void)r; (void)b;          /* empty in the reference too (:1527-1531) */
}
void spectrogramObj_xxccStandard(SpectrogramObj s, float *a, int *d, CepstralEnergyType *e, CepstralRectifyType *r, float *b) {
    (void)s; (void)a; (void)d; (void)e; (void)r; (void)b;          /* empty in the reference too (:1533-1537) */
}

/* ---- cepstral deconvolution of the band spectra (spectrogram_algorithm.c:1545-1612): the same per-frame transform
 * as cqtObj_deconv (rows zero-padded to ceilPow2(2 num); timbre = Re IFFT(|FFT(row)|), pitch = Re IFFT(FFT(row) /
 * max(|FFT(row)|, 1e-16))), so the same kernel (kernels/deconv.cu) ---- */
int spectrogramObj_deconvBatch(SpectrogramObj s, const float *in, int rows, float *timbre, float *pitch, int memKind, void *stream) {
    if (!s || !in || !timbre || !pitch || rows < 0) return af_fail(AF_ERR_ARG, "spectrogramObj_deconvBatch: bad argument");
    af_clear_error();
    int rc = af_device_ready();
    if (rc) return rc;
    if (rows == 0) return AF_OK;
    if (memKind == AFB200_MEM_DEVICE) return af_launch_cq_deconv(in, rows, s->num, 1, 0, 12, timbre, pitch, stream);
    if (!s->cuStream && (rc = af_stream_create(&s->cuStream))) return rc;
    void *st = stream ? stream : s->cuStream;
    const size_t bytes = sizeof(float) * (size_t)rows * s->num;
    if ((rc = af_devbuf_reserve(&s->dPostA, bytes)) || (rc = af_devbuf_reserve(&s->dPostOut, bytes)) ||
        (rc = af_devbuf_reserve(&s->dPostB, bytes))) return rc;
    if ((rc = af_memcpy_h2d(s->dPostA.ptr, in, bytes, st))) return rc;
    if ((rc = af_launch_cq_deconv((const float *)s->dPostA.ptr, rows, s->num, 1, 0, 12, (float *)s->dPostOut.ptr, (float *)s->dPostB.ptr, st))) return rc;
    if ((rc = af_memcpy_d2h(timbre, s->dPostOut.ptr, bytes, st)) || (rc = af_memcpy_d2h(pitch, s->dPostB.ptr, bytes, st))) return rc;
    return af_stream_sync(st);
}

/* mDataArr1: timeLength x num of the LAST spectrogram call -> mDataArr2 (timbre / tone), mDataArr3 (pitch) */
void spectrogramObj_deconv(SpectrogramObj s, float *mDataArr1, float *mDataArr2, float *mDataArr3) {
    if (!s || !mDataArr1 || !mDataArr2 || !mDataArr3 || s->timeLength <= 0) return;
    spectrogramObj_deconvBatch(s, mDataArr1, s->timeLength, mDataArr2, mDataArr3, AFB200_MEM_HOST, NULL);
}

void spectrogramObj_free(SpectrogramObj s) {
    if (!s) return;
    af_devbuf_free(&s->dPostA); af_devbuf_free(&s->dPostB); af_devbuf_free(&s->dPostOut);
    af_stream_destroy(s->cuStream);
    if (s->ownBands) { free(s->freBandArr); free(s->binBandArr); }
    xxccObj_free(s->cc);
    stftObj_free(s->stream);
    bftObj_free(s->core);
    free(s);
}
