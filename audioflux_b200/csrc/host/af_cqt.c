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
    float *dBfrag;                               /* tensor-core octave kernel: pre-split kernel fragments */
    unsigned char *dBimg;                        /* wgmma octave kernel: pre-swizzled shared-memory images of the kernels */
    float *dKappa2, *dLeft, *dRight, *dScale;    /* dScale: octaveNum x bpo, rebuilt when isScale flips */
    int scaleDirty;
    AfDevBuf dSigA, dSigB;                       /* decimated signal, octave after octave */
    /* post-processing of the last transform (chroma / cqcc) */
    int timeLength;                /* frames of the last cqtObj_cqt call (cqt_algorithm.c:463-478) */
    int chromaNum;
    float *dChromaBank, *dDctT;
    AfPipe pipe;
    /* streaming (isContinue, cqt_algorithm.c:346-456): full-rate samples that did not complete a hop wait for the next call */
    int isContinue;
    AfTail tail;
};

int cqtObj_newWith(CQTObj *out, int num, int *samplate, float *minFre, int *binPerOctave, float *factor,
                   float *beta, float *thresh, WindowType *windowType, int *slideLength, int *isContinue,
                   SpectralFilterBankNormalType *normalType, int *isScale) {
    af_clear_error();
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
    if (c->isContinue) return dataLength + c->tail.length <= 0 ? 0 : cqt_time_length(c, dataLength + c->tail.length, 1);
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

/* ---- octave plan: which kernel, which tile (the launchers in kernels/cqt.cu and cqt_wgmma.cu take it as given) ---- */
int af_cqt_tc_tables(int fftLength, int bpo) { return bpo == 12 && fftLength > 0 && fftLength % 64 == 0; }
int af_cqt_wgmma_tables(int fftLength, int bpo) { return bpo == 12 && fftLength % AF_CQT_WG_CHUNK_K == 0 && fftLength >= 2 * AF_CQT_WG_CHUNK_K; }

static int is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

/* wgmma: two warpgroups x AF_CQT_WG_MT m-tiles (256 frames) when the CTA fits ~113 KB (two CTAs per SM), else smaller
 * tiles, then the same shapes up to 227 KB; 0 when not even one 64-frame tile fits */
static int wgmma_geometry(int fftLength, int hop, AfCqtOctPlan *p) {
    static const int shapes[][2] = {{2, AF_CQT_WG_MT}, {2, 1}, {1, 1}};
    const size_t chunkBytes = (size_t)64 * AF_CQT_WG_CHUNK_K * 4;
    for (int pass = 0; pass < 2; pass++)
        for (int s = 0; s < 3; s++) {
            const int wg = shapes[s][0], mt = shapes[s][1], TT = wg * 64 * mt;
            int rowLen = TT + fftLength / hop + 1;
            rowLen = ((rowLen + 31) / 32) * 32 + 8;                           /* == 8 (mod 32): conflict-free fragment reads */
            const size_t sigFloats = hop >= 8 ? (size_t)hop * rowLen : (size_t)(TT - 1) * hop + fftLength;
            const size_t smem = 2 * chunkBytes + ((sigFloats * 4 + 15) & ~(size_t)15) + 16;
            if (smem <= (size_t)(pass == 0 ? 113 : 227) * 1024) {
                p->kernel = AF_CQT_WGMMA; p->wg = wg; p->mt = mt; p->TT = TT; p->threads = wg * 128;
                p->rowLen = rowLen; p->smem = (int)smem;
                return 1;
            }
        }
    return 0;
}

/* mma.sync: 8 warps x AF_CQT_TC_MT m-tiles = 256 frames when the signal tile fits ~100 KB (two CTAs per SM), else fewer
 * warps (one warp up to 227 KB); 0 when even one warp does not fit */
static int tc_geometry(int fftLength, int hop, AfCqtOctPlan *p) {
    const size_t bBytes = (size_t)16 * AF_CQT_TC_KC * 96;                    /* float4 B fragments of AF_CQT_TC_KC k-steps */
    for (int warps = 8; warps >= 1; warps /= 2) {
        const int TT = warps * 16 * AF_CQT_TC_MT;
        int rowLen = TT + fftLength / hop + 1;
        rowLen = ((rowLen + 31) / 32) * 32 + 8;                               /* == 8 (mod 32): conflict-free fragment reads */
        const size_t sigFloats = hop >= 8 ? (size_t)hop * rowLen : (size_t)(TT - 1) * hop + fftLength;
        const size_t smem = bBytes + sizeof(float) * sigFloats;
        if (smem <= (size_t)100 * 1024 || (warps == 1 && smem <= (size_t)227 * 1024)) {
            p->kernel = AF_CQT_TC; p->warps = warps; p->TT = TT; p->threads = warps * 32;
            p->rowLen = rowLen; p->smem = (int)smem;
            return 1;
        }
    }
    return 0;
}

/* FP32 loop: frames per CTA -- the largest tile that still lets two CTAs share an SM (<= 100 KB); if that would drop
 * below 256 frames (large hops: the polyphase signal tile is hop x TT floats) the largest tile that fits 200 KB at all;
 * 0 when none does */
static int loop_geometry(int fftLength, int hop, AfCqtOctPlan *p) {
    static const int ttChoices[] = {512, 256, 128, 64, 32, 16, 8};
    p->rowsA = (fftLength + hop - 1) / hop;
    p->nChunk = fftLength < 512 ? fftLength : 512;
    const size_t kBytes = 2 * sizeof(float) * (size_t)AF_CQT_BINS_PER_PASS * p->nChunk;
    for (int pass = 0; pass < 2; pass++) {
        for (int c = 0; c < 7; c++) {
            const int tt = ttChoices[c];
            if (pass == 0 && tt < 256) break;
            int rowLen = tt + p->rowsA + 1;
            /* pitch chosen so consecutive samples (r fastest) land in different banks while staging */
            if (hop >= 32) rowLen |= 1; else { int want = 32 / hop; rowLen = ((rowLen + 31) / 32) * 32 + want; }
            const size_t bytes = kBytes + sizeof(float) * (size_t)hop * rowLen;
            if (bytes <= (size_t)(pass == 0 ? 100 : 200) * 1024) {
                p->kernel = AF_CQT_LOOP; p->TT = tt; p->rowLen = rowLen; p->smem = (int)bytes;
                /* enough threads per CTA: split the taps of a frame over up to rowsA segments until the CTA has >= 512
                 * threads; the reduction scratch of the segments must fit the kernel buffer */
                p->segs = 1;
                while (p->segs * 2 <= p->rowsA && (tt / AF_CQT_FT) * AF_CQT_JG * p->segs * 2 <= 512) p->segs *= 2;
                if ((size_t)(tt / AF_CQT_FT) * AF_CQT_JG * 2 * AF_CQT_FT * AF_CQT_BT * sizeof(float) > kBytes) p->segs = 1;
                p->threads = (tt / AF_CQT_FT) * AF_CQT_JG * p->segs;
                return 1;
            }
        }
    }
    return 0;
}

void af_cqt_octave_plan(int fftLength, int hop, int bpo, AfCqtOctPlan *p) {
    memset(p, 0, sizeof(*p));
    p->segs = 1;
    if (af_cqt_wgmma_tables(fftLength, bpo) && hop >= 2 && hop <= 128 && is_pow2(hop) && wgmma_geometry(fftLength, hop, p)) return;
    if (af_cqt_tc_tables(fftLength, bpo) && hop >= 2 && is_pow2(hop) && tc_geometry(fftLength, hop, p)) return;
    if (loop_geometry(fftLength, hop, p)) return;
    /* no tile of the polyphase kernel fits: one warp per (frame, bin) */
    memset(p, 0, sizeof(*p));
    p->kernel = AF_CQT_DIRECT; p->threads = 256; p->segs = 1;
}

int cqtObj_octavePlan(CQTObj c, int *kernel, int *hop, int *framesPerCta, int *threadsPerCta, int *segs, int *smemBytes) {
    if (!c) { af_fail(AF_ERR_ARG, "cqtObj_octavePlan: bad argument"); return -1; }
    for (int k = 0; k < c->octaveNum; k++) {
        const int h = c->slideLength >> k;                                    /* the recursion halves the hop per octave */
        AfCqtOctPlan p;
        af_cqt_octave_plan(c->fftLength, h, c->binPerOctave, &p);
        if (kernel) kernel[k] = p.kernel;
        if (hop) hop[k] = h;
        if (framesPerCta) framesPerCta[k] = p.TT;
        if (threadsPerCta) threadsPerCta[k] = p.threads;
        if (segs) segs[k] = p.segs;
        if (smemBytes) smemBytes[k] = p.smem;
    }
    return c->octaveNum;
}

static int cqt_device(CQTObj c) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (!c->devReady) {
        /* kernel sets: one (the top octave's, shared) or -- VQT -- one per octave, set o at offset o * bpo rows */
        const int sets = c->bank.vqt ? c->octaveNum : 1;
        const size_t setFloats = 2 * (size_t)c->binPerOctave * c->fftLength;
        if ((rc = af_dev_upload((void **)&c->dKappa2, c->kappa2, sizeof(float) * setFloats * sets))) return rc;
        if (af_cqt_tc_tables(c->fftLength, c->binPerOctave)) {
            const size_t nf = (size_t)(c->fftLength / 8) * 96 * 4;
            float *bf = (float *)malloc(sizeof(float) * nf * sets);
            if (!bf) return AF_ERR_NOMEM;
            for (int s = 0; s < sets; s++) af_cqt_tc_fragments(c->kappa2 + setFloats * s, c->fftLength, bf + nf * s);
            rc = af_dev_upload((void **)&c->dBfrag, bf, sizeof(float) * nf * sets);
            free(bf);
            if (rc) return rc;
        }
        if (af_cqt_wgmma_tables(c->fftLength, c->binPerOctave)) {
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
        /* kernel set of this octave: the shared top-octave set, or -- VQT -- the octave's own */
        const size_t set = c->bank.vqt ? (size_t)o : 0;
        const unsigned char *bimg = c->dBimg ? c->dBimg + set * (size_t)(c->fftLength / 128) * 32768 : NULL;
        const float *bfrag = c->dBfrag ? c->dBfrag + set * (size_t)(c->fftLength / 8) * 96 * 4 : NULL;
        const float *kappa = c->dKappa2 + set * 2 * (size_t)c->binPerOctave * c->fftLength;
        /* wgmma where the hop allows it, else mma.sync 3xTF32, else the FP32 loop (cqtObj_octavePlan reports the same) */
        AfCqtOctPlan plan;
        af_cqt_octave_plan(c->fftLength, hop, c->binPerOctave, &plan);
        const float *scale = c->dScale + (size_t)k * c->binPerOctave;
        if (plan.kernel == AF_CQT_WGMMA)
            rc = af_launch_cqt_octave_wgmma(&plan, sig, stride, batch, valid, c->fftLength, hop, padLeft, T, bimg, scale, c->num,
                                            o * c->binPerOctave, dRe, dIm, st);
        else if (plan.kernel == AF_CQT_TC)
            rc = af_launch_cqt_octave_tc(&plan, sig, stride, batch, valid, c->fftLength, hop, padLeft, T, bfrag, scale, c->num,
                                         o * c->binPerOctave, dRe, dIm, st);
        else
            rc = af_launch_cqt_octave(&plan, sig, len, stride, batch, valid, c->fftLength, hop, padLeft, T, c->binPerOctave,
                                      kappa, scale, c->num, o * c->binPerOctave, dRe, dIm, st);
        if (rc) return rc;
    }
    return AF_OK;
}

typedef struct { CQTObj c; int dataLength, T, padLeft; } CqtCall;

static int cqt_chunk(void *p, int nb, float *const *d, void *st) {
    const CqtCall *a = (const CqtCall *)p;
    return cqt_compute_ex(a->c, d[0], a->dataLength, nb, a->T, a->padLeft, d[1], d[2], st);
}

static int cqt_run(CQTObj c, const float *data, int dataLength, int batch, int T, int padLeft, float *re, float *im,
                   int memKind, void *stream) {
    CqtCall a = {c, dataLength, T, padLeft};
    const size_t outPer = (size_t)T * c->num;
    const AfPlane pl[3] = {{data, (size_t)dataLength, AF_IN, 0}, {re, outPer, AF_OUT, 0}, {im, outPer, AF_OUT, 0}};
    return af_run_batch(&c->pipe, memKind, stream, cqt_chunk, &a, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

/* batched / device entry points are stateless: centre padding, every clip on its own */
int cqtObj_cqtBatch(CQTObj c, const float *data, int dataLength, int batch, float *mReal3, float *mImag3,
                    int memKind, void *stream) {
    if (!c || !data || !mReal3 || !mImag3 || dataLength <= 0 || batch <= 0) return af_fail(AF_ERR_ARG, "cqtObj_cqtBatch: bad argument");
    af_clear_error();
    int rc = cqt_device(c);
    if (rc) return rc;
    return cqt_run(c, data, dataLength, batch, cqt_time_length(c, dataLength, 0), c->fftLength / 2, mReal3, mImag3, memKind, stream);
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
    if (!af_tail_assemble(&c->tail, c->fftLength, c->slideLength, dataArr, dataLength, &x, &len)) { c->timeLength = 0; return; }
    af_clear_error();
    if (cqt_device(c)) return;
    c->timeLength = cqt_time_length(c, len, 1);
    if (c->timeLength <= 0) return;
    cqt_run(c, x, len, 1, c->timeLength, 0, mRealArr3, mImageArr3, AFB200_MEM_HOST, NULL);
}

/* ---- chroma: rows x num CQT planes -> rows x chromaNum (cqt_algorithm.c:484-600) ---- */
typedef struct { CQTObj c; int chromaNum, isMag, normType; } ChromaCall;

static int chroma_chunk(void *p, int nb, float *const *d, void *st) {
    const ChromaCall *a = (const ChromaCall *)p;
    return af_launch_chroma(d[0], d[1], nb, a->c->num, a->chromaNum, a->isMag, a->normType, a->c->dChromaBank, d[2], st);
}

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
    ChromaCall a = {c, chromaNum, dataType == SpectralData_Mag, normType};
    const AfPlane pl[3] = {{mReal, (size_t)c->num, AF_IN, 0}, {mImag, (size_t)c->num, AF_IN, 0}, {out, (size_t)chromaNum, AF_OUT, 0}};
    return af_run_batch(&c->pipe, memKind, stream, chroma_chunk, &a, pl, 3, rows, AF_PIPE_CHUNK_BYTES);
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
    if (!c->dDctT && (rc = af_dct2_upload_transposed(&c->dDctT, c->num))) return rc;
    return af_xxcc_batch(&c->pipe, in, rows, c->num, ccNum, rectifyType, c->dDctT, out, memKind, stream);
}

void cqtObj_cqcc(CQTObj c, float *mDataArr1, int ccNum, CepstralRectifyType *rectifyType, float *mDataArr2) {
    if (!c || !mDataArr1 || !mDataArr2) return;
    if (ccNum > c->num || ccNum < 1 || c->timeLength <= 0) return;     /* silent, like cqt_algorithm.c:625-627 */
    cqtObj_cqccBatch(c, mDataArr1, c->timeLength, ccNum, rectifyType ? (int)*rectifyType : CepstralRectify_Log,
                     mDataArr2, AFB200_MEM_HOST, NULL);
}

/* ---- cqhc / deconv: rows x num magnitudes (or powers) -> harmonic-index picks of the timbre sequence / timbre + pitch
 * (cqt_algorithm.c:662-781).  mode 0: out0 [rows x hcNum]; mode 1: out0 = timbre, out1 = pitch [rows x num] ---- */
typedef struct { int num, mode, hcNum, bpo; } DeconvCall;

static int deconv_chunk(void *p, int nb, float *const *d, void *st) {
    const DeconvCall *a = (const DeconvCall *)p;
    return af_launch_cq_deconv(d[0], nb, a->num, a->mode, a->hcNum, a->bpo, d[1], d[2], st);
}

int af_deconv_batch(AfPipe *pipe, const float *in, int rows, int num, int mode, int hcNum, int bpo, float *out0, float *out1,
                    int memKind, void *stream) {
    if (rows <= 0) return AF_OK;
    DeconvCall a = {num, mode, hcNum, bpo};
    const size_t outPer = (size_t)(mode ? num : hcNum);
    const AfPlane pl[3] = {{in, (size_t)num, AF_IN, 0}, {out0, outPer, AF_OUT, 0}, {mode ? out1 : NULL, outPer, AF_OUT, 0}};
    return af_run_batch(pipe, memKind, stream, deconv_chunk, &a, pl, 3, rows, AF_PIPE_CHUNK_BYTES);
}

static int cqt_deconv_batch(CQTObj c, const float *in, int rows, int mode, int hcNum, float *out0, float *out1, int memKind, void *stream) {
    af_clear_error();
    int rc = cqt_device(c);
    if (rc) return rc;
    return af_deconv_batch(&c->pipe, in, rows, c->num, mode, hcNum, c->binPerOctave, out0, out1, memKind, stream);
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
    af_devbuf_free(&c->dSigA); af_devbuf_free(&c->dSigB);
    af_pipe_free(&c->pipe);
    af_dev_free(c->dChromaBank); af_dev_free(c->dDctT);
    af_dev_free(c->dBfrag); af_dev_free(c->dBimg);
    af_dev_free(c->dKappa2); af_dev_free(c->dLeft); af_dev_free(c->dRight); af_dev_free(c->dScale);
    af_cqt_bank_free(&c->bank);
    free(c->kappa2);
    af_tail_free(&c->tail);
    free(c);
}
