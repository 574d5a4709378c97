/* af_nsgt.c -- NSGTObj of the C ABI (host C; compute = the forward FFT of af_launch_stft, then kernels/nsgt.cu).
 * Interface spec: src/nsgt_algorithm.h:14-57; behaviour src/nsgt_algorithm.c:72-637 (object, time grids, transform)
 * and src/filterbank/nsgt_filterBank.c:48-365 (bank).  Everything a call needs is built here at construction (and by
 * setMinLength): the band lengths, offsets and windows, the matrix column map and the per-length transform tables.
 * They go to the device at the first compute call after a rebuild. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueNSGT {
    int num, radix2Exp, fftLength, samplate, binPerOctave, minLength;
    float lowFre, highFre;
    int bankType, scaleType, styleType, normType;

    /* tables of the current minLength, built together by nsgt_build */
    int *lenArr, *binBandArr, *offArr, *cellOff;   /* num each */
    float *freBandArr;                             /* num */
    float *win;                                    /* totalLen: the band windows, band after band */
    int *map;                                      /* num x maxLen */
    int maxLen, totalLen;
    AfNsgtBand *bands;                             /* num: Bluestein groups, then the direct bands */
    int *groupStart;                               /* nGroups + 1 */
    int nGroups, nDirect, maxM, maxDirectL;
    float *tab, *filt;                             /* interleaved complex */
    size_t tabLen, filtLen;                        /* complex values */
    float *cellRe, *cellIm;                        /* totalLen: cells of the last nsgtObj_nsgt call */

    int dirty;                                     /* tables changed since the last upload */
    void *dWin, *dMap, *dBands, *dGroup, *dTab, *dFilt;
    AfDevBuf spec;                                 /* half spectra of the clips */
    AfPipe pipe;
};

/* ---------------- bank (nsgt_filterBank.c:48-239) ---------------- */

/* style -> window of __nsgt_standardFilterBank / __nsgt_efficientFilterBank1 (:265-294, :325-354): Slaney -> Triang,
 * ETSI -> Bartlett, Point / Rect (and anything else) -> ones */
static int style_window(int style) {
    switch (style) {
    case SpectralFilterBankStyle_Slaney: return Window_Triang;
    case SpectralFilterBankStyle_ETSI: return Window_Bartlett;
    case SpectralFilterBankStyle_Hann: return Window_Hann;
    case SpectralFilterBankStyle_Hamm: return Window_Hamm;
    case SpectralFilterBankStyle_Blackman: return Window_Blackman;
    case SpectralFilterBankStyle_Bohman: return Window_Bohman;
    case SpectralFilterBankStyle_Kaiser: return Window_Kaiser;
    case SpectralFilterBankStyle_Gauss: return Window_Gauss;
    default: return Window_Rect;
    }
}

/* __vlinspace(start, stop, length, 0) (src/vector/flux_vector.c:2145-2162) in float32, as the reference evaluates it */
static void linspace_ref(float start, float stop, int length, float *out) {
    float step = (stop - start) / (length - 1 > 0 ? length - 1 : 1);
    for (int i = 0; i < length; i++) out[i] = start + i * step;
}

/* iterative radix-2 forward DFT in double, n a power of two */
static void fft_double(double *re, double *im, int n) {
    for (int i = 1, j = 0; i < n; i++) {
        int bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) { double t = re[i]; re[i] = re[j]; re[j] = t; t = im[i]; im[i] = im[j]; im[j] = t; }
    }
    for (int len = 2; len <= n; len <<= 1) {
        for (int i = 0; i < n; i += len) {
            for (int k = 0; k < len / 2; k++) {
                const double a = -2.0 * M_PI * k / len, wr = cos(a), wi = sin(a);
                const int p = i + k, q = p + len / 2;
                const double xr = re[q] * wr - im[q] * wi, xi = re[q] * wi + im[q] * wr;
                re[q] = re[p] - xr; im[q] = im[p] - xi;
                re[p] += xr; im[p] += xi;
            }
        }
    }
}

typedef struct { int band; double cost; } GroupKey;
static int cmp_group(const void *a, const void *b) {
    const GroupKey *x = (const GroupKey *)a, *y = (const GroupKey *)b;
    if (x->cost != y->cost) return x->cost > y->cost ? -1 : 1;
    return x->band - y->band;
}
static int cmp_direct(const void *a, const void *b) {
    const AfNsgtBand *x = (const AfNsgtBand *)a, *y = (const AfNsgtBand *)b;
    return x->L != y->L ? y->L - x->L : x->band - y->band;
}

typedef struct {
    int *lenArr, *binBandArr, *offArr, *cellOff, *map, *groupStart;
    float *freBandArr, *win, *tab, *filt;
    AfNsgtBand *bands;
    int maxLen, totalLen, nGroups, nDirect, maxM, maxDirectL;
    size_t tabLen, filtLen;
} Tables;

static void tables_free(Tables *t) {
    free(t->lenArr); free(t->binBandArr); free(t->offArr); free(t->cellOff); free(t->map); free(t->groupStart);
    free(t->freBandArr); free(t->win); free(t->tab); free(t->filt); free(t->bands);
    memset(t, 0, sizeof(*t));
}

static int log2_ceil(int v) { int l = 0; while ((1 << l) < v) l++; return l; }

/* lengths, offsets, windows (nsgt_filterBank), the column map of nsgtObj_nsgt step 3 on the time grids of
 * __nsgtObj_dealTime (nsgt_algorithm.c:253-290, 585-604), and the transform tables.  Returns AF_OK, -2 for a window
 * longer than AF_NSGT_MAX_LEN, or AF_ERR_NOMEM. */
static int nsgt_build(const NSGTObj s, int minLength, Tables *t) {
    const int num = s->num, N = s->fftLength;
    memset(t, 0, sizeof(*t));
    float *fre = (float *)calloc((size_t)num + 2, sizeof(float));
    int *bin = (int *)calloc((size_t)num + 2, sizeof(int));
    t->lenArr = (int *)calloc((size_t)num, sizeof(int));
    t->binBandArr = (int *)calloc((size_t)num, sizeof(int));
    t->offArr = (int *)calloc((size_t)num, sizeof(int));
    t->cellOff = (int *)calloc((size_t)num, sizeof(int));
    t->freBandArr = (float *)calloc((size_t)num, sizeof(float));
    if (!fre || !bin || !t->lenArr || !t->binBandArr || !t->offArr || !t->cellOff || !t->freBandArr) goto nomem;

    /* num+2 edges, revised with isEdge = 0 and rounded to bins (:83-139, :482-555) */
    af_band_edges(num, N, s->samplate, s->lowFre, s->highFre, s->scaleType, s->binPerOctave, 0, 0, fre, bin);
    for (int i = 0; i < num; i++) {
        int len;
        if (s->bankType == NSGTFilterBank_Standard) {                 /* :145-152 */
            len = bin[i + 2] - bin[i] + 1;
        } else {                                                      /* :153-182 */
            const int left = bin[i], cur = bin[i + 1], right = bin[i + 2];
            const int v1 = cur - left, v2 = right - cur;
            len = right - left >= 1 ? 2 * (v2 >= v1 ? v2 : v1) + 1 : 0;
        }
        if (len < minLength) len = minLength;
        if (len > AF_NSGT_MAX_LEN) {
            free(fre); free(bin); tables_free(t);
            af_fail(-2, "NSGT: band %d needs a window of %d points; the longest supported is %d", i, len, AF_NSGT_MAX_LEN);
            return -2;
        }
        t->lenArr[i] = len;
        t->cellOff[i] = t->totalLen;
        t->totalLen += len;
        if (len > t->maxLen) t->maxLen = len;
        t->offArr[i] = bin[i + 1] - len / 2 < 0 ? 0 : bin[i + 1] - len / 2;     /* :259-263 */
        t->freBandArr[i] = fre[i + 1];
        t->binBandArr[i] = bin[i + 1];
    }
    free(fre); free(bin);
    fre = NULL; bin = NULL;

    /* windows: symmetric (Efficient) or periodic (Standard), BandWidth norm = / sqrtf(len) (:296-298, :356-358) */
    t->win = (float *)malloc(sizeof(float) * (size_t)t->totalLen);
    if (!t->win) goto nomem;
    for (int i = 0; i < num; i++) {
        const int len = t->lenArr[i];
        float *w = t->win + t->cellOff[i];
        if (af_window_create(style_window(s->styleType), len, s->bankType == NSGTFilterBank_Standard, w)) goto nomem;
        if (s->normType == SpectralFilterBankNormal_BandWidth) {
            const float d = sqrtf(len);
            for (int j = 0; j < len; j++) w[j] = w[j] / d;
        }
    }

    /* column map: out[i][j] = cell_i[k-1], k the first grid point with maxTime[j] < time_i[k] */
    t->map = (int *)malloc(sizeof(int) * (size_t)num * t->maxLen);
    float *maxTime = (float *)malloc(sizeof(float) * ((size_t)t->maxLen + 1));
    float *grid = (float *)malloc(sizeof(float) * ((size_t)t->maxLen + 1));
    if (!t->map || !maxTime || !grid) { free(maxTime); free(grid); goto nomem; }
    const float time = N / (float)s->samplate;
    linspace_ref(0, time, t->maxLen + 1, maxTime);
    for (int i = 0; i < num; i++) {
        const float curLen = t->lenArr[i];
        const float det = (curLen - 2 >= 0 ? curLen - 2 : 0);
        const float offset = time / (curLen + det);
        linspace_ref(-offset, time + offset, (int)(curLen + 1), grid);
        int *row = t->map + (size_t)i * t->maxLen;
        for (int j = 0, start = 0; j < t->maxLen; j++) {
            row[j] = -1;
            for (int k = start; k < t->lenArr[i] + 1; k++) {
                if (maxTime[j] < grid[k]) { row[j] = k - 1; start = k; break; }
            }
        }
    }
    free(maxTime); free(grid);

    /* transform tables per distinct length */
    int *tabAt = (int *)malloc(sizeof(int) * (AF_NSGT_MAX_LEN + 1));
    int *filtAt = (int *)malloc(sizeof(int) * (AF_NSGT_MAX_LEN + 1));
    if (!tabAt || !filtAt) { free(tabAt); free(filtAt); goto nomem; }
    for (int L = 0; L <= AF_NSGT_MAX_LEN; L++) tabAt[L] = filtAt[L] = -1;
    for (int i = 0; i < num; i++) {
        const int L = t->lenArr[i];
        if (tabAt[L] >= 0) continue;
        tabAt[L] = (int)t->tabLen;
        if (L <= AF_NSGT_BLUESTEIN_MAX) {
            filtAt[L] = (int)t->filtLen;
            t->tabLen += L;
            t->filtLen += (size_t)1 << log2_ceil(2 * L - 1);
        } else {
            t->tabLen += AF_NSGT_FINE + (L - 1) / AF_NSGT_FINE + 1;
        }
    }
    t->tab = (float *)malloc(sizeof(float) * 2 * (t->tabLen ? t->tabLen : 1));
    t->filt = (float *)malloc(sizeof(float) * 2 * (t->filtLen ? t->filtLen : 1));
    double *hr = (double *)malloc(sizeof(double) * 2 * (AF_NSGT_BLUESTEIN_MAX * 2));
    if (!t->tab || !t->filt || !hr) { free(tabAt); free(filtAt); free(hr); goto nomem; }
    double *hi = hr + AF_NSGT_BLUESTEIN_MAX * 2;
    for (int L = 1; L <= AF_NSGT_MAX_LEN; L++) {
        if (tabAt[L] < 0) continue;
        float *tb = t->tab + 2 * (size_t)tabAt[L];
        if (L <= AF_NSGT_BLUESTEIN_MAX) {
            /* chirp c_m = e^{i pi m^2 / L} (phase from m^2 mod 2L), filter h = conj(c) on -(L-1) .. L-1 wrapped to M */
            const int M = 1 << log2_ceil(2 * L - 1);
            memset(hr, 0, sizeof(double) * 2 * M);
            memset(hi, 0, sizeof(double) * M);
            for (int m = 0; m < L; m++) {
                const double a = M_PI * (double)(((long long)m * m) % (2LL * L)) / L;
                const double c = cos(a), sn = sin(a);
                tb[2 * m] = (float)c; tb[2 * m + 1] = (float)sn;
                hr[m] = c; hi[m] = -sn;
                if (m) { hr[M - m] = c; hi[M - m] = -sn; }
            }
            fft_double(hr, hi, M);
            float *fl = t->filt + 2 * (size_t)filtAt[L];
            const double scale = 1.0 / ((double)L * M);
            for (int k = 0; k < M; k++) { fl[2 * k] = (float)(hr[k] * scale); fl[2 * k + 1] = (float)(hi[k] * scale); }
        } else {
            /* fine[r] = e^{2 pi i r / L}, coarse[q] = e^{2 pi i 64 q / L} */
            for (int r = 0; r < AF_NSGT_FINE; r++) {
                const double a = 2.0 * M_PI * r / L;
                tb[2 * r] = (float)cos(a); tb[2 * r + 1] = (float)sin(a);
            }
            for (int q = 0; q <= (L - 1) / AF_NSGT_FINE; q++) {
                const double a = 2.0 * M_PI * (double)((long long)q * AF_NSGT_FINE % L) / L;
                tb[2 * (AF_NSGT_FINE + q)] = (float)cos(a); tb[2 * (AF_NSGT_FINE + q) + 1] = (float)sin(a);
            }
        }
    }
    free(hr);

    /* Bluestein groups: runs of consecutive bands with sum M <= AF_NSGT_GROUP_BUDGET, ordered largest first; then the
     * direct bands, longest first */
    t->bands = (AfNsgtBand *)calloc((size_t)num, sizeof(AfNsgtBand));
    AfNsgtBand *all = (AfNsgtBand *)calloc((size_t)num, sizeof(AfNsgtBand));
    GroupKey *keys = (GroupKey *)calloc((size_t)num + 1, sizeof(GroupKey));
    int *gFirst = (int *)calloc((size_t)num + 1, sizeof(int));
    t->groupStart = (int *)calloc((size_t)num + 2, sizeof(int));
    if (!t->bands || !all || !keys || !gFirst || !t->groupStart) {
        free(tabAt); free(filtAt); free(all); free(keys); free(gFirst); goto nomem;
    }
    int nb = 0, nd = 0, sum = 0;
    for (int i = 0; i < num; i++) {
        const int L = t->lenArr[i];
        AfNsgtBand b;
        b.L = L; b.off = t->offArr[i]; b.winOff = t->cellOff[i]; b.cellOff = t->cellOff[i];
        b.tabOff = tabAt[L]; b.filtOff = filtAt[L]; b.band = i;
        b.log2M = L <= AF_NSGT_BLUESTEIN_MAX ? log2_ceil(2 * L - 1) : 0;
        if (L > AF_NSGT_BLUESTEIN_MAX) {
            t->bands[num - 1 - nd++] = b;             /* direct bands collect at the back */
            if (L > t->maxDirectL) t->maxDirectL = L;
            continue;
        }
        const int M = 1 << b.log2M;
        if (M > t->maxM) t->maxM = M;
        if (nb == 0 || sum + M > AF_NSGT_GROUP_BUDGET) {
            gFirst[t->nGroups] = nb;
            keys[t->nGroups].band = t->nGroups;
            keys[t->nGroups].cost = 0;
            t->nGroups++;
            sum = 0;
        }
        sum += M;
        keys[t->nGroups - 1].cost += (double)M * (b.log2M > 0 ? b.log2M : 1);
        all[nb++] = b;
    }
    gFirst[t->nGroups] = nb;
    t->nDirect = nd;
    free(tabAt); free(filtAt);
    qsort(keys, (size_t)t->nGroups, sizeof(GroupKey), cmp_group);
    int at = 0;
    for (int g = 0; g < t->nGroups; g++) {
        const int src = keys[g].band;
        t->groupStart[g] = at;
        for (int k = gFirst[src]; k < gFirst[src + 1]; k++) t->bands[at++] = all[k];
    }
    t->groupStart[t->nGroups] = at;
    qsort(t->bands + at, (size_t)nd, sizeof(AfNsgtBand), cmp_direct);
    free(all); free(keys); free(gFirst);
    return AF_OK;

nomem:
    free(fre); free(bin);
    tables_free(t);
    return af_fail(AF_ERR_NOMEM, "NSGT: out of host memory");
}

static void nsgt_adopt(NSGTObj s, Tables *t, int minLength) {
    free(s->lenArr); free(s->binBandArr); free(s->offArr); free(s->cellOff); free(s->map); free(s->groupStart);
    free(s->freBandArr); free(s->win); free(s->tab); free(s->filt); free(s->bands);
    s->lenArr = t->lenArr; s->binBandArr = t->binBandArr; s->offArr = t->offArr; s->cellOff = t->cellOff;
    s->map = t->map; s->groupStart = t->groupStart; s->freBandArr = t->freBandArr; s->win = t->win;
    s->tab = t->tab; s->filt = t->filt; s->bands = t->bands;
    s->maxLen = t->maxLen; s->totalLen = t->totalLen; s->nGroups = t->nGroups; s->nDirect = t->nDirect;
    s->maxM = t->maxM; s->maxDirectL = t->maxDirectL; s->tabLen = t->tabLen; s->filtLen = t->filtLen;
    s->minLength = minLength;
    s->dirty = 1;
}

/* ---------------- the reference's entry points ---------------- */

int nsgtObj_new(NSGTObj *nsgtObj, int num, int radix2Exp, int *samplate, float *lowFre, float *highFre,
                int *binPerOctave, int *minLength, NSGTFilterBankType *nsgtFilterBankType,
                SpectralFilterBankScaleType *filterScaleType, SpectralFilterBankStyleType *filterStyleType,
                SpectralFilterBankNormalType *filterNormalType) {
    af_clear_error();
    int minLen = 3, sr = 32000, bpo = 12;
    int bank = NSGTFilterBank_Efficient, scale = SpectralFilterBankScale_Octave;
    int style = SpectralFilterBankStyle_Hann, norm = SpectralFilterBankNormal_BandWidth;
    if (!nsgtObj) return -1;
    if (minLength && *minLength > 0) minLen = *minLength;
    if (radix2Exp && (radix2Exp < 1 || radix2Exp > 30)) { printf("radix2Exp is error!\n"); return -100; }
    const int N = 1 << radix2Exp;
    if (samplate && *samplate > 0 && *samplate <= 196000) sr = *samplate;
    if (nsgtFilterBankType) bank = *nsgtFilterBankType;
    if (filterScaleType) {
        scale = *filterScaleType;
        if (scale > SpectralFilterBankScale_Log) { printf("scaleType is error!\n"); return 1; }
    }
    if (filterStyleType) {
        style = *filterStyleType;
        if (style == SpectralFilterBankStyle_Gammatone) style = SpectralFilterBankStyle_Hann;
    }
    if (filterNormalType) {
        norm = *filterNormalType;
        if (norm == SpectralFilterBankNormal_Area) norm = SpectralFilterBankNormal_BandWidth;
    }
    if (binPerOctave && *binPerOctave >= 4 && *binPerOctave <= 48) bpo = *binPerOctave;
    /* range defaults and the isEdge = 1 revision of Linear / Octave (:151-209) */
    AfRange r;
    if (af_revise_range(num, N, sr, lowFre, highFre, scale, bpo, &r)) {
        printf("scale %s: lowFre and num is large, overflow error!\n", scale == SpectralFilterBankScale_Linear ? "linear" : "log");
        return -1;
    }
    if (num < 2 || num > N / 2 + 1) { printf("num is error!\n"); return -1; }
    if (radix2Exp > 20) {
        af_fail(-2, "nsgtObj_new: radix2Exp=%d; the forward FFT supports at most 2^20 points", radix2Exp);
        return -2;
    }

    NSGTObj s = (NSGTObj)calloc(1, sizeof(struct OpaqueNSGT));
    if (!s) return -1;
    s->num = num; s->radix2Exp = radix2Exp; s->fftLength = N; s->samplate = sr; s->binPerOctave = bpo;
    s->lowFre = r.low; s->highFre = r.high;
    s->bankType = bank == NSGTFilterBank_Standard ? NSGTFilterBank_Standard : NSGTFilterBank_Efficient;
    s->scaleType = scale; s->styleType = style; s->normType = norm;
    Tables t;
    int rc = nsgt_build(s, minLen, &t);
    if (rc) { free(s); return rc == -2 ? -2 : -1; }
    nsgt_adopt(s, &t, minLen);
    s->cellRe = (float *)calloc((size_t)s->totalLen, sizeof(float));
    s->cellIm = (float *)calloc((size_t)s->totalLen, sizeof(float));
    if (!s->cellRe || !s->cellIm) { nsgtObj_free(s); return -1; }
    *nsgtObj = s;
    return 0;
}

int nsgtObj_getMaxTimeLength(NSGTObj s) { return s ? s->maxLen : 0; }
int nsgtObj_getTotalTimeLength(NSGTObj s) { return s ? s->totalLen : 0; }
int *nsgtObj_getTimeLengthArr(NSGTObj s) { return s ? s->lenArr : NULL; }
float *nsgtObj_getFreBandArr(NSGTObj s) { return s ? s->freBandArr : NULL; }
int *nsgtObj_getBinBandArr(NSGTObj s) { return s ? s->binBandArr : NULL; }

void nsgtObj_setMinLength(NSGTObj s, int minLength) {
    if (!s || minLength < 1 || minLength == s->minLength) return;      /* :447 */
    Tables t;
    if (nsgt_build(s, minLength, &t)) return;                           /* too long a window: the object stays as it was */
    float *re = (float *)calloc((size_t)t.totalLen, sizeof(float)), *im = (float *)calloc((size_t)t.totalLen, sizeof(float));
    if (!re || !im) { free(re); free(im); tables_free(&t); af_fail(AF_ERR_NOMEM, "NSGT: out of host memory"); return; }
    nsgt_adopt(s, &t, minLength);
    free(s->cellRe); free(s->cellIm);
    s->cellRe = re; s->cellIm = im;
}

void nsgtObj_getCellData(NSGTObj s, float **realArr3, float **imageArr3) {
    if (!s) return;
    if (realArr3) *realArr3 = s->cellRe;
    if (imageArr3) *imageArr3 = s->cellIm;
}

/* ---------------- device path ---------------- */

static void nsgt_device_tables_free(NSGTObj s) {
    af_dev_free(s->dWin); af_dev_free(s->dMap); af_dev_free(s->dBands); af_dev_free(s->dGroup);
    af_dev_free(s->dTab); af_dev_free(s->dFilt);
    s->dWin = s->dMap = s->dBands = s->dGroup = s->dTab = s->dFilt = NULL;
}

static int nsgt_device(NSGTObj s) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (!s->dirty) return AF_OK;
    nsgt_device_tables_free(s);
    if ((rc = af_dev_upload(&s->dWin, s->win, sizeof(float) * (size_t)s->totalLen)) ||
        (rc = af_dev_upload(&s->dMap, s->map, sizeof(int) * (size_t)s->num * s->maxLen)) ||
        (rc = af_dev_upload(&s->dBands, s->bands, sizeof(AfNsgtBand) * (size_t)s->num)) ||
        (rc = af_dev_upload(&s->dGroup, s->groupStart, sizeof(int) * ((size_t)s->nGroups + 1))) ||
        (rc = af_dev_upload(&s->dTab, s->tab, sizeof(float) * 2 * (s->tabLen ? s->tabLen : 1))) ||
        (rc = af_dev_upload(&s->dFilt, s->filt, sizeof(float) * 2 * (s->filtLen ? s->filtLen : 1))))
        return rc;
    s->dirty = 0;
    return AF_OK;
}

/* nb clips already on the device: forward FFT (one frame per clip) into the object's spectrum planes, then the bands */
static int nsgt_run(NSGTObj s, const float *dIn, int nb, float *re, float *im, float *cre, float *cim, void *st) {
    const int N = s->fftLength, width = N / 2 + 1;
    int rc;
    if ((rc = af_devbuf_reserve(&s->spec, sizeof(float) * 2 * (size_t)nb * width))) return rc;
    float *specRe = (float *)s->spec.ptr, *specIm = specRe + (size_t)nb * width;
    AfFrameSrc src;
    memset(&src, 0, sizeof(src));
    src.fftLength = N; src.slideLength = N; src.dataLength = N; src.timeLength = 1; src.batch = nb;
    src.validLength = N; src.padMode = PaddingMode_Constant; src.data = dIn;
    if ((rc = af_launch_stft(&src, AF_STFT_HALF, 1.0f, specRe, specIm, st))) return rc;
    AfNsgtArgs a;
    memset(&a, 0, sizeof(a));
    a.fftLength = N; a.num = s->num; a.maxLen = s->maxLen; a.totalLen = s->totalLen; a.batch = nb;
    a.specRe = specRe; a.specIm = specIm;
    a.win = (const float *)s->dWin; a.map = (const int *)s->dMap; a.bands = (const AfNsgtBand *)s->dBands;
    a.groupStart = (const int *)s->dGroup; a.tab = (const float *)s->dTab; a.filt = (const float *)s->dFilt;
    a.nGroups = s->nGroups; a.maxM = s->maxM; a.nDirect = s->nDirect; a.maxDirectL = s->maxDirectL;
    a.outRe = re; a.outIm = im; a.cellRe = cre; a.cellIm = cim;
    return af_launch_nsgt(&a, st);
}

static int nsgt_chunk(void *p, int nb, float *const *d, void *st) {
    return nsgt_run((NSGTObj)p, d[0], nb, d[1], d[2], d[3], d[4], st);
}

int nsgtObj_nsgtBatch(NSGTObj s, const float *data, int batch, float *mReal, float *mImag, float *cellReal,
                      float *cellImag, int memKind, void *stream) {
    if (!s || !data || !mReal || !mImag || batch < 0 || (!cellReal != !cellImag))
        return af_fail(AF_ERR_ARG, "nsgtObj_nsgtBatch: bad argument");
    af_clear_error();
    int rc = nsgt_device(s);
    if (rc) return rc;
    if (batch == 0) return AF_OK;
    const size_t outPer = (size_t)s->num * s->maxLen, cellPer = (size_t)s->totalLen;
    const AfPlane pl[5] = {{data, (size_t)s->fftLength, AF_IN, 0}, {mReal, outPer, AF_OUT, 0}, {mImag, outPer, AF_OUT, 0},
                           {cellReal, cellPer, AF_OUT, 0}, {cellImag, cellPer, AF_OUT, 0}};
    return af_run_batch(&s->pipe, memKind, stream, nsgt_chunk, s, pl, 5, batch, AF_PIPE_CHUNK_BYTES);
}

void nsgtObj_nsgt(NSGTObj s, float *dataArr, float *mRealArr3, float *mImageArr3) {
    if (!s || !dataArr || !mRealArr3 || !mImageArr3) return;
    nsgtObj_nsgtBatch(s, dataArr, 1, mRealArr3, mImageArr3, s->cellRe, s->cellIm, AFB200_MEM_HOST, NULL);
}

void nsgtObj_free(NSGTObj s) {
    if (!s) return;
    nsgt_device_tables_free(s);
    af_devbuf_free(&s->spec);
    af_pipe_free(&s->pipe);
    free(s->lenArr); free(s->binBandArr); free(s->offArr); free(s->cellOff); free(s->map); free(s->groupStart);
    free(s->freBandArr); free(s->win); free(s->tab); free(s->filt); free(s->bands);
    free(s->cellRe); free(s->cellIm);
    free(s);
}
