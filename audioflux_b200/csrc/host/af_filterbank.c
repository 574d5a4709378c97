/* af_filterbank.c -- auditory scales, band edges and dense filter banks (setup time, host).
 *
 * Behavioural spec (constants the device kernels consume; every integer outcome -- band-edge
 * bins, supports -- must equal the reference's, so the float32 evaluation order of the
 * published scale formulas is kept):
 *   scales      src/filterbank/auditory_filterBank.c:1023-1190
 *   band edges  :594-677      range revision :946-1021     bank styles :210-500
 *   range rules src/bft_algorithm.c:158-230, src/cwt_algorithm.c:137-196
 * Unlike the reference, writes are clipped to the bank's columns (the reference writes out of
 * bounds when a revised edge leaves [0, samplate/2], e.g. Linspace/Log with the default range).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

/* ---- Hz <-> scale value.  `ref` = bin spacing (Linear) or bins per octave (Octave). ---- */
static float fre_to_scale(float fre, int scale, float ref) {
    switch (scale) {
    case SpectralFilterBankScale_Linear: return roundf(fre / ref);
    case SpectralFilterBankScale_Mel: return 2595 * log10f(1 + fre / 700);            /* O'Shaughnessy */
    case SpectralFilterBankScale_Bark: {                                              /* Traunmueller */
        float z = 26.81 * fre / (1960 + fre) - 0.53;
        if (z < 2) z = z + 0.15 * (2 - z);
        else if (z > 20.1) z = z + 0.22 * (z - 20.1);
        return z;
    }
    case SpectralFilterBankScale_Erb: {                                               /* Glasberg-Moore */
        float a = 21.3654;
        return a * log10f(1 + fre * 0.004368);
    }
    case SpectralFilterBankScale_Octave: return roundf(ref * log2(fre / 440));
    case SpectralFilterBankScale_Log: return log2(fre / 440);
    default: return fre;                                                              /* Linspace */
    }
}

static float scale_to_fre(float v, int scale, float ref) {
    switch (scale) {
    case SpectralFilterBankScale_Linear: return v * ref;
    case SpectralFilterBankScale_Mel: return 700 * (powf(10, v / 2595) - 1);
    case SpectralFilterBankScale_Bark: {
        if (v < 2) v = (v - 0.3) / 0.85;
        else if (v > 20.1) v = (v + 4.422) / 1.22;
        return 1960 * (v + 0.53) / (26.28 - v);
    }
    case SpectralFilterBankScale_Erb: {
        float a = 21.3654;
        return (powf(10, v / a) - 1) / 0.004368;
    }
    case SpectralFilterBankScale_Octave: return pow(2, v / ref) * 440;
    case SpectralFilterBankScale_Log: return pow(2, v) * 440;
    default: return v;
    }
}

static void linspace_f32(float start, float stop, int n, float *out) {
    float step = (stop - start) / (n - 1 > 0 ? n - 1 : 1);
    for (int i = 0; i < n; i++) out[i] = start + i * step;
}

static void default_log_range(float *lo, float *hi) {
    *lo = powf(2, -45 / 12.0) * 440;      /* C1 */
    *hi = powf(2, 38 / 12.0) * 440;       /* B7 */
}

int af_revise_range(int num, int fftLength, int samplate, const float *lowFre, const float *highFre,
                    int scale, int bpo, AfRange *out) {
    const int logLike = (scale == SpectralFilterBankScale_Octave || scale == SpectralFilterBankScale_Log);
    float lo = 0, hi = samplate / 2.0;
    if (lowFre && *lowFre >= 0 && *lowFre < samplate / 2.0) lo = *lowFre;
    if (lo == 0 && logLike) default_log_range(&lo, &hi);
    if (highFre && *highFre > 0 && *highFre <= samplate / 2.0) hi = *highFre;
    if (hi < lo) {
        lo = 0; hi = samplate / 2.0;
        if (logLike) default_log_range(&lo, &hi);
    }
    out->lowIndex = out->highIndex = 0;
    if (scale == SpectralFilterBankScale_Linear) {
        float det = samplate / (float)fftLength;
        float l = roundf(lo / det), h = l + num - 1;
        lo = l * det; hi = h * det;
        out->lowIndex = roundf(lo / det);
        out->highIndex = roundf(hi / det);
        if (hi > samplate / 2.0) return -1;
    } else if (scale == SpectralFilterBankScale_Octave) {
        float l = fre_to_scale(lo, scale, bpo), h = l + num - 1;
        lo = scale_to_fre(l, scale, bpo); hi = scale_to_fre(h, scale, bpo);
        if (hi > samplate / 2.0) return -1;
    }
    out->low = lo; out->high = hi;
    return 0;
}

/* widen [low, high] so that the num centres sit inside num+2 edge points (non-edge styles);
 * edge-inclusive styles (gammatone: the num points ARE the centres) only snap Octave / Linear to their grids */
static float widen_range(int num, int lengthForLinear, int samplate, int scale, int bpo, int isEdge,
                         float *low, float *high) {
    float ref = 0, lo = *low, hi = *high;
    const int off = isEdge ? 0 : 1, det = isEdge ? 0 : 2;
    if (scale == SpectralFilterBankScale_Octave) {
        ref = (bpo >= 4 && bpo <= 48) ? bpo : 12;
        float l = fre_to_scale(lo, scale, ref) - off, h = l + num - 1 + det;
        lo = scale_to_fre(l, scale, ref); hi = scale_to_fre(h, scale, ref);
    } else if (scale == SpectralFilterBankScale_Linear) {
        ref = samplate * 1.0 / lengthForLinear;
        float l = roundf(lo / ref) - off, h = l + num - 1 + det;
        lo = l * ref; hi = h * ref;
    } else if (isEdge) {
        /* Linspace / Log keep the range as given */
    } else if (scale == SpectralFilterBankScale_Linspace) {
        float d = (hi - lo) / (num - 1);
        lo = lo - d; hi = hi + d;
    } else if (scale == SpectralFilterBankScale_Log) {
        float l = fre_to_scale(lo, scale, 0), h = fre_to_scale(hi, scale, 0);
        float d = (h - l) / (num - 1);
        lo = scale_to_fre(l - d, scale, 0); hi = scale_to_fre(h + d, scale, 0);
    }
    *low = lo; *high = hi;
    return ref;
}

void af_band_edges(int num, int fftLength, int samplate, float lowFre, float highFre, int scale,
                   int bpo, int slaneyBins, int isEdge, float *freEdge, int *binEdge) {
    float ref = widen_range(num, fftLength, samplate, scale, bpo, isEdge, &lowFre, &highFre);
    const int n = isEdge ? num : num + 2;
    linspace_f32(fre_to_scale(lowFre, scale, ref), fre_to_scale(highFre, scale, ref), n, freEdge);
    for (int i = 0; i < n; i++) freEdge[i] = scale_to_fre(freEdge[i], scale, ref);
    if (!binEdge) return;
    if (!slaneyBins) {
        for (int i = 0; i < n; i++) binEdge[i] = roundf(fftLength * freEdge[i] / samplate);
    } else {
        /* first FFT-grid frequency strictly above the edge; grid = linspace(0, sr - sr/n, n) */
        float step = ((samplate - samplate / (float)fftLength) - 0.0f) / (fftLength - 1 > 0 ? fftLength - 1 : 1);
        for (int i = 0; i < n; i++) {
            int j = 0;
            while (j < fftLength && !(0.0f + j * step > freEdge[i])) j++;
            binEdge[i] = j < fftLength ? j : 0;
        }
    }
}

/* Weights that fall above the Nyquist bin (band edges beyond samplate / 2: Log / Linspace scales with highFre at Nyquist)
 * have no place in the one-sided bank; they are counted so that callers whose reference counterpart keeps them -- the
 * pseudo banks of pwtObj_new span all fftLength bins -- can refuse instead of dropping them silently.  A weight at bin -1
 * (Linear scale starting at bin 0: the reference writes it in FRONT of its bank buffer, auditory_filterBank.c:358-364, so
 * the first band is empty there too) is dropped without counting. */
static __thread int g_clipped;
int af_filterbank_clipped(void) { return g_clipped; }

static void put(float *bank, int width, int row, int col, float v) {
    if (col >= 0 && col < width) bank[(size_t)row * width + col] = v;
    else if (col >= width && v != 0.0f) g_clipped++;
}

static void window_half_fill(float *bank, int width, int row, int style, int from, int to, int rising) {
    /* one flank of a window-designed filter (flux: auditory_filterBank.c:249-316) */
    static const int map[] = {0, 0, 0, 0, 0, Window_Hann, Window_Hamm, Window_Blackman, Window_Bohman,
                              Window_Kaiser, Window_Gauss};
    int span = to - from;               /* > 0 */
    int L = 2 * span + 1;
    double *w = (double *)malloc(sizeof(double) * (size_t)L);
    if (!w) return;
    af_window_symmetric(map[style], L, NULL, w);
    if (rising) for (int j = from, k = 0; j <= to; j++, k++) put(bank, width, row, j, (float)w[k]);
    else for (int j = from + 1, k = L / 2 + 1; j <= to; j++, k++) put(bank, width, row, j, (float)w[k]);
    free(w);
}

/* Gammatone bank: magnitude response of Slaney's 4th-order gammatone filter (four cascaded biquads,
 * "An efficient implementation of the Patterson-Holdsworth auditory filter bank", 1993) at the FFT bins.
 * Behavioural spec: src/filterbank/auditory_filterBank.c:509-591 (bank, norms, x2 interior),
 * :691-924 (coefficients), src/dsp/filterDesign_freqz.c:8-118 (response on
 * omega = linspace(0, 2 pi - 2 pi/n, n)[0 .. n/2]).
 * The lowest bands (centre frequency below ~100 Hz) are numerically degenerate: the gain and the biquad
 * responses lose most of their float32 digits to cancellation, and the reference's values there are what a
 * float32 evaluation in this order produces (a float64 evaluation differs by up to 2 % of the row maximum).
 * To stay within 1e-4 of the reference the evaluation below is deliberately float32, section by section. */
typedef struct { float re, im; } cf32;
static cf32 cf_mul(cf32 a, cf32 b) { cf32 r = {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; return r; }
static cf32 cf_div(cf32 a, cf32 b) {
    float d = b.re * b.re + b.im * b.im;
    cf32 r = {(a.re * b.re + a.im * b.im) / d, (a.im * b.re - a.re * b.im) / d};
    return r;
}
/* c0 + c1 e^{-jw} + c2 e^{-2jw}, accumulated term by term in float */
static cf32 poly3(const float *c, float w) {
    cf32 r = {0, 0};
    for (int j = 0; j < 3; j++) { r.re += cosf(-w * j) * c[j]; r.im += sinf(-w * j) * c[j]; }
    return r;
}

static void gammatone_bank(int num, int fftLength, int samplate, int norm, const float *fre, float *bank) {
    const int width = fftLength / 2 + 1;
    const float t = 1.0 / samplate;
    const float pv = sqrtf(3 + powf(2, 1.5)), nv = sqrtf(3 - powf(2, 1.5));
    const float wEnd = 2 * M_PI, wStep = (wEnd - wEnd / fftLength - 0.0f) / (fftLength - 1 > 0 ? fftLength - 1 : 1);
    for (int i = 0; i < num; i++) {
        const float cf = fre[i];
        const float bw = (cf / 9.26449 + 24.7) * 2 * M_PI * 1.019;         /* 2 pi * 1.019 * ERB(cf) */
        const float arg = cf * 2 * M_PI * t;
        const float v = -t * expf(-t * bw);
        const float cs = cosf(arg), sn = sinf(arg);
        const float c2r = cosf(4 * M_PI * t * cf), c2i = sinf(4 * M_PI * t * cf);   /* e^{i 4 pi cf t} */
        const float gr = 2 * t * expf(-bw * t) * cos(2 * M_PI * t * cf);
        const float gi = 2 * t * expf(-bw * t) * sin(2 * M_PI * t * cf);
        const float den1 = -2 * cs / expf(bw * t), den2 = expf(-2 * t * bw);        /* shared denominator */
        const float k[4] = {cs + pv * sn, cs - pv * sn, cs + nv * sn, cs - nv * sn};
        float num1[4];
        for (int s = 0; s < 4; s++) num1[s] = v * k[s];                             /* numerator z^-1 terms */
        float mags[4];
        for (int s = 0; s < 4; s++) {
            float re = -2 * t * c2r + gr * k[s], im = -2 * t * c2i + gi * k[s];
            mags[s] = sqrtf(re * re + im * im);
        }
        const float r5 = -2 / expf(2 * t * bw) - 2 * c2r + 2 * (1 + c2r) / expf(t * bw);
        const float i5 = -2 * c2i + 2 * c2i / expf(t * bw);
        const float gain = mags[0] * mags[1] * mags[2] * mags[3] / ((r5 * r5 + i5 * i5) * (r5 * r5 + i5 * i5));
        float sec[4][6];
        for (int s = 0; s < 4; s++) {
            sec[s][0] = s == 0 ? t / gain : t;
            sec[s][1] = s == 0 ? num1[0] / gain : num1[s];
            sec[s][2] = s == 0 ? 0.0f / gain : 0.0f;
            sec[s][3] = 1; sec[s][4] = den1; sec[s][5] = den2;
        }
        float *row = bank + (size_t)i * width;
        for (int kbin = 0; kbin < width; kbin++) {
            const float w = 0.0f + kbin * wStep;
            cf32 h = cf_div(poly3(sec[0], w), poly3(sec[0] + 3, w));
            for (int s = 1; s < 4; s++) h = cf_mul(h, cf_div(poly3(sec[s], w), poly3(sec[s] + 3, w)));
            row[kbin] = sqrtf(h.re * h.re + h.im * h.im);
        }
        if (norm == SpectralFilterBankNormal_Area || norm == SpectralFilterBankNormal_BandWidth) {
            float wt;
            if (norm == SpectralFilterBankNormal_Area) {
                float inner = 0;
                for (int j = 1; j < width - 1; j++) inner += row[j];
                wt = row[0] + row[width - 1];
                wt += inner * 2;
            } else {
                wt = 1.019 * 24.7 * (0.00437 * fre[i] + 1);
                wt = wt / 2;
            }
            for (int j = 0; j < width; j++) if (row[j]) row[j] = row[j] / wt;
        }
        for (int j = 1; j < width - 1; j++) row[j] *= 2;                            /* one-sided spectrum: double the interior */
    }
}

int af_auditory_filterbank(int num, int fftLength, int samplate, int scale, int style, int norm,
                           float lowFre, float highFre, int bpo, float *bank, float *freBandArr,
                           int *binBandArr) {
    if (num < 1 || fftLength < 2 || !bank) return AF_ERR_ARG;
    g_clipped = 0;
    if (style == SpectralFilterBankStyle_Gammatone) {
        float *cfre = (float *)calloc((size_t)num + 2, sizeof(float));
        int *cbin = (int *)calloc((size_t)num + 2, sizeof(int));
        if (!cfre || !cbin) { free(cfre); free(cbin); return AF_ERR_NOMEM; }
        af_band_edges(num, fftLength, samplate, lowFre, highFre, scale, bpo, 0, 1, cfre, cbin);
        gammatone_bank(num, fftLength, samplate, norm, cfre, bank);
        if (freBandArr) memcpy(freBandArr, cfre, sizeof(float) * (size_t)num);
        if (binBandArr) memcpy(binBandArr, cbin, sizeof(int) * (size_t)num);
        free(cfre); free(cbin);
        return AF_OK;
    }
    const int width = fftLength / 2 + 1;
    float *fre = (float *)calloc((size_t)num + 2, sizeof(float));
    int *bin = (int *)calloc((size_t)num + 2, sizeof(int));
    if (!fre || !bin) { free(fre); free(bin); return AF_ERR_NOMEM; }
    memset(bank, 0, sizeof(float) * (size_t)num * width);
    af_band_edges(num, fftLength, samplate, lowFre, highFre, scale, bpo,
                  style == SpectralFilterBankStyle_Slaney, 0, fre, bin);

    if (scale == SpectralFilterBankScale_Linear) {
        for (int i = 1; i <= num; i++) { bin[i] -= 1; put(bank, width, i - 1, bin[i], 1.0f); }
    } else if (style == SpectralFilterBankStyle_Slaney) {
        /* triangles measured in Hz on the FFT grid */
        float step = ((samplate - samplate / (float)fftLength) - 0.0f) / (fftLength - 1 > 0 ? fftLength - 1 : 1);
        for (int i = 0; i < num; i++) {
            float up = fre[i + 1] - fre[i], down = fre[i + 2] - fre[i + 1];
            for (int j = bin[i]; j < bin[i + 1]; j++) put(bank, width, i, j, ((0.0f + j * step) - fre[i]) / up);
            for (int j = bin[i + 1]; j < bin[i + 2]; j++) put(bank, width, i, j, (fre[i + 2] - (0.0f + j * step)) / down);
        }
    } else if (style == SpectralFilterBankStyle_ETSI) {
        /* triangles measured in bins */
        for (int i = 1; i <= num; i++) {
            int l = bin[i - 1], c = bin[i], r = bin[i + 1];
            if (c > l) for (int j = l; j <= c; j++) put(bank, width, i - 1, j, 1.0 * (j - l) / (c - l));
            for (int j = c + 1; j <= r; j++) put(bank, width, i - 1, j, 1.0 * (r - j) / (r - c));
        }
    } else if (style == SpectralFilterBankStyle_Point) {
        for (int i = 1; i <= num; i++) put(bank, width, i - 1, bin[i], 1.0f);
    } else if (style == SpectralFilterBankStyle_Rect) {
        for (int i = 1; i <= num; i++)
            for (int j = bin[i - 1]; j <= bin[i + 1]; j++) put(bank, width, i - 1, j, 1.0f);
    } else {
        for (int i = 1; i <= num; i++) {
            int l = bin[i - 1], c = bin[i], r = bin[i + 1];
            if (c > l) window_half_fill(bank, width, i - 1, style, l, c, 1);
            if (r > c) window_half_fill(bank, width, i - 1, style, c, r, 0);
        }
    }

    if (scale != SpectralFilterBankScale_Linear &&
        (norm == SpectralFilterBankNormal_Area || norm == SpectralFilterBankNormal_BandWidth)) {
        for (int i = 0; i < num; i++) {
            float wt = 0;
            float *row = bank + (size_t)i * width;
            if (norm == SpectralFilterBankNormal_Area) for (int j = 0; j < width; j++) wt += row[j];
            else wt = (fre[i + 2] - fre[i]) / 2;
            for (int j = 0; j < width; j++) if (row[j]) row[j] = row[j] / wt;   /* exact zeros stay zero */
        }
    }
    if (freBandArr) memcpy(freBandArr, fre + 1, sizeof(float) * (size_t)num);
    if (binBandArr) memcpy(binBandArr, bin + 1, sizeof(int) * (size_t)num);
    free(fre); free(bin);
    return AF_OK;
}

int afb200_auditoryFilterBank(int num, int fftLength, int samplate, int scaleType, int styleType,
                              int normType, float lowFre, float highFre, int binPerOctave,
                              float *bank, float *freBandArr, int *binBandArr) {
    return af_auditory_filterbank(num, fftLength, samplate, scaleType, styleType, normType, lowFre,
                                  highFre, binPerOctave, bank, freBandArr, binBandArr);
}

int af_bands_build(const float *bank, int num, int width, AfBands *b) {
    b->num = num; b->width = width; b->nnz = 0; b->maxLen = 0;
    b->start = (int *)calloc((size_t)num, sizeof(int));
    b->len = (int *)calloc((size_t)num, sizeof(int));
    if (!b->start || !b->len) return AF_ERR_NOMEM;
    for (int i = 0; i < num; i++) {
        const float *row = bank + (size_t)i * width;
        int first = -1, last = -1;
        for (int j = 0; j < width; j++) if (row[j] != 0.0f) { if (first < 0) first = j; last = j; }
        b->start[i] = first < 0 ? 0 : first;
        b->len[i] = first < 0 ? 0 : last - first + 1;
        b->nnz += b->len[i];
        if (b->len[i] > b->maxLen) b->maxLen = b->len[i];
    }
    return AF_OK;
}

void af_bands_free(AfBands *b) { free(b->start); free(b->len); b->start = b->len = NULL; }

/* ortho-normalised DCT-II rows: D[k][j] = s_k cos(pi (j + 1/2) k / N)
 * (reference: src/dsp/fft_algorithm.c:625-674, src/dsp/dct_algorithm.c:81-110, 170-181) */
void af_dct2_matrix(int num, int ccNum, float *out) {
    for (int k = 0; k < ccNum; k++) {
        double s = sqrt((k == 0 ? 1.0 : 2.0) / num);
        for (int j = 0; j < num; j++) out[(size_t)k * num + j] = (float)(s * cos(M_PI * (j + 0.5) * k / num));
    }
}

void af_fft_twiddles(int n, float *c, float *s) {
    for (int i = 0; i < n / 2; i++) { c[i] = (float)cos(2.0 * M_PI * i / n); s[i] = (float)-sin(2.0 * M_PI * i / n); }
}
