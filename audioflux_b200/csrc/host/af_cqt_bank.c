/* af_cqt_bank.c -- constant-Q kernels and the fixed /2 decimator taps (setup time, host).
 *
 * Behavioural spec:
 *   bin frequencies   src/filterbank/cqt_filterBank.c:159-184 (float32 running product:
 *                     the kernel phase 2*pi*j*f/sr reaches ~250 rad, so a 1-ulp change of f moves
 *                     kernel entries by ~2e-5 -- the float evaluation order is therefore kept)
 *   kernel lengths    :187-244      temporal kernels :253-336      spectral kernels + threshold :57-148
 *   object wiring     src/cqt_algorithm.c:1181-1265
 *   decimator         src/dsp/resample_algorithm.c:60-98 (quality Fast), :430-521, :546-634
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

/* in-place iterative radix-2 FFT in double (setup only; af_internal.h) */
void af_fft_double(double *re, double *im, int n) {
    for (int i = 1, j = 0; i < n; i++) {
        int bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) { double t = re[i]; re[i] = re[j]; re[j] = t; t = im[i]; im[i] = im[j]; im[j] = t; }
    }
    for (int len = 2; len <= n; len <<= 1) {
        double ang = -2.0 * M_PI / len;
        for (int i = 0; i < n; i += len)
            for (int k = 0; k < len / 2; k++) {
                double wr = cos(ang * k), wi = sin(ang * k);
                double ur = re[i + k], ui = im[i + k];
                double vr = re[i + k + len / 2] * wr - im[i + k + len / 2] * wi;
                double vi = re[i + k + len / 2] * wi + im[i + k + len / 2] * wr;
                re[i + k] = ur + vr; im[i + k] = ui + vi;
                re[i + k + len / 2] = ur - vr; im[i + k + len / 2] = ui - vi;
            }
    }
}

static int ceil_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }

int af_cqt_bank_build(AfCqtBank *b, int num, int samplate, float minFre, int bpo, float factor,
                      float beta, float thresh, int windowType, int normType) {
    memset(b, 0, sizeof(*b));
    const int octs = num / bpo;
    b->num = num; b->binPerOctave = bpo; b->octaveNum = octs; b->samplate = samplate;
    b->freBandArr = (float *)calloc((size_t)num + 2, sizeof(float));
    b->sLenArr = (float *)calloc((size_t)num, sizeof(float));
    if (!b->freBandArr || !b->sLenArr) return AF_ERR_NOMEM;

    float ratio = powf(2, 1.0 / bpo);
    for (int o = 0; o < octs; o++) {
        float f = minFre * (1 << o);
        b->freBandArr[o * bpo] = f;
        for (int j = 1; j < bpo; j++) { f *= ratio; b->freBandArr[o * bpo + j] = f; }
    }
    const float alpha = powf(2, 1.0 / bpo) - 1;
    const float q = factor / alpha;
    const float *top = b->freBandArr + (octs - 1) * bpo;
    int len0 = ceilf(q * samplate / (top[0] + beta / alpha));
    const int n = ceil_pow2(len0);
    b->fftLength = n;
    for (int i = 0; i < num; i++) b->sLenArr[i] = sqrtf(q * samplate / (b->freBandArr[i] + beta / alpha));

    /* beta != 0 (VQT, cqt_algorithm.c:186-193, 1208-1246): no sharing of the top octave's kernels -- every octave gets its
     * own `bpo` rows, built from its own float frequencies and the integer-halved sample rate, with the TOP octave's
     * kernel lengths (cqt_filterBank.c:57-124) */
    b->vqt = beta != 0;
    b->rows = b->vqt ? num : bpo;
    const int width = n / 2 + 1;
    b->kr = (float *)calloc((size_t)b->rows * width, sizeof(float));
    b->ki = (float *)calloc((size_t)b->rows * width, sizeof(float));
    double *re = (double *)malloc(sizeof(double) * n), *im = (double *)malloc(sizeof(double) * n);
    float *win = (float *)malloc(sizeof(float) * (n + 1));
    if (!b->kr || !b->ki || !re || !im || !win) { free(re); free(im); free(win); return AF_ERR_NOMEM; }
    if (windowType == Window_Rect) windowType = Window_Hann;
    const float thresh2 = thresh * thresh;
    int srOct = samplate;
    for (int oct = octs - 1; oct >= (b->vqt ? 0 : octs - 1); oct--, srOct /= 2)
    for (int i = 0; i < bpo; i++) {
        const float *fre = b->freBandArr + oct * bpo;
        const size_t row = b->vqt ? (size_t)oct * bpo + i : (size_t)i;
        const float lenF = q * samplate / (top[i] + beta / alpha);
        int len = ceilf(lenF);
        if (len > n) len = n;
        af_window_fft(windowType, len, win);
        memset(re, 0, sizeof(double) * n); memset(im, 0, sizeof(double) * n);
        const int st = (n - len) / 2;
        float area = 0;                                          /* float accumulation, like the reference */
        for (int j = 0; j < len; j++) {
            float phase = 2 * M_PI * j * fre[i] / srOct;        /* rounded to float like the reference */
            float w = (normType == SpectralFilterBankNormal_None) ? lenF : 1.0f;
            float tr = cosf(phase) * win[j] / w, ti = sinf(phase) * win[j] / w;
            re[st + j] = tr; im[st + j] = ti;
            area += sqrtf(tr * tr + ti * ti);
        }
        float div = 1.0f;
        if (normType == SpectralFilterBankNormal_Area) div = area;
        else if (normType == SpectralFilterBankNormal_BandWidth) {
            /* neighbours in the full list; the slot after the last bin is 0 (as in the reference) */
            int g = oct * bpo + i;
            float prev = g > 0 ? b->freBandArr[g - 1] : 0.0f;     /* (the reference reads one float before its array there) */
            div = (b->freBandArr[g + 1] - prev) / 2;
        }
        const float rescale = lenF / n;
        for (int j = 0; j < len; j++) {
            float tr = (float)re[st + j], ti = (float)im[st + j];
            if (normType != SpectralFilterBankNormal_None) { tr /= div; ti /= div; }
            re[st + j] = tr * rescale;
            im[st + j] = ti * rescale;
        }
        af_fft_double(re, im, n);
        for (int k = 0; k < width; k++) {
            float vr = (float)re[k], vi = (float)im[k];
            if (vr * vr + vi * vi > thresh2) { b->kr[row * width + k] = vr; b->ki[row * width + k] = vi; }
        }
    }
    free(re); free(im); free(win);
    return AF_OK;
}

void af_cqt_bank_free(AfCqtBank *b) {
    free(b->freBandArr); free(b->sLenArr); free(b->kr); free(b->ki);
    memset(b, 0, sizeof(*b));
}

/* kappa_b[n] = sum_{k=0}^{N/2} K_b[k] e^{-2 pi i k n / N}: the spectral dot sum_k X[k] K_b[k]
 * equals sum_n x[n] kappa_b[n] for a real frame x, which is what the device evaluates. */
int af_cqt_time_kernels(const AfCqtBank *b, float *kappaRe, float *kappaIm) {
    const int n = b->fftLength, width = n / 2 + 1;
    double *re = (double *)malloc(sizeof(double) * n), *im = (double *)malloc(sizeof(double) * n);
    if (!re || !im) { free(re); free(im); return AF_ERR_NOMEM; }
    for (int i = 0; i < b->rows; i++) {
        for (int k = 0; k < n; k++) {
            re[k] = k < width ? b->kr[(size_t)i * width + k] : 0.0;
            im[k] = k < width ? b->ki[(size_t)i * width + k] : 0.0;
        }
        af_fft_double(re, im, n);       /* forward DFT over k gives sum_k K[k] e^{-2 pi i k n/N} */
        for (int t = 0; t < n; t++) { kappaRe[(size_t)i * n + t] = (float)re[t]; kappaIm[(size_t)i * n + t] = (float)im[t]; }
    }
    free(re); free(im);
    return AF_OK;
}

/* Windowed-sinc table of the reference's "Fast" resampler (16 zero crossings x 512 samples,
 * Kaiser beta 8.5555046, roll-off 0.85) sampled for ratio 1/2: output i sits exactly on input 2i,
 * so the polyphase filter degenerates to fixed taps table[256*j].  The integer division
 * (tableLength - offset) / step gives 32 taps on the left (x[2i-j], j=0..31) and 31 on the right
 * (x[2i+1+j], j=0..30, table offset 256). */
void af_decimator_taps(float *left32, float *right31) {
    const int zeros = 16, per = 512, L = zeros * per + 1;
    const float beta = 8.5555046f, roll = 0.85f;
    double *win = (double *)malloc(sizeof(double) * (size_t)(2 * (L - 1) + 1));
    af_window_symmetric(Window_Kaiser, 2 * (L - 1) + 1, &beta, win);
    for (int j = 0; j < 32; j++) {
        for (int side = 0; side < 2; side++) {
            int idx = 256 * j + (side ? 256 : 0);
            if (side && j >= 31) continue;
            double t = (double)zeros * idx / (L - 1) * roll;
            double sinc = t == 0 ? 1.0 : sin(M_PI * t) / (M_PI * t);
            double v = sinc * roll * win[(L - 1) + idx] * 0.5;
            if (side) right31[j] = (float)v; else left32[j] = (float)v;
        }
    }
    free(win);
}

int afb200_decimatorTaps(float *left32, float *right31) {
    if (!left32 || !right31) return AF_ERR_ARG;
    af_decimator_taps(left32, right31);
    return AF_OK;
}

/* 0/1 folding matrix of CQT bins onto chroma classes, bank[num][cqtLength]
 * (chroma_cqtFilterBank, src/filterbank/chroma_filterBank.c:176-262).  With n = bpo/num bins per class, class 0
 * is centred on the first bin of every octave (ceil(n/2) bins from the octave start plus the last n-ceil(n/2) of
 * the octave), class i>0 takes the next n bins.  Rows are then rotated so that row 0 is pitch class C, using the
 * reference's folded MIDI index (values above 6 are mirrored) and its integer factor num/bpo. */
int af_chroma_cqt_bank(int num, int cqtLength, int bpo, float minFre, float *bank) {
    if (num < 1 || num > bpo || bpo % num != 0) return -1;
    const int n = bpo / num, offset = (int)ceilf(n / 2.0), sub = n - offset;
    float fmin = minFre > 0 ? minFre : 32.703196f;
    int midi = (int)roundf(12 * log2(fmin / 440) + 69);
    midi = midi % 12;
    if (midi > 6) midi = 12 - midi;
    const int shift = midi * (num / bpo);
    memset(bank, 0, sizeof(float) * (size_t)num * cqtLength);
    for (int k = 0; k < num; k++) {
        const int i = shift ? (k + shift) % num : k;          /* source class of output row k */
        const int start = i ? offset + (i - 1) * n : 0;
        for (int j = 0; j < cqtLength; j++) {
            const int mod = j % bpo;
            int hit;
            if (i) hit = mod >= start && mod < start + n;
            else hit = (mod >= 0 && mod < offset) || (sub && mod >= bpo - sub && mod < bpo);
            if (hit) bank[(size_t)k * cqtLength + j] = 1.0f;
        }
    }
    return 0;
}

int afb200_chromaCqtFilterBank(int num, int cqtLength, int binPerOctave, float minFre, float *bank) {
    if (!bank || cqtLength < 1) return af_fail(AF_ERR_ARG, "afb200_chromaCqtFilterBank: bad argument");
    if (af_chroma_cqt_bank(num, cqtLength, binPerOctave, minFre, bank))
        return af_fail(AF_ERR_ARG, "afb200_chromaCqtFilterBank: num=%d does not divide binPerOctave=%d", num, binPerOctave);
    return AF_OK;
}
