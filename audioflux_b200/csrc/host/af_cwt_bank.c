/* af_cwt_bank.c -- analytic wavelets in the frequency domain and the scale ladder (setup time, host).
 *
 * Behavioural spec: src/filterbank/cwt_filterBank.c:85-290 (scales, omega grid),
 * :361-640 (psi_hat of each family), src/cwt_algorithm.c:198-244 (family defaults).
 * The bank is a closed form in s*omega, so the device evaluates `af_wavelet_eval`'s twin on the
 * fly instead of reading a num x N table (176 MB per clip at N = 2^19).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

int af_wavelet_setup(AfWavelet *w, int type, const float *gamma, const float *beta) {
    float g = 3, b = 20;                                   /* Morse defaults */
    switch (type) {
    case WaveletContinue_Morse: break;
    case WaveletContinue_Morlet: g = 6; b = 2; break;
    case WaveletContinue_Bump: g = 5; b = 0.6f; break;
    case WaveletContinue_Paul: g = 4; break;
    case WaveletContinue_DOG: g = 2; b = 2; break;
    case WaveletContinue_Mexican: b = 2; break;
    case WaveletContinue_Hermit: g = 5; b = 2; break;
    case WaveletContinue_Ricker: g = 4; break;
    default: return AF_ERR_ARG;
    }
    if (gamma && *gamma > 0) {
        g = *gamma;
        if (type == WaveletContinue_DOG) { int p = (int)roundf(g); g = (p % 2 == 0) ? (float)p : 2.0f; }
    }
    if (beta && *beta > 0) b = *beta;
    w->waveletType = type; w->gamma = g; w->beta = b; w->factor = 1.0;
    switch (type) {
    case WaveletContinue_Morse:
        w->cf = expf(1.0 / g * (logf(b) - logf(g)));       /* peak frequency (beta/gamma)^(1/gamma) */
        w->factor = expf(-b * logf(w->cf) + powf(w->cf, g));
        break;
    case WaveletContinue_Morlet: case WaveletContinue_Bump: case WaveletContinue_Ricker: w->cf = g; break;
    case WaveletContinue_Paul: {
        w->cf = g + 0.5;
        int p = (int)roundf(g);
        long double prod = 1;
        for (int i = 2 * p - 1; i >= 2; i--) prod *= i;
        w->factor = (double)(powl(2, p) / sqrtl(p * prod));
    } break;
    case WaveletContinue_DOG: case WaveletContinue_Mexican: {
        float order = type == WaveletContinue_Mexican ? 2.0f : g;
        w->cf = sqrtf(order + 0.5);
        int p = (int)roundf(order);
        double f = -1.0 / sqrt(tgamma(p + 0.5));
        if ((p / 2) % 2 == 1) f = -f;
        w->factor = f;
        if (type == WaveletContinue_Mexican) w->gamma = 2.0f, w->cf = sqrtf(2 + 0.5);
    } break;
    case WaveletContinue_Hermit:
        w->cf = g + 1;
        w->factor = 2.0 / sqrtf(g) * pow(M_PI, -0.25);
        break;
    }
    if (type == WaveletContinue_Ricker) w->factor = 2.0 / sqrtf(M_PI);
    return AF_OK;
}

float af_wavelet_eval(const AfWavelet *w, float sw) {
    const float g = w->gamma, b = w->beta;
    if (w->waveletType == WaveletContinue_Bump) {
        float r = (sw - g) / b;
        if (!(fabsf(r) < 1 - 1e-6f)) return 0.0f;
        float v = 2 * M_E * expf(-1 / (1 - r * r));
        return isnan(v) ? 0.0f : v;
    }
    if (!(sw > 0)) return 0.0f;
    switch (w->waveletType) {
    case WaveletContinue_Morse: {
        float p = (g == 3) ? sw * sw * sw : powf(sw, g);
        return 2 * (float)w->factor * expf(b * logf(sw) - p);
    }
    case WaveletContinue_Morlet: return 2 * expf(-(sw - g) * (sw - g) / b);
    case WaveletContinue_Paul: return (float)(w->factor * pow(sw, g) * exp(-(double)sw));
    case WaveletContinue_DOG: case WaveletContinue_Mexican:
        return (float)(w->factor * pow(sw, g) * exp(-(double)sw * sw / b));
    case WaveletContinue_Hermit: {
        double d = (double)sw - g;
        return (float)(w->factor * d * (1 + d) * exp(-d * d / b));
    }
    case WaveletContinue_Ricker:
        return (float)(w->factor * (double)sw * sw / ((double)g * g * g) * exp(-(double)sw * sw / ((double)g * g)));
    }
    return 0.0f;
}

/* centre frequencies (low -> high), their bins, and scales s_i = cf / (2 pi f / sr) ordered
 * high -> low frequency (row 0 of the transform is the highest band). */
void af_cwt_scales(int num, int dataLength, int samplate, float lowFre, float highFre, int scale,
                   int bpo, float cf, float *freBandArr, int *binBandArr, float *scaleArr) {
    float *fre = (float *)calloc((size_t)num + 2, sizeof(float));
    int *bin = (int *)calloc((size_t)num + 2, sizeof(int));
    af_band_edges(num, dataLength, samplate, lowFre, highFre, scale, bpo, 0, 0, fre, bin);
    if (freBandArr) memcpy(freBandArr, fre + 1, sizeof(float) * (size_t)num);
    if (binBandArr) memcpy(binBandArr, bin + 1, sizeof(int) * (size_t)num);
    for (int i = num, j = 0; i >= 1; i--, j++) {
        float f = fre[i];
        if (f < 1e-6) f = 1e-6;
        scaleArr[j] = cf / (f / samplate * 2 * M_PI);
    }
    free(fre); free(bin);
}
