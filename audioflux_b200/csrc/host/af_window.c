/* af_window.c -- FFT analysis windows (setup time, host).
 *
 * Behavioural spec: src/dsp/flux_window.c:890-940 (`window_calFFTWindow`):
 * "periodic" = symmetric window of length n+1 with the last sample dropped, except
 * Bartlett / Triang / Bartlett-Hann / Bohman which stay symmetric.  Formulas are the textbook
 * ones, evaluated in double and rounded once to float (the reference evaluates in float; the
 * difference is < 2e-7 and is checked by tests/test_tables.py against oracle/_ref).
 */
#include <math.h>
#include <stdlib.h>
#include "../af_internal.h"

/* modified Bessel I0 by its power series truncated after 15 terms: the truncation is part of
 * the behaviour being reproduced (flux_window.c `__besselZeroOne`). */
static double bessel_i0_15(double a) {
    double half = 0.5 * a, term = 1.0, sum = 1.0;
    for (int k = 1; k < 16; k++) {
        term *= half / k;
        sum += term * term;
    }
    return sum;
}

static double cosine_sum(const double *a, int terms, double phase) {
    double s = 0.0, sign = 1.0;
    for (int t = 0; t < terms; t++) {
        s += sign * a[t] * cos(t * phase);
        sign = -sign;
    }
    return s;
}

int af_window_symmetric(int type, int L, const float *value, double *w) {
    if (L <= 0 || !w) return AF_ERR_ARG;
    if (L == 1) { w[0] = 1.0; return AF_OK; }
    const int M = L - 1;
    static const double hann[2] = {0.5, 0.5}, hamm[2] = {0.54, 0.46};
    static const double blackman[3] = {0.42, 0.5, 0.08};
    static const double flattop[5] = {0.21557895, 0.41663158, 0.277263158, 0.083578947, 0.006947368};
    static const double bharris[4] = {0.35875, 0.48829, 0.14128, 0.01168};
    static const double bnuttall[4] = {0.3635819, 0.4891775, 0.1365995, 0.0106411};
    for (int i = 0; i < L; i++) {
        const double x = (double)i / M;          /* 0..1 */
        const double ph = 2.0 * M_PI * x;
        double v = 1.0;
        switch (type) {
        case Window_Hann: v = cosine_sum(hann, 2, ph); break;
        case Window_Hamm: v = cosine_sum(hamm, 2, ph); break;
        case Window_Blackman: v = (i == 0 || i == M) ? 0.0 : cosine_sum(blackman, 3, ph); break;
        case Window_Flattop: v = cosine_sum(flattop, 5, ph); break;
        case Window_Blackman_Harris: v = cosine_sum(bharris, 4, ph); break;
        case Window_Blackman_Nuttall: v = cosine_sum(bnuttall, 4, ph); break;
        case Window_Kaiser: {
            double beta = (value && *value > 0) ? *value : 5.0;
            double r = 2.0 * x - 1.0, q = 1.0 - r * r;
            v = bessel_i0_15(beta * sqrt(q > 0 ? q : 0.0)) / bessel_i0_15(beta);
        } break;
        case Window_Gauss: {
            double alpha = (value && *value > 0) ? *value : 2.5;
            double r = alpha * (2.0 * x - 1.0);
            v = exp(-0.5 * r * r);
        } break;
        case Window_Bartlett: v = 1.0 - fabs(2.0 * x - 1.0); break;
        case Window_Triang: {
            /* peak never reaches the end points: even L -> (2k+1)/L, odd L -> 2(k+1)/(L+1) */
            int k = i < L - 1 - i ? i : L - 1 - i;
            v = (L % 2 == 0) ? (2.0 * k + 1.0) / L : 2.0 * (k + 1.0) / (L + 1.0);
        } break;
        case Window_Bartlett_Hann: {
            double r = x - 0.5;
            v = (i == 0 || i == M) ? 0.0 : 0.62 - 0.48 * fabs(r) + 0.38 * cos(2.0 * M_PI * r);
        } break;
        case Window_Bohman: {
            double r = fabs(2.0 * x - 1.0);
            v = (i == 0 || i == M) ? 0.0 : (1.0 - r) * cos(M_PI * r) + sin(M_PI * r) / M_PI;
        } break;
        case Window_Tukey: {
            double a = (value && *value >= 0 && *value <= 1) ? *value : 0.5;
            if (a <= 0) v = 1.0;
            else if (a >= 1) v = cosine_sum(hann, 2, ph);
            else if (x < a / 2) v = 0.5 * (1 + cos(2 * M_PI / a * (x - a / 2)));
            else if (x >= 1 - a / 2) v = 0.5 * (1 + cos(2 * M_PI / a * (x - 1 + a / 2)));
            else v = 1.0;
        } break;
        default: v = 1.0;
        }
        w[i] = v;
    }
    return AF_OK;
}

int af_window_fft(int type, int n, float *out) {
    if (n <= 0 || !out) return AF_ERR_ARG;
    if (type <= Window_Rect || type > Window_Tukey) {
        for (int i = 0; i < n; i++) out[i] = 1.0f;
        return AF_OK;
    }
    const int symmetric = (type == Window_Bartlett || type == Window_Triang ||
                           type == Window_Bartlett_Hann || type == Window_Bohman);
    const int L = symmetric ? n : n + 1;
    double *w = (double *)malloc(sizeof(double) * (size_t)L);
    if (!w) return AF_ERR_NOMEM;
    af_window_symmetric(type, L, NULL, w);
    for (int i = 0; i < n; i++) out[i] = (float)w[i];
    free(w);
    return AF_OK;
}

int afb200_window(int windowType, int length, float *out) { return af_window_fft(windowType, length, out); }
