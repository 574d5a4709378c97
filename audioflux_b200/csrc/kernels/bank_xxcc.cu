// bank_xxcc.cu -- filter-bank contraction and cepstral (rectify + DCT-II) kernels, general path.
//
// Replaces the reference's `__mdot1` / `__mcdot1` contractions of bftObj_bft
// (src/bft_algorithm.c:481-485, 515-518; src/vector/flux_vector.c:55-86) and the rectify + per-frame
// DCT loop of xxccObj_xxcc (src/feature/xxcc_algorithm.c:124-155).
//
// Slaney/ETSI banks are banded (2019 non-zeros of 131 200 at n=2048, num=128), so the banded kernel
// walks only each filter's support; dense banks (gammatone-like) use a tiled FP32 contraction.
#include <math.h>
#include "common.cuh"

namespace {

// one warp per row; lane m walks the support of filters m, m+32, ... (fixed order -> bit-stable)
__global__ void k_bank_banded(const float *__restrict__ in, long long rows, int width, int num,
                              const int *__restrict__ start, const int *__restrict__ len,
                              const float *__restrict__ packed, const int *__restrict__ off,
                              float postPow, float *__restrict__ out) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float *x = in + row * width;
    for (int m = lane; m < num; m += 32) {
        const int s = start[m], l = len[m];
        const float *w = packed + off[m];
        float acc = 0.0f;
        for (int i = 0; i < l; i++) acc = fmaf(x[s + i], w[i], acc);
        if (postPow != 1.0f) acc = powf(acc, postPow);
        out[row * num + m] = acc;
    }
}

// out[r][m] = sum_k in[r][k] * bank[m][k]; 64x64 output tile, K-slab 16, 4x4 register micro-tile
__global__ void __launch_bounds__(256) k_bank_dense(const float *__restrict__ in, long long rows, int width, int num,
                                                    const float *__restrict__ bank, float postPow,
                                                    float *__restrict__ out) {
    __shared__ float sa[16][64 + 1], sb[16][64 + 1];
    const long long r0 = (long long)blockIdx.x * 64;
    const int m0 = blockIdx.y * 64;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < width; k0 += 16) {
        for (int e = threadIdx.x; e < 64 * 16; e += 256) {
            int rr = e >> 4, kk = e & 15;
            long long r = r0 + rr; int k = k0 + kk;
            sa[kk][rr] = (r < rows && k < width) ? in[r * width + k] : 0.0f;
            int m = m0 + rr;
            sb[kk][rr] = (m < num && k < width) ? bank[(long long)m * width + k] : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; kk++) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { a[i] = sa[kk][ty * 4 + i]; b[i] = sb[kk][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            long long r = r0 + ty * 4 + i; int m = m0 + tx * 4 + j;
            if (r < rows && m < num) {
                float v = acc[i][j];
                if (postPow != 1.0f) v = powf(v, postPow);
                out[r * num + m] = v;
            }
        }
}

__global__ void k_copy_cols(const float *__restrict__ in, long long rows, int width, int lo, int count,
                            float *__restrict__ out) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * count) return;
    long long r = i / count; int c = (int)(i % count);
    out[i] = in[r * width + lo + c];
}

// one warp per row: rectify into shared memory, then lane c accumulates coefficient c, c+32, ...
// dctT is the transposed ortho DCT-II matrix [num][ccStride] so lanes read consecutive floats.
__global__ void k_xxcc(const float *__restrict__ in, long long rows, int num, int ccNum, int rectify,
                       const float *__restrict__ dctT, int ccStride, float *__restrict__ out) {
    extern __shared__ float sh[];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + wib;
    if (row >= rows) return;
    float *l = sh + (size_t)wib * num;
    for (int m = lane; m < num; m += 32) {
        float v = in[row * num + m];
        if (rectify == CepstralRectify_CubicRoot) v = powf(v, 1.0f / 3.0f);
        else v = log10f(v < 1e-8f ? 1e-8f : v);
        l[m] = v;
    }
    __syncwarp();
    for (int c = lane; c < ccNum; c += 32) {
        float acc = 0.0f;
        for (int m = 0; m < num; m++) acc = fmaf(l[m], dctT[(size_t)m * ccStride + c], acc);
        out[row * ccNum + c] = acc;
    }
}

// xxccObj_xxccStandard (src/feature/xxcc_algorithm.c:168-296): cepstra, then log-energy replace / append, then
// the reference's delta and delta-delta: a causal `order`-tap FIR b[j] = (m - j) / sum_{i<=m} i^2 run ALONG THE
// COEFFICIENT AXIS of each frame (util_delta, src/util/flux_util.c:803-815; filterDesign_filter,
// src/dsp/filterDesign_fir.c:229-248).  One warp per frame.
__global__ void k_xxcc_standard(const float *__restrict__ in, const float *__restrict__ energy, long long rows,
                                int num, int ccNum, int rectify, int energyType, int order,
                                const float *__restrict__ dctT, int ccStride,
                                float *__restrict__ coe, float *__restrict__ d1, float *__restrict__ d2) {
    extern __shared__ float sh[];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + wib;
    if (row >= rows) return;
    const int W = ccNum + (energyType == CepstralEnergy_Append ? 1 : 0);
    float *l = sh + (size_t)wib * (num + 2 * (num + 1));
    float *c0 = l + num, *c1 = c0 + (num + 1);
    for (int m = lane; m < num; m += 32) {
        float v = in[row * num + m];
        if (rectify == CepstralRectify_CubicRoot) v = powf(v, 1.0f / 3.0f);
        else v = log10f(v < 1e-8f ? 1e-8f : v);
        l[m] = v;
    }
    __syncwarp();
    float e = 0.0f;
    if (energyType != CepstralEnergy_Ignore) {
        e = energy[row];
        e = logf(e < 1e-8f ? 1e-8f : e);
    }
    for (int c = lane; c < ccNum; c += 32) {
        float acc = 0.0f;
        for (int m = 0; m < num; m++) acc = fmaf(l[m], dctT[(size_t)m * ccStride + c], acc);
        if (energyType == CepstralEnergy_Replace) c0[c] = c ? acc : e;
        else if (energyType == CepstralEnergy_Append) { c0[c + 1] = acc; if (!c) c0[0] = e; }
        else c0[c] = acc;
    }
    __syncwarp();
    const int half = order / 2;
    float v1 = 0.0f;
    for (int i = 1; i <= half; i++) v1 += (float)(i * i);
    for (int i = lane; i < W; i += 32) {
        float acc = 0.0f;
        for (int j = 0; j < order && j <= i; j++) acc = acc + ((float)(half - j) / v1) * c0[i - j];
        c1[i] = acc;
        coe[row * W + i] = c0[i];
        d1[row * W + i] = acc;
    }
    __syncwarp();
    for (int i = lane; i < W; i += 32) {
        float acc = 0.0f;
        for (int j = 0; j < order && j <= i; j++) acc = acc + ((float)(half - j) / v1) * c1[i - j];
        d2[row * W + i] = acc;
    }
}

// cqtObj_chroma (src/cqt_algorithm.c:484-600): |z|^2 or |z| of each CQT bin, folded onto chroma classes by a 0/1
// bank [chromaNum][num] (chroma_cqtFilterBank), then per-frame normalisation by max / min / L1 / L2 of |.|
// (__mnormalize axis 1, src/vector/flux_vector.c:1058-1150; a zero norm leaves the row as it is).  Warp per frame.
__global__ void k_chroma(const float *__restrict__ re, const float *__restrict__ im, long long rows, int num,
                         int chromaNum, int isMag, int normType, const float *__restrict__ bank,
                         float *__restrict__ out) {
    extern __shared__ float sh[];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + wib;
    if (row >= rows) return;
    float *sv = sh + (size_t)wib * (num + chromaNum), *cv = sv + num;
    for (int j = lane; j < num; j += 32) {
        const float a = re[row * num + j], b = im[row * num + j];
        float v = a * a + b * b;
        if (isMag) v = sqrtf(v);
        sv[j] = v;
    }
    __syncwarp();
    float red = 0.0f;
    int first = 1;
    for (int c = lane; c < chromaNum; c += 32) {
        double acc = 0.0;
        for (int j = 0; j < num; j++) acc += (double)sv[j] * (double)bank[c * num + j];
        const float v = (float)acc, a = fabsf(v);
        cv[c] = v;
        if (normType == ChromaDataNormal_Max) red = first ? a : fmaxf(red, a);
        else if (normType == ChromaDataNormal_Min) red = first ? a : fminf(red, a);
        else if (normType == ChromaDataNormal_P2) red += a * a;
        else red += a;
        first = 0;
    }
    if (first) red = (normType == ChromaDataNormal_Min) ? INFINITY : 0.0f;      /* lanes without a class */
    for (int o = 16; o > 0; o >>= 1) {
        const float other = __shfl_xor_sync(0xffffffffu, red, o);
        if (normType == ChromaDataNormal_Max) red = fmaxf(red, other);
        else if (normType == ChromaDataNormal_Min) red = fminf(red, other);
        else red += other;
    }
    if (normType == ChromaDataNormal_P2) red = sqrtf(red);
    __syncwarp();
    for (int c = lane; c < chromaNum; c += 32) {
        float v = cv[c];
        if (normType != ChromaDataNormal_None && red != 0.0f) v = v / red;
        out[row * chromaNum + c] = v;
    }
}

// spectrogramObj_spectrogram's Linear-scale phase (src/spectrogram_algorithm.c:1040-1056): the real part is
// clamped from below at 1e-16 BEFORE atan2f, so every bin with a negative real part reports +-pi/2.
__global__ void k_phase(const float *__restrict__ re, const float *__restrict__ im, long long rows, int width,
                        int lo, int count, float *__restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * count) return;
    const long long r = i / count;
    const int k = (int)(i - r * count) + lo;
    float a = re[r * width + k];
    if (a < 1e-16f) a = 1e-16f;
    out[i] = atan2f(im[r * width + k], a);
}

// spectrum planes -> what the bank consumes (bft_algorithm.c:456-497), in place: SQUARE (re, im) <- z^2; POWER re <- |z|^2
// (optionally ^normValue); MAG re <- |z|.  Used after the reassignment scatter (the STFT kernel fuses this step itself).
__global__ void k_spec_post(float *__restrict__ re, float *__restrict__ im, long long cells, int mode, float normValue) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cells) return;
    const float a = re[i], b = im[i];
    if (mode == AF_STFT_SQUARE) { re[i] = a * a - b * b; im[i] = 2.0f * a * b; return; }
    float v = a * a + b * b;
    if (mode == AF_STFT_MAG) v = sqrtf(v);
    else if (normValue != 1.0f) v = powf(v, normValue);
    re[i] = v;
}

// temporal descriptors of the windowed frames (src/temporal_algorithm.c:93-146): energy sum v^2, rms sqrt(E / n) and the
// zero-crossing rate #{v[i] v[i-1] < 0} / n, v = x . w.  One warp per frame.
__global__ void __launch_bounds__(256) k_temporal(const float *__restrict__ data, int n, int hop, int T, const float *__restrict__ window,
                                                  float *__restrict__ e, float *__restrict__ r, float *__restrict__ z) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (t >= T) return;
    const float *x = data + (size_t)t * hop;
    float acc = 0.0f;
    int cross = 0;
    for (int i = lane; i < n; i += 32) {
        const float v = x[i] * window[i];
        acc += v * v;
        if (i > 0 && v * (x[i - 1] * window[i - 1]) < 0.0f) cross++;
    }
    for (int o = 16; o; o >>= 1) { acc += __shfl_xor_sync(0xffffffffu, acc, o); cross += __shfl_xor_sync(0xffffffffu, cross, o); }
    if (lane == 0) { e[t] = acc; r[t] = sqrtf(acc / (float)n); z[t] = (float)(1.0 * cross / n); }
}

}  // namespace

extern "C" int af_launch_bank(const AfBankDev *bank, const float *in, int rows, float postPow, float *out, void *stream) {
    if (rows <= 0) return AF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (bank->banded) {
        const int warps = 8;
        k_bank_banded<<<(unsigned)((rows + warps - 1) / warps), warps * 32, 0, st>>>(
            in, rows, bank->width, bank->num, bank->start, bank->len, bank->packed, bank->packedOff, postPow, out);
        AF_LAUNCH_CHECK("k_bank_banded");
    } else {
        dim3 grid((unsigned)((rows + 63) / 64), (unsigned)((bank->num + 63) / 64));
        k_bank_dense<<<grid, 256, 0, st>>>(in, rows, bank->width, bank->num, bank->dense, postPow, out);
        AF_LAUNCH_CHECK("k_bank_dense");
    }
    return AF_OK;
}

extern "C" int af_launch_copy_cols(const float *in, int rows, int width, int lo, int count, float *out, void *stream) {
    long long total = (long long)rows * count;
    if (total <= 0) return AF_OK;
    k_copy_cols<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(in, rows, width, lo, count, out);
    AF_LAUNCH_CHECK("k_copy_cols");
    return AF_OK;
}

// warps (rows) per CTA of the warp-per-row cepstral kernels: `most` while they fit the default 48 KB of shared memory,
// else as many as fit the 227 KB opt-in; 0 when one row does not fit.  Each row is computed by its own warp in the same
// order whatever the CTA size, so the size only changes how many rows share an SM.
static int xxcc_warps(size_t perWarp, int most) {
    if (perWarp * most <= 48 * 1024) return most;
    const size_t fit = (size_t)227 * 1024 / perWarp;
    return fit < (size_t)most ? (int)fit : most;
}

extern "C" int af_launch_xxcc(const float *in, int rows, int num, int ccNum, int rectifyType, const float *dctT,
                              float *out, void *stream) {
    if (rows <= 0) return AF_OK;
    const int warps = xxcc_warps(sizeof(float) * (size_t)num, 8);
    if (!warps) return af_fail(AF_ERR_UNSUPPORTED, "xxcc: num=%d too large (one row must fit 227 KB of shared memory)", num);
    const size_t smem = sizeof(float) * (size_t)warps * num;
    const int rc = af_smem_optin(k_xxcc, smem, "k_xxcc");
    if (rc) return rc;
    k_xxcc<<<(unsigned)((rows + warps - 1) / warps), warps * 32, smem, (cudaStream_t)stream>>>(
        in, rows, num, ccNum, rectifyType, dctT, num, out);
    AF_LAUNCH_CHECK("k_xxcc");
    return AF_OK;
}

extern "C" int af_launch_xxcc_standard(const float *in, const float *energy, int rows, int num, int ccNum,
                                       int rectifyType, int energyType, int order, const float *dctT,
                                       float *coe, float *d1, float *d2, void *stream) {
    if (rows <= 0) return AF_OK;
    const size_t perWarp = sizeof(float) * ((size_t)num + 2 * ((size_t)num + 1));
    const int warps = xxcc_warps(perWarp, 4);
    if (!warps) return af_fail(AF_ERR_UNSUPPORTED, "xxccStandard: num=%d too large (one row must fit 227 KB of shared memory)", num);
    const size_t smem = perWarp * warps;
    const int rc = af_smem_optin(k_xxcc_standard, smem, "k_xxcc_standard");
    if (rc) return rc;
    k_xxcc_standard<<<(unsigned)((rows + warps - 1) / warps), warps * 32, smem, (cudaStream_t)stream>>>(
        in, energy, rows, num, ccNum, rectifyType, energyType, order, dctT, num, coe, d1, d2);
    AF_LAUNCH_CHECK("k_xxcc_standard");
    return AF_OK;
}

extern "C" int af_launch_chroma(const float *re, const float *im, int rows, int num, int chromaNum, int isMag,
                                int normType, const float *bank, float *out, void *stream) {
    if (rows <= 0) return AF_OK;
    const int warps = 8;
    size_t smem = sizeof(float) * (size_t)warps * (num + chromaNum);
    if (smem > 48 * 1024) return af_fail(AF_ERR_UNSUPPORTED, "chroma: num=%d too large", num);
    k_chroma<<<(unsigned)((rows + warps - 1) / warps), warps * 32, smem, (cudaStream_t)stream>>>(
        re, im, rows, num, chromaNum, isMag, normType, bank, out);
    AF_LAUNCH_CHECK("k_chroma");
    return AF_OK;
}

extern "C" int af_launch_phase(const float *re, const float *im, int rows, int width, int lo, int count, float *out, void *stream) {
    long long total = (long long)rows * count;
    if (total <= 0) return AF_OK;
    k_phase<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(re, im, rows, width, lo, count, out);
    AF_LAUNCH_CHECK("k_phase");
    return AF_OK;
}

extern "C" int af_launch_spec_post(float *re, float *im, long long cells, int mode, float normValue, void *stream) {
    if (cells <= 0 || mode == AF_STFT_HALF) return AF_OK;
    k_spec_post<<<(unsigned)((cells + 255) / 256), 256, 0, (cudaStream_t)stream>>>(re, im, cells, mode, normValue);
    AF_LAUNCH_CHECK("k_spec_post");
    return AF_OK;
}

extern "C" int af_launch_temporal(const float *data, int fftLength, int slideLength, int timeLength, const float *window,
                                  float *energy, float *rms, float *zcr, void *stream) {
    if (timeLength <= 0) return AF_OK;
    k_temporal<<<(unsigned)((timeLength + 7) / 8), 256, 0, (cudaStream_t)stream>>>(data, fftLength, slideLength, timeLength, window, energy, rms, zcr);
    AF_LAUNCH_CHECK("k_temporal");
    return AF_OK;
}
