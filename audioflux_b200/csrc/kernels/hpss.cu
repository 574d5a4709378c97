// hpss.cu -- the masks of harmonic-percussive separation (sm_90a), the middle step of hpssObj_hpss
// (src/mir/hpss_algorithm.c:192-326) between the forward STFT and the two inverse STFTs.
//
// k_hpss_mask: one CTA per tile of kTT frames x kKB bins of one clip (grid.x = clips x frame tiles, grid.y = bin tiles).
// Per bin: mag = sqrtf(re^2 + im^2); mH = the median of mag over hOrder frames of the same bin, mP = the median over
// pOrder bins of the same frame, both windows centred, with zeros beyond the clip's first and last frame and beyond
// bins 0 and W-1; then h1 = mH^2, p1 = mP^2, v = max(h1 + p1, 1e-16), H = h1 / v * mag, P = p1 / v * mag, each times
// the unit phase (re, im) / max(mag, 1e-16).  That is the reference's float order; the file is compiled with
// -fmad=false so that no multiply-add is contracted.  An order of 1 gives a median of 0 (the reference never runs its
// filter then and reads the zeros its buffer was allocated with).
//
// The medians cost O(order) per output, not a rank count over the window (O(order^2)).  A thread walks a run of
// consecutive outputs along one axis.  It finds the first window's median by rank counts, and from then on uses that
// one removal and one insertion move the median by at most one place in sorted order: one pass over the new window
// counts the values below and not above the old median m and finds the nearest values above and below it, and the new
// median is m, the nearest value above or the nearest value below.  The windows are read from shared memory:
//   1. the frequency strip: the tile's kTT frames, bins k0 - pOrder/2 .. k0 + kKB + pOrder/2 (row pitch odd, so that
//      the 32 lanes of a warp, one frame each, read 32 banks), where each warp walks kKB/4 bins of 32 frames; mP goes to
//      its own tile in shared memory;
//   2. the time strip, in the same buffer: frames t0 - hOrder/2 .. t0 + kTT + hOrder/2, the tile's kKB bins, where each
//      thread walks the kTT frames of one bin, then forms H and P from the strip's centre row, mP and the phase, and
//      writes them (each warp: 32 consecutive bins of one frame).
#include "common.cuh"

namespace {

constexpr int kKB = 128;                     // bins per tile = threads per CTA
constexpr int kTT = 32;                      // frames per tile = lanes of a warp
constexpr int kRun = kKB / (kKB / 32);       // bins walked by one thread of the frequency pass
static_assert(kKB % 32 == 0 && kRun * (kKB / 32) == kKB, "tile shape");

struct HpssParams {
    const float *re, *im;                    // [clips * T][W]
    float *hRe, *hIm, *pRe, *pIm;            // same layout; hRe == nullptr: no H, pRe == nullptr: no P
    int T, W, frameTiles;
    int hh, ph;                              // hOrder / 2, pOrder / 2
    int zeroH, zeroP;                        // order 1: that median is 0
    int pitch2;                              // row pitch of the frequency strip (odd)
};

__device__ __forceinline__ float mag_of(float r, float i) { return sqrtf(r * r + i * i); }

// median of the K = 2h + 1 values w[0], w[s], ..., w[(K-1) s]: the value with at most h values below it and more than h
// values not above it
__device__ float median_first(const float *w, int s, int K, int h) {
    for (int i = 0; i < K; i++) {
        const float v = w[i * s];
        int lt = 0, le = 0;
        for (int j = 0; j < K; j++) {
            const float x = w[j * s];
            lt += x < v;
            le += x <= v;
        }
        if (lt <= h && h < le) return v;
    }
    return 0.0f;                              // only NaN input gets here
}

// median of the window after it moved by one place, from the previous median m
__device__ __forceinline__ float median_next(const float *w, int s, int K, int h, float m) {
    int lt = 0, le = 0;
    float above = __int_as_float(0x7f800000), below = -1.0f;   // values are >= 0
    for (int j = 0; j < K; j++) {
        const float x = w[j * s];
        lt += x < m;
        le += x <= m;
        above = fminf(above, x > m ? x : __int_as_float(0x7f800000));
        below = fmaxf(below, x < m ? x : -1.0f);
    }
    return lt > h ? below : le <= h ? above : m;
}

__global__ void __launch_bounds__(kKB) k_hpss_mask(HpssParams p) {
    extern __shared__ float smem[];
    const int clip = blockIdx.x / p.frameTiles;
    const int t0 = (blockIdx.x - clip * p.frameTiles) * kTT, k0 = blockIdx.y * kKB;
    const int tid = threadIdx.x;
    const int nT = min(kTT, p.T - t0), nK = min(kKB, p.W - k0);
    const long long row0 = (long long)clip * p.T;
    float *strip = smem;
    float *mp = smem + max((kTT + 2 * p.hh) * kKB, kTT * p.pitch2);    // [kTT][kKB + 1]

    // 1. frequency medians
    if (!p.zeroP) {
        const int width = kKB + 2 * p.ph;
        for (int e = tid; e < kTT * width; e += kKB) {
            const int r = e / width, c = e - r * width, k = k0 - p.ph + c;
            float v = 0.0f;
            if (r < nT && k >= 0 && k < p.W) {
                const long long g = (row0 + t0 + r) * p.W + k;
                v = mag_of(p.re[g], p.im[g]);
            }
            strip[r * p.pitch2 + c] = v;
        }
        __syncthreads();
        const int r = tid & 31, c0 = (tid >> 5) * kRun, c1 = min(c0 + kRun, nK), K = 2 * p.ph + 1;
        if (r < nT && c0 < c1) {
            const float *w = strip + r * p.pitch2 + c0;
            float m = median_first(w, 1, K, p.ph);
            mp[r * (kKB + 1) + c0] = m;
            for (int c = c0 + 1; c < c1; c++) {
                m = median_next(strip + r * p.pitch2 + c, 1, K, p.ph, m);
                mp[r * (kKB + 1) + c] = m;
            }
        }
        __syncthreads();
    }

    // 2. time medians, masks and outputs
    const int rows = kTT + 2 * p.hh;
    for (int e = tid; e < rows * kKB; e += kKB) {
        const int r = e / kKB, c = e - r * kKB, t = t0 - p.hh + r;
        float v = 0.0f;
        if (t >= 0 && t < p.T && c < nK) {
            const long long g = (row0 + t) * p.W + k0 + c;
            v = mag_of(p.re[g], p.im[g]);
        }
        strip[e] = v;
    }
    __syncthreads();
    if (tid >= nK) return;
    const int K = 2 * p.hh + 1;
    float m = 0.0f;
    for (int t = 0; t < nT; t++) {
        if (!p.zeroH) m = t == 0 ? median_first(strip + tid, kKB, K, p.hh) : median_next(strip + t * kKB + tid, kKB, K, p.hh, m);
        const float mag = strip[(t + p.hh) * kKB + tid];
        const float mP = p.zeroP ? 0.0f : mp[t * (kKB + 1) + tid];
        const long long g = (row0 + t0 + t) * p.W + k0 + tid;
        const float d = mag < 1e-16f ? 1e-16f : mag;
        const float ur = p.re[g] / d, ui = p.im[g] / d;
        const float h1 = m * m, p1 = mP * mP;
        float v = h1 + p1;
        if (v < 1e-16f) v = 1e-16f;
        if (p.hRe) {
            const float a = h1 / v * mag;
            p.hRe[g] = ur * a;
            p.hIm[g] = ui * a;
        }
        if (p.pRe) {
            const float a = p1 / v * mag;
            p.pRe[g] = ur * a;
            p.pIm[g] = ui * a;
        }
    }
}

}  // namespace

static size_t hpss_smem_bytes(int hOrder, int pOrder) {
    const int hh = hOrder / 2, pitch2 = (kKB + 2 * (pOrder / 2)) | 1;
    const int strip = (kTT + 2 * hh) * kKB > kTT * pitch2 ? (kTT + 2 * hh) * kKB : kTT * pitch2;
    return sizeof(float) * ((size_t)strip + (size_t)kTT * (kKB + 1));
}

extern "C" int af_launch_hpss_mask(const AfHpssArgs *a, void *stream) {
    if (a->clips <= 0 || a->timeLength <= 0) return AF_OK;
    if (a->hOrder < 1 || a->pOrder < 1 || !(a->hOrder & 1) || !(a->pOrder & 1) || a->hOrder > AFB200_HPSS_MAX_ORDER ||
        a->pOrder > AFB200_HPSS_MAX_ORDER)
        return af_fail(AF_ERR_ARG, "hpss mask: orders %d / %d; odd orders 1 .. %d are supported", a->hOrder, a->pOrder,
                       AFB200_HPSS_MAX_ORDER);
    if (!a->hRe && !a->pRe) return af_fail(AF_ERR_ARG, "hpss mask: no output (hRe and pRe are both NULL)");
    HpssParams p;
    p.re = a->re; p.im = a->im;
    p.hRe = a->hRe; p.hIm = a->hIm; p.pRe = a->pRe; p.pIm = a->pIm;
    p.T = a->timeLength; p.W = a->width;
    p.frameTiles = (a->timeLength + kTT - 1) / kTT;
    p.hh = a->hOrder / 2; p.ph = a->pOrder / 2;
    p.zeroH = a->hOrder == 1; p.zeroP = a->pOrder == 1;
    p.pitch2 = (kKB + 2 * p.ph) | 1;
    const long long gx = (long long)a->clips * p.frameTiles;
    const int gy = (a->width + kKB - 1) / kKB;
    if (gx > 0x7fffffffLL || gy > 65535) return af_fail(AF_ERR_ARG, "hpss mask: too many tiles in one launch");
    const size_t smem = hpss_smem_bytes(a->hOrder, a->pOrder);
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = af_smem_optin(k_hpss_mask, smem, "k_hpss_mask");
    if (rc) return rc;
    k_hpss_mask<<<dim3((unsigned)gx, (unsigned)gy), kKB, smem, st>>>(p);
    AF_LAUNCH_CHECK("k_hpss_mask");
    return AF_OK;
}
