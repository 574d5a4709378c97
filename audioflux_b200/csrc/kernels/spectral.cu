// spectral.cu -- spectral descriptors of time-major spectrograms (src/flux_spectral.c, src/feature/spectral_algorithm.c).
//
// k_spectral computes every request of one spectralObj_spectralBatch call in one launch.  A CTA owns a tile of TILE
// consecutive frames of ONE clip; each of its warps takes one frame at a time.  Temporal features read the rows
// t-step, t-1 and t-2 of the same clip (never of the previous clip) through L1/L2, right behind the warps that brought
// them in, so HBM sees each row about once.
//   pass 1: the sums that need only the row: sum x, sum f x, the double sum of logf(x+2e-16), max / first argmax,
//           hfc, rms, sum x^2, decrease;
//   pass 2: what needs the pass-1 scalars: the moments about the centroid (spread, skewness, kurtosis), entropy,
//           slope and var;
//   then one loop per parameterised request (flux / sd / sf / novelty / mkl / broadband / pd / cd / log energy /
//   bandWidth) and rolloff, whose two float sums are sequential in list order on one lane as in the reference (a tree
//   sum can move the crossing by one bin).
// The file is compiled with -fmad=false: the reference is gcc -O3 without contraction, and rolloff / max / the counts of
// broadband and novelty are integer outcomes of float comparisons.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int WARPS = 8;
constexpr int TILE = 32;   // frames per CTA
constexpr int UNROLL = 4;  // pass-1 loads in flight per lane
constexpr unsigned FULL = 0xffffffffu;

enum : unsigned {
    N_SUM = 1u << 0, N_SF = 1u << 1, N_LOG = 1u << 2, N_MAX = 1u << 3, N_HFC = 1u << 4, N_RMS = 1u << 5,
    N_E2 = 1u << 6, N_DEC = 1u << 7, N_MOM = 1u << 8, N_ENT = 1u << 9, N_SLOPE = 1u << 10, N_VAR = 1u << 11,
    N_SEQ = 1u << 12,
};

__device__ unsigned needs_of(int f) {
    switch (f) {
    case AFB200_SPECTRAL_FLATNESS: return N_SUM | N_LOG;
    case AFB200_SPECTRAL_ROLLOFF: return N_SEQ;
    case AFB200_SPECTRAL_CENTROID: return N_SUM | N_SF;
    case AFB200_SPECTRAL_SPREAD: case AFB200_SPECTRAL_SKEWNESS: case AFB200_SPECTRAL_KURTOSIS: return N_SUM | N_SF | N_MOM;
    case AFB200_SPECTRAL_ENTROPY: return N_SUM | N_ENT;
    case AFB200_SPECTRAL_CREST: return N_SUM | N_MAX;
    case AFB200_SPECTRAL_SLOPE: return N_SUM | N_SLOPE;
    case AFB200_SPECTRAL_DECREASE: return N_SUM | N_DEC;
    case AFB200_SPECTRAL_BANDWIDTH: return N_SUM | N_SF;
    case AFB200_SPECTRAL_RMS: return N_RMS;
    case AFB200_SPECTRAL_HFC: return N_HFC;
    case AFB200_SPECTRAL_EEF: case AFB200_SPECTRAL_EER: return N_SUM | N_ENT | N_E2;
    case AFB200_SPECTRAL_MAX: return N_MAX;
    case AFB200_SPECTRAL_MEAN: return N_SUM;
    case AFB200_SPECTRAL_VAR: return N_SUM | N_VAR;
    default: return 0;
    }
}

__device__ __forceinline__ float wsum(float v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ double wsumd(double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ int bin_of(const AfSpectralArgs &a, int j) { return a.idx ? __ldg(a.idx + j) : a.start + j; }

// the reference's row sum (spectral_algorithm.c:975-983): float, in list order
__device__ float seq_sum(const AfSpectralArgs &a, const float *row) {
    float s = 0.f;
    for (int j = 0; j < a.nb; j++) s += __ldg(row + bin_of(a, j));
    return s;
}
// flux_spectral.c:116-142: first bin at which the running sum of |x| reaches m1, -1 when none does
__device__ int seq_cross(const AfSpectralArgs &a, const float *row, float m1) {
    float n1 = 0.f;
    for (int j = 0; j < a.nb; j++) {
        const int k = bin_of(a, j);
        n1 += fabsf(__ldg(row + k));
        if (n1 >= m1) return k;
    }
    return -1;
}

// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(WARPS * 32) k_spectral(const __grid_constant__ AfSpectralArgs a) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tilesPerClip = (a.T + TILE - 1) / TILE;
    const int b = blockIdx.x / tilesPerClip, t0 = (blockIdx.x % tilesPerClip) * TILE;
    const size_t num = (size_t)a.num;
    const float *clip = a.spec + (size_t)b * a.T * num;
    const float *pclip = a.phase ? a.phase + (size_t)b * a.T * num : nullptr;
    const size_t BT = (size_t)a.batch * a.T;
    const int nb = a.nb;
    const float fnb = (float)nb;

    unsigned need = 0;
    for (int r = 0; r < a.nReq; r++) need |= needs_of(a.req[r]);

    for (int t = t0 + warp; t < t0 + TILE && t < a.T; t += WARPS) {
        const float *x = clip + (size_t)t * num;
        const size_t o = (size_t)b * a.T + t;
        auto put = [&](int plane, float v) { if (lane == 0) a.out[(size_t)plane * BT + o] = v; };

        // ---- pass 1
        float S = 0.f, SF = 0.f, hfc = 0.f, rms = 0.f, e2 = 0.f, dec = 0.f, bv = 0.f;
        double L = 0.0;
        int bj = -1;
        const float x0 = __ldg(x + bin_of(a, 0));
        for (int j0 = lane; j0 < nb; j0 += 32 * UNROLL) {
          // the loads of UNROLL list positions go out together (memory-level parallelism), then the lane folds them
          // in increasing position order (the argmax tie rule needs that order within a lane)
          int kk[UNROLL];
          float vv[UNROLL];
#pragma unroll
          for (int u = 0; u < UNROLL; u++) {
              const int j = j0 + 32 * u;
              kk[u] = j < nb ? bin_of(a, j) : 0;
              vv[u] = j < nb ? __ldg(x + kk[u]) : 0.f;
          }
#pragma unroll
          for (int u = 0; u < UNROLL; u++) {
            const int j = j0 + 32 * u;
            if (j >= nb) break;
            const int k = kk[u];
            const float v = vv[u];
            S += v;
            if (need & N_SF) SF += __ldg(a.fre + k) * v;
            if (need & N_LOG) L += (double)logf((float)((double)v + 2.0e-16));
            if (need & N_HFC) hfc += v * (float)k;
            if (need & N_RMS) {
                float q = v * v;
                if (k == 0 || ((a.num & 1) == 0 && k == a.num - 1)) q *= 0.5f;
                rms += q;
            }
            if (need & N_E2) e2 += v * v;
            if ((need & N_DEC) && j >= 1) dec += (v - x0) / (float)k;
            if ((need & N_MAX) && !(v != v) && (bj < 0 || bv < v)) { bv = v; bj = j; }
          }
        }
        S = wsum(S);
        if (need & N_SF) SF = wsum(SF);
        if (need & N_LOG) L = wsumd(L);
        if (need & N_HFC) hfc = wsum(hfc);
        if (need & N_RMS) rms = wsum(rms);
        if (need & N_E2) e2 = wsum(e2);
        if (need & N_DEC) dec = wsum(dec);
        if (need & N_MAX) {
            for (int off = 16; off; off >>= 1) {    // ties go to the first list position (strict < in list order)
                const float ov = __shfl_xor_sync(FULL, bv, off);
                const int oj = __shfl_xor_sync(FULL, bj, off);
                if (oj >= 0 && (bj < 0 || bv < ov || (bv == ov && oj < bj))) { bv = ov; bj = oj; }
            }
            if (x0 != x0 || bj < 0) { bv = x0; bj = 0; }   // a NaN first element is never replaced
        }
        const float c = S != 0.f ? SF / S : 0.f;                  // centroid, flux_spectral.c:148-173
        const float meanV = S / fnb;                               // spectral_algorithm.c:1135-1144

        // ---- pass 2
        float m2 = 0.f, m3 = 0.f, m4 = 0.f, H = 0.f, sn = 0.f, sm = 0.f, v1s = 0.f, v2s = 0.f;
        if (need & (N_MOM | N_ENT | N_SLOPE | N_VAR)) {
            for (int j = lane; j < nb; j += 32) {
                const int k = bin_of(a, j);
                const float v = __ldg(x + k);
                if (need & N_MOM) {
                    const float d = __ldg(a.fre + k) - c;
                    m2 += d * d * v;
                    m3 += d * d * d * v;
                    m4 += d * d * d * d * v;
                }
                if (need & N_ENT) {
                    const float q = v / S;
                    H += q * log2f((float)((double)q + 1e-16));
                }
                if (need & (N_SLOPE | N_VAR)) {
                    const float f = __ldg(a.fre + k);
                    const float d = f - a.meanFre;
                    sn += d * (v - meanV);
                    sm += d * d;
                    const float u1 = meanV - v, u2 = a.meanFre - f;
                    v1s += u1 * u1;
                    v2s += u2 * u2;
                }
            }
            if (need & N_MOM) { m2 = wsum(m2); m3 = wsum(m3); m4 = wsum(m4); }
            if (need & N_ENT) H = wsum(H);
            if (need & (N_SLOPE | N_VAR)) { sn = wsum(sn); sm = wsum(sm); v1s = wsum(v1s); v2s = wsum(v2s); }
        }
        const float spread = S != 0.f ? sqrtf(m2 / S) : 0.f;
        auto entropy = [&](int isNorm) -> float {                 // flux_spectral.c:280-291
            if (!isNorm) return -H;
            const float m = log2f(fnb);
            return m != 0.f ? -H / m : 0.f;
        };
        float seqS = 0.f;
        if ((need & N_SEQ) && lane == 0) seqS = seq_sum(a, x);

        // ---- per request
        for (int r = 0; r < a.nReq; r++) {
            const int f = a.req[r], pl = a.plane[r];
            const float *pr = a.par + 4 * r;
            const int step = max((int)pr[0], 1), flags = (int)pr[3];
            const float p = pr[1], thr = pr[2];
            switch (f) {
            case AFB200_SPECTRAL_FLATNESS: {
                const double n1 = (double)expf((float)(L / nb));
                const float m1 = S / fnb;
                put(pl, m1 != 0.f ? (float)(n1 / (double)m1) : 0.f);
            } break;
            case AFB200_SPECTRAL_CENTROID: put(pl, c); break;
            case AFB200_SPECTRAL_SPREAD: put(pl, spread); break;
            case AFB200_SPECTRAL_SKEWNESS: { const float m1 = spread * spread * spread * S; put(pl, m1 != 0.f ? m3 / m1 : 0.f); } break;
            case AFB200_SPECTRAL_KURTOSIS: { const float m1 = spread * spread * spread * spread * S; put(pl, m1 != 0.f ? m4 / m1 : 0.f); } break;
            case AFB200_SPECTRAL_ENTROPY: put(pl, entropy(flags & 1)); break;
            case AFB200_SPECTRAL_CREST: { const float m1 = S / fnb; put(pl, m1 != 0.f ? bv / m1 : 0.f); } break;
            case AFB200_SPECTRAL_SLOPE: put(pl, sm != 0.f ? sn / sm : 0.f); break;
            case AFB200_SPECTRAL_DECREASE: { const float m1 = S - x0; put(pl, m1 != 0.f ? dec / m1 : 0.f); } break;
            case AFB200_SPECTRAL_RMS: {
                const int nn = (int)((unsigned)a.num * (unsigned)a.num);   // the reference's int product, wrapped
                put(pl, sqrtf(2.f * rms / (float)nn));
            } break;
            case AFB200_SPECTRAL_HFC: put(pl, hfc); break;
            case AFB200_SPECTRAL_EEF: put(pl, sqrtf(1.f + fabsf((e2 / fnb) * entropy(flags & 1)))); break;
            case AFB200_SPECTRAL_EER: put(pl, sqrtf(1.f + fabsf(logf(1.f + (e2 / fnb) * p) / entropy(flags & 1)))); break;
            case AFB200_SPECTRAL_MAX: put(pl, bv); put(pl + 1, __ldg(a.fre + bin_of(a, bj))); break;
            case AFB200_SPECTRAL_MEAN: put(pl, meanV); put(pl + 1, a.meanFre); break;
            case AFB200_SPECTRAL_VAR:
                if (nb >= 2) { put(pl, v1s / (float)(nb - 1)); put(pl + 1, v2s / (float)(nb - 1)); }
                break;
            case AFB200_SPECTRAL_ROLLOFF: {
                int k = -1;
                if (lane == 0) k = seq_cross(a, x, seqS * thr);
                k = __shfl_sync(FULL, k, 0);
                // no crossing: the reference keeps the bin of the last frame that crossed (`index` is not reset per
                // frame, flux_spectral.c:114), 0 before any.  The lanes look back 32 frames at a time.
                for (int base = t - 1; k < 0 && base >= 0; base -= 32) {
                    const int tt = base - lane;
                    int ck = -1;
                    if (tt >= 0) {
                        const float *row = clip + (size_t)tt * num;
                        ck = seq_cross(a, row, seq_sum(a, row) * thr);
                    }
                    const unsigned m = __ballot_sync(FULL, ck >= 0);
                    if (m) k = __shfl_sync(FULL, ck, __ffs(m) - 1);
                }
                if (k < 0) k = 0;
                put(pl, __ldg(a.fre + k));
            } break;
            case AFB200_SPECTRAL_ENERGY: {
                const int isLog = flags & 1;
                const float g = p <= 0.f ? 10.f : p;
                float s = 0.f;
                for (int j = lane; j < nb; j += 32) {
                    const float v = __ldg(x + bin_of(a, j));
                    float q = v * v;
                    if (isLog) q = logf(1.f + g * q);
                    s += q;
                }
                put(pl, wsum(s) / fnb);
            } break;
            case AFB200_SPECTRAL_BANDWIDTH: {
                float s = 0.f;
                for (int j = lane; j < nb; j += 32) {
                    const int k = bin_of(a, j);
                    float d = __ldg(a.fre + k) - c;
                    d = p == 2.f ? d * d : powf(d, p);
                    s += __ldg(x + k) * d;
                }
                s = wsum(s);
                if (p != 1.f) s = powf(s, (float)(1.0 / (double)p));
                put(pl, s);
            } break;
            case AFB200_SPECTRAL_FLUX: case AFB200_SPECTRAL_SD: case AFB200_SPECTRAL_SF: case AFB200_SPECTRAL_NOVELTY: {
                if (t < step) { put(pl, 0.f); break; }
                const float *xp = x - (size_t)step * num;
                const int isPos = flags & 1, method = flags & 3, isNum = (flags >> 2) & 1;
                float s = 0.f;
                for (int j = lane; j < nb; j += 32) {
                    const int k = bin_of(a, j);
                    const float cur = __ldg(x + k), pre = __ldg(xp + k);
                    if (f == AFB200_SPECTRAL_NOVELTY) {
                        float v1;
                        if (method == SpectralNoveltyMethod_Sub) v1 = cur - pre;
                        else {
                            const double q = (double)cur / ((double)pre + 1e-16);
                            const float lq = logf((float)q);
                            if (method == SpectralNoveltyMethod_Entroy) v1 = lq;
                            else if (method == SpectralNoveltyMethod_KL) v1 = cur * lq;
                            else v1 = (float)(q - (double)lq - 1.0);
                        }
                        if (v1 > thr) s += isNum ? 1.f : v1;
                    } else {
                        float v1 = cur - pre;
                        v1 = isPos ? (v1 > 0.f ? v1 : 0.f) : fabsf(v1);
                        if (f == AFB200_SPECTRAL_FLUX) v1 = p == 2.f ? v1 * v1 : powf(v1, p);
                        else if (f == AFB200_SPECTRAL_SF) v1 = v1 * v1;
                        s += v1;
                    }
                }
                s = wsum(s);
                if (f == AFB200_SPECTRAL_FLUX) {
                    if (flags & 4) s /= fnb;
                    if (flags & 2) s = powf(s, (float)(1.0 / (double)p));
                }
                put(pl, s);
            } break;
            case AFB200_SPECTRAL_MKL: {
                if (t == 0) { put(pl, 0.f); break; }
                const float *xp = x - num;
                float s = 0.f;
                for (int j = lane; j < nb; j += 32) {
                    const int k = bin_of(a, j);
                    const float v1 = (float)((double)__ldg(x + k) / ((double)__ldg(xp + k) + 1e-16));
                    s += logf(1.f + v1);
                }
                s = wsum(s);
                if (flags & 4) s /= fnb;
                put(pl, s);
            } break;
            case AFB200_SPECTRAL_BROADBAND: {
                if (t == 0) { put(pl, 0.f); break; }
                const float *xp = x - num;
                float s = 0.f;
                for (int j = lane; j < nb; j += 32) {
                    const int k = bin_of(a, j);
                    const float diff = (float)(10.0 * (double)log10f(__ldg(x + k) / __ldg(xp + k)));
                    if (diff > thr) s += 1.f;
                }
                s = wsum(s);
                if (lane == 0) {
                    if (a.fresh) a.out[(size_t)pl * BT + o] = s;
                    else a.out[(size_t)pl * BT + o] += s;          // counts into the caller's array
                }
            } break;
            case AFB200_SPECTRAL_PD: case AFB200_SPECTRAL_WPD: case AFB200_SPECTRAL_NWPD: {
                if (t == 0) { put(pl, 0.f); break; }
                if (t == 1) { if (a.fresh) put(pl, 0.f); break; }     // the reference never writes frame 1
                const float *ph = pclip + (size_t)t * num;
                const int weight = f != AFB200_SPECTRAL_PD, norm = f == AFB200_SPECTRAL_NWPD;
                float s = 0.f, sx = 0.f;
                for (int j = lane; j < nb; j += 32) {
                    const int k = bin_of(a, j);
                    float v1 = __ldg(ph + k) - 2.f * __ldg(ph - num + k) + __ldg(ph - 2 * num + k);
                    v1 = fabsf(v1);
                    const float v = __ldg(x + k);
                    if (weight) v1 = v1 * v;
                    s += v1;
                    sx += v;
                }
                s = wsum(s) / fnb;
                if (norm) {
                    const float m = wsum(sx) / fnb;
                    s = (float)((double)s / ((double)m + 1e-16));
                }
                put(pl, s);
            } break;
            case AFB200_SPECTRAL_CD: case AFB200_SPECTRAL_RCD: {
                if (t == 0) { put(pl, 0.f); break; }
                const float *ph = pclip + (size_t)t * num, *xp = x - num;
                float s = 0.f;
                for (int j = lane; j < nb; j += 32) {
                    const int k = bin_of(a, j);
                    const float v = __ldg(x + k), vp = __ldg(xp + k);
                    if (f == AFB200_SPECTRAL_RCD && v <= vp) continue;
                    const float p1 = __ldg(ph + k);
                    float re = v * cosf(p1), im = (float)((double)v * sin((double)p1));
                    if (t > 1) {
                        const float p2 = 2.f * __ldg(ph - num + k) - __ldg(ph - 2 * num + k);
                        re -= vp * cosf(p2);
                        im -= (float)((double)vp * sin((double)p2));
                    }
                    s += sqrtf(re * re + im * im);
                }
                put(pl, wsum(s));
            } break;
            default: break;
            }
        }
    }
}

}  // namespace

extern "C" int af_launch_spectral(const AfSpectralArgs *a, void *stream) {
    if (a->batch <= 0 || a->T <= 0) return AF_OK;
    const long long tiles = (long long)a->batch * ((a->T + TILE - 1) / TILE);
    if (tiles > 0x7fffffffLL) return af_fail(AF_ERR_UNSUPPORTED, "spectral: %lld frame tiles exceed one grid", tiles);
    k_spectral<<<(unsigned)tiles, WARPS * 32, 0, (cudaStream_t)stream>>>(*a);
    AF_LAUNCH_CHECK("k_spectral");
    return AF_OK;
}
