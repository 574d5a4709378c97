// nmf.cu -- non-negative matrix factorisation V ~ W H (sm_90a), replacing the iteration loop of nmf
// (src/classic/nmf.c:104-265), which runs six triple-loop products per iteration on one core.
//
// Every matrix of a call runs the same stages, one launch each, over the whole batch (blockIdx.x = matrix):
//   k_nmf_norm (first)  W /= its column norms (__mnorm p = 1 | 2, else __mmax), done = 0, iters = 0;
//   then per iteration:
//   k_nmf_d    D = W H, with D2 / D3 formed from it (KL: V/(D+eps) and 1; IS: V/(D^2+eps) and 1/(D+eps) in double;
//              Euclidean: V and D);
//   k_nmf_h    H <- H * (W^T D2) / (W^T D3 + eps), the old H kept for the stop test;
//   k_nmf_w    W <- W * (D2 H^T) / (D3 H^T + eps) with the new H, the old W kept;
//   k_nmf_norm W normalised again, ||W - W_prev||, ||H - H_prev|| (the squares summed in float in index order, as
//              __vnorm does: for the same W and H the stop decision is the reference's), the per-matrix stop flag
//              and iteration count.
// A matrix whose flag is set returns at the top of every later stage, so the host queues 1 + 4 maxIter launches
// without waiting and their number does not depend on the batch.
//
// Products are formed in float and summed in double, as __mdot / __mdot2 do; the sums run in a fixed order that depends
// only on the shapes, so a matrix gives the same bits in any batch.  D2 and D3 (n x m) live in a device workspace: they
// do not fit in shared memory for spectrogram-sized matrices.  The file is compiled with -fmad=false (Makefile): every
// float step is rounded on its own, as in the reference.
#include "common.cuh"

namespace {

constexpr float kEps = 1e-16f;
constexpr int kKC = 8;              // k-columns whose sums one thread carries at a time
constexpr int kSlices = 8;          // k_nmf_h: row slices (warps) per CTA, summed through shared memory
constexpr int kRowsPerCta = 8;      // k_nmf_w: one warp per row
constexpr int kNormThreads = 256;
constexpr int kChunk = 8 * kNormThreads;   // k_nmf_norm: squared differences staged per pass of the sequential sum
constexpr unsigned FULL = 0xffffffffu;

struct NmfParams {
    const float *V;
    float *W, *H, *Wp, *Hp, *D2, *D3, *colv;
    int *done, *iters;
    int n, m, k, type, norm, it;
    float thresh;
};

__device__ __forceinline__ double prod(float a, float b) { return (double)__fmul_rn(a, b); }

// W * A / (B + eps) (KL, IS: nmf.c:151,196) or W * (A / (B + eps)) (Euclidean: :234,255), each step rounded to float
__device__ __forceinline__ float update(float x, double a, double b, int type) {
    const float fa = (float)a, fb = __fadd_rn((float)b, kEps);
    return type == 0 || type == 1 ? __fdiv_rn(__fmul_rn(x, fa), fb) : __fmul_rn(x, __fdiv_rn(fa, fb));
}

__global__ void __launch_bounds__(256) k_nmf_d(NmfParams p) {
    const int b = blockIdx.x;
    if (p.done[b]) return;
    const size_t nm = (size_t)p.n * p.m;
    const float *W = p.W + (size_t)b * p.n * p.k, *H = p.H + (size_t)b * p.k * p.m, *V = p.V + (size_t)b * nm;
    for (size_t e = (size_t)blockIdx.y * blockDim.x + threadIdx.x; e < nm; e += (size_t)gridDim.y * blockDim.x) {
        const int i = (int)(e / p.m), j = (int)(e % p.m);
        double acc = 0.0;
        for (int c = 0; c < p.k; c++) acc += prod(W[(size_t)i * p.k + c], H[(size_t)c * p.m + j]);
        const float d = (float)acc;
        if (p.type == 0) {
            p.D2[(size_t)b * nm + e] = __fdiv_rn(V[e], __fadd_rn(d, kEps));
        } else if (p.type == 1) {                              // nmf.c:167-170: 1.0/(float) is a double division
            p.D2[(size_t)b * nm + e] = (float)(1.0 / (double)__fadd_rn(__fmul_rn(d, d), kEps) * (double)V[e]);
            p.D3[(size_t)b * nm + e] = (float)(1.0 / (double)__fadd_rn(d, kEps));
        } else {
            p.D3[(size_t)b * nm + e] = d;
        }
    }
}

// P2 / P3 of stage h and w: the planes that stand for D2 and D3 (NULL P3: all ones)
__device__ __forceinline__ const float *plane2(const NmfParams &p, int b) {
    return p.type == 2 ? p.V + (size_t)b * p.n * p.m : p.D2 + (size_t)b * p.n * p.m;
}
__device__ __forceinline__ const float *plane3(const NmfParams &p, int b) {
    return p.type == 0 ? nullptr : p.D3 + (size_t)b * p.n * p.m;
}

// H[c][j] for 32 columns j (lanes) and kKC columns c of W at a time; 8 warps sum 8 interleaved row slices, then the
// slices are added in order through shared memory
__global__ void __launch_bounds__(256) k_nmf_h(NmfParams p) {
    __shared__ double sa[kSlices][kKC][32], sb[kSlices][kKC][32];
    const int b = blockIdx.x;
    if (p.done[b]) return;
    const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
    const float *P2 = plane2(p, b), *P3 = plane3(p, b), *W = p.W + (size_t)b * p.n * p.k;
    float *H = p.H + (size_t)b * p.k * p.m, *Hp = p.Hp + (size_t)b * p.k * p.m;
    for (int j0 = blockIdx.y * 32; j0 < p.m; j0 += gridDim.y * 32) {
        const int j = j0 + lane;
        for (int c0 = 0; c0 < p.k; c0 += kKC) {
            const int kc = p.k - c0 < kKC ? p.k - c0 : kKC;
            double a[kKC], bb[kKC];
#pragma unroll
            for (int c = 0; c < kKC; c++) a[c] = bb[c] = 0.0;
            if (j < p.m) {
                for (int i = slice; i < p.n; i += kSlices) {
                    const float d2 = P2[(size_t)i * p.m + j], d3 = P3 ? P3[(size_t)i * p.m + j] : 1.f;
                    const float *w = W + (size_t)i * p.k + c0;
#pragma unroll
                    for (int c = 0; c < kKC; c++)
                        if (c < kc) { a[c] += prod(w[c], d2); bb[c] += prod(w[c], d3); }
                }
            }
#pragma unroll
            for (int c = 0; c < kKC; c++) { sa[slice][c][lane] = a[c]; sb[slice][c][lane] = bb[c]; }
            __syncthreads();
            const int c = threadIdx.x >> 5;                    // 256 threads: one (c, lane) each
            if (c < kc && j < p.m) {
                double sA = 0.0, sB = 0.0;
                for (int s = 0; s < kSlices; s++) { sA += sa[s][c][lane]; sB += sb[s][c][lane]; }
                const size_t o = (size_t)(c0 + c) * p.m + j;
                const float h = H[o];
                Hp[o] = h;
                H[o] = update(h, sA, sB, p.type);
            }
            __syncthreads();
        }
    }
}

// W[i][c]: one warp per row i, lanes over the columns j, kKC columns of H^T at a time, a fixed xor-tree over the lanes
__global__ void __launch_bounds__(256) k_nmf_w(NmfParams p) {
    const int b = blockIdx.x;
    if (p.done[b]) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float *P2 = plane2(p, b), *P3 = plane3(p, b), *H = p.H + (size_t)b * p.k * p.m;
    float *W = p.W + (size_t)b * p.n * p.k, *Wp = p.Wp + (size_t)b * p.n * p.k;
    for (int i = blockIdx.y * kRowsPerCta + warp; i < p.n; i += gridDim.y * kRowsPerCta) {
        const float *r2 = P2 + (size_t)i * p.m, *r3 = P3 ? P3 + (size_t)i * p.m : nullptr;
        for (int c0 = 0; c0 < p.k; c0 += kKC) {
            const int kc = p.k - c0 < kKC ? p.k - c0 : kKC;
            double a[kKC], bb[kKC];
#pragma unroll
            for (int c = 0; c < kKC; c++) a[c] = bb[c] = 0.0;
            for (int j = lane; j < p.m; j += 32) {
                const float d2 = r2[j], d3 = r3 ? r3[j] : 1.f;
#pragma unroll
                for (int c = 0; c < kKC; c++)
                    if (c < kc) {
                        const float h = H[(size_t)(c0 + c) * p.m + j];
                        a[c] += prod(d2, h); bb[c] += prod(d3, h);
                    }
            }
#pragma unroll
            for (int c = 0; c < kKC; c++)
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    a[c] += __shfl_xor_sync(FULL, a[c], o);
                    bb[c] += __shfl_xor_sync(FULL, bb[c], o);
                }
#pragma unroll
            for (int c = 0; c < kKC; c++)
                if (lane == c && c < kc) {
                    const size_t o = (size_t)i * p.k + c0 + c;
                    const float w = W[o];
                    Wp[o] = w;
                    W[o] = update(w, a[c], bb[c], p.type);
                }
        }
    }
}

// squares of a chunk of differences, written by all threads into sq[0 .. cnt), added in index order by thread 0 into
// *acc: the float32 sequential sum of __vsub + __vnorm (nmf.c:270-273)
__device__ __forceinline__ void add_chunk(const float *sq, int cnt, float *acc) {
    __syncthreads();
    if (threadIdx.x == 0)
        for (int t = 0; t < cnt; t++) *acc = __fadd_rn(*acc, sq[t]);
    __syncthreads();
}

// one CTA per matrix.  it < 0: the normalisation before the loop (nmf.c:95-102); else the end of iteration `it`
// (:259-275)
__global__ void __launch_bounds__(kNormThreads) k_nmf_norm(NmfParams p) {
    __shared__ float sq[kChunk];
    const int b = blockIdx.x;
    if (p.it >= 0 && p.done[b]) return;
    float *W = p.W + (size_t)b * p.n * p.k, *v = p.colv + (size_t)b * p.k;
    for (int c = threadIdx.x; c < p.k; c += blockDim.x) {     // column sums in row order, in float, as __mnorm / __mmax
        float s = 0.f;
        if (p.norm == 1 || p.norm == 2) {
            for (int i = 0; i < p.n; i++) {
                const float x = fabsf(W[(size_t)i * p.k + c]);
                s = __fadd_rn(s, p.norm == 1 ? x : __fmul_rn(x, x));
            }
            if (p.norm == 2) s = __fsqrt_rn(s);
        } else {
            s = W[c];
            for (int i = 1; i < p.n; i++) {
                const float x = W[(size_t)i * p.k + c];
                if (s < x) s = x;
            }
        }
        v[c] = s;
    }
    __syncthreads();
    const size_t nk = (size_t)p.n * p.k, km = (size_t)p.k * p.m;
    const float *Wp = p.Wp + (size_t)b * nk;
    float dw = 0.f, dh = 0.f;                                  // thread 0's sums
    for (size_t base = 0; base < nk; base += kChunk) {
        const int cnt = nk - base < (size_t)kChunk ? (int)(nk - base) : kChunk;
        for (int t = threadIdx.x; t < cnt; t += blockDim.x) {  // __mdiv_vector: a zero stays zero, no guard on v
            const size_t e = base + t;
            const float x = W[e], y = x != 0.f ? __fdiv_rn(x, v[e % p.k]) : 0.f;
            W[e] = y;
            if (p.it >= 0) {
                const float d = __fsub_rn(y, Wp[e]);
                sq[t] = __fmul_rn(d, d);
            }
        }
        if (p.it >= 0) add_chunk(sq, cnt, &dw);
    }
    if (p.it < 0) {
        if (threadIdx.x == 0) {
            p.done[b] = 0;
            if (p.iters) p.iters[b] = 0;
        }
        return;
    }
    const float *H = p.H + (size_t)b * km, *Hp = p.Hp + (size_t)b * km;
    for (size_t base = 0; base < km; base += kChunk) {
        const int cnt = km - base < (size_t)kChunk ? (int)(km - base) : kChunk;
        for (int t = threadIdx.x; t < cnt; t += blockDim.x) {
            const float d = __fsub_rn(H[base + t], Hp[base + t]);
            sq[t] = __fmul_rn(d, d);
        }
        add_chunk(sq, cnt, &dh);
    }
    if (threadIdx.x == 0) {
        if (p.iters) p.iters[b] = p.it + 1;
        if (__fsqrt_rn(dw) < p.thresh && __fsqrt_rn(dh) < p.thresh) p.done[b] = 1;
    }
}

int grid_y(long long units, long long perCta) {
    const long long g = (units + perCta - 1) / perCta;
    return (int)(g < 1 ? 1 : g > 65535 ? 65535 : g);
}

}  // namespace

extern "C" int af_launch_nmf(const AfNmfArgs *a, void *stream) {
    if (a->batch <= 0) return AF_OK;
    if (a->n < 1 || a->m < 1 || a->k < 1 || a->type < 0 || a->type > 2)
        return af_fail(AF_ERR_ARG, "nmf: n=%d m=%d k=%d batch=%d type=%d", a->n, a->m, a->k, a->batch, a->type);
    NmfParams p;
    p.V = a->V; p.W = a->W; p.H = a->H; p.iters = a->iters;
    p.n = a->n; p.m = a->m; p.k = a->k; p.type = a->type; p.norm = a->norm; p.thresh = a->thresh;
    cudaStream_t st = (cudaStream_t)stream;
    // workspace: D2 (KL, IS), D3 (IS, Euclidean), previous W and H, column norms, stop flags
    const size_t nm = (size_t)a->batch * a->n * a->m, nk = (size_t)a->batch * a->n * a->k,
                 km = (size_t)a->batch * a->k * a->m, bk = (size_t)a->batch * a->k;
    const size_t n2 = a->type == 2 ? 0 : nm, n3 = a->type == 0 ? 0 : nm;
    float *ws = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&ws, sizeof(float) * (n2 + n3 + nk + km + bk + a->batch), st);
    if (e != cudaSuccess) return af_cuda_check(e, "cudaMallocAsync(nmf workspace)");
    p.D2 = n2 ? ws : nullptr;
    p.D3 = n3 ? ws + n2 : nullptr;
    p.Wp = ws + n2 + n3;
    p.Hp = p.Wp + nk;
    p.colv = p.Hp + km;
    p.done = (int *)(p.colv + bk);
    const unsigned B = (unsigned)a->batch;
    const dim3 gd(B, grid_y((long long)a->n * a->m, 256)), gh(B, grid_y(a->m, 32)), gw(B, grid_y(a->n, kRowsPerCta));
    int rc = AF_OK;
    p.it = -1;
    k_nmf_norm<<<B, kNormThreads, 0, st>>>(p);
    af_count_launch(1);
    for (int it = 0; it < a->maxIter && (e = cudaGetLastError()) == cudaSuccess; it++) {
        p.it = it;
        k_nmf_d<<<gd, 256, 0, st>>>(p);
        k_nmf_h<<<gh, 256, 0, st>>>(p);
        k_nmf_w<<<gw, 256, 0, st>>>(p);
        k_nmf_norm<<<B, kNormThreads, 0, st>>>(p);
        af_count_launch(4);
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) rc = af_fail(AF_ERR_CUDA, "nmf launch: %s", cudaGetErrorString(e));
    const cudaError_t ef = cudaFreeAsync(ws, st);
    return rc ? rc : af_cuda_check(ef, "cudaFreeAsync(nmf workspace)");
}
