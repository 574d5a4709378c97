// block_reduce.cuh -- CTA-wide reductions shared by the kernels (sm_90a).  Each one reduces within every warp by
// shuffles, then over the warps' results in warp order, so its result does not depend on scheduling; every thread of the
// block must call it and every thread gets the result.  Each one starts with a barrier, so its scratch may still be read
// from the previous reduction.
#pragma once
#include "common.cuh"

namespace {

// (v, i) beats (w, j): i is a candidate and either j is none, v > w, or they tie and i comes first
__device__ __forceinline__ bool beats(float v, int i, float w, int j) {
    return i >= 0 && (j < 0 || v > w || (v == w && i < j));
}

// the reference's __vmax (`max < v` from the first value on) in three steps: each thread offers its values with
// vmax_take, block_argmax reduces the threads' candidates, and vmax_first applies the rule for the first value

// one value v at index i: NaN is passed over, a strictly larger value replaces the candidate (bv, bi), so the first
// maximum is kept.  Start with bi = -1
__device__ __forceinline__ void vmax_take(float v, int i, float &bv, int &bi) {
    const bool take = v == v && (bi < 0 || v > bv);
    bv = take ? v : bv;
    bi = take ? i : bi;
}

// __vmax's index from block_argmax's bi: the first index `first` when the first value v0 is NaN (it stays the maximum)
// or when there is no candidate
__device__ __forceinline__ int vmax_first(int bi, float v0, int first) { return v0 != v0 || bi < 0 ? first : bi; }

// first index of the block's maximum over the candidates (i >= 0); -1 when there is none.  redv / redi: 32 each
__device__ int block_argmax(float v, int i, float *redv, int *redi) {
    for (int o = 16; o; o >>= 1) {
        const float w = __shfl_xor_sync(0xffffffffu, v, o);
        const int j = __shfl_xor_sync(0xffffffffu, i, o);
        if (beats(w, j, v, i)) { v = w; i = j; }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) { redv[warp] = v; redi[warp] = i; }
    __syncthreads();
    v = redv[0]; i = redi[0];
    for (int k = 1; k < nw; k++)
        if (beats(redv[k], redi[k], v, i)) { v = redv[k]; i = redi[k]; }
    return i;
}

// block sum of a double in a fixed order (tree within each warp, then the warps in order).  red: 32 doubles
__device__ double block_sum(double v, double *red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = red[0];
    for (int k = 1; k < nw; k++) v += red[k];
    return v;
}

// block minimum (isMax = false) or maximum of an int.  red: 32 ints
__device__ int block_reduce_int(int v, bool isMax, int *red) {
    v = isMax ? __reduce_max_sync(0xffffffffu, v) : __reduce_min_sync(0xffffffffu, v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = red[0];
    for (int i = 1; i < nw; i++) v = isMax ? max(v, red[i]) : min(v, red[i]);
    return v;
}

// fminf (isMax = 0) or fmaxf (isMax = 1) over a block of kWarps warps.  red: kWarps floats
template <int kWarps>
__device__ float block_reduce_float(float v, int isMax, float *red) {
    for (int o = 16; o; o >>= 1) {
        const float w = __shfl_xor_sync(0xffffffffu, v, o);
        v = isMax ? fmaxf(v, w) : fminf(v, w);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = red[0];
    for (int w = 1; w < kWarps; w++) v = isMax ? fmaxf(v, red[w]) : fminf(v, red[w]);
    return v;
}

}  // namespace
