// c64.cuh -- complex fp32 values packed in one 64-bit register pair.  sm_90 has no packed-fp32 instructions, so each
// helper is two scalar IEEE operations with explicit rounding (__fadd_rn / __fmul_rn / __fmaf_rn): the compiler may
// not contract a separate multiply and add into an FMA, so every result is the one the element-wise (re, im) arithmetic
// below defines, bit for bit.
#pragma once
#include <stdint.h>

typedef unsigned long long c64;     // lo 32 bits = real, hi 32 bits = imaginary

__device__ __forceinline__ c64 c_pack(float re, float im) { c64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(re), "f"(im)); return r; }
__device__ __forceinline__ void c_unpack(c64 v, float &re, float &im) { asm("mov.b64 {%0, %1}, %2;" : "=f"(re), "=f"(im) : "l"(v)); }
__device__ __forceinline__ c64 c_from(float2 v) { return c_pack(v.x, v.y); }
__device__ __forceinline__ float c_re(c64 v) { float a, b; c_unpack(v, a, b); return a; }
__device__ __forceinline__ float c_im(c64 v) { float a, b; c_unpack(v, a, b); return b; }

__device__ __forceinline__ c64 c_add(c64 a, c64 b) {
    float ar, ai, br, bi; c_unpack(a, ar, ai); c_unpack(b, br, bi);
    return c_pack(__fadd_rn(ar, br), __fadd_rn(ai, bi));
}
__device__ __forceinline__ c64 c_sub(c64 a, c64 b) {
    float ar, ai, br, bi; c_unpack(a, ar, ai); c_unpack(b, br, bi);
    return c_pack(__fsub_rn(ar, br), __fsub_rn(ai, bi));
}
__device__ __forceinline__ c64 v_mul(c64 a, c64 b) {     // element-wise
    float ar, ai, br, bi; c_unpack(a, ar, ai); c_unpack(b, br, bi);
    return c_pack(__fmul_rn(ar, br), __fmul_rn(ai, bi));
}
__device__ __forceinline__ c64 v_fma(c64 a, c64 b, c64 c) {
    float ar, ai, br, bi, cr, ci; c_unpack(a, ar, ai); c_unpack(b, br, bi); c_unpack(c, cr, ci);
    return c_pack(__fmaf_rn(ar, br, cr), __fmaf_rn(ai, bi, ci));
}

__device__ __forceinline__ c64 c_swap(c64 v) { float a, b; c_unpack(v, a, b); return c_pack(b, a); }
__device__ __forceinline__ c64 c_conj(c64 v) { float a, b; c_unpack(v, a, b); return c_pack(a, -b); }
__device__ __forceinline__ c64 c_mul_mi(c64 v) { float a, b; c_unpack(v, a, b); return c_pack(b, -a); }   // * (-i)
__device__ __forceinline__ c64 c_mul_pi(c64 v) { float a, b; c_unpack(v, a, b); return c_pack(-b, a); }   // * (+i)
__device__ __forceinline__ c64 c_scale(c64 v, float s) { return v_mul(v, c_pack(s, s)); }
// v * (c - i s)  (forward twiddle e^{-i theta}, c = cos theta, s = sin theta)
__device__ __forceinline__ c64 c_mul_cs(c64 v, float c, float s) { return v_fma(c_swap(v), c_pack(s, -s), v_mul(v, c_pack(c, c))); }
// general complex product a * w
__device__ __forceinline__ c64 c_mul(c64 a, c64 w) {
    float wr, wi; c_unpack(w, wr, wi);
    return v_fma(c_swap(a), c_pack(-wi, wi), v_mul(a, c_pack(wr, wr)));
}
// |v|^2
__device__ __forceinline__ float c_norm2(c64 v) { float a, b; c_unpack(v_mul(v, v), a, b); return a + b; }

// FMA forms (the fused MFCC frame path only): fewer instructions, each product rounded once inside an FMA, so results
// differ from the helpers above in the last bits.
// a * w: FMUL + FFMA per component
__device__ __forceinline__ c64 c_mul_fma(c64 a, c64 w) {
    float ar, ai, wr, wi; c_unpack(a, ar, ai); c_unpack(w, wr, wi);
    return c_pack(__fmaf_rn(-ai, wi, __fmul_rn(ar, wr)), __fmaf_rn(ai, wr, __fmul_rn(ar, wi)));
}
// |v|^2: FMUL + FFMA
__device__ __forceinline__ float c_norm2_fma(c64 v) { float a, b; c_unpack(v, a, b); return __fmaf_rn(a, a, __fmul_rn(b, b)); }
