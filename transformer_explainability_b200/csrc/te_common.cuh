// Shared device helpers for the sm_90a transformer-attribution kernels.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define TE_OK 0
#define TE_ERR_ARG (-1)
#define TE_ERR_WORKSPACE (-2)
#define TE_ERR_CUDA (-3)
#define TE_ERR_UNSUPPORTED (-4)

#define TE_CUDA_CHECK_LAUNCH()                                   \
    do {                                                         \
        te_count_launch();                                       \
        cudaError_t e__ = cudaGetLastError();                    \
        if (e__ != cudaSuccess) { te_set_last_error(cudaGetErrorString(e__)); return TE_ERR_CUDA; } \
    } while (0)

#define TE_TRY(x)                                                \
    do { int r__ = (x); if (r__ != TE_OK) return r__; } while (0)

void te_set_last_error(const char* msg);
void te_count_launch();

// safe_divide of the reference (modules/layers_ours.py:10-13):
//   den = clamp(b,min=eps) + clamp(b,max=eps)  ( == b + eps ) ; den += eps where den == 0 ;
//   out = a / den * (b != 0)
template <typename T>
__device__ __forceinline__ T te_sd(T a, T b) {
    const T eps = (T)1e-9;
    T den = b + eps;
    den = (den == (T)0) ? eps : den;
    return (a / den) * ((b != (T)0) ? (T)1 : (T)0);
}

// same rule with the quotient as a * rcp.approx(den) (2 ulp; |den| < 2^126): epilogues of the tensor-core attention kernels, whose
// operands are already products of rounded factors
__device__ __forceinline__ float te_sd_fast(float a, float b) {
    const float eps = 1e-9f;
    float den = b + eps;
    den = (den == 0.f) ? eps : den;
    return __fdividef(a, den) * ((b != 0.f) ? 1.f : 0.f);          // non-finite a keeps the reference's NaN (x * 0)
}

// safe_divide for a denominator that is known to be >= 0 (the z+ rule: a clamped sum of non-negative products): b + eps > 0, so only
// the (b != 0) mask of the rule remains
__device__ __forceinline__ float te_sd_fast_nonneg(float a, float b) {
    return (b > 0.f) ? __fdividef(a, b + 1e-9f) : a * 0.f;            // a * 0 keeps the reference's NaN for a non-finite a
}

__device__ __forceinline__ float te_gelu(float x) {           // exact (erf) GELU, nn.GELU default
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float te_gelu_grad(float x) {
    const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
    const float pdf = 0.39894228040143267794f * expf(-0.5f * x * x);
    return cdf + x * pdf;
}

// QuickGELU of CLIP, q(x) = x sigma(1.702 x), and q'(x) = s (1 + 1.702 x (1 - s)) with s = sigma(1.702 x).  1 - s is taken as
// sigma(-1.702 x), not by cancellation, so the x (1 - s) term keeps its relative precision in the tails.  An overflowing
// exponential gives the limits (-0 and 0 for x -> -inf, x and 1 for x -> +inf).
__device__ __forceinline__ float te_quick_gelu(float x) { return x / (1.0f + expf(-1.702f * x)); }
__device__ __forceinline__ float te_quick_gelu_grad(float x) {
    const float a = 1.702f * x;
    const float s = 1.0f / (1.0f + expf(-a)), oms = 1.0f / (1.0f + expf(a));
    return s * fmaf(a, oms, 1.0f);
}

// GELU'(x) = Phi(x) + x phi(x) for the single-pass (TF32-grade) backward epilogues: erf by Abramowitz-Stegun 7.1.26 (absolute
// error 1.5e-7), one ex2.approx shared by erf's exp(-x^2/2) and the density — ~15 instructions against ~45 for erff + expf.
__device__ __forceinline__ float te_gelu_grad_fast(float x) {
    const float ax = fabsf(x);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-0.72134752044448170368f * x * x));        // exp(-x^2 / 2)
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f)));    // argument in [1, inf)
    float p = fmaf(1.061405429f, t, -1.453152027f);
    p = fmaf(p, t, 1.421413741f);
    p = fmaf(p, t, -0.284496736f);
    p = fmaf(p, t, 0.254829592f);
    const float erfa = fmaf(-p * t, e, 1.0f);                     // erf(|x| / sqrt 2)
    const float cdf = 0.5f * (1.0f + copysignf(erfa, x));
    return fmaf(x * 0.39894228040143267794f, e, cdf);
}

__device__ __forceinline__ float te_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double te_warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float te_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---- block-scaled fp16 (hi, lo) split: the operand format of the fp16-split Linear GEMM (te_tc_wgmma.cu) -------------------
// A block of values with largest magnitude m is stored as 2^-e (hi + lo) with 2^e m in [2^14, 2^15): hi = fp16(2^e x),
// lo = fp16(2^e x - hi).  s = 2^e, si = 2^-e (exact powers of two).  Zero / non-finite blocks keep e = 0.
__device__ __forceinline__ void te_f16_block_scale(float m, float& s, float& si) {
    s = 1.f; si = 1.f;
    if (m > 0.f && m < 3.0e38f) {
        int e;
        frexpf(m, &e);                           // m = f 2^e, f in [0.5, 1)
        e = max(e, -100);
        s = ldexpf(1.f, 15 - e);
        si = ldexpf(1.f, e - 15);
    }
}
__device__ __forceinline__ float te_absmax4(const float4 v) {
    return fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
}
__device__ __forceinline__ void te_f16_split4(const float4 v, float s, uint2& hi, uint2& lo) {
    const float a0 = v.x * s, a1 = v.y * s, a2 = v.z * s, a3 = v.w * s;
    const __half2 h01 = __floats2half2_rn(a0, a1), h23 = __floats2half2_rn(a2, a3);
    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    const __half2 l01 = __floats2half2_rn(a0 - f01.x, a1 - f01.y), l23 = __floats2half2_rn(a2 - f23.x, a3 - f23.y);
    hi.x = *reinterpret_cast<const uint32_t*>(&h01); hi.y = *reinterpret_cast<const uint32_t*>(&h23);
    lo.x = *reinterpret_cast<const uint32_t*>(&l01); lo.y = *reinterpret_cast<const uint32_t*>(&l23);
}

static inline int te_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
