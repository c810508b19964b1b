// Activation math shared by the GEMM epilogues (gemm_sm90.cu) and their stand-alone counterparts (elementwise.cu):
// exact GELU / dGELU through an Abramowitz-Stegun erf, and the SiLU sigmoid.
#pragma once
#include <cuda_runtime.h>

namespace b200 {

__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// erf via Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7, far below bf16 resolution): 1 rcp + 1 exp + 6 FMA.
// e = exp(-z^2) is returned too: for z = x/sqrt(2) it is exactly the Gaussian factor gelu'(x) needs.
// Two variants that differ only in the reciprocal, so they can round differently: erf_as (GEMM epilogue) uses rcp.approx,
// erf_poly (stand-alone kernels) the correctly rounded __frcp_rn.
__device__ __forceinline__ float erf_as(float z, float& e) {
    const float az = fabsf(z);
    // rcp.approx (relative error <= 2^-23, below the 1.5e-7 of the formula) rather than __frcp_rn: the correctly
    // rounded reciprocal calls a slow-path subroutine, and the GEMM kernel must stay free of calls (see its body).
    // The argument is >= 1, never in that slow range.
    const float t = rcp_approx(fmaf(0.3275911f, az, 1.0f));
    e = __expf(-az * az);
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float y = 1.0f - poly * t * e;
    return copysignf(y, z);
}
__device__ __forceinline__ float erf_poly(float z, float& e) {
    const float az = fabsf(z);
    const float t = __frcp_rn(fmaf(0.3275911f, az, 1.0f));
    e = __expf(-az * az);
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    return copysignf(1.0f - poly * t * e, z);
}

__device__ __forceinline__ float gelu_erf(float x) {
    float e;
    return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752f, e));
}
__device__ __forceinline__ float dgelu_erf(float x) {
    float e;
    const float cdf = 0.5f * (1.0f + erf_as(x * 0.70710678118654752f, e));
    return fmaf(x * 0.3989422804014327f, e, cdf);  // cdf + x * pdf,  pdf = exp(-x^2/2)/sqrt(2 pi)
}

// sigmoid(x) = 1 / (1 + exp(-x)) with ex2.approx and rcp.approx: no call.  exp(-x) overflows to inf for x < -88 and the
// reciprocal of inf is 0, so silu(x) = x * sigmoid(x) and silu'(x) = s (1 + x (1 - s)) go to -0 / 0 there, as they should.
// The SwiGLU epilogues and the stand-alone SwiGLU kernels both use it, so the fused and unfused routes agree.
__device__ __forceinline__ float sigmoid_approx(float x) { return rcp_approx(1.0f + __expf(-x)); }

}  // namespace b200
