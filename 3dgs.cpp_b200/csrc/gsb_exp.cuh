// gsb_exp.cuh -- the blend's bit-defined exp, shared by k_blend (gsb_blend.cu) and its reverse pass (gsb_backward.cu), which
// must re-evaluate every alpha of the frame bit for bit to find the same contributors.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gsb {

// Bit-defined exp for x in [-87, 0] without the clamp; mirrors gso_exp_shared() in oracle/gs_oracle.c op for op: Cody-Waite
// reduction, degree-5 Horner with the constant term 1, 2^n applied through the exponent bits (12 instructions).  The blend
// only uses results with power in [cut, 0] (cut >= -87), where the oracle's clamp is the identity.
__device__ __forceinline__ float exp_shared_inrange(float x) {
    const float t = __fmul_rn(x, 1.44269504088896341f);
    const float tm = __fadd_rn(t, 12582912.0f);  // low mantissa bits = rint(t) in two's complement
    const float n = __fsub_rn(tm, 12582912.0f);
    float r = __fmaf_rn(n, -0.693359375f, x);
    r = __fmaf_rn(n, 2.12194440e-4f, r);
    float p = __fmaf_rn(8.290082216262817e-3f, r, 4.1899293661117554e-2f);
    p = __fmaf_rn(p, r, 1.6667647659778595e-1f);
    p = __fmaf_rn(p, r, 4.9999138712882996e-1f);
    p = __fmaf_rn(p, r, 9.999997019767761e-1f);
    p = __fmaf_rn(p, r, 1.0f);
    return __uint_as_float(__float_as_uint(p) + (__float_as_uint(tm) << 23));
}

}  // namespace gsb
