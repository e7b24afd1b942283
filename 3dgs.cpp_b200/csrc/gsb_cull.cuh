// gsb_cull.cuh -- conservative "can this Gaussian contribute anywhere in this pixel rectangle?" test of
// k_blend (8x8 pixel blocks, one per warp); its per-Gaussian cut power_cut() is also the threshold of
// k_emit's instance culling (16x16 tiles, gsb_set_tile_cull level 1).
//
// render.comp:66-80 skips a (pixel, Gaussian) pair when alpha = opacity * exp(power) < 1/255; with
// opacity <= 1 (sigmoid, GSScene.cpp:44) that is implied by power < POWER_CUT = -5.55.  The exponent
// is power = -q/2 with q(dx, dy) = A dx^2 + 2 B dx dy + C dy^2 (the conic), convex, so its minimum over a
// rectangle of pixel centres is bounded below by the minimum over the continuous rectangle, which lies at
// the centre (0) or on one of the four edges (four 1-D quadratics).  A rectangle is declared dead only if
// -q_min/2, widened by a bound on the fp32 rounding error of the shader's evaluation order, is still below
// POWER_CUT; every pair inside a dead rectangle is therefore one the shader itself skips and dropping it
// leaves the image bit-identical.
#pragma once
#include <cuda_runtime.h>

namespace gsb {

constexpr float POWER_CUT = -5.55f;  // for opacity <= 1: alpha = opacity * exp(power) <= exp(-5.55) < 1/255 (documentation only)

// Per-Gaussian version of the same cut: power < power_cut(opacity) implies opacity * exp(power) < 1/255 in the
// kernel's arithmetic (the 1e-3 margin dwarfs the error of __logf, of the shared-definition exp and of the final
// multiply).  For opacity <= 1 (what GSScene::load produces) it is >= -log(255) - 1e-3 = -5.5423; gsb_scene_upload
// does not validate opacities, so the bound is NOT clamped at POWER_CUT: for opacity > 1 it is simply lower (down to
// the exp's own clamp at -87), and the kernel keeps every pair render.comp:77-80 would blend.  Clamped to <= 0.
__device__ __forceinline__ float power_cut(float opacity) {
    const float c = -__logf(255.0f * opacity) - 1e-3f;  // opacity <= 0 / NaN -> +inf / NaN -> clamped to 0 below
    return fminf(fmaxf(c, -87.0f), 0.0f);
}

// Minimum over [lo, hi] of the 1-D quadratic  q(t) = a t^2 + 2 b t + c  (a > 0, inv_a ~ 1/a).
// An inexact minimiser only moves the result by a (t - t*)^2, second order in the rounding error.
__device__ __forceinline__ float min_quad_1d(float a, float inv_a, float b, float c, float lo, float hi) {
    const float t = fminf(fmaxf(-b * inv_a, lo), hi);
    return fmaf(fmaf(a, t, 2.0f * b), t, c);
}

// Pixels [x0, x0 + w - 1] x [y0, y0 + h - 1] (as floats); (ux, uy) = Gaussian centre; A, B, C = conic; A, C > 0.
__device__ __forceinline__ bool rect_may_contribute(float ux, float uy, float A, float B, float C, float inv_a, float inv_c,
                                                    float x0, float y0, float w, float h, float cut) {
    // d = uv - pixel
    const float dx_lo = ux - (x0 + (w - 1.0f)), dx_hi = ux - x0, dy_lo = uy - (y0 + (h - 1.0f)), dy_hi = uy - y0;
    float qmin;
    if (dx_lo <= 0.0f && dx_hi >= 0.0f && dy_lo <= 0.0f && dy_hi >= 0.0f) {
        qmin = 0.0f;  // centre inside the rectangle
    } else {
        const float e0 = min_quad_1d(C, inv_c, B * dx_lo, A * dx_lo * dx_lo, dy_lo, dy_hi);  // edge dx = dx_lo
        const float e1 = min_quad_1d(C, inv_c, B * dx_hi, A * dx_hi * dx_hi, dy_lo, dy_hi);  // edge dx = dx_hi
        const float e2 = min_quad_1d(A, inv_a, B * dy_lo, C * dy_lo * dy_lo, dx_lo, dx_hi);  // edge dy = dy_lo
        const float e3 = min_quad_1d(A, inv_a, B * dy_hi, C * dy_hi * dy_hi, dx_lo, dx_hi);  // edge dy = dy_hi
        qmin = fminf(fminf(e0, e1), fminf(e2, e3));
    }
    const float dxm = fmaxf(fabsf(dx_lo), fabsf(dx_hi)), dym = fmaxf(fabsf(dy_lo), fabsf(dy_hi));
    const float mag = 0.5f * (A * dxm * dxm + C * dym * dym) + fabsf(B) * dxm * dym;  // sum of |terms| of render.comp:66
    const float margin = 0.02f + 2e-6f * mag;  // >= 32 ulp of the largest term: covers both evaluations' rounding
    return !(-0.5f * qmin < cut - margin);  // NaN -> keep
}

}  // namespace gsb
