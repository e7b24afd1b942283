// gsb_geom.cuh -- the forward's per-Gaussian geometry (preprocess.comp, precomp_cov3d.comp, common.glsl), stated once: k_project
// and k_ingest_cov3d compute the frame with it and k_preprocess_backward recomputes the same values, which the reverse pass
// needs bit for bit.  Every fp32 operation is a single IEEE op (-fmad=false) in the order of the GLSL source.
#pragma once
#include <cuda_runtime.h>

#include "gs_b200.h"

namespace gsb {

// common.glsl:16-33
__device__ constexpr float SH_C0 = 0.28209479177387814f;
__device__ constexpr float SH_C1 = 0.4886025119029199f;
__device__ constexpr float SH_C2_0 = 1.0925484305920792f, SH_C2_1 = -1.0925484305920792f, SH_C2_2 = 0.31539156525252005f,
                           SH_C2_3 = -1.0925484305920792f, SH_C2_4 = 0.5462742152960396f;
__device__ constexpr float SH_C3_0 = -0.5900435899266435f, SH_C3_1 = 2.890611442640554f, SH_C3_2 = -0.4570457994644658f,
                           SH_C3_3 = 0.3731763325901154f, SH_C3_4 = -0.4570457994644658f, SH_C3_5 = 1.445305721320277f,
                           SH_C3_6 = -0.5900435899266435f;

// preprocess.comp:130-134: h = proj (p, 1) (p_w = 1 / h.w, ndc = h.xy p_w) and v = view (p, 1), each
// mat4 * vec4(p, 1) = ((m0*x + m1*y) + m2*z) + m3*1
struct ClipView {
    float p_w, ndcx, ndcy, vx, vy, vz;
};
__device__ __forceinline__ ClipView clip_view(const gsb_uniforms& U, float px, float py, float pz) {
    const float *pm = U.proj_mat, *vm = U.view_mat;
    const float hx = ((pm[0] * px + pm[4] * py) + pm[8] * pz) + pm[12];
    const float hy = ((pm[1] * px + pm[5] * py) + pm[9] * pz) + pm[13];
    const float hw = ((pm[3] * px + pm[7] * py) + pm[11] * pz) + pm[15];
    ClipView c;
    c.p_w = 1.0f / hw;
    c.ndcx = hx * c.p_w, c.ndcy = hy * c.p_w;
    c.vx = ((vm[0] * px + vm[4] * py) + vm[8] * pz) + vm[12];
    c.vy = ((vm[1] * px + vm[5] * py) + vm[9] * pz) + vm[13];
    c.vz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14];
    return c;
}

// get_projection_jacobian_approx (:34-50), t = clamp(v.xy / v.z, +-1.3 tan_fov) v.z, and the rows of T = J W (:55,:61), W the
// view rotation: T0[r] = V[r][0]*ja + V[r][2]*g0, T1[r] = V[r][1]*jb + V[r][2]*g1
struct Jacobian {
    float limx, limy, txtz, tytz, tx, ty, focal_x, focal_y, ja, jb, g0, g1, T0[3], T1[3];
};
__device__ __forceinline__ Jacobian jacobian(const gsb_uniforms& U, float vx, float vy, float vz) {
    const float* vm = U.view_mat;
    Jacobian j;
    j.limx = 1.3f * U.tan_fovx, j.limy = 1.3f * U.tan_fovy;
    j.txtz = vx / vz, j.tytz = vy / vz;
    j.tx = fminf(j.limx, fmaxf(-j.limx, j.txtz)) * vz;
    j.ty = fminf(j.limy, fmaxf(-j.limy, j.tytz)) * vz;
    j.focal_x = (float)U.width / (2.0f * U.tan_fovx);
    j.focal_y = (float)U.height / (2.0f * U.tan_fovy);
    j.ja = j.focal_x / vz, j.jb = j.focal_y / vz;
    j.g0 = -(j.focal_x * j.tx) / (vz * vz), j.g1 = -(j.focal_y * j.ty) / (vz * vz);
#pragma unroll
    for (int r = 0; r < 3; r++) {
        j.T0[r] = vm[r * 4 + 0] * j.ja + vm[r * 4 + 2] * j.g0;
        j.T1[r] = vm[r * 4 + 1] * j.jb + vm[r * 4 + 2] * j.g1;
    }
    return j;
}

// The fisheye lens of gsb_set_camera_model (DESIGN.md section 19), for t = (x, y, z) in view space: r = |(x, y)|, d = |t|,
// theta = atan2(r, z), t2 = theta^2, rho = theta P(t2), rho' = Q(t2), P = 1 + t2 P1, Q = 1 + t2 Q1.  Everything is written in
// b = theta / r (1 / d on the axis) and S = (sin(2 theta) / 2 - theta) / theta^3, so that nothing divides 0 by 0 on the axis:
//   s = rho / r = P b,   c = (rho' cos sin - rho) / r^3 = B b^3 with B = S + Q1 sin(2 theta) / (2 theta) - P1,   e = Q / d^2
//   J = d uv / d t = [fx (s + x^2 c), fx x y c, -fx x e; fy x y c, fy (s + y^2 c), -fy y e]
// S cancels catastrophically in the direct form for small theta (its numerator is O(theta^3) against O(theta) terms): below
// FISHEYE_SERIES_THETA it is summed from its Taylor series in t2 (7 terms, truncation < 2e-10 relative at theta = 1), above it
// the direct form loses at most a few ulps.
constexpr float FISHEYE_SERIES_THETA = 1.0f;
__device__ constexpr float FS_A1 = -0.6666666666666666f, FS_A2 = 0.13333333333333333f, FS_A3 = -0.012698412698412698f,
                           FS_A4 = 0.0007054673721340388f, FS_A5 = -2.565335898669232e-05f, FS_A6 = 6.577784355562133e-07f,
                           FS_A7 = -1.2529113058213587e-08f;
struct FisheyeGeo {
    float r, d, theta, t2, b, P1, Q1, S, scth, s, c, e;  // scth = sin(2 theta) / (2 theta) = 1 + t2 S
};
__device__ __forceinline__ FisheyeGeo fisheye_geo(const gsb_camera_model& M, float x, float y, float z) {
    FisheyeGeo g;
    const float r2 = x * x + y * y;
    g.r = sqrtf(r2);
    g.d = sqrtf(r2 + z * z);
    g.theta = atan2f(g.r, z);
    g.t2 = g.theta * g.theta;
    const float t2 = g.t2;
    g.b = g.r > 0.0f ? g.theta / g.r : 1.0f / g.d;
    g.P1 = M.k[0] + t2 * (M.k[1] + t2 * (M.k[2] + t2 * M.k[3]));
    g.Q1 = 3.0f * M.k[0] + t2 * (5.0f * M.k[1] + t2 * (7.0f * M.k[2] + t2 * (9.0f * M.k[3])));
    if (g.theta < FISHEYE_SERIES_THETA) {
        g.S = FS_A1 + t2 * (FS_A2 + t2 * (FS_A3 + t2 * (FS_A4 + t2 * (FS_A5 + t2 * (FS_A6 + t2 * FS_A7)))));
        g.scth = 1.0f + t2 * g.S;
    } else {
        g.scth = ((g.r * z) / (g.d * g.d)) / g.theta;
        g.S = (g.scth - 1.0f) / t2;
    }
    const float B = (g.S + g.Q1 * g.scth) - g.P1;
    g.s = (1.0f + t2 * g.P1) * g.b;
    g.c = B * ((g.b * g.b) * g.b);
    g.e = (1.0f + t2 * g.Q1) / (g.d * g.d);
    return g;
}
// J and the rows of T = J W (T0[r] = V[r][0] J[0][0] + V[r][1] J[0][1] + V[r][2] J[0][2], as jacobian() for its two terms)
struct FisheyeJ {
    float J[2][3], T0[3], T1[3];
};
__device__ __forceinline__ FisheyeJ fisheye_jacobian(const gsb_camera_model& M, const float* vm, const FisheyeGeo& g, float x, float y) {
    FisheyeJ j;
    const float xyc = (x * y) * g.c;
    j.J[0][0] = M.fx * (g.s + (x * x) * g.c), j.J[0][1] = M.fx * xyc, j.J[0][2] = -M.fx * (x * g.e);
    j.J[1][0] = M.fy * xyc, j.J[1][1] = M.fy * (g.s + (y * y) * g.c), j.J[1][2] = -M.fy * (y * g.e);
#pragma unroll
    for (int r = 0; r < 3; r++) {
        j.T0[r] = (vm[r * 4 + 0] * j.J[0][0] + vm[r * 4 + 1] * j.J[0][1]) + vm[r * 4 + 2] * j.J[0][2];
        j.T1[r] = (vm[r * 4 + 0] * j.J[1][0] + vm[r * 4 + 1] * j.J[1][1]) + vm[r * 4 + 2] * j.J[1][2];
    }
    return j;
}
// The backward's share: dL/dt of Phi = sum_{a,i} dJ[a][i] J[a][i] (dJ = dL/dJ, J's second derivatives) plus J^T duv.  With
// c_x = dc/dx / x, c_z = dc/dz, e_x = de/dx / x, e_z = de/dz (ds/dx = x c, ds/dz = -e), all stable on the axis:
//   c_x = 2 B' z b^4 / d^2 + 3 B S b^5,   c_z = -(2 B' theta r b^3 + 3 B b^2) / d^2,   B' = dB / dt2
//   e_x = (z b R2 - 2 Q) / d^4,           e_z = -(R2 theta r + 2 Q z) / d^4,             R2 = rho'' / theta = 2 dQ / dt2
__device__ __forceinline__ void fisheye_grad(const gsb_camera_model& M, const FisheyeGeo& g, const FisheyeJ& j, float x, float y,
                                             float z, const float (&dJ)[2][3], float du, float dv, float& dx, float& dy, float& dz) {
    const float t2 = g.t2, b = g.b;
    float dS;
    if (g.theta < FISHEYE_SERIES_THETA) {
        dS = FS_A2 + t2 * (2.0f * FS_A3 + t2 * (3.0f * FS_A4 + t2 * (4.0f * FS_A5 + t2 * (5.0f * FS_A6 + t2 * (6.0f * FS_A7)))));
    } else {  // d scth / d t2 = (cos 2 theta - scth) / (2 t2)
        const float cos2 = ((z - g.r) * (z + g.r)) / (g.d * g.d);
        dS = (0.5f * (cos2 - g.scth) - (g.scth - 1.0f)) / (t2 * t2);
    }
    const float dP1 = M.k[1] + t2 * (2.0f * M.k[2] + t2 * (3.0f * M.k[3]));
    const float dQ1 = 5.0f * M.k[1] + t2 * (14.0f * M.k[2] + t2 * (27.0f * M.k[3]));
    const float B = (g.S + g.Q1 * g.scth) - g.P1;
    const float dB = ((dS + dQ1 * g.scth) + g.Q1 * (g.S + t2 * dS)) - dP1;
    const float d2 = g.d * g.d, b2 = b * b, b3 = b2 * b;
    const float Q = 1.0f + t2 * g.Q1, R2 = 2.0f * (g.Q1 + t2 * dQ1);
    const float cx = (2.0f * dB * z) * (b3 * b) / d2 + (3.0f * B * g.S) * (b3 * b2);
    const float cz = -((2.0f * dB * g.theta) * (g.r * b3) + 3.0f * B * b2) / d2;
    const float ex = ((z * b) * R2 - 2.0f * Q) / (d2 * d2);
    const float ez = -((R2 * g.theta) * g.r + 2.0f * Q * z) / (d2 * d2);
    const float A0 = M.fx * dJ[0][0], A1 = M.fx * dJ[0][1], A2 = M.fx * dJ[0][2];
    const float B0 = M.fy * dJ[1][0], B1 = M.fy * dJ[1][1], B2 = M.fy * dJ[1][2];
    const float sig = A0 + B1, m = A1 + B0;
    const float q = ((A0 * x) * x + (m * x) * y) + (B1 * y) * y, l = A2 * x + B2 * y;
    dx = (((sig * x) * g.c + (q * x) * cx) + g.c * (2.0f * A0 * x + m * y)) - ((l * x) * ex + g.e * A2);
    dy = (((sig * y) * g.c + (q * y) * cx) + g.c * (2.0f * B1 * y + m * x)) - ((l * y) * ex + g.e * B2);
    dz = (q * cz - sig * g.e) - l * ez;
    dx += du * j.J[0][0] + dv * j.J[1][0];
    dy += du * j.J[0][1] + dv * j.J[1][1];
    dz += du * j.J[0][2] + dv * j.J[1][2];
}

// cov2d = transpose(T) Sigma T + 0.3 I (:56-65), Sigma = the cov3d words ca.xyzw, cb.xy; tm0 / tm1 = Sigma T0 / Sigma T1 (S[k] =
// column k).  m01 and m10 round differently, so each caller states its own determinant.  c00 and c11 are the diagonal before
// the dilation (the anti-aliased mode's opacity compensation reads them; m01 and m10 are not dilated).
struct Cov2d {
    float tm0[3], tm1[3], m00, m01, m10, m11, c00, c11;
};
__device__ __forceinline__ Cov2d cov2d(const float (&T0)[3], const float (&T1)[3], float4 ca, float2 cb) {
    const float S[3][3] = {{ca.x, ca.y, ca.z}, {ca.y, ca.w, cb.x}, {ca.z, cb.x, cb.y}};
    Cov2d c;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        c.tm0[k] = (T0[0] * S[k][0] + T0[1] * S[k][1]) + T0[2] * S[k][2];
        c.tm1[k] = (T1[0] * S[k][0] + T1[1] * S[k][1]) + T1[2] * S[k][2];
    }
    const float c00 = (c.tm0[0] * T0[0] + c.tm0[1] * T0[1]) + c.tm0[2] * T0[2];
    const float c01 = (c.tm1[0] * T0[0] + c.tm1[1] * T0[1]) + c.tm1[2] * T0[2];  // [0][1]: col 0, row 1
    const float c10 = (c.tm0[0] * T1[0] + c.tm0[1] * T1[1]) + c.tm0[2] * T1[2];  // [1][0]
    const float c11 = (c.tm1[0] * T1[0] + c.tm1[1] * T1[1]) + c.tm1[2] * T1[2];
    c.m00 = c00 + 0.3f, c.m01 = c01, c.m10 = c10, c.m11 = c11 + 0.3f;
    c.c00 = c00, c.c11 = c11;
    return c;
}

// The anti-aliased mode (gsb_set_antialiased): the opacity factor sqrt(det(cov2d) / det(cov2d + 0.3 I)) that keeps a
// Gaussian's integral what it was before the dilation.  det is the caller's dilated determinant (m00 m11 - m10 m01, > 0);
// det0 is the same product order over the undilated entries.  A NaN ratio gives 0.
__device__ __forceinline__ float aa_det0(const Cov2d& c) { return c.c00 * c.c11 - c.m10 * c.m01; }
__device__ __forceinline__ float aa_compensation(float det0, float det) { return sqrtf(fmaxf(0.0f, det0 / det)); }

// rotationFromQuaternion, common.glsl:51-75: R[c][r] of the quaternion as stored (not normalised)
__device__ __forceinline__ void rotation_from_quaternion(float qw, float qx, float qy, float qz, float (&R)[3][3]) {
    const float qx2 = qx * qx, qy2 = qy * qy, qz2 = qz * qz;
    R[0][0] = (1.0f - 2.0f * qy2) - 2.0f * qz2;
    R[0][1] = (2.0f * qx) * qy - (2.0f * qz) * qw;
    R[0][2] = (2.0f * qx) * qz + (2.0f * qy) * qw;
    R[1][0] = (2.0f * qx) * qy + (2.0f * qz) * qw;
    R[1][1] = (1.0f - 2.0f * qx2) - 2.0f * qz2;
    R[1][2] = (2.0f * qy) * qz - (2.0f * qx) * qw;
    R[2][0] = (2.0f * qx) * qz - (2.0f * qy) * qw;
    R[2][1] = (2.0f * qy) * qz + (2.0f * qx) * qw;
    R[2][2] = (1.0f - 2.0f * qx2) - 2.0f * qy2;
}

// The scene words of one record (GSScene.cpp:157-184, precomp_cov3d.comp:25-48): pos_op[o] = (p.xyz, opacity) and Sigma =
// transpose(M) M with M = S R, S = diag(scale * scale_factor), stored as cov_a[o], cov_b[o].  p, so, q are the record's first
// three float4 (position, scale_opacity, rotation wxyz as stored).  k_ingest_cov3d and k_adam_step both store through it, so a
// step leaves the words a gsb_scene_upload of the same records would.
__device__ __forceinline__ void store_cov3d(float4 p, float4 so, float4 q, uint64_t o, float4* __restrict__ pos_op,
                                            float4* __restrict__ cov_a, float2* __restrict__ cov_b, float scale_factor) {
    float R[3][3];
    rotation_from_quaternion(q.x, q.y, q.z, q.w, R);
    // M = S * R  (precomp_cov3d.comp:39), S diagonal => M[c][r] = s_r * R[c][r]
    const float s[3] = {so.x * scale_factor, so.y * scale_factor, so.z * scale_factor};
    float M[3][3];
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int r = 0; r < 3; r++) M[c][r] = s[r] * R[c][r];
        // cov3d = transpose(M) * M (:40): cov[c][r] = sum_k M[r][k] * M[c][k]
#define COV(c, r) ((M[r][0] * M[c][0] + M[r][1] * M[c][1]) + M[r][2] * M[c][2])
    const float c0 = COV(0, 0), c1 = COV(0, 1), c2 = COV(0, 2), c3 = COV(1, 1), c4 = COV(1, 2), c5 = COV(2, 2);
#undef COV
    pos_op[o] = make_float4(p.x, p.y, p.z, so.w);
    cov_a[o] = make_float4(c0, c1, c2, c3);
    cov_b[o] = make_float2(c4, c5);
}

// preprocess.comp:73-78: (x, y, z) = normalize(p - camera_position); returns |p - camera_position|
__device__ __forceinline__ float view_direction(const float* cam, float px, float py, float pz, float& x, float& y, float& z) {
    const float dx = px - cam[0], dy = py - cam[1], dz = pz - cam[2];
    const float len = sqrtf((dx * dx + dy * dy) + dz * dz);
    x = dx / len, y = dy / len, z = dz / len;
    return len;
}

}  // namespace gsb
