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
// J of a lens frame (fisheye or OpenCV) and the rows of T = J W (T0[r] = V[r][0] J[0][0] + V[r][1] J[0][1] + V[r][2] J[0][2],
// as jacobian() for its two terms)
struct LensJ {
    float J[2][3], T0[3], T1[3];
};
__device__ __forceinline__ LensJ fisheye_jacobian(const gsb_camera_model& M, const float* vm, const FisheyeGeo& g, float x, float y) {
    LensJ j;
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
__device__ __forceinline__ void fisheye_grad(const gsb_camera_model& M, const FisheyeGeo& g, const LensJ& j, float x, float y,
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
// The lens's share (gsb_render_backward_fisheye): adds dL/d(fx, fy, cx, cy, k1..k4) of uv and J to dl.  With P = 1 + t2 P1 and
// Q = 1 + t2 Q1, s = P b, c = B b^3, e = Q / d^2 as in fisheye_geo:
//   d uv / d(fx, fy) = (s x, 0), (0, s y);  d uv / d(cx, cy) = (1, 0), (0, 1);  d J / d fx = J's row 0 / fx (row 1 for fy)
//   d s / d k_j = b t2^j,  d c / d k_j = t2^(j-1) ((2j + 1) scth - 1) b^3,  d e / d k_j = (2j + 1) t2^j / d^2
// so that, with fisheye_grad's sig, q, l (dJ weighted by fx, fy) and Ls = fx du x + fy dv y + sig,
//   dL/dk_j = t2^(j-1) ((t2 b Ls - b^3 q) + (2j + 1) (scth b^3 q - t2 l / d^2)).
// Every factor is finite on the axis (b = 1 / d, x = y = 0 there).
__device__ __forceinline__ void fisheye_lens_grad(const gsb_camera_model& M, const FisheyeGeo& g, float x, float y,
                                                  const float (&dJ)[2][3], float du, float dv, float* dl) {
    const float xyc = (x * y) * g.c, j00 = g.s + (x * x) * g.c, j11 = g.s + (y * y) * g.c;
    dl[0] += du * (g.s * x) + ((dJ[0][0] * j00 + dJ[0][1] * xyc) - dJ[0][2] * (x * g.e));
    dl[1] += dv * (g.s * y) + ((dJ[1][0] * xyc + dJ[1][1] * j11) - dJ[1][2] * (y * g.e));
    dl[2] += du;
    dl[3] += dv;
    const float A0 = M.fx * dJ[0][0], A1 = M.fx * dJ[0][1], A2 = M.fx * dJ[0][2];
    const float B0 = M.fy * dJ[1][0], B1 = M.fy * dJ[1][1], B2 = M.fy * dJ[1][2];
    const float sig = A0 + B1, m = A1 + B0;
    const float q = ((A0 * x) * x + (m * x) * y) + (B1 * y) * y, l = A2 * x + B2 * y;
    const float Ls = ((M.fx * du) * x + (M.fy * dv) * y) + sig;
    const float b3 = (g.b * g.b) * g.b;
    const float al = (g.t2 * g.b) * Ls, be = b3 * q, ga = (g.t2 * l) / (g.d * g.d);
    const float base = al - be, odd = g.scth * be - ga;
    float pw = 1.0f;  // t2^(j-1)
#pragma unroll
    for (int j = 1; j <= 4; j++) {
        dl[3 + j] += pw * (base + (float)(2 * j + 1) * odd);
        pw *= g.t2;
    }
}

// The OpenCV (Brown-Conrady radial-tangential) lens of gsb_set_camera_model (DESIGN.md section 23), for t = (x, y, z) in view
// space with z > 0.2 and k = (k1, k2, p1, p2):
//   xn = x / z, yn = y / z, r2 = xn^2 + yn^2, R = 1 + k1 r2 + k2 r2^2, R' = dR / dr2 = k1 + 2 k2 r2
//   xd = xn R + 2 p1 xn yn + p2 (r2 + 2 xn^2),   yd = yn R + p1 (r2 + 2 yn^2) + 2 p2 xn yn,   uv = (fx xd + cx, fy yd + cy)
//   D = d(xd, yd) / d(xn, yn), symmetric:  D00 = R + 2 xn^2 R' + 2 p1 yn + 6 p2 xn,  D11 = R + 2 yn^2 R' + 6 p1 yn + 2 p2 xn,
//                                          D01 = D10 = 2 xn yn R' + 2 p1 xn + 2 p2 yn
//   J = d uv / d t = diag(fx, fy) D N,  N = d(xn, yn) / dt = [1, 0, -xn; 0, 1, -yn] / z,  so with (e0, e1) = D (xn, yn):
//   J = [fx D00, fx D01, -fx e0; fy D01, fy D11, -fy e1] / z
// Polynomial in (xn, yn): no series and no singularity inside the cull (z > 0.2, r2 <= tan^2 max_theta, det D > 0).
struct OpencvGeo {
    float xn, yn, r2, R, Rp, xd, yd, D00, D01, D11, e0, e1, det;
};
__device__ __forceinline__ OpencvGeo opencv_geo(const gsb_camera_model& M, float x, float y, float z) {
    const float k1 = M.k[0], k2 = M.k[1], p1 = M.k[2], p2 = M.k[3];
    OpencvGeo g;
    g.xn = x / z, g.yn = y / z;
    const float xn = g.xn, yn = g.yn, xx = xn * xn, yy = yn * yn, xy = xn * yn;
    g.r2 = xx + yy;
    g.R = 1.0f + g.r2 * (k1 + g.r2 * k2);
    g.Rp = k1 + (2.0f * k2) * g.r2;
    g.xd = xn * g.R + ((2.0f * p1) * xy + p2 * (g.r2 + 2.0f * xx));
    g.yd = yn * g.R + (p1 * (g.r2 + 2.0f * yy) + (2.0f * p2) * xy);
    g.D00 = ((g.R + (2.0f * xx) * g.Rp) + (2.0f * p1) * yn) + (6.0f * p2) * xn;
    g.D11 = ((g.R + (2.0f * yy) * g.Rp) + (6.0f * p1) * yn) + (2.0f * p2) * xn;
    g.D01 = ((2.0f * xy) * g.Rp + (2.0f * p1) * xn) + (2.0f * p2) * yn;
    g.e0 = g.D00 * xn + g.D01 * yn;
    g.e1 = g.D01 * xn + g.D11 * yn;
    g.det = g.D00 * g.D11 - g.D01 * g.D01;
    return g;
}
__device__ __forceinline__ LensJ opencv_jacobian(const gsb_camera_model& M, const float* vm, const OpencvGeo& g, float z) {
    LensJ j;
    j.J[0][0] = (M.fx * g.D00) / z, j.J[0][1] = (M.fx * g.D01) / z, j.J[0][2] = -(M.fx * g.e0) / z;
    j.J[1][0] = (M.fy * g.D01) / z, j.J[1][1] = (M.fy * g.D11) / z, j.J[1][2] = -(M.fy * g.e1) / z;
#pragma unroll
    for (int r = 0; r < 3; r++) {
        j.T0[r] = (vm[r * 4 + 0] * j.J[0][0] + vm[r * 4 + 1] * j.J[0][1]) + vm[r * 4 + 2] * j.J[0][2];
        j.T1[r] = (vm[r * 4 + 0] * j.J[1][0] + vm[r * 4 + 1] * j.J[1][1]) + vm[r * 4 + 2] * j.J[1][2];
    }
    return j;
}
// dL/dJ weighted by the focal lengths, (A, B) = (fx dJ[0], fy dJ[1]), folded through N: the J term of the loss is
// Psi / z with Psi = a D00 + m D01 + c D11, a = A0 - A2 xn, m = A1 + B0 - A2 yn - B2 xn, c = B1 - B2 yn.
struct OpencvDJ {
    float A2, B2, a, m, c;
};
__device__ __forceinline__ OpencvDJ opencv_dj(const gsb_camera_model& M, const OpencvGeo& g, const float (&dJ)[2][3]) {
    const float A0 = M.fx * dJ[0][0], A1 = M.fx * dJ[0][1], A2 = M.fx * dJ[0][2];
    const float B0 = M.fy * dJ[1][0], B1 = M.fy * dJ[1][1], B2 = M.fy * dJ[1][2];
    return OpencvDJ{A2, B2, A0 - A2 * g.xn, (A1 + B0) - (A2 * g.yn + B2 * g.xn), B1 - B2 * g.yn};
}
// The backward's share: dL/dt of Phi = Psi / z + du u + dv v.  D's derivatives are the third derivatives of one potential, so
// four numbers hold them (R'' = 2 k2):
//   H000 = dD00/dxn = 6 xn R' + 8 k2 xn^3 + 6 p2,        H001 = dD00/dyn = dD01/dxn = 2 yn R' + 8 k2 xn^2 yn + 2 p1
//   H011 = dD11/dxn = dD01/dyn = 2 xn R' + 8 k2 xn yn^2 + 2 p2,   H111 = dD11/dyn = 6 yn R' + 8 k2 yn^3 + 6 p1
// Then G = dPhi/d(xn, yn) = (dPsi/d(xn, yn)) / z + D (fx du, fy dv), and through (xn, yn, 1 / z) = (x, y, 1) / z:
//   dx = Gx / z,  dy = Gy / z,  dz = -(Gx xn + Gy yn + Psi / z) / z.
__device__ __forceinline__ void opencv_grad(const gsb_camera_model& M, const OpencvGeo& g, float z, const float (&dJ)[2][3], float du,
                                            float dv, float& dx, float& dy, float& dz) {
    const float k8 = 8.0f * M.k[1], p1 = M.k[2], p2 = M.k[3], xn = g.xn, yn = g.yn;
    const OpencvDJ w = opencv_dj(M, g, dJ);
    const float psi = (w.a * g.D00 + w.m * g.D01) + w.c * g.D11;
    const float H000 = ((6.0f * xn) * g.Rp + ((k8 * xn) * xn) * xn) + 6.0f * p2;
    const float H001 = ((2.0f * yn) * g.Rp + ((k8 * xn) * xn) * yn) + 2.0f * p1;
    const float H011 = ((2.0f * xn) * g.Rp + ((k8 * yn) * yn) * xn) + 2.0f * p2;
    const float H111 = ((6.0f * yn) * g.Rp + ((k8 * yn) * yn) * yn) + 6.0f * p1;
    const float psx = ((w.a * H000 + w.m * H001) + w.c * H011) - (w.A2 * g.D00 + w.B2 * g.D01);
    const float psy = ((w.a * H001 + w.m * H011) + w.c * H111) - (w.A2 * g.D01 + w.B2 * g.D11);
    const float Lu = M.fx * du, Lv = M.fy * dv;
    const float gx = psx / z + (Lu * g.D00 + Lv * g.D01);
    const float gy = psy / z + (Lu * g.D01 + Lv * g.D11);
    dx = gx / z;
    dy = gy / z;
    dz = -((gx * xn + gy * yn) + psi / z) / z;
}
// The lens's share (gsb_render_backward_fisheye on an OpenCV frame): adds dL/d(fx, fy, cx, cy, k1, k2, p1, p2) of uv and J to
// dl.  d J / d fx = J's row 0 / fx (row 1 for fy), d uv / d(fx, fy) = (xd, 0), (0, yd), and with s = a + c,
// q = a xn^2 + m xn yn + c yn^2, Ld = fx du xn + fy dv yn (opencv_dj's a, m, c):
//   dL/dk1 = (r2 s + 2 q) / z + r2 Ld,   dL/dk2 = r2 ((r2 s + 4 q) / z + r2 Ld)
//   dL/dp1 = (2 a yn + 2 m xn + 6 c yn) / z + fx du 2 xn yn + fy dv (r2 + 2 yn^2)
//   dL/dp2 = (6 a xn + 2 m yn + 2 c xn) / z + fx du (r2 + 2 xn^2) + fy dv 2 xn yn
__device__ __forceinline__ void opencv_lens_grad(const gsb_camera_model& M, const OpencvGeo& g, float z, const float (&dJ)[2][3],
                                                 float du, float dv, float* dl) {
    const float xn = g.xn, yn = g.yn, xx = xn * xn, yy = yn * yn, xy = xn * yn, r2 = g.r2;
    dl[0] += du * g.xd + ((dJ[0][0] * g.D00 + dJ[0][1] * g.D01) - dJ[0][2] * g.e0) / z;
    dl[1] += dv * g.yd + ((dJ[1][0] * g.D01 + dJ[1][1] * g.D11) - dJ[1][2] * g.e1) / z;
    dl[2] += du;
    dl[3] += dv;
    const OpencvDJ w = opencv_dj(M, g, dJ);
    const float Lu = M.fx * du, Lv = M.fy * dv;
    const float s = w.a + w.c, q = ((w.a * xx + w.m * xy) + w.c * yy), Ld = Lu * xn + Lv * yn;
    dl[4] += (r2 * s + 2.0f * q) / z + r2 * Ld;
    dl[5] += r2 * ((r2 * s + 4.0f * q) / z + r2 * Ld);
    dl[6] += (((2.0f * w.a) * yn + (2.0f * w.m) * xn) + (6.0f * w.c) * yn) / z + (Lu * (2.0f * xy) + Lv * (r2 + 2.0f * yy));
    dl[7] += (((6.0f * w.a) * xn + (2.0f * w.m) * yn) + (2.0f * w.c) * xn) / z + (Lu * (r2 + 2.0f * xx) + Lv * (2.0f * xy));
}

// The orthographic camera of gsb_set_camera_model (DESIGN.md section 26), for t = (x, y, z) in view space with z > 0.2:
//   uv = (fx x + cx, fy y + cy),   J = d uv / d t = [fx, 0, 0; 0, fy, 0],   T = J W: T0 = fx (view row 0), T1 = fy (view row 1)
// J is constant, so the backward has no second-derivative term: dL/dt = J^T duv (ortho_grad), plus dL/df on t.z for the
// depth key f = z.
__device__ __forceinline__ LensJ ortho_jacobian(const gsb_camera_model& M, const float* vm) {
    LensJ j;
    j.J[0][0] = M.fx, j.J[0][1] = 0.0f, j.J[0][2] = 0.0f;
    j.J[1][0] = 0.0f, j.J[1][1] = M.fy, j.J[1][2] = 0.0f;
#pragma unroll
    for (int r = 0; r < 3; r++) {
        j.T0[r] = M.fx * vm[r * 4 + 0];
        j.T1[r] = M.fy * vm[r * 4 + 1];
    }
    return j;
}
__device__ __forceinline__ void ortho_grad(const gsb_camera_model& M, float du, float dv, float& dx, float& dy, float& dz) {
    dx = M.fx * du;
    dy = M.fy * dv;
    dz = 0.0f;
}
// The lens's share (gsb_render_backward_fisheye on an orthographic frame): adds dL/d(fx, fy, cx, cy) of uv and J to dl:
// d uv / d(fx, fy) = (x, 0), (0, y);  d uv / d(cx, cy) = I;  d J / d fx = J's row 0 / fx = (1, 0, 0), d J / d fy = (0, 1, 0).
__device__ __forceinline__ void ortho_lens_grad(float x, float y, const float (&dJ)[2][3], float du, float dv, float* dl) {
    dl[0] += du * x + dJ[0][0];
    dl[1] += dv * y + dJ[1][1];
    dl[2] += du;
    dl[3] += dv;
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

// The SH view direction of an orthographic frame: every ray is parallel to the camera's forward axis, so the direction is
// view row 2 normalised, the same for every Gaussian.  view_direction of the point (row 2) from the origin: p - 0 = p exactly,
// so this is view_direction's fp32 normalisation of the row, and its gradient goes to the row (not to p or camera_position).
__device__ __forceinline__ float ortho_direction(const float* vm, float& x, float& y, float& z) {
    const float origin[3] = {0.0f, 0.0f, 0.0f};
    return view_direction(origin, vm[2], vm[6], vm[10], x, y, z);
}

// One element of torch.optim.Adam (no weight decay): gsb_adam_step's and gsb_adam_step_features' update.
struct AdamUpdate {
    float w1, w2, beta2, eps, bc2_sqrt;
    // torch's exp_avg.lerp_(g, 1 - beta1); exp_avg_sq.mul_(beta2).addcmul_(g, g, value=1 - beta2);
    // denom = sqrt(exp_avg_sq) / bc2_sqrt + eps; param.addcdiv_(exp_avg, denom, value=-step_size)
    __device__ __forceinline__ void operator()(float g, float& x, float& m, float& v, float step_size) const {
        m = w1 < 0.5f ? fmaf(w1, g - m, m) : fmaf(w1 - 1.0f, g - m, g);
        v = fmaf(w2 * g, g, v * beta2);
        const float denom = sqrtf(v) / bc2_sqrt + eps;
        x = fmaf(-step_size, m / denom, x);
    }
};

}  // namespace gsb
