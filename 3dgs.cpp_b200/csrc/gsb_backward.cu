// gsb_backward.cu -- reverse mode of one whole frame: dL/d(image) -> dL/d(GSScene::Vertex records).  No reference counterpart
// (3DGS.cpp only renders); this differentiates the function the forward computes, quirks included (DESIGN.md section 10):
// no background term, only the red channel clamped at 0, integer pixel centres, alpha = min(0.99, .), the T' < 1e-4 break and
// the per-tile lists of the frame.
//
//   k_blend_backward      one CTA per 16 x 16 tile, one pixel per thread.  The tile's list is walked back to front from the
//                         largest last-contributor position among its pixels (recorded by k_blend<..., RECORD>), in batches
//                         staged into shared memory.  Every (pixel, entry) pair re-evaluates power and alpha with the frame's
//                         own arithmetic (EXACT: the ops of k_blend + exp_shared_inrange; FAST: the same FMAs + __expf), so the
//                         contributor set is the forward's bit for bit; T is recovered by division, T_i = T_{i+1} / (1 - alpha_i).
//                         Per survivor it accumulates d uv (2), d conic (3), d opacity (1), d colour (3): reduced over the warp
//                         (fp32 shuffles), then over the CTA (fp64 shared-memory atomics), then one global fp64 atomic per value
//                         and tile.  fp64 keeps the order-dependent rounding of the sums over warps and tiles ~1e-16 relative.
//   k_preprocess_backward one thread per survivor (grid-stride over N_v, read on the device): recomputes preprocess.comp for the
//                         survivor's Gaussian from the scene and the frame's camera and chains colour -> SH + view direction,
//                         conic -> cov2d -> (Sigma, J) -> position, uv -> ndc -> clip position -> position,
//                         Sigma -> scale and (stored, unnormalised) rotation.  It writes the Gaussian's 60-float gradient
//                         record and returns its scratch accumulators to zero for the next call.
//
// The atomics make the sums depend on the order in which warps and CTAs add their partial sums: gradients are NOT guaranteed
// to be bitwise reproducible from run to run (fp64 accumulation makes a difference in the final fp32 value rare).
// Compiled with -fmad=false like the forward.
#include "gsb_cull.cuh"
#include "gsb_exp.cuh"
#include "gsb_internal.cuh"

namespace gsb {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int BW_THREADS = 256;  // one pixel per thread of a 16 x 16 tile
constexpr int BW_BATCH = 256;    // list entries staged per batch (one per thread)
constexpr int BW_NACC = 9;       // per-survivor accumulators: uv (2), conic (3), opacity, colour (3)
constexpr int PB_THREADS = 256;

struct __align__(16) BwRec {  // the staged record in k_blend's pre-scaled form (render.comp:66 evaluated identically)
    float4 q0;                // ux uy -A/2 -B
    float4 q1;                // -C/2 opacity r g
    float4 q2;                // b power_cut bits(compact id) -
};

template <int MODE>
__global__ void __launch_bounds__(BW_THREADS) k_blend_backward(const __grid_constant__ BackwardParams P) {
    __shared__ BwRec s_rec[BW_BATCH];
    __shared__ double s_acc[BW_BATCH][BW_NACC];
    __shared__ uint32_t s_max;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.x;
    const uint32_t tx = tile % P.tiles_x, ty = tile / P.tiles_x;
    uint2 range = P.ranges[tile];
    range.y = ~range.y;
    // warp w owns the 8 x 4 pixel block at (8 (w & 1), 4 (w >> 1)): a compact footprint, so a warp shares most records' fate
    const uint32_t px = tx * GSB_TILE + (warp & 1) * 8 + (lane & 7);
    const uint32_t py = ty * GSB_TILE + (warp >> 1) * 4 + (lane >> 3);
    const bool inside = px < P.width && py < P.height;
    const float fx = (float)px, fy = (float)py;

    float T = 1.0f, gr = 0.f, gg = 0.f, gb = 0.f;
    uint32_t last = 0;
    if (inside) {
        const uint2 r = P.record[(size_t)py * P.width + px];
        T = __uint_as_float(r.x);
        last = r.y;
        const float4 g = *reinterpret_cast<const float4*>(reinterpret_cast<const unsigned char*>(P.grad_image) + (size_t)py * P.row_pitch_bytes +
                                                          (size_t)px * sizeof(float4));
        gr = g.x, gg = g.y, gb = g.z;  // A is constant 1 in the forward: no gradient
    }
    if (tid == 0) s_max = 0;
    __syncthreads();
    const uint32_t wmax = __reduce_max_sync(FULL, last);
    if (lane == 0 && wmax) atomicMax(&s_max, wmax);
    __syncthreads();
    const uint32_t max_last = s_max;
    if (range.x >= range.y) return;  // empty list: every pixel has last == 0

    float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f;  // colour behind the current entry, per unit of its transmittance
    for (uint32_t hi = max_last; hi > 0;) {
        const uint32_t lo = hi > (uint32_t)BW_BATCH ? hi - (uint32_t)BW_BATCH : 0u;
        const uint32_t cnt = hi - lo;
        __syncthreads();  // the previous batch's walk and flush are done with s_rec / s_acc
        if ((uint32_t)tid < cnt) {
            const uint32_t cid = __ldg(P.vals + range.x + lo + (uint32_t)tid);
            const float4* rec = P.recs + (size_t)cid * GSB_REC_F4;
            const float4 a = __ldg(rec), col = __ldg(rec + 2);
            const float2 b = __ldg(reinterpret_cast<const float2*>(rec + 1));  // conic.z, opacity
            s_rec[tid].q0 = make_float4(a.x, a.y, -0.5f * a.z, -a.w);
            s_rec[tid].q1 = make_float4(-0.5f * b.x, b.y, col.x, col.y);
            s_rec[tid].q2 = make_float4(col.z, power_cut(b.y), __uint_as_float(cid), 0.f);
#pragma unroll
            for (int k = 0; k < BW_NACC; k++) s_acc[tid][k] = 0.0;
        }
        __syncthreads();
        for (int k = (int)cnt - 1; k >= 0; k--) {
            const uint32_t pos = lo + (uint32_t)k + 1u;  // list position + 1, as recorded
            const float4 q0 = s_rec[k].q0, q1 = s_rec[k].q1, q2 = s_rec[k].q2;
            const float dx = q0.x - fx, dy = q0.y - fy;
            float pw, e;
            if (MODE == GSB_MODE_EXACT) {  // k_blend's EXACT walk, op for op
                pw = ((q0.z * dx) * dx + (q1.x * dy) * dy) + (q0.w * dx) * dy;
                e = exp_shared_inrange(pw);
            } else {
                pw = fmaf(q0.z * dx, dx, fmaf(q1.x * dy, dy, (q0.w * dx) * dy));
                e = __expf(pw);
            }
            const float raw = q1.y * e;
            const float al = fminf(0.99f, raw);
            const bool contrib = pos <= last && !(pw > 0.0f || pw < q2.y) && !(al < 1.0f / 255.0f);
            if (!__any_sync(FULL, contrib)) continue;
            float v[BW_NACC];
#pragma unroll
            for (int j = 0; j < BW_NACC; j++) v[j] = 0.f;
            if (contrib) {
                T = T / (1.0f - al);  // transmittance in front of this entry
                const float w = al * T;
                v[6] = gr * w;  // d colour
                v[7] = gg * w;
                v[8] = gb * w;
                const float dal = T * ((gr * (q1.z - acc_r) + gg * (q1.w - acc_g)) + gb * (q2.x - acc_b));
                acc_r = q1.z * al + (1.0f - al) * acc_r;
                acc_g = q1.w * al + (1.0f - al) * acc_g;
                acc_b = q2.x * al + (1.0f - al) * acc_b;
                if (!(raw > 0.99f)) {           // alpha clamped at 0.99: no gradient through it
                    const float dpw = dal * raw;  // d alpha / d power = opacity * exp(power)
                    v[5] = dal * e;               // d opacity
                    // power = -A/2 dx^2 - C/2 dy^2 - B dx dy with (dx, dy) = uv - pixel
                    v[0] = dpw * (2.0f * q0.z * dx + q0.w * dy);  // d u
                    v[1] = dpw * (2.0f * q1.x * dy + q0.w * dx);  // d v
                    v[2] = dpw * (-0.5f * dx * dx);               // d A
                    v[3] = dpw * (-dx * dy);                      // d B
                    v[4] = dpw * (-0.5f * dy * dy);               // d C
                }
            }
#pragma unroll
            for (int j = 0; j < BW_NACC; j++) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(FULL, v[j], o);
            }
            if (lane == 0) {
#pragma unroll
                for (int j = 0; j < BW_NACC; j++)
                    if (v[j] != 0.f) atomicAdd(&s_acc[k][j], (double)v[j]);
            }
        }
        __syncthreads();
        if ((uint32_t)tid < cnt) {
            double* dst = P.scratch + (size_t)__float_as_uint(s_rec[tid].q2.z) * BW_NACC;
#pragma unroll
            for (int j = 0; j < BW_NACC; j++) {
                const double a = s_acc[tid][j];
                if (a != 0.0) atomicAdd(dst + j, a);
            }
        }
        hi = lo;
    }
}

// common.glsl:16-33
__device__ constexpr float SH_C0 = 0.28209479177387814f;
__device__ constexpr float SH_C1 = 0.4886025119029199f;
__device__ constexpr float SH_C2_0 = 1.0925484305920792f, SH_C2_1 = -1.0925484305920792f, SH_C2_2 = 0.31539156525252005f,
                           SH_C2_3 = -1.0925484305920792f, SH_C2_4 = 0.5462742152960396f;
__device__ constexpr float SH_C3_0 = -0.5900435899266435f, SH_C3_1 = 2.890611442640554f, SH_C3_2 = -0.4570457994644658f,
                           SH_C3_3 = 0.3731763325901154f, SH_C3_4 = -0.4570457994644658f, SH_C3_5 = 1.445305721320277f,
                           SH_C3_6 = -0.5900435899266435f;

__global__ void __launch_bounds__(PB_THREADS) k_preprocess_backward(const __grid_constant__ BackwardParams P) {
    const uint32_t nv = P.ctl->num_visible;
    const gsb_uniforms& U = P.ubo;
    const float* pm = U.proj_mat;
    const float* vm = U.view_mat;
    for (uint32_t cid = blockIdx.x * blockDim.x + threadIdx.x; cid < nv; cid += gridDim.x * blockDim.x) {
        double* sc = P.scratch + (size_t)cid * BW_NACC;
        float d[BW_NACC];
        bool any = false;
#pragma unroll
        for (int k = 0; k < BW_NACC; k++) {
            const double a = sc[k];
            d[k] = (float)a;
            any |= a != 0.0;
        }
        if (!any) continue;  // in no pixel's contributor set (or every gradient it received was zero)
#pragma unroll
        for (int k = 0; k < BW_NACC; k++) sc[k] = 0.0;
        const float4 r2 = __ldg(P.recs + (size_t)cid * GSB_REC_F4 + 2), r3 = __ldg(P.recs + (size_t)cid * GSB_REC_F4 + 3);
        const uint32_t i = __float_as_uint(r3.y);
        const float* v = P.vertices + (size_t)i * 60;
        float* gv = P.grad_vertices + (size_t)i * 60;
        const float px = v[0], py = v[1], pz = v[2];

        // ---- forward of preprocess.comp:130-157 (k_project's expressions) ----
        const float hx = ((pm[0] * px + pm[4] * py) + pm[8] * pz) + pm[12];
        const float hy = ((pm[1] * px + pm[5] * py) + pm[9] * pz) + pm[13];
        const float hw = ((pm[3] * px + pm[7] * py) + pm[11] * pz) + pm[15];
        const float p_w = 1.0f / hw;
        const float ndcx = hx * p_w, ndcy = hy * p_w;
        const float vx = ((vm[0] * px + vm[4] * py) + vm[8] * pz) + vm[12];
        const float vy = ((vm[1] * px + vm[5] * py) + vm[9] * pz) + vm[13];
        const float vz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14];
        const float limx = 1.3f * U.tan_fovx, limy = 1.3f * U.tan_fovy;
        const float txtz = vx / vz, tytz = vy / vz;
        const float tx = fminf(limx, fmaxf(-limx, txtz)) * vz;
        const float ty = fminf(limy, fmaxf(-limy, tytz)) * vz;
        const float focal_x = (float)U.width / (2.0f * U.tan_fovx);
        const float focal_y = (float)U.height / (2.0f * U.tan_fovy);
        const float ja = focal_x / vz, jb = focal_y / vz;
        const float g0 = -(focal_x * tx) / (vz * vz), g1 = -(focal_y * ty) / (vz * vz);
        float T0[3], T1[3];  // rows of J W (W = the view rotation)
#pragma unroll
        for (int r = 0; r < 3; r++) {
            T0[r] = vm[r * 4 + 0] * ja + vm[r * 4 + 2] * g0;
            T1[r] = vm[r * 4 + 1] * jb + vm[r * 4 + 2] * g1;
        }
        const float4 ca = __ldg(P.cov_a + i);
        const float2 cb = __ldg(P.cov_b + i);
        const float S[3][3] = {{ca.x, ca.y, ca.z}, {ca.y, ca.w, cb.x}, {ca.z, cb.x, cb.y}};
        float ST0[3], ST1[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            ST0[k] = (S[k][0] * T0[0] + S[k][1] * T0[1]) + S[k][2] * T0[2];
            ST1[k] = (S[k][0] * T1[0] + S[k][1] * T1[1]) + S[k][2] * T1[2];
        }
        const float a = ((T0[0] * ST0[0] + T0[1] * ST0[1]) + T0[2] * ST0[2]) + 0.3f;
        const float b = (T1[0] * ST0[0] + T1[1] * ST0[1]) + T1[2] * ST0[2];
        const float c = ((T1[0] * ST1[0] + T1[1] * ST1[1]) + T1[2] * ST1[2]) + 0.3f;
        const float det = a * c - b * b;

        // ---- conic = (c, -b, a) / det  ->  cov2d (a, b, c) ----
        const float id2 = 1.0f / (det * det);
        const float dA = d[2], dB = d[3], dC = d[4];
        const float da = id2 * ((-c * c * dA + b * c * dB) - b * b * dC);
        const float db = id2 * ((2.0f * b * c * dA - (det + 2.0f * b * b) * dB) + 2.0f * a * b * dC);
        const float dc = id2 * ((-b * b * dA + a * b * dB) - a * a * dC);
        // cov2d = (J W) Sigma (J W)^T: dL/dSigma (symmetric) and dL/d(J W)
        float G[3][3];
#pragma unroll
        for (int j = 0; j < 3; j++)
#pragma unroll
            for (int k = 0; k < 3; k++) G[j][k] = (da * T0[j] * T0[k] + dc * T1[j] * T1[k]) + 0.5f * db * (T0[j] * T1[k] + T1[j] * T0[k]);
        float dT0[3], dT1[3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            dT0[j] = 2.0f * da * ST0[j] + db * ST1[j];
            dT1[j] = 2.0f * dc * ST1[j] + db * ST0[j];
        }
        // J W -> J = (ja, 0, g0; 0, jb, g1) -> view-space position
        float dja = 0.f, dg0 = 0.f, djb = 0.f, dg1 = 0.f;
#pragma unroll
        for (int r = 0; r < 3; r++) {
            dja += dT0[r] * vm[r * 4 + 0];
            dg0 += dT0[r] * vm[r * 4 + 2];
            djb += dT1[r] * vm[r * 4 + 1];
            dg1 += dT1[r] * vm[r * 4 + 2];
        }
        float dvx = 0.f, dvy = 0.f, dvz = -(ja / vz) * dja - (jb / vz) * djb;
        const float dtx = -(focal_x / (vz * vz)) * dg0, dty = -(focal_y / (vz * vz)) * dg1;
        dvz += -(2.0f * g0 / vz) * dg0 - (2.0f * g1 / vz) * dg1;
        // t.x = clamp(v.x / v.z, +-1.3 tan_fovx) v.z: identity in v.x inside the clamp, +-lim v.z outside it
        if (txtz < -limx || txtz > limx) dvz += (txtz > 0.0f ? limx : -limx) * dtx;
        else dvx += dtx;
        if (tytz < -limy || tytz > limy) dvz += (tytz > 0.0f ? limy : -limy) * dty;
        else dvy += dty;
        // uv = ((ndc + 1) size - 1) / 2, ndc = h.xy / h.w
        const float dndcx = d[0] * (0.5f * (float)U.width), dndcy = d[1] * (0.5f * (float)U.height);
        const float dhx = dndcx * p_w, dhy = dndcy * p_w, dhw = -(dndcx * ndcx + dndcy * ndcy) * p_w;
        float dp[3];
#pragma unroll
        for (int k = 0; k < 3; k++)
            dp[k] = ((pm[k * 4 + 0] * dhx + pm[k * 4 + 1] * dhy) + pm[k * 4 + 3] * dhw) + ((vm[k * 4 + 0] * dvx + vm[k * 4 + 1] * dvy) + vm[k * 4 + 2] * dvz);

        // ---- colour (preprocess.comp:73-108) -> SH coefficients and the view direction ----
        const float dcr = r2.x > 0.0f ? d[6] : 0.0f;  // :102-104 red clamped at 0 (the record holds the clamped value)
        const float dcg = d[7], dcb = d[8];
        const float ex = px - U.camera_position[0], ey = py - U.camera_position[1], ez = pz - U.camera_position[2];
        const float len = sqrtf((ex * ex + ey * ey) + ez * ez);
        const float x = ex / len, y = ey / len, z = ez / len;
        const float xx = x * x, yy = y * y, zz = z * z;
        const float basis[16] = {SH_C0,
                                 -SH_C1 * y,
                                 SH_C1 * z,
                                 -SH_C1 * x,
                                 SH_C2_0 * x * y,
                                 SH_C2_1 * y * z,
                                 SH_C2_2 * ((2.0f * zz - xx) - yy),
                                 SH_C2_3 * z * x,
                                 SH_C2_4 * (xx - yy),
                                 SH_C3_0 * (3.0f * xx - yy) * y,
                                 SH_C3_1 * x * y * z,
                                 SH_C3_2 * ((4.0f * zz - xx) - yy) * y,
                                 SH_C3_3 * z * ((2.0f * zz - 3.0f * xx) - 3.0f * yy),
                                 SH_C3_4 * x * ((4.0f * zz - xx) - yy),
                                 SH_C3_5 * (xx - yy) * z,
                                 SH_C3_6 * x * (xx - 3.0f * yy)};
        const float* sh = v + 12;
        float vk[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            gv[12 + 3 * k + 0] = basis[k] * dcr;
            gv[12 + 3 * k + 1] = basis[k] * dcg;
            gv[12 + 3 * k + 2] = basis[k] * dcb;
            vk[k] = (sh[3 * k] * dcr + sh[3 * k + 1] * dcg) + sh[3 * k + 2] * dcb;
        }
        const float ddx = -SH_C1 * vk[3] + SH_C2_0 * y * vk[4] - 2.0f * SH_C2_2 * x * vk[6] + SH_C2_3 * z * vk[7] + 2.0f * SH_C2_4 * x * vk[8] +
                          6.0f * SH_C3_0 * x * y * vk[9] + SH_C3_1 * y * z * vk[10] - 2.0f * SH_C3_2 * x * y * vk[11] -
                          6.0f * SH_C3_3 * x * z * vk[12] + SH_C3_4 * ((4.0f * zz - 3.0f * xx) - yy) * vk[13] + 2.0f * SH_C3_5 * x * z * vk[14] +
                          3.0f * SH_C3_6 * (xx - yy) * vk[15];
        const float ddy = -SH_C1 * vk[1] + SH_C2_0 * x * vk[4] + SH_C2_1 * z * vk[5] - 2.0f * SH_C2_2 * y * vk[6] - 2.0f * SH_C2_4 * y * vk[8] +
                          3.0f * SH_C3_0 * (xx - yy) * vk[9] + SH_C3_1 * x * z * vk[10] + SH_C3_2 * ((4.0f * zz - xx) - 3.0f * yy) * vk[11] -
                          6.0f * SH_C3_3 * y * z * vk[12] - 2.0f * SH_C3_4 * x * y * vk[13] - 2.0f * SH_C3_5 * y * z * vk[14] -
                          6.0f * SH_C3_6 * x * y * vk[15];
        const float ddz = SH_C1 * vk[2] + SH_C2_1 * y * vk[5] + 4.0f * SH_C2_2 * z * vk[6] + SH_C2_3 * x * vk[7] + SH_C3_1 * x * y * vk[10] +
                          8.0f * SH_C3_2 * y * z * vk[11] + SH_C3_3 * ((6.0f * zz - 3.0f * xx) - 3.0f * yy) * vk[12] + 8.0f * SH_C3_4 * x * z * vk[13] +
                          SH_C3_5 * (xx - yy) * vk[14];
        const float dot = (x * ddx + y * ddy) + z * ddz;  // d (e / |e|) = (I - dir dir^T) / |e|
        dp[0] += (ddx - x * dot) / len;
        dp[1] += (ddy - y * dot) / len;
        dp[2] += (ddz - z * dot) / len;

        // ---- Sigma = M^T M, M = diag(s) R(q) (precomp_cov3d.comp:25-48, the quaternion as stored) ----
        const float s[3] = {v[4], v[5], v[6]};
        const float qw = v[8], qx = v[9], qy = v[10], qz = v[11];
        float R[3][3];  // R[c][r] as in k_ingest_cov3d
        R[0][0] = (1.0f - 2.0f * qy * qy) - 2.0f * qz * qz;
        R[0][1] = (2.0f * qx) * qy - (2.0f * qz) * qw;
        R[0][2] = (2.0f * qx) * qz + (2.0f * qy) * qw;
        R[1][0] = (2.0f * qx) * qy + (2.0f * qz) * qw;
        R[1][1] = (1.0f - 2.0f * qx * qx) - 2.0f * qz * qz;
        R[1][2] = (2.0f * qy) * qz - (2.0f * qx) * qw;
        R[2][0] = (2.0f * qx) * qz - (2.0f * qy) * qw;
        R[2][1] = (2.0f * qy) * qz + (2.0f * qx) * qw;
        R[2][2] = (1.0f - 2.0f * qx * qx) - 2.0f * qy * qy;
        float ds[3] = {0.f, 0.f, 0.f}, dR[3][3];
#pragma unroll
        for (int r = 0; r < 3; r++) {  // row r of M: M_rc = s_r R[c][r];  dL/dM = 2 M G
#pragma unroll
            for (int cc = 0; cc < 3; cc++) {
                const float dm = 2.0f * s[r] * ((R[0][r] * G[0][cc] + R[1][r] * G[1][cc]) + R[2][r] * G[2][cc]);
                ds[r] += dm * R[cc][r];
                dR[cc][r] = s[r] * dm;
            }
        }
        const float dqw = 2.0f * (((-qz * dR[0][1] + qy * dR[0][2]) + (qz * dR[1][0] - qx * dR[1][2])) + (-qy * dR[2][0] + qx * dR[2][1]));
        const float dqx = 2.0f * (((qy * dR[0][1] + qz * dR[0][2]) + (qy * dR[1][0] - 2.0f * qx * dR[1][1] - qw * dR[1][2])) +
                                  (qz * dR[2][0] + qw * dR[2][1] - 2.0f * qx * dR[2][2]));
        const float dqy = 2.0f * (((-2.0f * qy * dR[0][0] + qx * dR[0][1] + qw * dR[0][2]) + (qx * dR[1][0] + qz * dR[1][2])) +
                                  (-qw * dR[2][0] + qz * dR[2][1] - 2.0f * qy * dR[2][2]));
        const float dqz = 2.0f * (((-2.0f * qz * dR[0][0] - qw * dR[0][1] + qx * dR[0][2]) + (qw * dR[1][0] - 2.0f * qz * dR[1][1] + qy * dR[1][2])) +
                                  (qx * dR[2][0] + qy * dR[2][1]));

        gv[0] = dp[0];
        gv[1] = dp[1];
        gv[2] = dp[2];
        gv[4] = ds[0];
        gv[5] = ds[1];
        gv[6] = ds[2];
        gv[7] = d[5];
        gv[8] = dqw;
        gv[9] = dqx;
        gv[10] = dqy;
        gv[11] = dqz;
    }
}

}  // namespace

cudaError_t launch_backward(const BackwardParams& p, cudaStream_t s) {
    if (p.num_tiles) {
        if (p.mode == GSB_MODE_EXACT) k_blend_backward<GSB_MODE_EXACT><<<p.num_tiles, BW_THREADS, 0, s>>>(p);
        else k_blend_backward<GSB_MODE_FAST><<<p.num_tiles, BW_THREADS, 0, s>>>(p);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    // grid-stride over N_v, which stays on the device: the grid comes from the SM count
    k_preprocess_backward<<<(unsigned)p.num_sms * 4u, PB_THREADS, 0, s>>>(p);
    return cudaGetLastError();
}

}  // namespace gsb
