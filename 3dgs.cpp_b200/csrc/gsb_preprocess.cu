// gsb_preprocess.cu -- the reference's first three stages, re-cut for a two-level LSD sort.
//
//   k_project  = preprocess.comp:115-182 (project, cull, EWA cov2d, conic, radius, tile AABB,
//                degree-3 SH colour) + stream compaction of the cull survivors (single-pass
//                decoupled look-back scan).  Per survivor it writes the 48-B blend record, the
//                tile AABB and the 32-bit depth key of the Gaussian-level sort.
//   k_emit     = prefix_sum.comp:32-58 (x (log2 N + 1) dispatches, Renderer.cpp:497-526) +
//                preprocess_sort.comp:31-60: one single-pass decoupled look-back scan of the tile
//                counts and the emission of one (tile id, payload) pair per covered tile -- but
//                over the survivors in DEPTH order (after the Gaussian-level sort), so the low 32
//                key bits of the reference's 64-bit (tile << 32 | depth) key are already in order
//                and only the tile id is left to sort at instance granularity (DESIGN.md).
// Both remove the mid-frame fence + host read of M (Renderer.cpp:391,538): counts stay in HBM.
//
// Arithmetic: compiled with -fmad=false; every fp32 operation is a single IEEE op in the order
// of the GLSL source, so results are value-identical to the oracle (bit-exact parity).
#include <cuda_fp16.h>

#include <cmath>

#include "gsb_cull.cuh"
#include "gsb_geom.cuh"
#include "gsb_internal.cuh"

namespace gsb {

namespace {

constexpr int PRE_THREADS = 256;
constexpr unsigned FULL = 0xffffffffu;

template <typename T>
__device__ __forceinline__ T ld_vol(const T* p) {
    return *reinterpret_cast<const volatile T*>(p);
}
template <typename T>
__device__ __forceinline__ void st_vol(T* p, T v) {
    *reinterpret_cast<volatile T*>(p) = v;
}

// Single-pass decoupled look-back scan over chunks.  One status word per chunk: the top two bits are the flag (0 = nothing
// published yet, AGG = the chunk's own count, PREFIX = the inclusive prefix up to and including the chunk), the rest the
// count.  k_project scans survivors with u32 words ([29:0]), k_emit instances with u64 words ([61:0]).
template <typename W>
struct Lookback {
    static constexpr int SHIFT = 8 * sizeof(W) - 2;
    static constexpr W AGG = W(1) << SHIFT, PREFIX = W(2) << SHIFT, FLAGS = W(3) << SHIFT, COUNT = AGG - W(1);
    // the word a chunk publishes as soon as it knows its own count (chunk 0's count is its inclusive prefix)
    static __device__ __forceinline__ W aggregate(uint32_t chunk, W count) { return (chunk == 0 ? PREFIX : AGG) | count; }
};

// Run by all 32 lanes of one warp: returns the exclusive prefix of `chunk` and publishes its inclusive prefix (+ `total`, the
// chunk's own count).  Chunk k's word is status[k * stride] (the routed k_project keeps one column per destination).  The
// predecessors are polled 32 at a time; the sum stops at the nearest one that has published its inclusive prefix.
template <typename W>
__device__ __forceinline__ W lookback_exclusive(W* status, uint32_t stride, uint32_t chunk, int lane, W total) {
    using L = Lookback<W>;
    W ex = 0;
    if (chunk != 0) {
        int look = (int)chunk - 1;
        while (true) {
            const int idx = look - lane;
            W st = L::PREFIX;  // virtual predecessor of chunk 0
            if (idx >= 0) {
                st = ld_vol(status + (size_t)idx * stride);
                while ((st & L::FLAGS) == 0) st = ld_vol(status + (size_t)idx * stride);
            }
            const unsigned pm = __ballot_sync(FULL, (st & L::FLAGS) == L::PREFIX);
            const int first = pm ? (__ffs(pm) - 1) : 32;
            W cs = (lane <= first) ? (st & L::COUNT) : W(0);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) cs += __shfl_xor_sync(FULL, cs, o);
            ex += cs;
            if (pm) break;
            look -= 32;
        }
        if (lane == 0) st_vol(status + (size_t)chunk * stride, L::PREFIX | (ex + total));
    }
    return ex;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

struct ShDir {
    float x, y, z, w6, w8, w9, w11, w12, w15;
};

// one term of preprocess.comp:80-98, in the shader's association order
template <int K>
__device__ __forceinline__ float sh_term(float a, float s, const ShDir& d) {
    if constexpr (K == 0) return SH_C0 * s;
    else if constexpr (K == 1) return a - (SH_C1 * s) * d.y;
    else if constexpr (K == 2) return a + (SH_C1 * s) * d.z;
    else if constexpr (K == 3) return a - (SH_C1 * s) * d.x;
    else if constexpr (K == 4) return a + ((SH_C2_0 * s) * d.x) * d.y;
    else if constexpr (K == 5) return a + ((SH_C2_1 * s) * d.y) * d.z;
    else if constexpr (K == 6) return a + (SH_C2_2 * s) * d.w6;
    else if constexpr (K == 7) return a + ((SH_C2_3 * s) * d.z) * d.x;
    else if constexpr (K == 8) return a + (SH_C2_4 * s) * d.w8;
    else if constexpr (K == 9) return a + ((SH_C3_0 * s) * d.w9) * d.y;
    else if constexpr (K == 10) return a + (((SH_C3_1 * s) * d.x) * d.y) * d.z;
    else if constexpr (K == 11) return a + ((SH_C3_2 * s) * d.w11) * d.y;
    else if constexpr (K == 12) return a + ((SH_C3_3 * s) * d.z) * d.w12;
    else if constexpr (K == 13) return a + ((SH_C3_4 * s) * d.x) * d.w11;
    else if constexpr (K == 14) return a + ((SH_C3_5 * s) * d.w8) * d.z;
    else return a + ((SH_C3_6 * s) * d.x) * d.w15;
}

template <int G, bool SH16>
__device__ __forceinline__ void sh_group(const float4* __restrict__ sh4, float (&c)[3], const ShDir& d) {
    // coefficients 4G .. 4G+3 = floats 12G .. 12G+11 = three float4 (SH16, non-parity: 12 halves = three 8-B words)
    float f[12];
    if constexpr (SH16) {
        const uint2* sh2 = reinterpret_cast<const uint2*>(sh4);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const uint2 w = __ldg(sh2 + 3 * G + k);
            const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&w.x)), hi = __half22float2(*reinterpret_cast<const __half2*>(&w.y));
            f[4 * k + 0] = lo.x, f[4 * k + 1] = lo.y, f[4 * k + 2] = hi.x, f[4 * k + 3] = hi.y;
        }
    } else {
        const float4 t0 = __ldg(sh4 + 3 * G), t1 = __ldg(sh4 + 3 * G + 1), t2 = __ldg(sh4 + 3 * G + 2);
        f[0] = t0.x, f[1] = t0.y, f[2] = t0.z, f[3] = t0.w, f[4] = t1.x, f[5] = t1.y, f[6] = t1.z, f[7] = t1.w;
        f[8] = t2.x, f[9] = t2.y, f[10] = t2.z, f[11] = t2.w;
    }
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
        c[ch] = sh_term<4 * G + 0>(c[ch], f[0 + ch], d);
        c[ch] = sh_term<4 * G + 1>(c[ch], f[3 + ch], d);
        c[ch] = sh_term<4 * G + 2>(c[ch], f[6 + ch], d);
        c[ch] = sh_term<4 * G + 3>(c[ch], f[9 + ch], d);
    }
}

// preprocess.comp:73-108 compute_sh(); sh = 48 floats RGB-interleaved, as 12 float4 (SH16: 48 halves).
template <bool SH16>
__device__ __forceinline__ void compute_sh(const float4* __restrict__ sh4, float px, float py, float pz,
                                           const float* cam, float& r, float& g, float& b) {
    ShDir d;
    view_direction(cam, px, py, pz, d.x, d.y, d.z);
    const float xx = d.x * d.x, yy = d.y * d.y;
    d.w6 = ((2.0f * d.z) * d.z - xx) - yy;
    d.w8 = xx - yy;
    d.w9 = (3.0f * d.x) * d.x - yy;
    d.w11 = ((4.0f * d.z) * d.z - xx) - yy;
    d.w12 = ((2.0f * d.z) * d.z - (3.0f * d.x) * d.x) - (3.0f * d.y) * d.y;
    d.w15 = xx - (3.0f * d.y) * d.y;
    float c[3] = {0.f, 0.f, 0.f};
    sh_group<0, SH16>(sh4, c, d);
    sh_group<1, SH16>(sh4, c, d);
    sh_group<2, SH16>(sh4, c, d);
    sh_group<3, SH16>(sh4, c, d);
    c[0] = c[0] + 0.5f;
    c[1] = c[1] + 0.5f;
    c[2] = c[2] + 0.5f;
    r = c[0] < 0.0f ? 0.0f : c[0];  // :102-104 only the red channel is clamped
    g = c[1];
    b = c[2];
}

// The first coefficient 4G of group G alone: floats 12G .. 12G+2 of the first of the group's three words.
template <int G, bool SH16>
__device__ __forceinline__ void sh_group_head(const float4* __restrict__ sh4, float (&c)[3], const ShDir& d) {
    float f[3];
    if constexpr (SH16) {
        const uint2 w = __ldg(reinterpret_cast<const uint2*>(sh4) + 3 * G);
        const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&w.x)), hi = __half22float2(*reinterpret_cast<const __half2*>(&w.y));
        f[0] = lo.x, f[1] = lo.y, f[2] = hi.x;
    } else {
        const float4 t0 = __ldg(sh4 + 3 * G);
        f[0] = t0.x, f[1] = t0.y, f[2] = t0.z;
    }
#pragma unroll
    for (int ch = 0; ch < 3; ch++) c[ch] = sh_term<4 * G>(c[ch], f[ch], d);
}

// compute_sh at gsb_set_sh_degree's degree deg in 0..2 (warp-uniform): the sum over the (deg + 1)^2 coefficients of bands <= deg
// only, in compute_sh's order, reading only the words that hold them -- 1 float4 (SH16: uint2) at degree 0, 3 at 1, 7 at 2
// (degree 2 ends at coefficient 8, the head of group 2).  Degree 0 needs no view direction.  Each dropped term of compute_sh is
// a + (C 0) w = a for a finite direction, so this is compute_sh of the scene with the dropped bands zeroed (DESIGN.md section 25).
template <bool SH16>
__device__ __forceinline__ void compute_sh_degree(const float4* __restrict__ sh4, float px, float py, float pz, const float* cam, int deg,
                                                  float& r, float& g, float& b) {
    float c[3] = {0.f, 0.f, 0.f};
    ShDir d{};
    if (deg == 0) {
        sh_group_head<0, SH16>(sh4, c, d);  // SH_C0 s: the direction takes no part
    } else {
        view_direction(cam, px, py, pz, d.x, d.y, d.z);
        const float xx = d.x * d.x, yy = d.y * d.y;
        d.w6 = ((2.0f * d.z) * d.z - xx) - yy;
        d.w8 = xx - yy;
        sh_group<0, SH16>(sh4, c, d);
        if (deg >= 2) {
            sh_group<1, SH16>(sh4, c, d);
            sh_group_head<2, SH16>(sh4, c, d);
        }
    }
    c[0] = c[0] + 0.5f;
    c[1] = c[1] + 0.5f;
    c[2] = c[2] + 0.5f;
    r = c[0] < 0.0f ? 0.0f : c[0];
    g = c[1];
    b = c[2];
}

// ------------------------------------------------------------------------------------------
// k_project
// ------------------------------------------------------------------------------------------
#ifndef GSB_PROJECT_MIN_BLOCKS
#define GSB_PROJECT_MIN_BLOCKS 6  // <= 42 registers: 6 CTAs (48 warps) per SM hide the SH gather latency
#endif
#ifndef GSB_PROJECT_FISHEYE_MIN_BLOCKS
#define GSB_PROJECT_FISHEYE_MIN_BLOCKS 4
#endif
#ifndef GSB_PROJECT_OPENCV_MIN_BLOCKS
#define GSB_PROJECT_OPENCV_MIN_BLOCKS 4
#endif
// ROUTED (frame sharding, gsb_shard.cu): the single stream compaction becomes one compaction per destination band -- G
// simultaneous decoupled look-back scans over G-wide status vectors, warp d walking column d -- and the record goes straight
// from registers into the exchange buffer of every rank whose band the AABB touches (stores into peer-mapped memory over
// NVLink).  Slots are deterministic (Gaussian-index order inside this source's region), so every band's survivor list is
// ordered exactly like the single-GPU compaction and the band's pixels are bit-identical.
// AA (gsb_set_antialiased, plain contexts only): the stored opacity is scaled by sqrt(det(cov2d) / det(cov2d + 0.3 I)); the
// conic, radius, AABB and survivor set are those of AA = false.
// FISHEYE (gsb_set_camera_model, plain contexts only): the projection, Jacobian and cull of the fisheye lens (gsb_geom.cuh's
// fisheye_geo / fisheye_jacobian) and the depth key d = |t| instead of z; everything from cov2d on is the pinhole path's.
// OPENCV (gsb_set_camera_model, plain contexts only): the projection, Jacobian and cull of the OpenCV lens (opencv_geo /
// opencv_jacobian); the depth key stays z.
// SHDEG (gsb_set_sh_degree below 3, plain contexts only): the colour is compute_sh_degree's at P.sh_degree; the launch bounds
// are the lens family's.
// ORTHO (gsb_set_camera_model, plain contexts only): the orthographic camera (ortho_jacobian): uv = (fx x + cx, fy y + cy),
// culled unless z > 0.2 (NaN culled), depth key z, and the SH colour seen along the camera's forward axis (ortho_direction)
// rather than from camera_position.  It takes the pinhole's launch bounds.
template <bool FISHEYE, bool OPENCV = false>
struct ProjectBounds {
    static constexpr int MIN_BLOCKS = GSB_PROJECT_MIN_BLOCKS;
};
template <>
struct ProjectBounds<true> {
    static constexpr int MIN_BLOCKS = GSB_PROJECT_FISHEYE_MIN_BLOCKS;
};
template <>
struct ProjectBounds<false, true> {
    static constexpr int MIN_BLOCKS = GSB_PROJECT_OPENCV_MIN_BLOCKS;
};
template <bool DEBUG, bool ROUTED, bool SH16, bool AA, bool FISHEYE = false, bool OPENCV = false, bool SHDEG = false, bool ORTHO = false>
__global__ void __launch_bounds__(PRE_THREADS, ProjectBounds<FISHEYE, OPENCV>::MIN_BLOCKS)
    k_project(const __grid_constant__ ProjectParams P) {
    static_assert(!(ROUTED && AA), "sharded contexts have no anti-aliased mode");
    static_assert(!(ROUTED && FISHEYE), "sharded contexts have no fisheye camera");
    static_assert(!(ROUTED && OPENCV) && !(FISHEYE && OPENCV), "sharded contexts have no OpenCV camera; one lens per frame");
    static_assert(!(ROUTED && SHDEG), "sharded contexts have only degree 3");
    static_assert(!(ROUTED && ORTHO) && !((FISHEYE || OPENCV) && ORTHO), "sharded contexts have no orthographic camera; one lens per frame");
    __shared__ uint32_t s_chunk;
    __shared__ uint32_t s_wsurv[PRE_THREADS / 32];
    __shared__ uint32_t s_base_surv;
    __shared__ uint32_t s_rcnt[ROUTED ? PRE_THREADS / 32 : 1][GSB_MAX_SHARDS];  // per warp, per destination: touching lanes
    __shared__ uint32_t s_rbase[GSB_MAX_SHARDS];                                // chunk total, then exclusive base

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_chunk = atomicAdd(&P.ctl->project_ticket, 1u);
    __syncthreads();
    const uint32_t chunk = s_chunk;
    const uint32_t num_chunks = (P.n + PRE_THREADS - 1) / PRE_THREADS;
    const uint32_t i = chunk * PRE_THREADS + tid;

    const gsb_uniforms& U = P.ubo;
    const int W = (int)U.width, H = (int)U.height;
    const int tiles_x = (int)((U.width + GSB_TILE - 1) / GSB_TILE);
    const int tiles_y = (int)((U.height + GSB_TILE - 1) / GSB_TILE);

    bool surv = false;
    uint32_t nt = 0;
    float uvx = 0.f, uvy = 0.f, conx = 0.f, cony = 0.f, conz = 0.f, opac = 0.f, depth = 0.f, radii = 0.f;
    float px = 0.f, py = 0.f, pz = 0.f;
    int bx0 = 0, by0 = 0, bx1 = 0, by1 = 0;

    if (i < P.n) {
        const float4 po = __ldg(P.pos_op + i);
        px = po.x;
        py = po.y;
        pz = po.z;
        opac = po.w;
        const ClipView cv = clip_view(U, px, py, pz);
        const float ndcx = cv.ndcx, ndcy = cv.ndcy, vz = cv.vz;
        FisheyeGeo F;
        OpencvGeo O;
        bool front;
        if constexpr (FISHEYE) {
            F = fisheye_geo(P.camera, cv.vx, cv.vy, vz);
            front = F.d > 0.2f && F.theta <= P.camera.max_theta;  // NaN is culled
        } else if constexpr (OPENCV) {
            O = opencv_geo(P.camera, cv.vx, cv.vy, vz);
            front = vz > 0.2f && O.r2 <= P.tan2_max && O.det > 0.0f;  // NaN is culled; so is a tangential fold
        } else if constexpr (ORTHO) {
            front = vz > 0.2f;  // NaN is culled
        } else {
            front = !(vz <= 0.2f);  // :135 (NaN is not culled by the shader's test either)
        }
        if (front) {
            Cov2d cov;
            if constexpr (FISHEYE) {
                const LensJ J = fisheye_jacobian(P.camera, U.view_mat, F, cv.vx, cv.vy);
                cov = cov2d(J.T0, J.T1, __ldg(P.cov_a + i), __ldg(P.cov_b + i));
            } else if constexpr (OPENCV) {
                const LensJ J = opencv_jacobian(P.camera, U.view_mat, O, vz);
                cov = cov2d(J.T0, J.T1, __ldg(P.cov_a + i), __ldg(P.cov_b + i));
            } else if constexpr (ORTHO) {
                const LensJ J = ortho_jacobian(P.camera, U.view_mat);
                cov = cov2d(J.T0, J.T1, __ldg(P.cov_a + i), __ldg(P.cov_b + i));
            } else {
                const Jacobian J = jacobian(U, cv.vx, cv.vy, vz);
                cov = cov2d(J.T0, J.T1, __ldg(P.cov_a + i), __ldg(P.cov_b + i));
            }
            const float m00 = cov.m00, m01 = cov.m01, m10 = cov.m10, m11 = cov.m11;
            const float det = m00 * m11 - m10 * m01;  // :138
            if (!(det <= 0.0f)) {                                                  // :139-141
                const float ood = 1.0f / det;
                conx = m11 * ood;
                cony = -m01 * ood;
                conz = m00 * ood;  // :142-143
                if constexpr (AA) opac = opac * aa_compensation(aa_det0(cov), det);
                const float mid = 0.5f * (m00 + m11);
                const float sq = sqrtf(fmaxf(0.1f, mid * mid - det));
                const float lambda = fmaxf(mid + sq, mid - sq);
                radii = ceilf(3.0f * sqrtf(lambda));                     // :146-151
                if constexpr (FISHEYE) {
                    uvx = P.camera.fx * (F.s * cv.vx) + P.camera.cx;
                    uvy = P.camera.fy * (F.s * cv.vy) + P.camera.cy;
                } else if constexpr (OPENCV) {
                    uvx = P.camera.fx * O.xd + P.camera.cx;
                    uvy = P.camera.fy * O.yd + P.camera.cy;
                } else if constexpr (ORTHO) {
                    uvx = P.camera.fx * cv.vx + P.camera.cx;
                    uvy = P.camera.fy * cv.vy + P.camera.cy;
                } else {
                    uvx = ((ndcx + 1.0f) * (float)W - 1.0f) * 0.5f;  // :157 ndc2Pix
                    uvy = ((ndcy + 1.0f) * (float)H - 1.0f) * 0.5f;
                }
                // :159-164; cvt.rzi.s32.f32 saturates where GLSL int() is undefined
                bx0 = clampi(__float2int_rz((uvx - radii) / 16.0f), 0, tiles_x);
                by0 = clampi(__float2int_rz((uvy - radii) / 16.0f), 0, tiles_y);
                bx1 = clampi(__float2int_rz((((uvx + radii) + 16.0f) - 1.0f) / 16.0f), 0, tiles_x);  // "+ TILE_WIDTH - 1"
                by1 = clampi(__float2int_rz((((uvy + radii) + 16.0f) - 1.0f) / 16.0f), 0, tiles_y);
                // multi-GPU band clip (identity for the whole frame)
                if ((uint32_t)by0 < P.tile_row_begin) by0 = (int)P.tile_row_begin;
                if ((uint32_t)by1 > P.tile_row_end) by1 = (int)P.tile_row_end;
                if (by1 < by0) by1 = by0;
                nt = (uint32_t)(bx1 - bx0) * (uint32_t)(by1 - by0);  // :168
                surv = nt != 0;                                      // :169-171
                depth = FISHEYE ? F.d : vz;
            }
        }
    }

    if constexpr (ROUTED) {
        const int G = P.route_world;
        // ---- per destination band: does the AABB touch it, rank among the warp's touching lanes (5 bits each, packed) ----
        uint32_t touch = 0;
        unsigned long long ranks = 0ull;
#pragma unroll
        for (int d = 0; d < GSB_MAX_SHARDS; d++) {
            if (d < G) {
                const int b0 = d * (int)P.band_rows, b1 = b0 + (int)P.band_rows;
                const bool t = surv && max(by0, b0) < min(by1, b1);
                const unsigned bits = __ballot_sync(FULL, t);
                if (t) touch |= 1u << d;
                ranks |= (unsigned long long)__popc(bits & ((1u << lane) - 1u)) << (5 * d);
                if (lane == 0) s_rcnt[warp][d] = __popc(bits);
            }
        }
        __syncthreads();
        if (tid < G) {  // thread d: exclusive scan over the warps, chunk total, publish the aggregate as early as possible
            uint32_t run = 0;
#pragma unroll
            for (int w = 0; w < PRE_THREADS / 32; w++) {
                const uint32_t c = s_rcnt[w][tid];
                s_rcnt[w][tid] = run;
                run += c;
            }
            s_rbase[tid] = run;
            st_vol(P.route_status + (size_t)chunk * GSB_MAX_SHARDS + tid, Lookback<uint32_t>::aggregate(chunk, run));
        }
        // ---- SH colour of survivors (overlaps the look-back of other chunks) ----
        float colr = 0.f, colg = 0.f, colb = 0.f;
        if (surv) compute_sh<SH16>(reinterpret_cast<const float4*>(P.sh) + (size_t)i * (SH16 ? 6 : 12), px, py, pz, U.camera_position, colr, colg, colb);
        __syncthreads();
        // ---- decoupled look-back: warp d walks column d of the status vectors, 32 predecessors per step ----
        if (warp < G) {
            const int d = warp;
            const uint32_t total = s_rbase[d];
            const uint32_t ex = lookback_exclusive(P.route_status + d, GSB_MAX_SHARDS, chunk, lane, total);
            __syncwarp();
            if (lane == 0) {
                s_rbase[d] = ex;
                if (chunk == num_chunks - 1) P.ctl->route_total[d] = ex + total;
            }
        }
        __syncthreads();
        // ---- deliver: one 64-B record + depth key per touched band, straight from registers ----
        if (touch) {
            const float4 q0 = make_float4(uvx, uvy, conx, cony);
            const float4 q2 = make_float4(colr, colg, colb, depth);
            const float4 q3 = make_float4(radii, __uint_as_float(P.index_base + i), 0.f, 0.f);
            const uint32_t dk = __float_as_uint(depth);
#pragma unroll
            for (int d = 0; d < GSB_MAX_SHARDS; d++) {
                if (d < G && ((touch >> d) & 1u)) {
                    const uint32_t pos = s_rbase[d] + s_rcnt[warp][d] + (uint32_t)((ranks >> (5 * d)) & 31ull);
                    const int b0 = d * (int)P.band_rows, b1 = b0 + (int)P.band_rows;
                    const int cy0 = max(by0, b0), cy1 = min(by1, b1);  // the band clip k_project applies on one GPU
                    float4* dst = P.route_dst_recs[d] + (size_t)pos * GSB_REC_F4;
                    dst[0] = q0;
                    dst[1] = make_float4(conz, opac, __uint_as_float((uint32_t)bx0 | ((uint32_t)cy0 << 16)),
                                         __uint_as_float((uint32_t)(bx1 - bx0) | ((uint32_t)(cy1 - cy0) << 16)));
                    dst[2] = q2;
                    dst[3] = q3;
                    P.route_dst_dkeys[d][pos] = dk;
                }
            }
        }
    } else {
    // ---- block scan of the survivor flags ----
    const unsigned surv_mask = __ballot_sync(FULL, surv);
    const uint32_t surv_rank_w = __popc(surv_mask & ((1u << lane) - 1u));
    if (lane == 0) s_wsurv[warp] = __popc(surv_mask);
    __syncthreads();
    uint32_t surv_before = 0, blk_surv = 0;
#pragma unroll
    for (int w = 0; w < PRE_THREADS / 32; w++) {
        const uint32_t a = s_wsurv[w];
        if (w < warp) surv_before += a;
        blk_surv += a;
    }
    // publish this chunk's aggregate as early as possible
    if (tid == 0) st_vol(P.status + chunk, Lookback<uint32_t>::aggregate(chunk, blk_surv));

    // ---- SH colour of survivors (overlaps the look-back of other chunks) ----
    float colr = 0.f, colg = 0.f, colb = 0.f;
    if constexpr (ORTHO) {  // the direction from the origin to view row 2: ortho_direction's, the same for every Gaussian
        const float origin[3] = {0.0f, 0.0f, 0.0f};
        const float fx = U.view_mat[2], fy = U.view_mat[6], fz = U.view_mat[10];
        const float4* sh4 = reinterpret_cast<const float4*>(P.sh) + (size_t)i * (SH16 ? 6 : 12);
        if constexpr (SHDEG) {
            if (surv) compute_sh_degree<SH16>(sh4, fx, fy, fz, origin, P.sh_degree, colr, colg, colb);
        } else {
            if (surv) compute_sh<SH16>(sh4, fx, fy, fz, origin, colr, colg, colb);
        }
    } else if constexpr (SHDEG) {
        if (surv)
            compute_sh_degree<SH16>(reinterpret_cast<const float4*>(P.sh) + (size_t)i * (SH16 ? 6 : 12), px, py, pz, U.camera_position,
                                    P.sh_degree, colr, colg, colb);
    } else {
        if (surv) compute_sh<SH16>(reinterpret_cast<const float4*>(P.sh) + (size_t)i * (SH16 ? 6 : 12), px, py, pz, U.camera_position, colr, colg, colb);
    }

    // ---- decoupled look-back by warp 0: 32 predecessors per step ----
    if (warp == 0) {
        const uint32_t ex = lookback_exclusive(P.status, 1u, chunk, lane, blk_surv);
        if (lane == 0) {
            s_base_surv = ex;
            if (chunk == num_chunks - 1) P.ctl->num_visible = ex + blk_surv;
        }
    }
    __syncthreads();

    // ---- compacted per-survivor outputs ----
    if (surv) {
        const uint32_t cid = s_base_surv + surv_before + surv_rank_w;
        float4* rec = P.recs + (size_t)cid * GSB_REC_F4;
        rec[0] = make_float4(uvx, uvy, conx, cony);
        rec[1] = make_float4(conz, opac, __uint_as_float((uint32_t)bx0 | ((uint32_t)by0 << 16)),
                             __uint_as_float((uint32_t)(bx1 - bx0) | ((uint32_t)(by1 - by0) << 16)));
        rec[2] = make_float4(colr, colg, colb, depth);
        rec[3] = make_float4(radii, __uint_as_float(P.index_base + i), 0.f, 0.f);  // global Gaussian index (the sort payload of the reference)
        P.dkeys[cid] = __float_as_uint(depth);  // depth > 0.2 (z, or d for a fisheye): the IEEE bits are monotone as unsigned
        P.dvals[cid] = cid;
    }
    }
    if (DEBUG && i < P.n) {
        P.dbg_tiles[i] = nt;
        P.dbg_aabb[i] = surv ? make_uint4(bx0, by0, bx1, by1) : make_uint4(0, 0, 0, 0);
    }
}

// ------------------------------------------------------------------------------------------
// k_emit
// ------------------------------------------------------------------------------------------
#ifndef GSB_EMIT_WIN
#define GSB_EMIT_WIN 4096
#endif
#ifndef GSB_EMIT_MIN_BLOCKS
#define GSB_EMIT_MIN_BLOCKS 5  // k_emit<true>: <= 51 registers (an unannotated kernel got 48; minBlocks = 1 makes ptxas take 69)
#endif
constexpr int EMIT_WIN = GSB_EMIT_WIN;   // instances staged in shared memory per window
constexpr uint32_t EMIT_BIG = 128;  // Gaussians covering more tiles than this are expanded by the whole block

// The last chunk's inclusive prefix is M, the frame's instance count (Renderer.cpp:538 reads it back; here it stays in HBM).
__device__ __forceinline__ void emit_store_total(const EmitParams& P, unsigned long long total) {
    P.ctl->instances_total = total;
    P.ctl->num_instances = total > P.capacity ? P.capacity : (uint32_t)total;
    P.ctl->overflow = total > P.capacity ? 1u : 0u;
    if (total > P.capacity) atomicOr(&P.ctl->overflow_sticky, 1u);  // survives the next frames' k_frame_init
}

// Coalesced copy-out of one window of n staged instances to slots first_slot ..; slots past the capacity are dropped.
__device__ __forceinline__ void emit_copy_out(const EmitParams& P, const uint32_t* s_key, const uint32_t* s_val,
                                              unsigned long long first_slot, uint32_t n, int tid) {
    for (uint32_t i = tid; i < n; i += PRE_THREADS) {
        const unsigned long long slot = first_slot + i;
        if (slot < P.capacity) {
            P.keys[slot] = s_key[i];
            P.vals[slot] = s_val[i];
        }
    }
}

// COARSE (gsb_set_tile_cull level 2): the emitted unit is a block of 2^cs x 2^cs tiles (cs = 1 or 2) instead of a tile.  The key is
// (block id) | (mask << 16): bit (ly << cs | lx) of the mask says that tile (lx, ly) of the block lies inside the Gaussian's
// tile AABB, i.e. that preprocess_sort.comp:47-48 would have emitted that (Gaussian, tile) instance.  The radix passes only
// look at the low 16 bits, the mask rides along, and the blend of a tile keeps exactly the entries whose mask has its bit.
__device__ __forceinline__ uint32_t coarse_tile_mask(uint32_t cs, uint32_t bx, uint32_t by, uint32_t x0, uint32_t y0, uint32_t x1, uint32_t y1) {
    const uint32_t ox = bx << cs, oy = by << cs, n = 1u << cs;
    const uint32_t lx0 = max(x0, ox) - ox, lx1 = min(x1, ox + n) - ox, ly0 = max(y0, oy) - oy, ly1 = min(y1, oy + n) - oy;
    const uint32_t cols = (1u << lx1) - (1u << lx0);                       // tiles lx0 .. lx1-1 of one block row
    const uint32_t rows = (1u << (ly1 << cs)) - (1u << (ly0 << cs));       // bit ranges of block rows ly0 .. ly1-1
    return (cols * (cs == 2 ? 0x1111u : 0x5u)) & rows;
}

// ------------------------------------------------------------------------------------------
// Exact instance culling (gsb_set_tile_cull level 1, k_emit<true>).  A (Gaussian, tile) instance
// is dropped when the Gaussian provably cannot reach alpha >= 1/255 on any pixel of the 16x16 tile: the
// blend would `continue` over it for all 256 pixels (render.comp:78), so the image is bit-identical, but
// scan / sort / ranges / blend staging see fewer instances.  The reference has no such cull
// (preprocess_sort.comp emits the whole AABB), so M and the key buffers differ from it when enabled.
//
// The set {q <= c} (q = the conic's quadratic form, c = 2 * (|POWER_CUT| + rounding margin)) is an ellipse;
// intersected with one tile row (a slab of pixel-centre ordinates) it is convex, so the tiles of that row it
// touches are exactly one contiguous span [xa, xb], computed in closed form per row (no per-tile test):
//   dx_max(dy) = (-B dy + sqrt(A c - det dy^2)) / A  is concave with its maximum at dy* = -(B/C) sqrt(c C / det),
// so over the slab it is attained at dy* clamped to the slab (and to |dy| <= sqrt(A c / det)); same for the minimum.
// Emission order inside one Gaussian becomes row-major; that cannot change the sorted result (all instances of a
// Gaussian have distinct tiles).  Gaussians covering more than EMIT_BIG tiles are emitted un-culled by the block.
// ------------------------------------------------------------------------------------------
struct CullGauss {
    float ux, uy, A, B, C, inv_a, c2, dy_ext, dy_star;  // c2 = c, dy_ext = sqrt(A c / det), dy_star = (B / C) sqrt(c C / det)
    bool ok;                                            // false: not positive definite / NaN -> never cull
};

__device__ __forceinline__ CullGauss cull_setup(float4 r0, float C, float opacity, float reach_x, float reach_y) {
    CullGauss g;
    g.ux = r0.x;
    g.uy = r0.y;
    g.A = r0.z;
    g.B = r0.w;
    g.C = C;
    const float det = g.A * g.C - g.B * g.B;
    g.ok = g.A > 0.0f && g.C > 0.0f && det > 0.0f;
    // bound on the fp32 rounding error of render.comp:66 anywhere inside the AABB (|dx| <= reach_x, |dy| <= reach_y)
    const float mag = 0.5f * (g.A * reach_x * reach_x + g.C * reach_y * reach_y) + fabsf(g.B) * reach_x * reach_y;
    const float margin = 0.03f + 4e-6f * mag;
    g.c2 = 2.0f * (-power_cut(opacity) + margin);
    g.inv_a = 1.0f / g.A;
    g.dy_ext = sqrtf(g.A * g.c2 / det) * 1.0001f + 1e-3f;
    g.dy_star = (g.B / g.C) * sqrtf(g.c2 * g.C / det);
    return g;
}

// Tile span [xa, xb] (inclusive, clipped to [x0, x1]) of tile row ty that the ellipse may touch; xa > xb = empty.
__device__ __forceinline__ void cull_row_span(const CullGauss& g, uint32_t ty, int x0, int x1, int& xa, int& xb) {
    if (!g.ok) {
        xa = x0;
        xb = x1;
        return;
    }
    // d = uv - pixel; the row's pixel centres are y in [16 ty, 16 ty + 15]
    const float dy_lo = g.uy - (float)(ty * GSB_TILE + (GSB_TILE - 1)), dy_hi = g.uy - (float)(ty * GSB_TILE);
    const float lo = fmaxf(dy_lo, -g.dy_ext), hi = fminf(dy_hi, g.dy_ext);
    if (!(lo <= hi)) {  // the slab misses the ellipse (NaN -> keep everything)
        if (lo > hi) {
            xa = 1;
            xb = 0;
        } else {
            xa = x0;
            xb = x1;
        }
        return;
    }
    // dx range: dx = (-B dy -+ sqrt(A c - det dy^2)) / A.  max at dy = -dy_star, min at dy = +dy_star (clamped)
    const float det = g.A * g.C - g.B * g.B;
    const float dy1 = fminf(fmaxf(-g.dy_star, lo), hi), dy2 = fminf(fmaxf(g.dy_star, lo), hi);
    const float dx_max = (-g.B * dy1 + sqrtf(fmaxf(0.0f, g.A * g.c2 - det * dy1 * dy1))) * g.inv_a;
    const float dx_min = (-g.B * dy2 - sqrtf(fmaxf(0.0f, g.A * g.c2 - det * dy2 * dy2))) * g.inv_a;
    // pixel x = ux - dx in [ux - dx_max, ux - dx_min], widened by a slack that dwarfs the rounding of this formula
    const float slack = 0.01f + 1e-4f * (fabsf(dx_max) + fabsf(dx_min));
    const float px_lo = g.ux - dx_max - slack, px_hi = g.ux - dx_min + slack;
    // tile tx holds pixel centres [16 tx, 16 tx + 15]: keep tx with 16 tx <= px_hi and 16 tx + 15 >= px_lo
    const int ta = (int)ceilf((px_lo - (float)(GSB_TILE - 1)) * (1.0f / GSB_TILE));
    const int tb = (int)floorf(px_hi * (1.0f / GSB_TILE));
    xa = max(x0, ta);
    xb = min(x1, tb);
    if (!(px_lo <= px_hi)) {  // NaN safety
        xa = x0;
        xb = x1;
    }
}

// ------------------------------------------------------------------------------------------
// k_emit<CULL> -- gsb_set_tile_cull levels 0 and 1.  Per ticketed chunk of 256 depth-sorted survivors: block scan of their
// instance counts, the chunk's base by decoupled look-back, and the expansion into (tile id, compact id) pairs through
// shared memory, window by window.  A Gaussian covering more than EMIT_BIG tiles is expanded by the whole block (its whole
// AABB), the others by their own thread: level 0 the whole AABB, x outer / y inner (:47-48, the reference's order, which
// GSB_BUF_KEYS_UNSORTED exposes), level 1 the culled row spans, row-major.
// ------------------------------------------------------------------------------------------
// (Level 0 needs no minimum-blocks bound: 38 KB of shared memory per CTA already cap it at 5 CTAs per H100 SM.)
template <bool CULL>
__global__ void __launch_bounds__(PRE_THREADS, CULL ? GSB_EMIT_MIN_BLOCKS : 0) k_emit(const __grid_constant__ EmitParams P) {
    __shared__ uint32_t s_chunk;
    __shared__ uint32_t s_wnt[PRE_THREADS / 32];
    __shared__ unsigned long long s_base;
    __shared__ uint32_t s_nbig;
    __shared__ uint32_t s_big[PRE_THREADS];  // lanes of the chunk holding "big" Gaussians
    __shared__ uint4 s_info[PRE_THREADS];    // x0 | y0 << 16, w | h << 16, local offset, compact id (big Gaussians)
    __shared__ uint32_t s_key[EMIT_WIN];
    __shared__ uint32_t s_val[EMIT_WIN];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t nv = P.ctl->num_visible;
    const uint32_t num_chunks = (nv + PRE_THREADS - 1) / PRE_THREADS;
    const uint32_t tiles_x = P.tiles_x;

    while (true) {
        if (tid == 0) {
            s_chunk = atomicAdd(&P.ctl->emit_ticket, 1u);
            s_nbig = 0;
        }
        __syncthreads();
        const uint32_t chunk = s_chunk;
        if (chunk >= num_chunks) break;
        const uint32_t j = chunk * PRE_THREADS + tid;

        uint32_t nt = 0, cand = 0, cid = 0, xy = 0, wh = 0;
        CullGauss g{};
        if (j < nv) {
            cid = __ldg(P.sorted_cid + j);
            const float4 q1 = __ldg(P.recs + (size_t)cid * GSB_REC_F4 + 1);  // conic.z, opacity, AABB: same 32-B sector as q0
            xy = __float_as_uint(q1.z);
            wh = __float_as_uint(q1.w);
            cand = (wh & 0xffffu) * (wh >> 16);  // tiles of the AABB = the reference's instance count for this Gaussian
            nt = cand;
            if (CULL && cand != 0 && cand <= EMIT_BIG) {  // the tiles of the AABB's row spans
                const float4 r0 = __ldg(P.recs + (size_t)cid * GSB_REC_F4);
                // |uv - pixel centre| over the pixels of the AABB's tiles (the rounding bound of cull_setup needs it)
                const float px0 = (float)((xy & 0xffffu) * GSB_TILE), px1 = (float)(((xy & 0xffffu) + (wh & 0xffffu)) * GSB_TILE);
                const float py0 = (float)((xy >> 16) * GSB_TILE), py1 = (float)(((xy >> 16) + (wh >> 16)) * GSB_TILE);
                const float reach_x = fmaxf(fabsf(r0.x - px0), fabsf(px1 - r0.x)) + 1.0f;
                const float reach_y = fmaxf(fabsf(r0.y - py0), fabsf(py1 - r0.y)) + 1.0f;
                g = cull_setup(r0, q1.x, q1.y, reach_x, reach_y);
                const int gx0 = (int)(xy & 0xffffu), gx1 = gx0 + (int)(wh & 0xffffu) - 1;
                nt = 0;
                for (uint32_t r = 0; r < (wh >> 16); r++) {
                    int xa, xb;
                    cull_row_span(g, (xy >> 16) + r, gx0, gx1, xa, xb);
                    nt += (uint32_t)max(0, xb - xa + 1);
                }
            }
        }
        // ---- block scan of the tile counts (prefix_sum.comp's job) ----
        uint32_t nt_incl = nt, cand_sum = cand;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, nt_incl, o);
            if (lane >= o) nt_incl += t;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cand_sum += __shfl_xor_sync(FULL, cand_sum, o);
        if (lane == 31) s_wnt[warp] = nt_incl;
        if (lane == 0 && cand_sum) atomicAdd(&P.ctl->candidates_total, (unsigned long long)cand_sum);
        __syncthreads();
        uint32_t nt_before = 0, blk_nt = 0;
#pragma unroll
        for (int w = 0; w < PRE_THREADS / 32; w++) {
            const uint32_t b = s_wnt[w];
            if (w < warp) nt_before += b;
            blk_nt += b;
        }
        const uint32_t off = nt_before + (nt_incl - nt);  // exclusive offset inside the chunk
        if (tid == 0) st_vol(P.status + chunk, Lookback<unsigned long long>::aggregate(chunk, blk_nt));
        if (cand > EMIT_BIG) {
            s_info[tid] = make_uint4(xy, wh, off, cid);
            s_big[atomicAdd(&s_nbig, 1u)] = (uint32_t)tid;
        }
        __syncthreads();
        const uint32_t nbig = s_nbig;
        unsigned long long base = 0;

        const uint32_t x0 = xy & 0xffffu, y0 = xy >> 16, h = wh >> 16;
        for (uint32_t w0 = 0; w0 == 0 || w0 < blk_nt; w0 += EMIT_WIN) {  // at least once: the look-back lives inside
            const uint32_t w1 = min(blk_nt, w0 + (uint32_t)EMIT_WIN);
            if (nt != 0 && cand <= EMIT_BIG) {  // small Gaussians: each thread writes its own tiles
                if constexpr (CULL) {  // row-major over the row spans
                    if (off < w1 && off + nt > w0) {
                        const int gx0 = (int)x0, gx1 = gx0 + (int)(wh & 0xffffu) - 1;
                        uint32_t o = off;
                        for (uint32_t r = 0; r < h; r++) {
                            const uint32_t ty = y0 + r;
                            int xa, xb;
                            cull_row_span(g, ty, gx0, gx1, xa, xb);
                            for (int x = xa; x <= xb; x++, o++) {
                                if (o >= w0 && o < w1) {
                                    s_key[o - w0] = (uint32_t)x + ty * tiles_x;
                                    s_val[o - w0] = cid;
                                }
                            }
                        }
                    }
                } else {  // x outer / y inner
                    const uint32_t lo = max(off, w0), hi = min(off + nt, w1);
                    if (lo < hi) {
                        uint32_t k = lo - off;
                        uint32_t q = k / h, r = k - q * h;
                        uint32_t t = (x0 + q) + (y0 + r) * tiles_x;
                        for (uint32_t o = lo; o < hi; o++) {
                            s_key[o - w0] = t;  // :49 tile index (the high 32 bits of the reference key)
                            s_val[o - w0] = cid;
                            t += tiles_x;
                            if (++r == h) {  // next column: y back to y0, x + 1
                                r = 0;
                                t = t - h * tiles_x + 1;
                            }
                        }
                    }
                }
            }
            for (uint32_t b = 0; b < nbig; b++) {  // big Gaussians: whole AABB, expanded by the whole block
                const uint4 inf = s_info[s_big[b]];
                const uint32_t bh = inf.y >> 16, bnt = (inf.y & 0xffffu) * bh;
                const uint32_t lo = max(inf.z, w0), hi = min(inf.z + bnt, w1);
                for (uint32_t o = lo + tid; o < hi; o += PRE_THREADS) {
                    const uint32_t k = o - inf.z, q = k / bh, r = k - q * bh;
                    s_key[o - w0] = ((inf.x & 0xffffu) + q) + ((inf.x >> 16) + r) * tiles_x;
                    s_val[o - w0] = inf.w;
                }
            }
            if (w0 == 0 && warp == 0) {  // look-back after the first fill: the predecessors' latency overlaps local work
                const unsigned long long ex = lookback_exclusive(P.status, 1u, chunk, lane, (unsigned long long)blk_nt);
                if (lane == 0) {
                    s_base = ex;
                    if (chunk == num_chunks - 1) emit_store_total(P, ex + blk_nt);
                }
            }
            __syncthreads();
            if (w0 == 0) {
                base = s_base;
                if (P.dbg_offsets != nullptr && j < nv) P.dbg_offsets[j] = base + off;  // the device scan, for gsb_debug_download
            }
            emit_copy_out(P, s_key, s_val, base + w0, w1 - w0, tid);
            __syncthreads();
        }
    }
}

// ------------------------------------------------------------------------------------------
// k_emit_coarse -- k_emit for gsb_set_tile_cull level 2: one entry per (Gaussian, block of 2^cs x 2^cs tiles), key =
// block id | tile mask << 16 (coarse_tile_mask).  Entries per Gaussian are few (2.4 on the bench scene), so the kernel is
// bound by the latency of the record gather, the look-back and the barriers, not by the expansion: every thread handles
// EC_IPT consecutive survivors (four independent gathers in flight, a quarter of the chunks / tickets / barriers).
// ------------------------------------------------------------------------------------------
#ifndef GSB_EMIT_COARSE_IPT
#define GSB_EMIT_COARSE_IPT 4  // survivors per thread (a multiple of 4: the sorted ids are read 16 B at a time)
#endif
constexpr int EC_IPT = GSB_EMIT_COARSE_IPT;
static_assert(EC_IPT % 4 == 0, "k_emit_coarse reads the sorted ids as uint4");
constexpr int EC_CHUNK = PRE_THREADS * EC_IPT;
constexpr int EC_MAXBIG = 32;  // block-expanded Gaussians per chunk; more than that (never seen) fall back to the thread loop

__global__ void __launch_bounds__(PRE_THREADS) k_emit_coarse(const __grid_constant__ EmitParams P) {
    __shared__ uint32_t s_chunk;
    __shared__ uint32_t s_wnt[PRE_THREADS / 32];
    __shared__ unsigned long long s_base;
    __shared__ uint32_t s_nbig;
    __shared__ uint4 s_info[EC_MAXBIG];  // x0 | y0 << 16 (blocks), w | h << 16 (blocks), local offset, compact id
    __shared__ uint2 s_fine[EC_MAXBIG];  // the tile AABB (x0 | y0 << 16, x1 | y1 << 16)
    __shared__ uint32_t s_key[EMIT_WIN];
    __shared__ uint32_t s_val[EMIT_WIN];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t nv = P.ctl->num_visible;
    const uint32_t num_chunks = (nv + EC_CHUNK - 1) / EC_CHUNK;
    const uint32_t bins_x = P.tiles_x, cs = P.coarse_shift;

    while (true) {
        if (tid == 0) {
            s_chunk = atomicAdd(&P.ctl->emit_ticket, 1u);
            s_nbig = 0;
        }
        __syncthreads();
        const uint32_t chunk = s_chunk;
        if (chunk >= num_chunks) break;
        const uint32_t j0 = chunk * EC_CHUNK + tid * EC_IPT;  // this thread's survivors j0 .. j0 + EC_IPT - 1 (depth order)

        uint32_t cid[EC_IPT], nt[EC_IPT], bxy[EC_IPT], bwh[EC_IPT], f0[EC_IPT], f1[EC_IPT];
        if (j0 + EC_IPT <= nv) {
#pragma unroll
            for (int k = 0; k < EC_IPT; k += 4) {
                const uint4 c4 = __ldg(reinterpret_cast<const uint4*>(P.sorted_cid + j0 + k));
                cid[k] = c4.x, cid[k + 1] = c4.y, cid[k + 2] = c4.z, cid[k + 3] = c4.w;
            }
        } else {
#pragma unroll
            for (int k = 0; k < EC_IPT; k++) cid[k] = j0 + k < nv ? __ldg(P.sorted_cid + j0 + k) : 0u;
        }
        float4 q1[EC_IPT];
#pragma unroll
        for (int k = 0; k < EC_IPT; k++) q1[k] = j0 + k < nv ? __ldg(P.recs + (size_t)cid[k] * GSB_REC_F4 + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
        uint32_t cand = 0, mine = 0;
#pragma unroll
        for (int k = 0; k < EC_IPT; k++) {
            const uint32_t xy = __float_as_uint(q1[k].z), wh = __float_as_uint(q1[k].w);
            const uint32_t c = (wh & 0xffffu) * (wh >> 16);  // tiles of the AABB = the reference's instance count for this Gaussian
            cand += c;
            nt[k] = 0, bxy[k] = 0, bwh[k] = 0, f0[k] = 0, f1[k] = 0;
            if (c != 0) {
                const uint32_t x0 = xy & 0xffffu, y0 = xy >> 16, x1 = x0 + (wh & 0xffffu), y1 = y0 + (wh >> 16);
                const uint32_t cx0 = x0 >> cs, cy0 = y0 >> cs, cx1 = ((x1 - 1) >> cs) + 1, cy1 = ((y1 - 1) >> cs) + 1;
                bxy[k] = cx0 | (cy0 << 16);
                bwh[k] = (cx1 - cx0) | ((cy1 - cy0) << 16);
                f0[k] = x0 | (y0 << 16);
                f1[k] = x1 | (y1 << 16);
                nt[k] = (cx1 - cx0) * (cy1 - cy0);
            }
            mine += nt[k];
        }
        // ---- block scan of the entry counts ----
        uint32_t incl = mine, cand_sum = cand;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, incl, o);
            if (lane >= o) incl += t;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cand_sum += __shfl_xor_sync(FULL, cand_sum, o);
        if (lane == 31) s_wnt[warp] = incl;
        if (lane == 0 && cand_sum) atomicAdd(&P.ctl->candidates_total, (unsigned long long)cand_sum);
        __syncthreads();
        uint32_t before = 0, blk_nt = 0;
#pragma unroll
        for (int w = 0; w < PRE_THREADS / 32; w++) {
            const uint32_t b = s_wnt[w];
            if (w < warp) before += b;
            blk_nt += b;
        }
        if (tid == 0) st_vol(P.status + chunk, Lookback<unsigned long long>::aggregate(chunk, blk_nt));
        uint32_t off[EC_IPT];
        {
            uint32_t run = before + (incl - mine);
#pragma unroll
            for (int k = 0; k < EC_IPT; k++) {
                off[k] = run;
                run += nt[k];
            }
        }
        uint32_t big = 0;  // bit k: item k is expanded by the whole block
#pragma unroll
        for (int k = 0; k < EC_IPT; k++) {
            if (nt[k] > EMIT_BIG) {
                const uint32_t slot = atomicAdd(&s_nbig, 1u);
                if (slot < EC_MAXBIG) {
                    s_info[slot] = make_uint4(bxy[k], bwh[k], off[k], cid[k]);
                    s_fine[slot] = make_uint2(f0[k], f1[k]);
                    big |= 1u << k;
                }
            }
        }
        __syncthreads();
        const uint32_t nbig = min(s_nbig, (uint32_t)EC_MAXBIG);
        unsigned long long base = 0;

        for (uint32_t w0 = 0; w0 == 0 || w0 < blk_nt; w0 += EMIT_WIN) {  // at least once: the look-back lives inside
            const uint32_t w1 = min(blk_nt, w0 + (uint32_t)EMIT_WIN);
#pragma unroll
            for (int k = 0; k < EC_IPT; k++) {  // x outer / y inner inside a Gaussian, like preprocess_sort.comp:47-48
                if (nt[k] == 0 || ((big >> k) & 1u)) continue;
                const uint32_t lo = max(off[k], w0), hi = min(off[k] + nt[k], w1);
                if (lo >= hi) continue;
                const uint32_t x0 = bxy[k] & 0xffffu, y0 = bxy[k] >> 16, h = bwh[k] >> 16;
                uint32_t e = lo - off[k];
                uint32_t q = e / h, r = e - q * h;
                for (uint32_t o = lo; o < hi; o++) {
                    const uint32_t m = coarse_tile_mask(cs, x0 + q, y0 + r, f0[k] & 0xffffu, f0[k] >> 16, f1[k] & 0xffffu, f1[k] >> 16);
                    s_key[o - w0] = ((x0 + q) + (y0 + r) * bins_x) | (m << 16);
                    s_val[o - w0] = cid[k];
                    if (++r == h) {
                        r = 0;
                        q++;
                    }
                }
            }
            for (uint32_t b = 0; b < nbig; b++) {
                const uint4 inf = s_info[b];
                const uint2 f = s_fine[b];
                const uint32_t bh = inf.y >> 16, bnt = (inf.y & 0xffffu) * bh;
                const uint32_t lo = max(inf.z, w0), hi = min(inf.z + bnt, w1);
                for (uint32_t o = lo + tid; o < hi; o += PRE_THREADS) {
                    const uint32_t e = o - inf.z, q = e / bh, r = e - q * bh;
                    const uint32_t bx = (inf.x & 0xffffu) + q, by = (inf.x >> 16) + r;
                    s_key[o - w0] = (bx + by * bins_x) | (coarse_tile_mask(cs, bx, by, f.x & 0xffffu, f.x >> 16, f.y & 0xffffu, f.y >> 16) << 16);
                    s_val[o - w0] = inf.w;
                }
            }
            if (w0 == 0 && warp == 0) {  // look-back after the first fill: the predecessors' latency overlaps local work
                const unsigned long long ex = lookback_exclusive(P.status, 1u, chunk, lane, (unsigned long long)blk_nt);
                if (lane == 0) {
                    s_base = ex;
                    if (chunk == num_chunks - 1) emit_store_total(P, ex + blk_nt);
                }
            }
            __syncthreads();
            if (w0 == 0) base = s_base;
            emit_copy_out(P, s_key, s_val, base + w0, w1 - w0, tid);
            __syncthreads();
        }
    }
}

}  // namespace

template <bool AA, bool FISHEYE, bool OPENCV, bool SHDEG, bool ORTHO>
void launch_project_as(const ProjectParams& p, bool debug, unsigned blocks, cudaStream_t s) {
    if (p.sh_half) {  // fp16 SH storage (non-parity)
        if (debug) k_project<true, false, true, AA, FISHEYE, OPENCV, SHDEG, ORTHO><<<blocks, PRE_THREADS, 0, s>>>(p);
        else k_project<false, false, true, AA, FISHEYE, OPENCV, SHDEG, ORTHO><<<blocks, PRE_THREADS, 0, s>>>(p);
    } else if (debug) k_project<true, false, false, AA, FISHEYE, OPENCV, SHDEG, ORTHO><<<blocks, PRE_THREADS, 0, s>>>(p);
    else k_project<false, false, false, AA, FISHEYE, OPENCV, SHDEG, ORTHO><<<blocks, PRE_THREADS, 0, s>>>(p);
}

template <bool FISHEYE, bool OPENCV = false, bool ORTHO = false>
void launch_project_camera(const ProjectParams& p, bool debug, unsigned blocks, cudaStream_t s) {
    const bool shdeg = p.sh_degree < 3;
    if (p.antialiased) {
        if (shdeg) launch_project_as<true, FISHEYE, OPENCV, true, ORTHO>(p, debug, blocks, s);
        else launch_project_as<true, FISHEYE, OPENCV, false, ORTHO>(p, debug, blocks, s);
    } else if (shdeg) launch_project_as<false, FISHEYE, OPENCV, true, ORTHO>(p, debug, blocks, s);
    else launch_project_as<false, FISHEYE, OPENCV, false, ORTHO>(p, debug, blocks, s);
}

cudaError_t launch_project(const ProjectParams& p, bool debug, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    const unsigned blocks = (p.n + PRE_THREADS - 1) / PRE_THREADS;
    if (p.route_world > 0) {  // the routed kernel has no AA, lens or degree instantiation
        if (p.antialiased || p.camera.kind != GSB_CAMERA_PINHOLE || p.sh_degree < 3) return cudaErrorInvalidValue;
        if (p.sh_half) k_project<false, true, true, false><<<blocks, PRE_THREADS, 0, s>>>(p);
        else k_project<false, true, false, false><<<blocks, PRE_THREADS, 0, s>>>(p);
    } else if (p.camera.kind == GSB_CAMERA_FISHEYE) {
        launch_project_camera<true>(p, debug, blocks, s);
    } else if (p.camera.kind == GSB_CAMERA_OPENCV) {
        ProjectParams q = p;
        const double t = std::tan((double)p.camera.max_theta);
        q.tan2_max = (float)(t * t);
        launch_project_camera<false, true>(q, debug, blocks, s);
    } else if (p.camera.kind == GSB_CAMERA_ORTHO) {
        launch_project_camera<false, false, true>(p, debug, blocks, s);
    } else {
        launch_project_camera<false>(p, debug, blocks, s);
    }
    return cudaGetLastError();
}

cudaError_t launch_emit(const EmitParams& p, cudaStream_t s) {
    uint32_t blocks = (p.nv_hint + PRE_THREADS - 1) / PRE_THREADS;
    const uint32_t cap = (uint32_t)p.num_sms * 8;  // ticket loop: any grid size is correct
    if (blocks > cap) blocks = cap;
    if (blocks == 0) blocks = 1;
    if (p.cull) k_emit<true><<<blocks, PRE_THREADS, 0, s>>>(p);
    else if (p.coarse_shift) k_emit_coarse<<<std::max<uint32_t>(1u, std::min<uint32_t>((p.nv_hint + EC_CHUNK - 1) / EC_CHUNK, cap)), PRE_THREADS, 0, s>>>(p);
    else k_emit<false><<<blocks, PRE_THREADS, 0, s>>>(p);
    return cudaGetLastError();
}

}  // namespace gsb
