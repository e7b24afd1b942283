// gsb_backward.cu -- reverse mode of one whole frame: dL/d(image) -> dL/d(GSScene::Vertex records).  No reference counterpart
// (3DGS.cpp only renders); this differentiates the function the forward computes, quirks included (DESIGN.md section 10):
// only the red channel clamped at 0, integer pixel centres, alpha = min(0.99, .), the T' < 1e-4 break and the per-tile lists
// of the frame.  A frame of gsb_set_background composites c + T_final bg (DESIGN.md section 15): the BG instantiations of
// k_blend_backward start the colour behind every pixel's last contributor at bg instead of 0, and
//   k_background_grad + k_background_reduce  (gsb_background_gradient) sum T_final g over the frame's pixels for dL/d bg, in
//                         fp64 in an order fixed by the frame size: one row of partials per CTA, then one CTA.
//
//   k_blend_backward      one CTA per 16 x 16 tile, one pixel per thread.  The tile's list is walked back to front from the
//                         largest last-contributor position among its pixels (recorded by k_blend<..., RECORD>), in batches
//                         staged into shared memory.  Every (pixel, entry) pair re-evaluates power and alpha with the frame's
//                         own arithmetic (EXACT: the ops of k_blend + exp_shared_inrange; FAST: the same FMAs + __expf), so the
//                         contributor set is the forward's bit for bit; T is recovered by division, T_i = T_{i+1} / (1 - alpha_i).
//                         Per survivor it accumulates d uv (2), d conic (3), d opacity (1), d colour (3): reduced over the warp
//                         (fp32 shuffles), then over the CTA (fp64 shared-memory atomics), then one global fp64 atomic per value
//                         and tile.  fp64 keeps the order-dependent rounding of the sums over warps and tiles ~1e-16 relative.
//                         The ABSGRAD instantiation (gsb_render_backward_density) also sums |d u|, |d v| of each pixel.
//   k_density_accumulate  one thread per survivor (gsb_render_backward_density only): adds the frame's screen-space gradient
//                         norms, one view and the max pixel radius to the caller's n x 4 statistics.
//   k_preprocess_backward one thread per survivor (grid-stride over N_v, read on the device): recomputes preprocess.comp for the
//                         survivor's Gaussian from the scene and the frame's camera and chains colour -> SH + view direction,
//                         conic -> cov2d -> (Sigma, J) -> position, uv -> ndc -> clip position -> position,
//                         Sigma -> scale and (stored, unnormalised) rotation.  It writes the Gaussian's 60-float gradient
//                         record and returns its scratch accumulators to zero for the next call.  The CAMERA instantiation
//                         (gsb_render_backward_camera) also keeps the camera's share of that chain rule -- view matrix,
//                         projection matrix, camera position, tan_fov -- summed per thread, then per CTA into one fp64 row.
//   k_camera_reduce       one CTA: sums those rows in a fixed order into the fp32 gsb_uniforms of gradients.
//
// The atomics make the sums depend on the order in which warps and CTAs add their partial sums: by default gradients are NOT
// guaranteed to be bitwise reproducible from run to run (fp64 accumulation makes a difference in the final fp32 value rare).
// gsb_set_backward_deterministic(ctx, 1) replaces that reduction, and only it (DESIGN.md section 10):
//   k_blend_backward<MODE, ABSGRAD, DET = true>  the same walk; per-warp partials summed in warp order, one fp64 slot per
//                         (tile, list entry) stored at the entry's list position, +0 for entries that contributed nothing.
//   k_det_prepare + the Onesweep sort (k_sort_hist, k_onesweep_pass)  a stable sort of (compact id, list position) over the
//                         frame's M entries; its last pass publishes each survivor's run, in tile order.
//   k_det_reduce          one thread per survivor: the run's slots summed in order in fp64, stored into the scratch that
//                         k_density_accumulate and k_preprocess_backward read.  Every output is then order-fixed.
// Compiled with -fmad=false like the forward.
#include <algorithm>
#include <type_traits>

#include "gsb_cull.cuh"
#include "gsb_exp.cuh"
#include "gsb_geom.cuh"
#include "gsb_internal.cuh"

namespace gsb {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int BW_THREADS = 256;  // one pixel per thread of a 16 x 16 tile
constexpr int BW_BATCH = 256;    // list entries staged per batch (one per thread)
constexpr int BW_NACC = 9;       // per-survivor accumulators: uv (2), conic (3), opacity, colour (3)
constexpr int BW_NABS = 2;       // ABSGRAD: sum over pixels of |d u|, |d v| (gsb_render_backward_density)
constexpr int BW_DET_BATCH = 128;  // DET: list entries per batch, so that the per-warp partials fit 4-5 CTAs per SM
constexpr int BW_WARPS = BW_THREADS / 32;
template <bool DET>
constexpr uint32_t bw_batch = DET ? BW_DET_BATCH : BW_BATCH;
constexpr int PB_THREADS = 256;

struct __align__(16) BwRec {  // the staged record in k_blend's pre-scaled form (render.comp:66 evaluated identically)
    float4 q0;                // ux uy -A/2 -B
    float4 q1;                // -C/2 opacity r g
    float4 q2;                // b power_cut bits(compact id) -
};

// ABSGRAD (gsb_render_backward_density): each lane's d u and d v -- one pixel's own terms -- also go through the same
// reduction as absolute values, into P.abs_scratch.
// DET (gsb_set_backward_deterministic): the same walk, reduced without atomics.  Lane 0 of each warp stores the warp's
// shuffle sums into its own fp32 row of det_partials() (dynamic shared memory, [warp][NACC][BW_DET_BATCH]); at the flush
// thread k sums the 8 warps in warp order in fp64 and stores the tile's partial of entry k into P.det_slots at its list
// position.  Every position of the tile's list is stored, +0 for entries no pixel of the tile has as contributor.
// DET = false is the atomic reduction.  The DET-only constants and the shared-memory pointer live outside the kernel: a new
// local, even unused, changes ptxas' allocation of the DET = false instantiations.
__device__ __forceinline__ float* det_partials() {
    extern __shared__ float s_dyn[];  // referenced by the DET instantiations only
    return s_dyn;
}

// BG (a frame of gsb_set_background): the colour behind every pixel's last contributor is P.bg instead of 0.  Only the BG
// instantiations take the larger argument: the others keep BackwardParams as it was, and with it their code.
struct BackwardBgParams : BackwardParams {
    float3 bg;
};
template <bool BG>
using BwParams = std::conditional_t<BG, BackwardBgParams, BackwardParams>;
template <bool BG>
BwParams<BG> bw_params(const BackwardParams& p, float3 bg) {
    if constexpr (BG) return BackwardBgParams{p, bg};
    else return p;
}

template <int MODE, bool ABSGRAD, bool DET = false, bool BG = false>
__global__ void __launch_bounds__(BW_THREADS) k_blend_backward(const __grid_constant__ BwParams<BG> P) {
    constexpr int NACC = BW_NACC + (ABSGRAD ? BW_NABS : 0);  // shared-memory columns: the extra two in ABSGRAD only
    __shared__ BwRec s_rec[bw_batch<DET>];
    __shared__ double s_acc[DET ? 1 : BW_BATCH][NACC];
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
    if constexpr (BG) {  // the background is behind every pixel's last contributor
        acc_r = P.bg.x;
        acc_g = P.bg.y;
        acc_b = P.bg.z;
    }
    for (uint32_t hi = max_last; hi > 0;) {
        const uint32_t lo = hi > bw_batch<DET> ? hi - bw_batch<DET> : 0u;
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
            if constexpr (!DET) {
#pragma unroll
                for (int k = 0; k < NACC; k++) s_acc[tid][k] = 0.0;
            }
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
            if (!__any_sync(FULL, contrib)) {
                if constexpr (DET) {
                    if (lane == 0) {
#pragma unroll
                        for (int j = 0; j < NACC; j++) det_partials()[(warp * NACC + j) * bw_batch<true> + k] = 0.f;
                    }
                }
                continue;
            }
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
            float va[BW_NABS];
            if constexpr (ABSGRAD) {  // this pixel's own |d u|, |d v|, taken before the sum over pixels
                va[0] = fabsf(v[0]);
                va[1] = fabsf(v[1]);
            }
#pragma unroll
            for (int j = 0; j < BW_NACC; j++) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(FULL, v[j], o);
            }
            if constexpr (ABSGRAD) {
#pragma unroll
                for (int j = 0; j < BW_NABS; j++) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) va[j] += __shfl_xor_sync(FULL, va[j], o);
                }
            }
            if constexpr (DET) {
                if (lane == 0) {
#pragma unroll
                    for (int j = 0; j < BW_NACC; j++) det_partials()[(warp * NACC + j) * bw_batch<true> + k] = v[j];
                    if constexpr (ABSGRAD) {
#pragma unroll
                        for (int j = 0; j < BW_NABS; j++) det_partials()[(warp * NACC + BW_NACC + j) * bw_batch<true> + k] = va[j];
                    }
                }
            } else if (lane == 0) {
#pragma unroll
                for (int j = 0; j < BW_NACC; j++)
                    if (v[j] != 0.f) atomicAdd(&s_acc[k][j], (double)v[j]);
                if constexpr (ABSGRAD) {
#pragma unroll
                    for (int j = 0; j < BW_NABS; j++)
                        if (va[j] != 0.f) atomicAdd(&s_acc[k][BW_NACC + j], (double)va[j]);
                }
            }
        }
        __syncthreads();
        if constexpr (DET) {
            if ((uint32_t)tid < cnt) {  // warps 0..7 in order, in fp64 from +0.0: the slot is never -0
                double* dst = P.det_slots + (size_t)(range.x + lo + (uint32_t)tid) * NACC;
#pragma unroll
                for (int j = 0; j < NACC; j++) {
                    double a = 0.0;
#pragma unroll
                    for (int w = 0; w < BW_WARPS; w++) a += (double)det_partials()[(w * NACC + j) * bw_batch<true> + tid];
                    dst[j] = a;
                }
            }
        } else if ((uint32_t)tid < cnt) {
            double* dst = P.scratch + (size_t)__float_as_uint(s_rec[tid].q2.z) * BW_NACC;
#pragma unroll
            for (int j = 0; j < BW_NACC; j++) {
                const double a = s_acc[tid][j];
                if (a != 0.0) atomicAdd(dst + j, a);
            }
            if constexpr (ABSGRAD) {
                double* dabs = P.abs_scratch + (size_t)__float_as_uint(s_rec[tid].q2.z) * BW_NABS;
#pragma unroll
                for (int j = 0; j < BW_NABS; j++) {
                    const double a = s_acc[tid][BW_NACC + j];
                    if (a != 0.0) atomicAdd(dabs + j, a);
                }
            }
        }
        hi = lo;
    }
    if constexpr (DET) {  // the entries behind every pixel's last contributor: +0, so k_det_reduce reads no stale slot
        const uint32_t len = range.y - range.x;
        for (uint32_t p = max_last + (uint32_t)tid; p < len; p += BW_THREADS) {
            double* dst = P.det_slots + (size_t)(range.x + p) * NACC;
#pragma unroll
            for (int j = 0; j < NACC; j++) dst[j] = 0.0;
        }
    }
}

// gsb_render_backward_density, between k_blend_backward<MODE, true> and k_preprocess_backward: one thread per survivor
// (grid-stride over N_v, read on the device) adds the frame's statistics to the Gaussian's row of P.density:
// |d uv| and |sum_p |d uv_p|| in NDC units (d u / d ndc.x = W / 2 exactly), one view, and the max of the pixel radius.
// Every survivor is counted, zero gradient or not -- which is why this is not folded into k_preprocess_backward, whose
// threads skip such survivors.  It reads d uv without clearing it (k_preprocess_backward still consumes the scratch) and
// returns abs_scratch to zero.  Plain loads and stores suffice: a Gaussian is at most one survivor of a frame.
__global__ void __launch_bounds__(PB_THREADS) k_density_accumulate(const __grid_constant__ BackwardParams P) {
    const uint32_t nv = P.ctl->num_visible;
    const double hw = 0.5 * (double)P.width, hh = 0.5 * (double)P.height;
    for (uint32_t cid = blockIdx.x * blockDim.x + threadIdx.x; cid < nv; cid += gridDim.x * blockDim.x) {
        const double* sc = P.scratch + (size_t)cid * BW_NACC;
        double* ab = P.abs_scratch + (size_t)cid * BW_NABS;
        const double gx = sc[0] * hw, gy = sc[1] * hh;
        const double ax = ab[0] * hw, ay = ab[1] * hh;
        ab[0] = 0.0;
        ab[1] = 0.0;
        const float4 r3 = __ldg(P.recs + (size_t)cid * GSB_REC_F4 + 3);
        float* d = P.density + (size_t)__float_as_uint(r3.y) * 4;
        d[0] += (float)sqrt(gx * gx + gy * gy);
        d[1] += (float)sqrt(ax * ax + ay * ay);
        d[2] += 1.0f;
        d[3] = fmaxf(d[3], r3.x);
    }
}

// gsb_set_backward_deterministic, before the sort that groups the slots by survivor: the sort's input pairs (compact id of
// list position p, p) over the frame's M entries -- a copy, so the frame's lists survive for a repeated backward -- and the
// per-survivor runs set to all ones (= no entry) for the sort's last pass to fill.  M and N_v are read on the device.
__global__ void __launch_bounds__(PB_THREADS) k_det_prepare(const uint32_t* __restrict__ vals, const Control* ctl, uint32_t* __restrict__ keys,
                                                            uint32_t* __restrict__ pos, uint2* __restrict__ runs) {
    const uint32_t m = ctl->num_instances, nv = ctl->num_visible;
    const uint32_t i0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    for (uint32_t p = i0; p < m; p += stride) {
        keys[p] = __ldg(vals + p);
        pos[p] = p;
    }
    for (uint32_t c = i0; c < nv; c += stride) runs[c] = make_uint2(0xffffffffu, 0xffffffffu);
}

// gsb_set_backward_deterministic, after the sort: one thread per survivor (grid-stride over N_v, read on the device) sums its
// slots in run order -- ascending list position, which is tile order -- in fp64 from +0.0, and STORES the totals into
// P.scratch (and P.abs_scratch), where k_density_accumulate and k_preprocess_backward read them as they read the atomic sums.
// The sum is sequential so that an entry whose slot is +0 changes nothing: tile-cull level 1's list is level 0's with such
// entries removed, and both give the same bits.  Loads run UNROLL entries ahead of the adds.
template <bool ABSGRAD>
__global__ void __launch_bounds__(PB_THREADS) k_det_reduce(const __grid_constant__ BackwardParams P, const uint32_t* __restrict__ pos,
                                                           const uint2* __restrict__ runs) {
    constexpr int NACC = BW_NACC + (ABSGRAD ? BW_NABS : 0);
    constexpr uint32_t UNROLL = 4;
    const uint32_t nv = P.ctl->num_visible;
    const double* __restrict__ slots = P.det_slots;
    for (uint32_t cid = blockIdx.x * blockDim.x + threadIdx.x; cid < nv; cid += gridDim.x * blockDim.x) {
        double s[NACC];
#pragma unroll
        for (int k = 0; k < NACC; k++) s[k] = 0.0;
        const uint2 r = __ldg(runs + cid);
        if (r.x != 0xffffffffu) {  // a survivor in no list (level 1 culled it from every tile) keeps zeros
            const uint32_t end = ~r.y;
            uint32_t j = r.x;
            for (; j + UNROLL <= end; j += UNROLL) {
                double x[UNROLL][NACC];
#pragma unroll
                for (uint32_t u = 0; u < UNROLL; u++) {
                    const double* sl = slots + (size_t)__ldg(pos + j + u) * NACC;
#pragma unroll
                    for (int k = 0; k < NACC; k++) x[u][k] = __ldg(sl + k);
                }
#pragma unroll
                for (uint32_t u = 0; u < UNROLL; u++)
#pragma unroll
                    for (int k = 0; k < NACC; k++) s[k] += x[u][k];
            }
            for (; j < end; j++) {
                const double* sl = slots + (size_t)__ldg(pos + j) * NACC;
#pragma unroll
                for (int k = 0; k < NACC; k++) s[k] += __ldg(sl + k);
            }
        }
        double* sc = P.scratch + (size_t)cid * BW_NACC;
#pragma unroll
        for (int k = 0; k < BW_NACC; k++) sc[k] = s[k];
        if constexpr (ABSGRAD) {
            double* ab = P.abs_scratch + (size_t)cid * BW_NABS;
#pragma unroll
            for (int k = 0; k < BW_NABS; k++) ab[k] = s[BW_NACC + k];
        }
    }
}

// gsb_uniforms word offsets of the fields the camera gradient has
constexpr int U_CAMPOS = 0, U_PROJ = 4, U_VIEW = 20, U_TANX = 38, U_TANY = 39;
// Words of dL/d(UBO) that can be non-zero: camera_position.xyz, proj_mat rows 0, 1, 3, view_mat rows 0-2, tan_fovx / tan_fovy.
// The rest (camera_position.w, proj row 2 = depth, view row 3, width, height) feed only step functions or nothing.
__host__ __device__ constexpr bool cam_word_live(int j) {
    return j < 3 || (j >= U_PROJ && j < U_VIEW && (j & 3) != 2) || (j >= U_VIEW && j < 36 && (j & 3) != 3) || j >= U_TANX;
}

// CAMERA (gsb_render_backward_camera): each thread also accumulates, over its survivors, their share of dL/d(UBO) in the
// UBO's word layout (fp32), and each CTA writes one fp64 row of partial sums (warp shuffles, then a fixed-order sum over the
// warps) into P.cam_partials for k_camera_reduce.  The vertex gradient is written only when P.grad_vertices is set.
// AA (a frame of gsb_set_antialiased): d[5] is dL/d(o comp), comp = sqrt(det0 / det).  The opacity gets d[5] comp, and
// g = d[5] o reaches both determinants: dL/d det0 = g comp / (2 det0), dL/d det = -g comp / (2 det), 0 where comp = 0.
// FISHEYE (a frame of gsb_set_camera_model's fisheye, CAMERA = false only): J and uv are the lens's (fisheye_geo,
// fisheye_jacobian), dL/d(J W) goes to J through the view rotation and on to the view-space position through J's second
// derivatives (fisheye_grad), and that position to the Gaussian's through the view rotation; the projection matrix takes no
// part.  Only these instantiations take the larger argument, so the others keep their code.
struct BackwardFisheyeParams : BackwardParams {
    gsb_camera_model cam;
};
template <bool FISHEYE>
using PbParams = std::conditional_t<FISHEYE, BackwardFisheyeParams, BackwardParams>;
template <bool CAMERA, bool AA, bool FISHEYE = false>
__global__ void __launch_bounds__(PB_THREADS) k_preprocess_backward(const __grid_constant__ PbParams<FISHEYE> P) {
    static_assert(!(CAMERA && FISHEYE), "no camera gradient through the fisheye lens");
    const uint32_t nv = P.ctl->num_visible;
    const gsb_uniforms& U = P.ubo;
    const float* pm = U.proj_mat;
    const float* vm = U.view_mat;
    const bool store_v = !CAMERA || P.grad_vertices != nullptr;  // frozen scene: camera only
    float cam[GSB_UBO_WORDS];
    if constexpr (CAMERA) {
#pragma unroll
        for (int j = 0; j < GSB_UBO_WORDS; j++) cam[j] = 0.f;
    }
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

        // ---- forward of preprocess.comp:130-157 (k_project's values) ----
        const ClipView cv = clip_view(U, px, py, pz);
        const float p_w = cv.p_w, ndcx = cv.ndcx, ndcy = cv.ndcy, vz = cv.vz;
        const Jacobian J = jacobian(U, cv.vx, cv.vy, vz);
        const float limx = J.limx, limy = J.limy, txtz = J.txtz, tytz = J.tytz, tx = J.tx, ty = J.ty;
        const float focal_x = J.focal_x, focal_y = J.focal_y, ja = J.ja, jb = J.jb, g0 = J.g0, g1 = J.g1;
        FisheyeGeo F;
        FisheyeJ FJ;
        if constexpr (FISHEYE) {
            F = fisheye_geo(P.cam, cv.vx, cv.vy, vz);
            FJ = fisheye_jacobian(P.cam, vm, F, cv.vx, cv.vy);
        }
        const auto& JW = [&]() -> const auto& {
            if constexpr (FISHEYE) return FJ;
            else return J;
        }();
        const float(&T0)[3] = JW.T0, (&T1)[3] = JW.T1;  // rows of J W (W = the view rotation)
        const Cov2d cov = cov2d(T0, T1, __ldg(P.cov_a + i), __ldg(P.cov_b + i));
        const float(&ST0)[3] = cov.tm0, (&ST1)[3] = cov.tm1;  // Sigma T0, Sigma T1
        const float a = cov.m00, b = cov.m10, c = cov.m11;  // b: the [1][0] entry, rounded like k_project's m10
        const float det = a * c - b * b;

        // ---- conic K = (c, -b, a) / det  ->  cov2d (a, b, c): dL/dcov2d = -K dL/dK K ----
        // From k_project's conic (ood = 1 / det) rather than 1 / det^2: det^2 overflows past det ~ 1.8e19 (an isotropic sigma of
        // ~6.5e4 px), while the products of K stay normal from the 0.3 dilation floor to sigma ~ 1e9 px.
        const float ood = 1.0f / det;
        const float k00 = c * ood, k01 = -b * ood, k11 = a * ood;
        const float dA = d[2], dB = d[3], dC = d[4];
        float da = -((k00 * k00 * dA + k00 * k01 * dB) + k01 * k01 * dC);
        float db = -((2.0f * k00 * k01 * dA + (k00 * k11 + k01 * k01) * dB) + 2.0f * k01 * k11 * dC);
        float dc = -((k01 * k01 * dA + k01 * k11 * dB) + k11 * k11 * dC);
        float comp = 1.0f;
        if constexpr (AA) {  // det0 = c00 c11 - b^2, det = a c - b^2 (a = c00 + 0.3, c = c11 + 0.3): k_project's own values
            const float det_f = a * c - cov.m10 * cov.m01, det0 = aa_det0(cov);
            comp = aa_compensation(det0, det_f);
            if (comp > 0.0f) {
                const float h = 0.5f * (d[5] * v[7]) * comp;
                const float gdet0 = h / det0, gdet = -h / det_f;  // dL/d det0, dL/d det
                da += gdet0 * cov.c11 + gdet * c;
                dc += gdet0 * cov.c00 + gdet * a;
                db -= 2.0f * b * (gdet0 + gdet);
            }
        }
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
        if constexpr (FISHEYE) {  // J W -> J -> view-space position (with uv's own share) -> position
            float dJ[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
            for (int r = 0; r < 3; r++) {
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    dJ[0][k] += dT0[r] * vm[r * 4 + k];
                    dJ[1][k] += dT1[r] * vm[r * 4 + k];
                }
            }
            float ftx, fty, ftz;
            fisheye_grad(P.cam, F, FJ, cv.vx, cv.vy, vz, dJ, d[0], d[1], ftx, fty, ftz);
#pragma unroll
            for (int k = 0; k < 3; k++) dp[k] = (vm[k * 4 + 0] * ftx + vm[k * 4 + 1] * fty) + vm[k * 4 + 2] * ftz;
        }

        // ---- colour (preprocess.comp:73-108) -> SH coefficients and the view direction ----
        const float dcr = r2.x > 0.0f ? d[6] : 0.0f;  // :102-104 red clamped at 0 (the record holds the clamped value)
        const float dcg = d[7], dcb = d[8];
        float x, y, z;
        const float len = view_direction(U.camera_position, px, py, pz, x, y, z);
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
            if (store_v) {
                gv[12 + 3 * k + 0] = basis[k] * dcr;
                gv[12 + 3 * k + 1] = basis[k] * dcg;
                gv[12 + 3 * k + 2] = basis[k] * dcb;
            }
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

        if constexpr (CAMERA) {  // ---- this survivor's share of dL/d(UBO), the UBO's fields taken as independent inputs ----
            const float p3[3] = {px, py, pz}, dv[3] = {dvx, dvy, dvz}, dh[4] = {dhx, dhy, 0.f, dhw};
#pragma unroll
            for (int r = 0; r < 3; r++) {
                // v = V p (rows 0-2), through J's dependence on v
#pragma unroll
                for (int c = 0; c < 3; c++) cam[U_VIEW + c * 4 + r] += dv[r] * p3[c];
                cam[U_VIEW + 12 + r] += dv[r];
                // the view rotation inside J W
                cam[U_VIEW + r * 4 + 0] += dT0[r] * ja;
                cam[U_VIEW + r * 4 + 1] += dT1[r] * jb;
                cam[U_VIEW + r * 4 + 2] += dT0[r] * g0 + dT1[r] * g1;
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {  // h = P p (rows 0, 1, 3)
                if (k == 2) continue;
#pragma unroll
                for (int c = 0; c < 3; c++) cam[U_PROJ + c * 4 + k] += dh[k] * p3[c];
                cam[U_PROJ + 12 + k] += dh[k];
            }
            // the view direction p - camera_position
            cam[U_CAMPOS + 0] -= (ddx - x * dot) / len;
            cam[U_CAMPOS + 1] -= (ddy - y * dot) / len;
            cam[U_CAMPOS + 2] -= (ddz - z * dot) / len;
            // focal = size / (2 tan_fov) feeds ja / jb and g0 / g1; the clamp limit is 1.3 tan_fov
            const float dfx = dja / vz - (tx / (vz * vz)) * dg0, dfy = djb / vz - (ty / (vz * vz)) * dg1;
            float dtfx = -(focal_x / U.tan_fovx) * dfx, dtfy = -(focal_y / U.tan_fovy) * dfy;
            if (txtz < -limx || txtz > limx) dtfx += (txtz > 0.0f ? 1.3f : -1.3f) * vz * dtx;
            if (tytz < -limy || tytz > limy) dtfy += (tytz > 0.0f ? 1.3f : -1.3f) * vz * dty;
            cam[U_TANX] += dtfx;
            cam[U_TANY] += dtfy;
        }
        if (!store_v) continue;

        // ---- Sigma = M^T M, M = diag(s) R(q) (precomp_cov3d.comp:25-48, the quaternion as stored) ----
        const float s[3] = {v[4], v[5], v[6]};
        const float qw = v[8], qx = v[9], qy = v[10], qz = v[11];
        float R[3][3];  // R[c][r] as in k_ingest_cov3d
        rotation_from_quaternion(qw, qx, qy, qz, R);
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
        gv[7] = AA ? d[5] * comp : d[5];
        gv[8] = dqw;
        gv[9] = dqx;
        gv[10] = dqy;
        gv[11] = dqz;
    }
    if constexpr (CAMERA) {  // one row of fp64 partial sums per CTA
        __shared__ double s_cam[PB_THREADS / 32][GSB_UBO_WORDS];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int j = 0; j < GSB_UBO_WORDS; j++) {
            double a = 0.0;
            if (cam_word_live(j)) {
                a = (double)cam[j];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(FULL, a, o);
            }
            if (lane == 0) s_cam[warp][j] = a;
        }
        __syncthreads();
        if (threadIdx.x < GSB_UBO_WORDS) {
            double a = 0.0;
#pragma unroll
            for (int w = 0; w < PB_THREADS / 32; w++) a += s_cam[w][threadIdx.x];
            P.cam_partials[(size_t)blockIdx.x * GSB_UBO_WORDS + threadIdx.x] = a;
        }
    }
}

// Sums the `rows` partial rows of k_preprocess_backward<true> in a fixed order (warp w owns words w and w + 32; each lane a
// strided set of rows, then a shuffle tree) and writes the whole fp32 gsb_uniforms of gradients, zero words included.
constexpr int CR_THREADS = 1024;
__global__ void __launch_bounds__(CR_THREADS) k_camera_reduce(const double* __restrict__ partials, uint32_t rows, gsb_uniforms* out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = warp; j < GSB_UBO_WORDS; j += CR_THREADS / 32) {
        double a = 0.0;
        for (uint32_t r = lane; r < rows; r += 32) a += partials[(size_t)r * GSB_UBO_WORDS + j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(FULL, a, o);
        if (lane == 0) reinterpret_cast<float*>(out)[j] = (float)a;  // 0.0f is also the bit pattern of width = height = 0
    }
}

template <int MODE, bool ABSGRAD, bool BG>
cudaError_t launch_blend_det(const BackwardParams& p, float3 bg, cudaStream_t s) {
    constexpr int NACC = BW_NACC + (ABSGRAD ? BW_NABS : 0);
    const size_t smem = (size_t)BW_WARPS * NACC * BW_DET_BATCH * sizeof(float);  // 36 KB, or 44 KB with ABSGRAD
    cudaError_t e = cudaFuncSetAttribute(k_blend_backward<MODE, ABSGRAD, true, BG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k_blend_backward<MODE, ABSGRAD, true, BG><<<p.num_tiles, BW_THREADS, smem, s>>>(bw_params<BG>(p, bg));
    return cudaGetLastError();
}

template <int MODE, bool ABSGRAD>
cudaError_t launch_blend_det(const BackwardParams& p, float3 bg, cudaStream_t s) {
    return has_background(bg) ? launch_blend_det<MODE, ABSGRAD, true>(p, bg, s) : launch_blend_det<MODE, ABSGRAD, false>(p, bg, s);
}

template <bool BG>
void launch_blend_backward(const BackwardParams& p, float3 bg, cudaStream_t s) {
    const bool density = p.density != nullptr;
    if (p.mode == GSB_MODE_EXACT) {
        if (density) k_blend_backward<GSB_MODE_EXACT, true, false, BG><<<p.num_tiles, BW_THREADS, 0, s>>>(bw_params<BG>(p, bg));
        else k_blend_backward<GSB_MODE_EXACT, false, false, BG><<<p.num_tiles, BW_THREADS, 0, s>>>(bw_params<BG>(p, bg));
    } else {
        if (density) k_blend_backward<GSB_MODE_FAST, true, false, BG><<<p.num_tiles, BW_THREADS, 0, s>>>(bw_params<BG>(p, bg));
        else k_blend_backward<GSB_MODE_FAST, false, false, BG><<<p.num_tiles, BW_THREADS, 0, s>>>(bw_params<BG>(p, bg));
    }
}

// gsb_background_gradient: one CTA per row r, r + grid, ... of the frame (grid = background_grad_rows(H)); each thread sums
// T_final * g of its pixels x = tid, tid + 256, ... in fp64 (the products of two floats are exact), then a shuffle tree and
// the 8 warps in order give the CTA's row of 3 partials.  k_background_reduce sums the rows in a fixed order.
constexpr int BG_THREADS = 256;
constexpr uint32_t BG_MAX_ROWS = 2048;
__global__ void __launch_bounds__(BG_THREADS) k_background_grad(const uint2* __restrict__ record, const unsigned char* __restrict__ grad_image,
                                                                size_t pitch, uint32_t width, uint32_t height, double* __restrict__ partials) {
    __shared__ double s_w[BG_THREADS / 32][3];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    for (uint32_t y = blockIdx.x; y < height; y += gridDim.x) {
        const uint2* rec = record + (size_t)y * width;
        const float4* g = reinterpret_cast<const float4*>(grad_image + (size_t)y * pitch);
        for (uint32_t x = threadIdx.x; x < width; x += BG_THREADS) {
            const double t = (double)__uint_as_float(__ldg(&rec[x].x));
            const float4 v = __ldg(g + x);  // A is ignored: the output's A is constant
            a0 = __dadd_rn(a0, __dmul_rn(t, (double)v.x));
            a1 = __dadd_rn(a1, __dmul_rn(t, (double)v.y));
            a2 = __dadd_rn(a2, __dmul_rn(t, (double)v.z));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(FULL, a0, o);
        a1 += __shfl_xor_sync(FULL, a1, o);
        a2 += __shfl_xor_sync(FULL, a2, o);
    }
    if (lane == 0) {
        s_w[warp][0] = a0;
        s_w[warp][1] = a1;
        s_w[warp][2] = a2;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        double a = 0.0;
#pragma unroll
        for (int w = 0; w < BG_THREADS / 32; w++) a += s_w[w][threadIdx.x];
        partials[(size_t)blockIdx.x * 3 + threadIdx.x] = a;
    }
}

// One CTA of three warps: warp c sums column c of the `rows` partial rows (lane-strided, then a shuffle tree) and stores it,
// rounded once, into out[c].
__global__ void __launch_bounds__(96) k_background_reduce(const double* __restrict__ partials, uint32_t rows, float* out) {
    const int lane = threadIdx.x & 31, c = threadIdx.x >> 5;
    double a = 0.0;
    for (uint32_t r = lane; r < rows; r += 32) a += partials[(size_t)r * 3 + c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(FULL, a, o);
    if (lane == 0) out[c] = (float)a;
}

// gsb_set_backward_deterministic: the per-survivor sums of the blend backward without atomics.  The blend stores one slot
// per (tile, entry); a stable sort of (compact id, list position) over the M entries groups each survivor's slots in tile
// order, its last pass publishing each survivor's run; k_det_reduce sums every run in order.  Integer atomics remain
// (the sort's counters and the runs' atomicMin), but their results do not depend on the order they land in.
cudaError_t launch_det_sums(const BackwardParams& p, float3 bg, const DetBackward& d, unsigned grid, cudaStream_t s) {
    const bool density = p.density != nullptr;
    cudaError_t e = cudaMemsetAsync(d.sc, 0, sizeof(SortCtl), s);
    if (e != cudaSuccess) return e;
    // look-back words no earlier call has tagged: zeroed here, tagged 1.. by this sort's passes (epoch 0 = not published)
    if ((e = cudaMemsetAsync(d.status, 0, (size_t)d.status_tiles * 256 * sizeof(unsigned long long), s)) != cudaSuccess) return e;
    k_det_prepare<<<grid, PB_THREADS, 0, s>>>(p.vals, p.ctl, d.keys[0], d.pos[0], d.runs);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    SortParams sp;
    sp.keys[0] = d.keys[0];
    sp.keys[1] = d.keys[1];
    sp.vals[0] = d.pos[0];
    sp.vals[1] = d.pos[1];
    sp.d_m = &p.ctl->num_instances;
    sp.m_hint = d.m_hint;
    sp.key_bits = d.key_bits;
    sp.status = d.status;
    sp.status_tiles = d.status_tiles;
    sp.epoch_base = 1;
    sp.sc = d.sc;
    sp.num_sms = p.num_sms;
    sp.ranges = d.runs;  // the last pass: (start, ~end) of each compact id's run
    sp.discard_sorted_keys = true;
    uint32_t passes = 0;
    if ((e = launch_sort(sp, &passes, s)) != cudaSuccess) return e;
    if (passes == 0) return cudaErrorInvalidValue;  // key_bits >= 1: the runs come from the last pass
    if (p.num_tiles) {
        if (p.mode == GSB_MODE_EXACT) e = density ? launch_blend_det<GSB_MODE_EXACT, true>(p, bg, s) : launch_blend_det<GSB_MODE_EXACT, false>(p, bg, s);
        else e = density ? launch_blend_det<GSB_MODE_FAST, true>(p, bg, s) : launch_blend_det<GSB_MODE_FAST, false>(p, bg, s);
        if (e != cudaSuccess) return e;
    }
    const uint32_t* sorted_pos = d.pos[passes & 1];
    if (density) k_det_reduce<true><<<grid, PB_THREADS, 0, s>>>(p, sorted_pos, d.runs);
    else k_det_reduce<false><<<grid, PB_THREADS, 0, s>>>(p, sorted_pos, d.runs);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_backward(const BackwardParams& p, bool antialiased, float3 background, cudaStream_t s, const DetBackward* det,
                            const gsb_camera_model* fisheye) {
    if (fisheye && p.grad_ubo) return cudaErrorInvalidValue;
    const bool density = p.density != nullptr;
    // grid-stride over N_v, which stays on the device: the grid comes from the SM count
    const unsigned grid = (unsigned)p.num_sms * 4u;
    if (det) {
        cudaError_t e = launch_det_sums(p, background, *det, grid, s);
        if (e != cudaSuccess) return e;
    } else if (p.num_tiles) {
        if (has_background(background)) launch_blend_backward<true>(p, background, s);  // a frame of gsb_set_background
        else launch_blend_backward<false>(p, background, s);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    if (density) {  // reads d uv before k_preprocess_backward clears it
        k_density_accumulate<<<grid, PB_THREADS, 0, s>>>(p);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    if (fisheye) {  // vertex gradients only (checked above)
        const BackwardFisheyeParams fp{p, *fisheye};
        if (antialiased) k_preprocess_backward<false, true, true><<<grid, PB_THREADS, 0, s>>>(fp);
        else k_preprocess_backward<false, false, true><<<grid, PB_THREADS, 0, s>>>(fp);
        return cudaGetLastError();
    }
    if (!p.grad_ubo) {
        if (antialiased) k_preprocess_backward<false, true><<<grid, PB_THREADS, 0, s>>>(p);
        else k_preprocess_backward<false, false><<<grid, PB_THREADS, 0, s>>>(p);
        return cudaGetLastError();
    }
    if (antialiased) k_preprocess_backward<true, true><<<grid, PB_THREADS, 0, s>>>(p);
    else k_preprocess_backward<true, false><<<grid, PB_THREADS, 0, s>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k_camera_reduce<<<1, CR_THREADS, 0, s>>>(p.cam_partials, grid, p.grad_ubo);
    return cudaGetLastError();
}

uint32_t background_grad_rows(uint32_t height) { return std::min(height, BG_MAX_ROWS); }

cudaError_t launch_background_grad(const uint2* record, const float* grad_image, size_t row_pitch_bytes, uint32_t width,
                                   uint32_t height, double* partials, float* out, cudaStream_t s) {
    const uint32_t rows = background_grad_rows(height);
    k_background_grad<<<rows, BG_THREADS, 0, s>>>(record, reinterpret_cast<const unsigned char*>(grad_image), row_pitch_bytes, width,
                                                  height, partials);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k_background_reduce<<<1, 96, 0, s>>>(partials, rows, out);
    return cudaGetLastError();
}

}  // namespace gsb
