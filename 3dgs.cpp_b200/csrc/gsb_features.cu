// gsb_features.cu -- rendered feature maps of a recorded frame and their gradients (DESIGN.md section 21): C per-Gaussian
// channels composited over 0 with the frame's own contributors, F_c = sum_i f_ic alpha_i T_i.
//
// The channel count is a runtime value up to 128, so these are kernels of their own over the last recorded frame -- its
// per-tile lists, survivor records and per-pixel (T_final, last) -- and not instantiations of k_blend / k_blend_backward:
// those keep their register and shared-memory budgets and their code.  Channels are processed FW at a time (4 when C <= 4,
// 16 otherwise), each chunk walking the tile's list again, so registers, shared memory and the deterministic slots are
// bounded independently of C.
//
//   k_render_features   one CTA per 16 x 16 tile, one pixel per thread, front to back up to the tile's largest recorded
//                       last-contributor position.  Every (pixel, entry) pair re-evaluates power and alpha with the frame's
//                       arithmetic (EXACT: k_blend's ops + exp_shared_inrange; FAST: the same FMAs + __expf) and takes the
//                       entry iff its position is at most the pixel's recorded last and it passes the power and 1/255 tests:
//                       exactly the frame's contributor set, whose T' < 1e-4 break lies behind `last`.  T is the forward's
//                       product, so with f = the record's colour (depth key) F is the image's RGB over black (gsb_render_depth's
//                       D) bit for bit: EXACT adds (f * alpha) * T, FAST f * (alpha * T), each with __fadd_rn.
//   k_feature_backward  the same tile walk back to front from T_final, T recovered by division like k_blend_backward.  With
//                       g = dL/dF of the pixel's chunk and acc_c its features behind the entry (from 0, one register per
//                       channel), dL/dalpha_i gains T_i sum_c g_c (f_ic - acc_c) in k_blend_backward's order of operations,
//                       acc_c <- f_ic alpha + (1 - alpha) acc_c, and dL/df_ic = g_c alpha_i T_i.  dL/dalpha goes on to d uv, d conic, d opacity as in k_blend_backward (no
//                       gradient through a clamped alpha), and |d u|, |d v| per pixel for the density statistics.  Per entry the
//                       warp reduces its 8 + FW values by shuffles; then
//                         atomic:        fp64 shared-memory atomics per CTA, one global fp64 atomic per value and tile into
//                                        the n x 9 geometry scratch of the colour pass (columns 0-5), the n x 2 density scratch
//                                        and an n x FW feature scratch, which k_feature_flush rounds into grad_features;
//                         deterministic: per-warp partials summed in warp order into one fp64 slot row per list position, and
//                                        k_feature_det_reduce sums each survivor's run -- the sorted positions and runs of the
//                                        colour pass's deterministic sort -- in order and adds it to the same scratch.
//   k_adam_features     torch.optim.Adam on the n x C raw features (identity activation), dense or over the last frame's
//                       survivors.
// Compiled with -fmad=false like the forward.
#include <algorithm>

#include "gsb_cull.cuh"
#include "gsb_exp.cuh"
#include "gsb_geom.cuh"
#include "gsb_internal.cuh"

namespace gsb {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int FT_THREADS = 256;  // one pixel per thread of a 16 x 16 tile
constexpr int FT_WARPS = FT_THREADS / 32;
constexpr int FT_BATCH = 64;     // list entries staged per batch
constexpr int FT_GEOM = 8;       // per-entry geometry columns: d uv (2), d conic (3), d opacity, |d u|, |d v|
constexpr int FB_THREADS = 256;

struct __align__(16) FtRec {  // k_blend's pre-scaled record: ux uy -A/2 -B | -C/2 opacity power_cut -
    float4 q0, q1;
};

// The tile's staged batch: records and the chunk's FW feature columns of list entries [lo, lo + cnt) (features of rows past C
// are 0).  Also returns the entries' compact ids in s_cid.
template <int FW>
__device__ __forceinline__ void stage_batch(const FeatureParams& P, uint32_t first, uint32_t cnt, FtRec* s_rec, float (*s_f)[FW],
                                            uint32_t* s_cid, uint32_t* s_row) {
    const int tid = threadIdx.x;
    if ((uint32_t)tid < cnt) {
        const uint32_t cid = __ldg(P.vals + first + (uint32_t)tid);
        const float4* rec = P.recs + (size_t)cid * GSB_REC_F4;
        const float4 a = __ldg(rec);
        const float2 b = __ldg(reinterpret_cast<const float2*>(rec + 1));  // conic.z, opacity
        s_rec[tid].q0 = make_float4(a.x, a.y, -0.5f * a.z, -a.w);
        s_rec[tid].q1 = make_float4(-0.5f * b.x, b.y, power_cut(b.y), 0.f);
        s_cid[tid] = cid;
        s_row[tid] = __float_as_uint(__ldg(rec + 3).y);
    }
    __syncthreads();
    for (uint32_t i = (uint32_t)tid; i < cnt * FW; i += FT_THREADS) {
        const uint32_t e = i / FW, c = P.c0 + i % FW;
        s_f[e][i % FW] = c < P.channels ? __ldg(P.features + (size_t)s_row[e] * P.channels + c) : 0.f;
    }
    __syncthreads();
}

// power, exp(power), the unclamped and the clamped alpha of one (pixel, entry) pair, and whether it passes the frame's
// power and 1/255 tests: k_blend's EXACT walk op for op, or its FAST FMAs
template <int MODE>
__device__ __forceinline__ bool eval_alpha(const FtRec& r, float fx, float fy, float& dx, float& dy, float& e, float& raw, float& al) {
    dx = r.q0.x - fx;
    dy = r.q0.y - fy;
    float pw;
    if (MODE == GSB_MODE_EXACT) {
        pw = ((r.q0.z * dx) * dx + (r.q1.x * dy) * dy) + (r.q0.w * dx) * dy;
        e = exp_shared_inrange(pw);
    } else {
        pw = fmaf(r.q0.z * dx, dx, fmaf(r.q1.x * dy, dy, (r.q0.w * dx) * dy));
        e = __expf(pw);
    }
    raw = r.q1.y * e;
    al = fminf(0.99f, raw);
    return !(pw > 0.0f || pw < r.q1.z) && !(al < 1.0f / 255.0f);
}

// The pixel this thread owns (warp w: the 8 x 4 block at (8 (w & 1), 4 (w >> 1)), as in k_blend_backward), its recorded
// (T_final, last), and the largest `last` of the tile.
struct FtPixel {
    uint32_t px, py;
    bool inside;
    float T;
    uint32_t last, max_last;
};
__device__ __forceinline__ FtPixel tile_pixel(const FeatureParams& P, uint32_t* s_max) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tx = blockIdx.x % P.tiles_x, ty = blockIdx.x / P.tiles_x;
    FtPixel q;
    q.px = tx * GSB_TILE + (warp & 1) * 8 + (lane & 7);
    q.py = ty * GSB_TILE + (warp >> 1) * 4 + (lane >> 3);
    q.inside = q.px < P.width && q.py < P.height;
    q.T = 1.0f;
    q.last = 0;
    if (q.inside) {
        const uint2 r = P.record[(size_t)q.py * P.width + q.px];
        q.T = __uint_as_float(r.x);
        q.last = r.y;
    }
    if (tid == 0) *s_max = 0;
    __syncthreads();
    const uint32_t wmax = __reduce_max_sync(FULL, q.last);
    if (lane == 0 && wmax) atomicMax(s_max, wmax);
    __syncthreads();
    q.max_last = *s_max;
    return q;
}

template <int MODE, int FW>
__global__ void __launch_bounds__(FT_THREADS) k_render_features(const __grid_constant__ FeatureParams P) {
    __shared__ FtRec s_rec[FT_BATCH];
    __shared__ float s_f[FT_BATCH][FW];
    __shared__ uint32_t s_cid[FT_BATCH], s_row[FT_BATCH];
    __shared__ uint32_t s_max;
    const FtPixel q = tile_pixel(P, &s_max);
    uint2 range = P.ranges[blockIdx.x];
    range.y = ~range.y;
    const float fx = (float)q.px, fy = (float)q.py;
    float acc[FW];
#pragma unroll
    for (int c = 0; c < FW; c++) acc[c] = 0.f;
    float T = 1.0f;  // the forward's transmittance, front to back
    if (range.x < range.y) {
        for (uint32_t lo = 0; lo < q.max_last; lo += FT_BATCH) {
            const uint32_t cnt = min((uint32_t)FT_BATCH, q.max_last - lo);
            __syncthreads();  // the previous batch's walk is done with the staging
            stage_batch<FW>(P, range.x + lo, cnt, s_rec, s_f, s_cid, s_row);
            for (uint32_t k = 0; k < cnt; k++) {
                float dx, dy, e, raw, al;
                const bool pass = eval_alpha<MODE>(s_rec[k], fx, fy, dx, dy, e, raw, al);
                if (!(pass && lo + k + 1u <= q.last)) continue;
                if (MODE == GSB_MODE_EXACT) {
#pragma unroll
                    for (int c = 0; c < FW; c++) acc[c] = __fadd_rn(acc[c], (s_f[k][c] * al) * T);
                } else {
                    const float w = al * T;
#pragma unroll
                    for (int c = 0; c < FW; c++) acc[c] = __fadd_rn(acc[c], s_f[k][c] * w);
                }
                T = T * (1.0f - al);
            }
        }
    }
    if (!q.inside) return;
    float* out = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(P.map) + (size_t)q.py * P.map_pitch) + (size_t)q.px * P.channels + P.c0;
#pragma unroll
    for (int c = 0; c < FW; c++)
        if (P.c0 + c < P.channels) out[c] = acc[c];
}

// DET: lane 0 of each warp keeps the warp's shuffle sums in its own fp32 row of dynamic shared memory,
// [warp][FT_GEOM + FW][FT_BATCH]; at the flush thread k sums the 8 warps in order in fp64 into the slot row of entry k's list
// position.  Every position of the tile's list is stored, +0 for entries no pixel of the tile has as contributor, so that
// tile-cull levels 0 and 1 give the same sums.
__device__ __forceinline__ float* ft_partials() {
    extern __shared__ float s_ft_dyn[];
    return s_ft_dyn;
}

template <int MODE, int FW, bool DET>
__global__ void __launch_bounds__(FT_THREADS) k_feature_backward(const __grid_constant__ FeatureParams P) {
    constexpr int NCOL = FT_GEOM + FW;
    __shared__ FtRec s_rec[FT_BATCH];
    __shared__ float s_f[FT_BATCH][FW];
    __shared__ uint32_t s_cid[FT_BATCH], s_row[FT_BATCH];
    __shared__ double s_acc[DET ? 1 : FT_BATCH][NCOL];
    __shared__ uint32_t s_max;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    FtPixel q = tile_pixel(P, &s_max);
    uint2 range = P.ranges[blockIdx.x];
    range.y = ~range.y;
    if (range.x >= range.y) return;  // empty list: every pixel has last == 0
    const float fx = (float)q.px, fy = (float)q.py;
    float g[FW];
#pragma unroll
    for (int c = 0; c < FW; c++) g[c] = 0.f;
    if (q.inside) {
        const float* gm = reinterpret_cast<const float*>(reinterpret_cast<const unsigned char*>(P.grad_map) + (size_t)q.py * P.grad_pitch) +
                          (size_t)q.px * P.channels + P.c0;
#pragma unroll
        for (int c = 0; c < FW; c++)
            if (P.c0 + c < P.channels) g[c] = gm[c];
    }
    float T = q.T, acc[FW];  // the chunk's features behind the current entry, per unit of its transmittance
#pragma unroll
    for (int c = 0; c < FW; c++) acc[c] = 0.f;
    for (uint32_t hi = q.max_last; hi > 0;) {
        const uint32_t lo = hi > (uint32_t)FT_BATCH ? hi - FT_BATCH : 0u;
        const uint32_t cnt = hi - lo;
        __syncthreads();  // the previous batch's walk and flush are done with the staging and s_acc
        if constexpr (!DET) {
            if ((uint32_t)tid < cnt) {
#pragma unroll
                for (int j = 0; j < NCOL; j++) s_acc[tid][j] = 0.0;
            }
        }
        stage_batch<FW>(P, range.x + lo, cnt, s_rec, s_f, s_cid, s_row);
        for (int k = (int)cnt - 1; k >= 0; k--) {
            float dx, dy, e, raw, al;
            const bool contrib = eval_alpha<MODE>(s_rec[k], fx, fy, dx, dy, e, raw, al) && lo + (uint32_t)k + 1u <= q.last;
            if (!__any_sync(FULL, contrib)) {
                if constexpr (DET) {
                    if (lane == 0) {
#pragma unroll
                        for (int j = 0; j < NCOL; j++) ft_partials()[(warp * NCOL + j) * FT_BATCH + k] = 0.f;
                    }
                }
                continue;
            }
            float v[NCOL];
#pragma unroll
            for (int j = 0; j < NCOL; j++) v[j] = 0.f;
            if (contrib) {
                T = T / (1.0f - al);  // transmittance in front of this entry
                const float w = al * T;
                // k_blend_backward's colour terms, channel for channel: with f = the colours (and g = 0 past them) the sum is
                // its dL/dalpha bit for bit
                float sum = 0.f;
#pragma unroll
                for (int c = 0; c < FW; c++) {
                    const float f = s_f[k][c];
                    sum += g[c] * (f - acc[c]);
                    acc[c] = f * al + (1.0f - al) * acc[c];
                    v[FT_GEOM + c] = g[c] * w;  // d f
                }
                const float dal = T * sum;
                if (!(raw > 0.99f)) {  // alpha clamped at 0.99: no gradient through it
                    const FtRec& r = s_rec[k];
                    const float dpw = dal * raw;
                    v[5] = dal * e;                               // d opacity
                    v[0] = dpw * (2.0f * r.q0.z * dx + r.q0.w * dy);  // d u
                    v[1] = dpw * (2.0f * r.q1.x * dy + r.q0.w * dx);  // d v
                    v[2] = dpw * (-0.5f * dx * dx);                   // d A
                    v[3] = dpw * (-dx * dy);                          // d B
                    v[4] = dpw * (-0.5f * dy * dy);                   // d C
                    v[6] = fabsf(v[0]);                               // this pixel's own |d u|, |d v|
                    v[7] = fabsf(v[1]);
                }
            }
#pragma unroll
            for (int j = 0; j < NCOL; j++) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(FULL, v[j], o);
            }
            if (lane == 0) {
#pragma unroll
                for (int j = 0; j < NCOL; j++) {
                    if constexpr (DET) ft_partials()[(warp * NCOL + j) * FT_BATCH + k] = v[j];
                    else if (v[j] != 0.f) atomicAdd(&s_acc[k][j], (double)v[j]);
                }
            }
        }
        __syncthreads();
        if ((uint32_t)tid < cnt) {
            if constexpr (DET) {  // warps 0..7 in order, in fp64 from +0.0
                double* dst = P.det_slots + (size_t)(range.x + lo + (uint32_t)tid) * NCOL;
#pragma unroll
                for (int j = 0; j < NCOL; j++) {
                    double a = 0.0;
#pragma unroll
                    for (int w = 0; w < FT_WARPS; w++) a += (double)ft_partials()[(w * NCOL + j) * FT_BATCH + tid];
                    dst[j] = a;
                }
            } else {
                const uint32_t cid = s_cid[tid];
                if (P.scratch) {
#pragma unroll
                    for (int j = 0; j < 6; j++)
                        if (s_acc[tid][j] != 0.0) atomicAdd(P.scratch + (size_t)cid * 9 + j, s_acc[tid][j]);
                }
                if (P.abs_scratch) {
#pragma unroll
                    for (int j = 0; j < 2; j++)
                        if (s_acc[tid][6 + j] != 0.0) atomicAdd(P.abs_scratch + (size_t)cid * 2 + j, s_acc[tid][6 + j]);
                }
                if (P.feat_scratch) {
#pragma unroll
                    for (int c = 0; c < FW; c++)
                        if (s_acc[tid][FT_GEOM + c] != 0.0) atomicAdd(P.feat_scratch + (size_t)cid * FW + c, s_acc[tid][FT_GEOM + c]);
                }
            }
        }
        hi = lo;
    }
    if constexpr (DET) {  // the entries behind every pixel's last contributor: +0, so the reduction reads no stale slot
        const uint32_t len = range.y - range.x;
        for (uint32_t p = q.max_last + (uint32_t)tid; p < len; p += FT_THREADS) {
            double* dst = P.det_slots + (size_t)(range.x + p) * NCOL;
#pragma unroll
            for (int j = 0; j < NCOL; j++) dst[j] = 0.0;
        }
    }
}

// Atomic path, after a chunk's k_feature_backward: one thread per survivor rounds its FW feature sums into its grad_features
// row and returns the scratch to zero.
template <int FW>
__global__ void __launch_bounds__(FB_THREADS) k_feature_flush(const __grid_constant__ FeatureParams P) {
    const uint32_t nv = P.ctl->num_visible;
    for (uint32_t cid = blockIdx.x * blockDim.x + threadIdx.x; cid < nv; cid += gridDim.x * blockDim.x) {
        double* sc = P.feat_scratch + (size_t)cid * FW;
        const uint32_t row = __float_as_uint(__ldg(P.recs + (size_t)cid * GSB_REC_F4 + 3).y);
        float* gf = P.grad_features + (size_t)row * P.channels + P.c0;
#pragma unroll
        for (int c = 0; c < FW; c++) {
            const double a = sc[c];
            sc[c] = 0.0;
            if (P.c0 + c < P.channels) gf[c] = (float)a;
        }
    }
}

// Deterministic path, after a chunk's k_feature_backward<..., DET = true>: one thread per survivor sums its slots in run order
// (ascending list position = tile order) in fp64 from +0.0 and adds them to the geometry and density scratch (after the
// colour pass's sums, or the earlier chunks'), and stores its feature gradient.
template <int FW>
__global__ void __launch_bounds__(FB_THREADS) k_feature_det_reduce(const __grid_constant__ FeatureParams P) {
    constexpr int NCOL = FT_GEOM + FW;
    const uint32_t nv = P.ctl->num_visible;
    for (uint32_t cid = blockIdx.x * blockDim.x + threadIdx.x; cid < nv; cid += gridDim.x * blockDim.x) {
        double s[NCOL];
#pragma unroll
        for (int j = 0; j < NCOL; j++) s[j] = 0.0;
        const uint2 r = __ldg(P.runs + cid);
        if (r.x != 0xffffffffu) {  // a survivor in no list keeps zeros
            for (uint32_t j = r.x, end = ~r.y; j < end; j++) {
                const double* sl = P.det_slots + (size_t)__ldg(P.pos + j) * NCOL;
#pragma unroll
                for (int k = 0; k < NCOL; k++) s[k] += __ldg(sl + k);
            }
        }
        if (P.scratch) {
#pragma unroll
            for (int j = 0; j < 6; j++) P.scratch[(size_t)cid * 9 + j] += s[j];
        }
        if (P.abs_scratch) {
            P.abs_scratch[(size_t)cid * 2] += s[6];
            P.abs_scratch[(size_t)cid * 2 + 1] += s[7];
        }
        if (P.grad_features) {
            const uint32_t row = __float_as_uint(__ldg(P.recs + (size_t)cid * GSB_REC_F4 + 3).y);
            float* gf = P.grad_features + (size_t)row * P.channels + P.c0;
#pragma unroll
            for (int c = 0; c < FW; c++)
                if (P.c0 + c < P.channels) gf[c] = (float)s[FT_GEOM + c];
        }
    }
}

template <int FW>
cudaError_t feature_backward_chunk(const FeatureParams& p, bool det, cudaStream_t s) {
    const unsigned grid = (unsigned)p.num_sms * 4u;
    if (det) {
        constexpr size_t smem = (size_t)FT_WARPS * (FT_GEOM + FW) * FT_BATCH * sizeof(float);  // 48 KB at FW = 16
        auto k = p.mode == GSB_MODE_EXACT ? k_feature_backward<GSB_MODE_EXACT, FW, true> : k_feature_backward<GSB_MODE_FAST, FW, true>;
        cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        k<<<p.num_tiles, FT_THREADS, smem, s>>>(p);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        k_feature_det_reduce<FW><<<grid, FB_THREADS, 0, s>>>(p);
        return cudaGetLastError();
    }
    if (p.mode == GSB_MODE_EXACT) k_feature_backward<GSB_MODE_EXACT, FW, false><<<p.num_tiles, FT_THREADS, 0, s>>>(p);
    else k_feature_backward<GSB_MODE_FAST, FW, false><<<p.num_tiles, FT_THREADS, 0, s>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || !p.grad_features) return e;
    k_feature_flush<FW><<<grid, FB_THREADS, 0, s>>>(p);
    return cudaGetLastError();
}

// ---- gsb_adam_step_features: one thread per feature, grid-stride over n x C (or N_v x C, read on the device) ----
__global__ void __launch_bounds__(FB_THREADS) k_adam_features(const __grid_constant__ FeatureAdamParams P) {
    const AdamUpdate adam{1.0f - P.beta1, 1.0f - P.beta2, P.beta2, P.eps, P.bias_correction2_sqrt};
    const float step = P.lr / P.bias_correction1;
    const uint64_t rows = P.recs ? (uint64_t)P.ctl->num_visible : P.n;
    const uint64_t count = rows * P.channels;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = i / P.channels, c = i - r * P.channels;
        const uint64_t row = P.recs ? __float_as_uint(__ldg(P.recs + r * GSB_REC_F4 + 3).y) : r;
        const uint64_t w = row * P.channels + c;
        float x = P.features[w], m = P.exp_avg[w], v = P.exp_avg_sq[w];
        adam(P.grad[w], x, m, v, step);
        P.features[w] = x;
        P.exp_avg[w] = m;
        P.exp_avg_sq[w] = v;
    }
}

}  // namespace

uint32_t feature_chunk(uint32_t channels) { return channels <= 4 ? 4u : 16u; }

cudaError_t launch_render_features(FeatureParams p, cudaStream_t s) {
    if (p.num_tiles == 0) return cudaSuccess;
    const uint32_t fw = feature_chunk(p.channels);
    for (p.c0 = 0; p.c0 < p.channels; p.c0 += fw) {
        if (fw == 4) {
            if (p.mode == GSB_MODE_EXACT) k_render_features<GSB_MODE_EXACT, 4><<<p.num_tiles, FT_THREADS, 0, s>>>(p);
            else k_render_features<GSB_MODE_FAST, 4><<<p.num_tiles, FT_THREADS, 0, s>>>(p);
        } else {
            if (p.mode == GSB_MODE_EXACT) k_render_features<GSB_MODE_EXACT, 16><<<p.num_tiles, FT_THREADS, 0, s>>>(p);
            else k_render_features<GSB_MODE_FAST, 16><<<p.num_tiles, FT_THREADS, 0, s>>>(p);
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_feature_backward(FeatureParams p, bool det, cudaStream_t s) {
    if (p.num_tiles == 0) return cudaSuccess;
    const uint32_t fw = feature_chunk(p.channels);
    for (p.c0 = 0; p.c0 < p.channels; p.c0 += fw) {
        const cudaError_t e = fw == 4 ? feature_backward_chunk<4>(p, det, s) : feature_backward_chunk<16>(p, det, s);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_adam_features(const FeatureAdamParams& p, int num_sms, cudaStream_t s) {
    if (p.n == 0 || p.channels == 0) return cudaSuccess;
    const uint64_t blocks = std::min<uint64_t>((p.n * p.channels + FB_THREADS - 1) / FB_THREADS, (uint64_t)num_sms * 8);
    k_adam_features<<<(unsigned)blocks, FB_THREADS, 0, s>>>(p);
    return cudaGetLastError();
}

}  // namespace gsb
