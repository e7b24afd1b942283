// gsb_optim.cu -- k_adam_step: one Adam step (torch.optim.Adam, no weight decay) of the scene's raw parameters from the
// gradient of the activated records, which also writes the new activated records and the context's scene words, so that
// the next frame needs no upload (DESIGN.md section 12).
//
// One thread per float4 of a row: the 15 float4 of a row are independent through the chain rule, Adam and the activation
// (position, scale + opacity, quaternion, and 12 of SH each stay inside one float4), so every array is read and written
// with 240 contiguous bytes per row.  Only the scene's Sigma needs position, scale + opacity and quaternion together: those
// three threads leave their activated float4 in shared memory and one thread per row stores the scene words.  No atomics.
// FILTER (gsb_adam_step_filter3d, DESIGN.md section 18): the scale and opacity of each row go through Mip-Splatting's 3D
// smoothing filter of its variance v, in the activation and in the chain rule; only the k == 1 thread reads v.
// Compiled with -fmad=false: every fp32 operation is one IEEE operation unless spelled fmaf().
#include <algorithm>

#include "gsb_geom.cuh"
#include "gsb_internal.cuh"

namespace gsb {
namespace {

constexpr int AD_ROWS = 16;                // rows per CTA and loop trip
constexpr int AD_THREADS = AD_ROWS * 15;   // one thread per float4 of a row

using Adam = AdamUpdate;

__device__ __forceinline__ float sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float4 normalise(float4 q, float& norm) {
    norm = sqrtf(((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w);
    return make_float4(q.x / norm, q.y / norm, q.z / norm, q.w / norm);
}

// Mip-Splatting's filtered scale and opacity of log scales (lx, ly, lz), opacity logit lw and filter variance var, each
// operation one IEEE op in this order: s = exp(l), q = s s, d = q + v, e = sqrt(d), r = q / d; c = sqrt((r0 r1) r2), the
// opacity factor as a product of per-axis ratios (prod q / prod d underflows once prod s^2 < 1e-38).  With v = 0 every
// value is the plain activation's: sqrt(fl(s s)) = s, r = 1, c = 1.
struct Filtered {
    float s[3], d[3], e[3], o, c, of;
    __device__ __forceinline__ Filtered(float4 x, float var) {
        const float l[3] = {x.x, x.y, x.z};
        float r[3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            s[j] = expf(l[j]);
            const float q = s[j] * s[j];
            d[j] = q + var;
            e[j] = sqrtf(d[j]);
            r[j] = q / d[j];
        }
        c = sqrtf((r[0] * r[1]) * r[2]);
        o = sigmoid(x.w);
        of = o * c;
    }
};

template <bool FILTER>
__global__ void __launch_bounds__(AD_THREADS) k_adam_step(const AdamParams P) {
    __shared__ float4 s_rec[AD_ROWS][3];  // activated position, scale_opacity, rotation of the trip's rows
    __shared__ uint32_t s_row[AD_ROWS];
    const uint32_t t = threadIdx.x, r = t / 15, k = t - r * 15;
    const Adam adam{1.0f - P.beta1, 1.0f - P.beta2, P.beta2, P.eps, P.bias_correction2_sqrt};
    // step sizes lr / bc1 of the float4's columns x, y, z and w: float4 1 is (scale, opacity), float4 3 (SH DC, SH rest)
    const int group_xyz = k == 0 ? 0 : k == 1 ? 1 : k == 2 ? 3 : k == 3 ? 4 : 5;
    const int group_w = k == 1 ? 2 : k == 2 ? 3 : 5;
    const float step = P.lr[group_xyz] / P.bias_correction1, step_w = P.lr[group_w] / P.bias_correction1;
    const uint64_t count = P.recs ? (uint64_t)P.ctl->num_visible : P.n;
    for (uint64_t base = (uint64_t)blockIdx.x * AD_ROWS; base < count; base += (uint64_t)gridDim.x * AD_ROWS) {
        const uint64_t i = base + r;
        if (i < count) {
            const uint32_t row = P.recs ? __float_as_uint(P.recs[i * GSB_REC_F4 + 3].y) : (uint32_t)i;
            const uint64_t w = (uint64_t)row * 15 + k;
            const float4 g = P.grad[w];
            float4 x = P.params[w], m = P.exp_avg[w], v = P.exp_avg_sq[w];
            float4 a;  // the activated float4
            if (k == 0) {  // position (column 3 is neither read as a parameter nor stored)
                adam(g.x, x.x, m.x, v.x, step);
                adam(g.y, x.y, m.y, v.y, step);
                adam(g.z, x.z, m.z, v.z, step);
                float* px = reinterpret_cast<float*>(P.params + w);
                float* pm = reinterpret_cast<float*>(P.exp_avg + w);
                float* pv = reinterpret_cast<float*>(P.exp_avg_sq + w);
                px[0] = x.x, px[1] = x.y, px[2] = x.z;
                pm[0] = m.x, pm[1] = m.y, pm[2] = m.z;
                pv[0] = v.x, pv[1] = v.y, pv[2] = v.z;
                a = make_float4(x.x, x.y, x.z, 1.0f);
            } else {
                if (FILTER && k == 1) {  // the record holds e = sqrt(s^2 + v) and o c; v is held constant
                    // d log s = (de s) (s / e) + (d(oc) oc) (v / d), d logit = ((d(oc) c) o) (1 - o)
                    const float var = P.variance[row];
                    const Filtered f(x, var);
                    adam((g.x * f.s[0]) * (f.s[0] / f.e[0]) + (g.w * f.of) * (var / f.d[0]), x.x, m.x, v.x, step);
                    adam((g.y * f.s[1]) * (f.s[1] / f.e[1]) + (g.w * f.of) * (var / f.d[1]), x.y, m.y, v.y, step);
                    adam((g.z * f.s[2]) * (f.s[2] / f.e[2]) + (g.w * f.of) * (var / f.d[2]), x.z, m.z, v.z, step);
                    adam(((g.w * f.c) * f.o) * (1.0f - f.o), x.w, m.w, v.w, step_w);
                    const Filtered a1(x, var);
                    a = make_float4(a1.e[0], a1.e[1], a1.e[2], a1.of);
                } else if (k == 1) {  // log scale, opacity logit: d log s = ds s, d logit = (do o) (1 - o)
                    const float o = sigmoid(x.w);
                    adam(g.x * expf(x.x), x.x, m.x, v.x, step);
                    adam(g.y * expf(x.y), x.y, m.y, v.y, step);
                    adam(g.z * expf(x.z), x.z, m.z, v.z, step);
                    adam((g.w * o) * (1.0f - o), x.w, m.w, v.w, step_w);
                    a = make_float4(expf(x.x), expf(x.y), expf(x.z), sigmoid(x.w));
                } else if (k == 2) {  // quaternion: d q = (d q^ - q^ (q^ . d q^)) / |q|
                    float norm;
                    const float4 qh = normalise(x, norm);
                    const float dot = ((qh.x * g.x + qh.y * g.y) + qh.z * g.z) + qh.w * g.w;
                    adam((g.x - qh.x * dot) / norm, x.x, m.x, v.x, step);
                    adam((g.y - qh.y * dot) / norm, x.y, m.y, v.y, step);
                    adam((g.z - qh.z * dot) / norm, x.z, m.z, v.z, step);
                    adam((g.w - qh.w * dot) / norm, x.w, m.w, v.w, step);
                    a = normalise(x, norm);
                } else {  // SH: the coefficients themselves
                    adam(g.x, x.x, m.x, v.x, step);
                    adam(g.y, x.y, m.y, v.y, step);
                    adam(g.z, x.z, m.z, v.z, step);
                    adam(g.w, x.w, m.w, v.w, step_w);
                    a = x;
                }
                P.params[w] = x;
                P.exp_avg[w] = m;
                P.exp_avg_sq[w] = v;
            }
            P.vertices[w] = a;
            if (k < 3) s_rec[r][k] = a;
            else P.sh[(uint64_t)row * 12 + (k - 3)] = a;
            if (k == 0) s_row[r] = row;
        }
        __syncthreads();
        if (t < AD_ROWS && base + t < count)  // scale_factor 1: gsb_scene_upload's
            store_cov3d(s_rec[t][0], s_rec[t][1], s_rec[t][2], s_row[t], P.pos_op, P.cov_a, P.cov_b, 1.0f);
        __syncthreads();
    }
}

template <bool FILTER>
cudaError_t launch_adam_t(const AdamParams& p, int num_sms, cudaStream_t s) {
    static int per_sm = 0;  // resident CTAs per SM: the grid is one wave, walking the rows grid-stride
    if (per_sm == 0) {
        const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_adam_step<FILTER>, AD_THREADS, 0);
        if (e != cudaSuccess) return e;
        per_sm = per_sm > 0 ? per_sm : 1;
    }
    const uint64_t trips = (p.n + AD_ROWS - 1) / AD_ROWS;  // selective mode: N_v <= n
    const unsigned blocks = (unsigned)std::min<uint64_t>(trips, (uint64_t)num_sms * per_sm);
    k_adam_step<FILTER><<<blocks, AD_THREADS, 0, s>>>(p);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_adam(const AdamParams& p, int num_sms, cudaStream_t s) {
    if (p.n == 0) return cudaSuccess;
    return p.variance ? launch_adam_t<true>(p, num_sms, s) : launch_adam_t<false>(p, num_sms, s);
}

}  // namespace gsb
