// gsb_filter3d.cu -- gsb_filter3d_variance: the per-Gaussian variance of Mip-Splatting's 3D smoothing filter (Yu et al.
// 2024, compute_3D_filter) from the training cameras, in the frame's own camera arithmetic (DESIGN.md section 18).
//
// k_filter3d_depth: one thread per F3_ROWS rows; the cameras pass through shared memory in chunks of F3_CHUNK, of which
// only the 18 words clip_view and ndc2Pix read are staged.  Each row keeps the least view depth over the cameras that see
// it and writes its variance, or -1 when no camera sees it; each CTA folds the largest seen depth of its rows into one word
// with an integer atomicMax (positive floats order as their bits).  k_filter3d_fill then gives the unseen rows that
// depth's variance.  Min and max are exact, so every output word is a function of the inputs on any grid or stream.
// k_filter3d_lens (gsb_filter3d_variance_lens, DESIGN.md section 24) does the same with each camera's own lens model and the
// footprint scale 1 / sigma_min(J) in place of the depth.
// Compiled with -fmad=false: every fp32 operation is one IEEE operation.
#include <algorithm>

#include "gsb_geom.cuh"
#include "gsb_internal.cuh"

namespace gsb {
namespace {

constexpr int F3_THREADS = 256;
constexpr int F3_ROWS = 4;     // rows per thread: one staging of a chunk serves 1024 rows
constexpr int F3_CHUNK = 64;   // cameras per staging (10 KB of shared memory)
constexpr uint32_t F3_WORDS = 18;

// The j-th of the 18 gsb_uniforms words the test reads (j < 18): proj_mat rows x, y and w (words 4-19), view_mat row z
// (words 20-35), width and height (words 36, 37).
__device__ __forceinline__ uint32_t camera_word(uint32_t j) {
    if (j < 12) return 4 + (j & 3) * 4 + ((j >> 2) == 2 ? 3 : (j >> 2));  // proj_mat[4 c + r], r = 0, 1, 3
    if (j < 16) return 20 + (j - 12) * 4 + 2;                              // view_mat[4 c + 2]
    return 36 + (j - 16);
}

// The filter's variance of a Gaussian whose least seen view depth is d: t = d / f, v = (t t) 0.2 (filter_3D =
// d / f sqrt(0.2), used squared).
__device__ __forceinline__ float filter_variance(float d, float focal) {
    const float t = d / focal;
    return (t * t) * 0.2f;
}

__global__ void __launch_bounds__(F3_THREADS) k_filter3d_depth(const float4* __restrict__ vertices, uint64_t n,
                                                               const gsb_uniforms* __restrict__ cams, uint32_t k, float focal,
                                                               uint32_t* __restrict__ dmax, float* __restrict__ variance) {
    __shared__ gsb_uniforms s_cam[F3_CHUNK];
    __shared__ uint32_t s_max[F3_THREADS / 32];
    const uint64_t base = (uint64_t)blockIdx.x * (F3_THREADS * F3_ROWS) + threadIdx.x;
    float px[F3_ROWS], py[F3_ROWS], pz[F3_ROWS], d[F3_ROWS];
    bool seen[F3_ROWS];
#pragma unroll
    for (int j = 0; j < F3_ROWS; j++) {
        const uint64_t i = base + (uint64_t)j * F3_THREADS;
        const float4 p = i < n ? vertices[i * 15] : make_float4(__int_as_float(0x7fffffff), 0.0f, 0.0f, 0.0f);  // NaN: never seen
        px[j] = p.x, py[j] = p.y, pz[j] = p.z;
        d[j] = __int_as_float(0x7f800000);
        seen[j] = false;
    }
    uint32_t* sw = reinterpret_cast<uint32_t*>(s_cam);
    for (uint32_t c0 = 0; c0 < k; c0 += F3_CHUNK) {
        const uint32_t cnt = min((uint32_t)F3_CHUNK, k - c0);
        const uint32_t* gw = reinterpret_cast<const uint32_t*>(cams + c0);
        __syncthreads();  // the previous chunk is read
        for (uint32_t w = threadIdx.x; w < cnt * F3_WORDS; w += F3_THREADS) {
            const uint32_t c = w / F3_WORDS, o = c * 40 + camera_word(w - c * F3_WORDS);
            sw[o] = gw[o];
        }
        __syncthreads();
        for (uint32_t c = 0; c < cnt; c++) {
            const gsb_uniforms& U = s_cam[c];
            const float W = (float)U.width, H = (float)U.height;
            const float xlo = -0.15f * W, xhi = 1.15f * W, ylo = -0.15f * H, yhi = 1.15f * H;
#pragma unroll
            for (int j = 0; j < F3_ROWS; j++) {
                const ClipView cv = clip_view(U, px[j], py[j], pz[j]);
                const float u = ((cv.ndcx + 1.0f) * W - 1.0f) * 0.5f;  // the frame's ndc2Pix
                const float v = ((cv.ndcy + 1.0f) * H - 1.0f) * 0.5f;
                if (cv.vz > 0.2f && u >= xlo && u <= xhi && v >= ylo && v <= yhi) {  // false for NaN
                    d[j] = fminf(d[j], cv.vz);
                    seen[j] = true;
                }
            }
        }
    }
    uint32_t mx = 0;  // bits of the largest seen depth (> 0.2, so positive); 0 = none
#pragma unroll
    for (int j = 0; j < F3_ROWS; j++) {
        const uint64_t i = base + (uint64_t)j * F3_THREADS;
        if (i < n) variance[i] = seen[j] ? filter_variance(d[j], focal) : -1.0f;
        if (seen[j]) mx = max(mx, __float_as_uint(d[j]));
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = threadIdx.x < F3_THREADS / 32 ? s_max[threadIdx.x] : 0;
        mx = __reduce_max_sync(0xffffffffu, mx);
        if (threadIdx.x == 0 && mx) atomicMax(dmax, mx);
    }
}

// Rows no camera sees (variance -1) take the variance of the largest seen depth, or 0 when no row is seen.
// k_filter3d_lens passes its largest seen scale with focal = 1 (d / 1 = d exactly), so both entries share this kernel.
__global__ void k_filter3d_fill(uint64_t n, float focal, const uint32_t* __restrict__ dmax, float* __restrict__ variance) {
    const uint32_t dm = *dmax;
    const float fill = dm ? filter_variance(__uint_as_float(dm), focal) : 0.0f;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        if (variance[i] < 0.0f) variance[i] = fill;
}

// ---- gsb_filter3d_variance_lens (DESIGN.md section 24): each camera with its own lens model ----
//
// k_filter3d_lens has k_filter3d_depth's shape.  Per camera it stages 28 gsb_uniforms words (proj_mat rows x, y, w for a
// pinhole camera's clip_view; view_mat rows x, y, z; width, height, tan_fovx, tan_fovy) and the 10 words of its model, and
// branches on the model's kind, which is the same for every thread.  Each row keeps the least footprint scale s (world
// units per pixel at the camera's finest image axis) over the cameras that see it; the CTA folds the largest seen s into
// one word as k_filter3d_depth folds the depth.
constexpr uint32_t F3L_WORDS = 28;
constexpr uint32_t F3L_MODEL_WORDS = sizeof(gsb_camera_model) / 4;

// The j-th of the 28 gsb_uniforms words k_filter3d_lens reads (j < 28).
__device__ __forceinline__ uint32_t lens_camera_word(uint32_t j) {
    if (j < 12) return camera_word(j);                         // proj_mat rows x, y, w
    if (j < 24) return 20 + ((j - 12) / 3) * 4 + (j - 12) % 3;  // view_mat[4 c + r], r = 0, 1, 2
    return 36 + (j - 24);                                      // width, height, tan_fovx, tan_fovy
}

// 1 / sigma_min of a lens's 2 x 3 J: with a = |J0|^2, c = |J1|^2, b = J0 . J1, lambda_min(J J^T) = det / lambda_max,
// det = |J0 x J1|^2 and lambda_max = (a + c + sqrt((a - c)^2 + 4 b^2)) / 2.  The textbook (a + c - sqrt(...)) / 2 cancels
// when a >> c, which is what a lens that compresses its periphery gives.
__device__ __forceinline__ float lens_scale(const float (&J)[2][3]) {
    const float a = (J[0][0] * J[0][0] + J[0][1] * J[0][1]) + J[0][2] * J[0][2];
    const float c = (J[1][0] * J[1][0] + J[1][1] * J[1][1]) + J[1][2] * J[1][2];
    const float b = (J[0][0] * J[1][0] + J[0][1] * J[1][1]) + J[0][2] * J[1][2];
    const float x0 = J[0][1] * J[1][2] - J[0][2] * J[1][1];
    const float x1 = J[0][2] * J[1][0] - J[0][0] * J[1][2];
    const float x2 = J[0][0] * J[1][1] - J[0][1] * J[1][0];
    const float det = (x0 * x0 + x1 * x1) + x2 * x2;
    const float dd = a - c;
    const float lmax = ((a + c) + sqrtf(dd * dd + (4.0f * b) * b)) * 0.5f;
    return 1.0f / sqrtf(det / lmax);
}

__device__ __forceinline__ void keep_scale(float sc, float& s, bool& seen) {
    if (sc > 0.0f && sc < __int_as_float(0x7f800000)) {  // false for NaN; a camera whose scale is 0 or inf does not count
        s = fminf(s, sc);
        seen = true;
    }
}

__global__ void __launch_bounds__(F3_THREADS) k_filter3d_lens(const float4* __restrict__ vertices, uint64_t n,
                                                              const gsb_uniforms* __restrict__ cams,
                                                              const gsb_camera_model* __restrict__ models, uint32_t k,
                                                              uint32_t* __restrict__ smax, float* __restrict__ variance) {
    __shared__ gsb_uniforms s_cam[F3_CHUNK];
    __shared__ gsb_camera_model s_model[F3_CHUNK];
    __shared__ uint32_t s_max[F3_THREADS / 32];
    const uint64_t base = (uint64_t)blockIdx.x * (F3_THREADS * F3_ROWS) + threadIdx.x;
    float px[F3_ROWS], py[F3_ROWS], pz[F3_ROWS], s[F3_ROWS];
    bool seen[F3_ROWS];
#pragma unroll
    for (int j = 0; j < F3_ROWS; j++) {
        const uint64_t i = base + (uint64_t)j * F3_THREADS;
        const float4 p = i < n ? vertices[i * 15] : make_float4(__int_as_float(0x7fffffff), 0.0f, 0.0f, 0.0f);  // NaN: never seen
        px[j] = p.x, py[j] = p.y, pz[j] = p.z;
        s[j] = __int_as_float(0x7f800000);
        seen[j] = false;
    }
    uint32_t* sw = reinterpret_cast<uint32_t*>(s_cam);
    uint32_t* smw = reinterpret_cast<uint32_t*>(s_model);
    for (uint32_t c0 = 0; c0 < k; c0 += F3_CHUNK) {
        const uint32_t cnt = min((uint32_t)F3_CHUNK, k - c0);
        const uint32_t* gw = reinterpret_cast<const uint32_t*>(cams + c0);
        const uint32_t* gmw = reinterpret_cast<const uint32_t*>(models + c0);
        __syncthreads();  // the previous chunk is read
        for (uint32_t w = threadIdx.x; w < cnt * F3L_WORDS; w += F3_THREADS) {
            const uint32_t c = w / F3L_WORDS, o = c * 40 + lens_camera_word(w - c * F3L_WORDS);
            sw[o] = gw[o];
        }
        for (uint32_t w = threadIdx.x; w < cnt * F3L_MODEL_WORDS; w += F3_THREADS) smw[w] = gmw[w];
        __syncthreads();
        for (uint32_t c = 0; c < cnt; c++) {
            const gsb_uniforms& U = s_cam[c];
            const gsb_camera_model& M = s_model[c];
            const float W = (float)U.width, H = (float)U.height;
            const float xlo = -0.15f * W, xhi = 1.15f * W, ylo = -0.15f * H, yhi = 1.15f * H;
            if (M.kind == GSB_CAMERA_FISHEYE) {
#pragma unroll
                for (int j = 0; j < F3_ROWS; j++) {
                    const ClipView cv = clip_view(U, px[j], py[j], pz[j]);
                    const FisheyeGeo F = fisheye_geo(M, cv.vx, cv.vy, cv.vz);
                    if (F.d > 0.2f && F.theta <= M.max_theta) {  // k_project's cull; NaN is culled
                        const float u = M.fx * (F.s * cv.vx) + M.cx, v = M.fy * (F.s * cv.vy) + M.cy;
                        if (u >= xlo && u <= xhi && v >= ylo && v <= yhi)
                            keep_scale(lens_scale(fisheye_jacobian(M, U.view_mat, F, cv.vx, cv.vy).J), s[j], seen[j]);
                    }
                }
            } else if (M.kind == GSB_CAMERA_OPENCV) {  // M.max_theta holds tan^2(max_theta), rounded to fp32 on the host
#pragma unroll
                for (int j = 0; j < F3_ROWS; j++) {
                    const ClipView cv = clip_view(U, px[j], py[j], pz[j]);
                    const OpencvGeo O = opencv_geo(M, cv.vx, cv.vy, cv.vz);
                    if (cv.vz > 0.2f && O.r2 <= M.max_theta && O.det > 0.0f) {  // k_project's cull; NaN is culled
                        const float u = M.fx * O.xd + M.cx, v = M.fy * O.yd + M.cy;
                        if (u >= xlo && u <= xhi && v >= ylo && v <= yhi)
                            keep_scale(lens_scale(opencv_jacobian(M, U.view_mat, O, cv.vz).J), s[j], seen[j]);
                    }
                }
            } else if (M.kind == GSB_CAMERA_ORTHO) {  // s = 1 / sigma_min(J) = 1 / min(fx, fy) at every depth
                const float so = 1.0f / fminf(M.fx, M.fy);
#pragma unroll
                for (int j = 0; j < F3_ROWS; j++) {
                    const ClipView cv = clip_view(U, px[j], py[j], pz[j]);
                    const float u = M.fx * cv.vx + M.cx, v = M.fy * cv.vy + M.cy;
                    if (cv.vz > 0.2f && u >= xlo && u <= xhi && v >= ylo && v <= yhi) keep_scale(so, s[j], seen[j]);  // NaN is culled
                }
            } else {  // pinhole: k_filter3d_depth's test; s = vz / min(focal_x, focal_y), the focals as jacobian() has them
                const float f = fminf(W / (2.0f * U.tan_fovx), H / (2.0f * U.tan_fovy));
#pragma unroll
                for (int j = 0; j < F3_ROWS; j++) {
                    const ClipView cv = clip_view(U, px[j], py[j], pz[j]);
                    const float u = ((cv.ndcx + 1.0f) * W - 1.0f) * 0.5f;  // the frame's ndc2Pix
                    const float v = ((cv.ndcy + 1.0f) * H - 1.0f) * 0.5f;
                    if (cv.vz > 0.2f && u >= xlo && u <= xhi && v >= ylo && v <= yhi) keep_scale(cv.vz / f, s[j], seen[j]);
                }
            }
        }
    }
    uint32_t mx = 0;  // bits of the largest seen scale (positive and finite); 0 = none
#pragma unroll
    for (int j = 0; j < F3_ROWS; j++) {
        const uint64_t i = base + (uint64_t)j * F3_THREADS;
        if (i < n) variance[i] = seen[j] ? filter_variance(s[j], 1.0f) : -1.0f;
        if (seen[j]) mx = max(mx, __float_as_uint(s[j]));
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = threadIdx.x < F3_THREADS / 32 ? s_max[threadIdx.x] : 0;
        mx = __reduce_max_sync(0xffffffffu, mx);
        if (threadIdx.x == 0 && mx) atomicMax(smax, mx);
    }
}

}  // namespace

cudaError_t launch_filter3d(const float4* vertices, uint64_t n, const gsb_uniforms* cams, uint32_t k, float focal,
                            uint32_t* dmax, float* variance, int num_sms, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const uint64_t blocks = (n + F3_THREADS * F3_ROWS - 1) / (F3_THREADS * F3_ROWS);
    k_filter3d_depth<<<(unsigned)blocks, F3_THREADS, 0, s>>>(vertices, n, cams, k, focal, dmax, variance);
    const uint64_t fill_blocks = std::min<uint64_t>((n + 255) / 256, (uint64_t)num_sms * 8);
    k_filter3d_fill<<<(unsigned)fill_blocks, 256, 0, s>>>(n, focal, dmax, variance);
    return cudaGetLastError();
}

cudaError_t launch_filter3d_lens(const float4* vertices, uint64_t n, const gsb_uniforms* cams, const gsb_camera_model* models,
                                 uint32_t k, uint32_t* smax, float* variance, int num_sms, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const uint64_t blocks = (n + F3_THREADS * F3_ROWS - 1) / (F3_THREADS * F3_ROWS);
    k_filter3d_lens<<<(unsigned)blocks, F3_THREADS, 0, s>>>(vertices, n, cams, models, k, smax, variance);
    const uint64_t fill_blocks = std::min<uint64_t>((n + 255) / 256, (uint64_t)num_sms * 8);
    k_filter3d_fill<<<(unsigned)fill_blocks, 256, 0, s>>>(n, 1.0f, smax, variance);
    return cudaGetLastError();
}

}  // namespace gsb
