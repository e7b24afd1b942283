// gsb_filter3d.cu -- gsb_filter3d_variance: the per-Gaussian variance of Mip-Splatting's 3D smoothing filter (Yu et al.
// 2024, compute_3D_filter) from the training cameras, in the frame's own camera arithmetic (DESIGN.md section 18).
//
// k_filter3d_depth: one thread per F3_ROWS rows; the cameras pass through shared memory in chunks of F3_CHUNK, of which
// only the 18 words clip_view and ndc2Pix read are staged.  Each row keeps the least view depth over the cameras that see
// it and writes its variance, or -1 when no camera sees it; each CTA folds the largest seen depth of its rows into one word
// with an integer atomicMax (positive floats order as their bits).  k_filter3d_fill then gives the unseen rows that
// depth's variance.  Min and max are exact, so every output word is a function of the inputs on any grid or stream.
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
__global__ void k_filter3d_fill(uint64_t n, float focal, const uint32_t* __restrict__ dmax, float* __restrict__ variance) {
    const uint32_t dm = *dmax;
    const float fill = dm ? filter_variance(__uint_as_float(dm), focal) : 0.0f;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        if (variance[i] < 0.0f) variance[i] = fill;
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

}  // namespace gsb
