// gsb_loss.cu -- gsb_image_loss: the photometric loss of 3DGS training (Kerbl et al. 2023), (1 - lambda) L1 + lambda (1 - SSIM),
// of a frame against a target, and its gradient with respect to the frame.  No reference counterpart (3DGS.cpp only renders).
// SSIM is the Inria definition: an 11 x 11 Gaussian window (sigma 1.5) applied as a zero-padded correlation to the five moment
// maps of each RGB channel, C1 = 0.01^2, C2 = 0.03^2; every term is a mean over the 3 W H RGB values (DESIGN.md section 11).
//
//   k_loss_forward   one CTA per 32 x 16 tile.  The tile's x and y plus a halo of 5 are staged into shared memory (16-B
//                    loads of the float4 image), then per channel a horizontal and a vertical pass of the separable window
//                    give the five moments of every pixel.  Per pixel it evaluates S, |x - y| and (x - y)^2 and, when a
//                    gradient is wanted, the gather terms A, B, C of S's derivative into the context's scratch.  Per CTA it
//                    stores fp64 sums of |d|, d^2 and S, reduced in a fixed order.
//   k_loss_backward  one CTA per tile (gradient only): stages A, B, C with a halo of 5, blurs them with the same window and
//                    stores d loss / d x = (1 - lambda)/N sign(x - y) - lambda/N (w*A + 2 x (w*B) + y (w*C)) as float4(r, g, b, 0).
//   k_loss_reduce    one CTA: sums the per-tile rows in a fixed order in fp64 and writes loss, L1, SSIM, MSE.
//
// The moments are taken of x - 1/2 and y - 1/2 (the zero padding then reads -1/2): sigma^2 = E[x^2] - mu^2 cancels less in
// fp32 around 0 than around 1/2, and the variances and covariance do not depend on the shift (mu is corrected back).  The
// gather terms use the shifted values as well, which keeps w*A and 2 x (w*B) small.  No atomics: every output word is a
// function of the inputs alone.  Compiled with -fmad=false like the rest of the library; fused ops are spelled fmaf.
#include "gsb_ctx.cuh"

namespace gsb {
namespace {

constexpr int LT_W = 32, LT_H = 16;          // output tile
constexpr int L_R = 5;                       // window radius
constexpr int L_K = 2 * L_R + 1;             // window taps
constexpr int LS_W = LT_W + 2 * L_R;         // staged tile with its halo: 42 x 26
constexpr int LS_H = LT_H + 2 * L_R;
constexpr int LS_N = LS_W * LS_H;
constexpr int LH_N = LS_H * LT_W;            // horizontal pass output: 26 rows x 32 columns
constexpr int L_THREADS = 256;               // two output pixels per thread: rows r and r + 8 of column lane
constexpr int L_PIX = LT_W * LT_H / L_THREADS;
constexpr int LR_THREADS = 1024;
constexpr float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
constexpr unsigned FULL = 0xffffffffu;

// g[i] = exp(-(i - 5)^2 / 4.5) / sum, rounded once from the float64 values
__constant__ float c_win[L_K] = {1.028380124e-03f, 7.598758209e-03f, 3.600077331e-02f, 1.093606874e-01f, 2.130055428e-01f,
                                 2.660117149e-01f, 2.130055428e-01f, 1.093606874e-01f, 3.600077331e-02f, 7.598758209e-03f,
                                 1.028380124e-03f};

struct LossParams {
    const float4* image;
    size_t image_pitch;
    const void* target;
    size_t target_pitch;
    int target_u8;            // GSB_FORMAT_RGBA8 (v / 255.0f), else RGBA32F
    uint32_t width, height, tiles_x;
    float* abc;               // 9 planes of W x H floats (A, B, C of r, then g, then b); null: no gradient
    size_t plane;             // W * H
    double* partials;         // 3 planes of num_tiles doubles: sum |d|, sum d^2, sum S of each tile
    uint32_t num_tiles;
    float4* grad;
    size_t grad_pitch;
    float k_l1, k_ssim;       // (1 - lambda) / N, lambda / N
};

__device__ __forceinline__ float4 load_target(const LossParams& P, uint32_t x, uint32_t y) {
    const unsigned char* row = static_cast<const unsigned char*>(P.target) + (size_t)y * P.target_pitch;
    if (P.target_u8) {
        const uchar4 t = reinterpret_cast<const uchar4*>(row)[x];
        return make_float4(t.x / 255.0f, t.y / 255.0f, t.z / 255.0f, 0.0f);
    }
    return reinterpret_cast<const float4*>(row)[x];
}

__device__ __forceinline__ float4 load_image(const LossParams& P, uint32_t x, uint32_t y) {
    return reinterpret_cast<const float4*>(reinterpret_cast<const unsigned char*>(P.image) + (size_t)y * P.image_pitch)[x];
}

__device__ __forceinline__ float chan(const float4& v, int c) { return c == 0 ? v.x : (c == 1 ? v.y : v.z); }

// Sums v over the CTA in a fixed order: a shuffle tree per warp, then the warps in order by thread 0.
__device__ __forceinline__ double cta_sum(double v, double* s_warp) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    double a = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < L_THREADS / 32; w++) a += s_warp[w];
    __syncthreads();
    return a;
}

__global__ void __launch_bounds__(L_THREADS) k_loss_forward(const __grid_constant__ LossParams P) {
    __shared__ float s_x[3][LS_N], s_y[3][LS_N];  // unshifted values, 0 outside the frame
    __shared__ float s_h[5][LH_N];                 // horizontal pass: x, y, x^2, y^2, x y (shifted)
    __shared__ double s_warp[L_THREADS / 32];
    const uint32_t tx = blockIdx.x % P.tiles_x, ty = blockIdx.x / P.tiles_x;
    const int x0 = (int)(tx * LT_W) - L_R, y0 = (int)(ty * LT_H) - L_R;
    for (int i = threadIdx.x; i < LS_N; i += L_THREADS) {
        const int gx = x0 + i % LS_W, gy = y0 + i / LS_W;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
        if (gx >= 0 && gy >= 0 && gx < (int)P.width && gy < (int)P.height) {
            a = load_image(P, gx, gy);
            b = load_target(P, gx, gy);
        }
        s_x[0][i] = a.x; s_x[1][i] = a.y; s_x[2][i] = a.z;
        s_y[0][i] = b.x; s_y[1][i] = b.y; s_y[2][i] = b.z;
    }
    const int col = threadIdx.x & 31, row0 = threadIdx.x >> 5;
    double sum_abs = 0.0, sum_sq = 0.0, sum_s = 0.0;
    for (int c = 0; c < 3; c++) {
        __syncthreads();  // staging done / the previous channel's vertical pass has read s_h
        for (int i = threadIdx.x; i < LH_N; i += L_THREADS) {
            const int r = i / LT_W, cc = i % LT_W;
            const float* px = &s_x[c][r * LS_W + cc];
            const float* py = &s_y[c][r * LS_W + cc];
            float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
            for (int k = 0; k < L_K; k++) {
                const float w = c_win[k], a = px[k] - 0.5f, b = py[k] - 0.5f;
                const float wa = w * a, wb = w * b;
                m0 += wa;
                m1 += wb;
                m2 = fmaf(wa, a, m2);
                m3 = fmaf(wb, b, m3);
                m4 = fmaf(wa, b, m4);
            }
            s_h[0][i] = m0; s_h[1][i] = m1; s_h[2][i] = m2; s_h[3][i] = m3; s_h[4][i] = m4;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < L_PIX; j++) {
            const int r = row0 + j * (L_THREADS / 32);
            const uint32_t gx = tx * LT_W + col, gy = ty * LT_H + r;
            if (gx >= P.width || gy >= P.height) continue;
            float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < L_K; k++) {
                const float w = c_win[k];
#pragma unroll
                for (int q = 0; q < 5; q++) m[q] = fmaf(w, s_h[q][(r + k) * LT_W + col], m[q]);
            }
            const float mx = m[0], my = m[1];                      // shifted means
            const float vx = fmaf(-mx, mx, m[2]), vy = fmaf(-my, my, m[3]), cxy = fmaf(-mx, my, m[4]);
            const float ux = mx + 0.5f, uy = my + 0.5f;            // the means themselves
            const float a1 = fmaf(2.0f * ux, uy, C1), a2 = fmaf(2.0f, cxy, C2);
            const float b1 = fmaf(ux, ux, fmaf(uy, uy, C1)), b2 = vx + vy + C2;
            const float inv = 1.0f / (b1 * b2);
            const float s = a1 * a2 * inv;
            const int si = (r + L_R) * LS_W + col + L_R;
            const float xv = s_x[c][si], yv = s_y[c][si], d = xv - yv;
            sum_abs += (double)fabsf(d);
            sum_sq += (double)d * (double)d;
            sum_s += (double)s;
            if (P.abc) {
                const float dmx = 2.0f * uy * a2 * inv - 2.0f * ux * s / b1;  // dS / d mu_x
                const float B = -s / b2;                                     // dS / d sigma_x^2
                const float Cc = 2.0f * a1 * inv;                            // dS / d sigma_xy
                const float A = dmx - 2.0f * mx * B - my * Cc;
                const size_t p = (size_t)gy * P.width + gx;
                P.abc[(3 * c + 0) * P.plane + p] = A;
                P.abc[(3 * c + 1) * P.plane + p] = B;
                P.abc[(3 * c + 2) * P.plane + p] = Cc;
            }
        }
    }
    const double t0 = cta_sum(sum_abs, s_warp), t1 = cta_sum(sum_sq, s_warp), t2 = cta_sum(sum_s, s_warp);
    if (threadIdx.x == 0) {
        P.partials[blockIdx.x] = t0;
        P.partials[P.num_tiles + blockIdx.x] = t1;
        P.partials[2 * (size_t)P.num_tiles + blockIdx.x] = t2;
    }
}

__global__ void __launch_bounds__(L_THREADS) k_loss_backward(const __grid_constant__ LossParams P) {
    __shared__ float s_t[3][LS_N];   // A, B, C of one channel, 0 outside the frame
    __shared__ float s_h[3][LH_N];
    const uint32_t tx = blockIdx.x % P.tiles_x, ty = blockIdx.x / P.tiles_x;
    const int x0 = (int)(tx * LT_W) - L_R, y0 = (int)(ty * LT_H) - L_R;
    const int col = threadIdx.x & 31, row0 = threadIdx.x >> 5;
    float4 xs[L_PIX], ys[L_PIX], out[L_PIX];
#pragma unroll
    for (int j = 0; j < L_PIX; j++) {
        const uint32_t gx = tx * LT_W + col, gy = ty * LT_H + row0 + j * (L_THREADS / 32);
        const bool in = gx < P.width && gy < P.height;
        xs[j] = in ? load_image(P, gx, gy) : make_float4(0.f, 0.f, 0.f, 0.f);
        ys[j] = in ? load_target(P, gx, gy) : make_float4(0.f, 0.f, 0.f, 0.f);
        out[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int c = 0; c < 3; c++) {
        if (c) __syncthreads();  // the previous channel's passes have read s_t and s_h
        for (int i = threadIdx.x; i < LS_N; i += L_THREADS) {
            const int gx = x0 + i % LS_W, gy = y0 + i / LS_W;
            const bool in = gx >= 0 && gy >= 0 && gx < (int)P.width && gy < (int)P.height;
            const size_t p = in ? (size_t)gy * P.width + gx : 0;
#pragma unroll
            for (int q = 0; q < 3; q++) s_t[q][i] = in ? P.abc[(3 * c + q) * P.plane + p] : 0.0f;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < LH_N; i += L_THREADS) {
            const int r = i / LT_W, cc = i % LT_W;
#pragma unroll
            for (int q = 0; q < 3; q++) {
                const float* pt = &s_t[q][r * LS_W + cc];
                float m = 0.f;
#pragma unroll
                for (int k = 0; k < L_K; k++) m = fmaf(c_win[k], pt[k], m);
                s_h[q][i] = m;
            }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < L_PIX; j++) {
            const int r = row0 + j * (L_THREADS / 32);
            float m[3] = {0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < L_K; k++) {
                const float w = c_win[k];
#pragma unroll
                for (int q = 0; q < 3; q++) m[q] = fmaf(w, s_h[q][(r + k) * LT_W + col], m[q]);
            }
            const float xv = chan(xs[j], c), yv = chan(ys[j], c);
            const float a = xv - 0.5f, b = yv - 0.5f;
            const float g = fmaf(2.0f * a, m[1], fmaf(b, m[2], m[0]));
            const float sgn = xv > yv ? 1.0f : (xv < yv ? -1.0f : 0.0f);
            const float v = fmaf(P.k_l1, sgn, -P.k_ssim * g);
            if (c == 0) out[j].x = v;
            else if (c == 1) out[j].y = v;
            else out[j].z = v;
        }
    }
#pragma unroll
    for (int j = 0; j < L_PIX; j++) {
        const uint32_t gx = tx * LT_W + col, gy = ty * LT_H + row0 + j * (L_THREADS / 32);
        if (gx < P.width && gy < P.height)
            reinterpret_cast<float4*>(reinterpret_cast<unsigned char*>(P.grad) + (size_t)gy * P.grad_pitch)[gx] = out[j];
    }
}

// Sums the three planes of per-tile partials in a fixed order (thread t a strided set of tiles, a shuffle tree per warp, then
// the warps in order) and writes loss, L1, SSIM, MSE.
__global__ void __launch_bounds__(LR_THREADS) k_loss_reduce(const double* __restrict__ partials, uint32_t tiles, double inv_n, double lambda,
                                                            double* __restrict__ result) {
    __shared__ double s_w[3][LR_THREADS / 32];
    double a[3] = {0.0, 0.0, 0.0};
    for (uint32_t t = threadIdx.x; t < tiles; t += LR_THREADS)
#pragma unroll
        for (int q = 0; q < 3; q++) a[q] += partials[(size_t)q * tiles + t];
#pragma unroll
    for (int q = 0; q < 3; q++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[q] += __shfl_xor_sync(FULL, a[q], o);
        if ((threadIdx.x & 31) == 0) s_w[q][threadIdx.x >> 5] = a[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s[3] = {0.0, 0.0, 0.0};
        for (int q = 0; q < 3; q++)
            for (int w = 0; w < LR_THREADS / 32; w++) s[q] += s_w[q][w];
        const double l1 = s[0] * inv_n, mse = s[1] * inv_n, ssim = s[2] * inv_n;
        result[0] = (1.0 - lambda) * l1 + lambda * (1.0 - ssim);
        result[1] = l1;
        result[2] = ssim;
        result[3] = mse;
    }
}

bool aligned(const void* p, size_t a) { return reinterpret_cast<uintptr_t>(p) % a == 0; }

}  // namespace
}  // namespace gsb

extern "C" int gsb_image_loss(gsb_ctx* ctx, uint32_t width, uint32_t height, const float* image, size_t image_pitch,
                              const void* target, size_t target_pitch, gsb_format target_fmt, float lambda_dssim, float* grad_image,
                              size_t grad_pitch, double* result, void* stream) {
    using namespace gsb;
    if (!ctx) return GSB_ERR_INVALID;
    auto bad = [&](const char* what) { return fail(ctx, GSB_ERR_INVALID, (std::string("gsb_image_loss: ") + what).c_str()); };
    if (!image || !target || !result) return bad("null argument");
    if (width == 0 || height == 0) return bad("bad image size");
    if (!(lambda_dssim >= 0.0f && lambda_dssim <= 1.0f)) return bad("lambda_dssim outside [0, 1]");
    if (target_fmt != GSB_FORMAT_RGBA32F && target_fmt != GSB_FORMAT_RGBA8) return bad("target format is neither RGBA32F nor RGBA8");
    const size_t row = (size_t)width * sizeof(float4);
    const size_t target_row = (size_t)width * bytes_per_pixel(target_fmt);
    const size_t target_align = target_fmt == GSB_FORMAT_RGBA32F ? 16 : 4;
    if (image_pitch == 0) image_pitch = row;
    if (target_pitch == 0) target_pitch = target_row;
    if (grad_pitch == 0) grad_pitch = row;
    if (image_pitch < row || target_pitch < target_row || (grad_image && grad_pitch < row)) return bad("row pitch below the row size");
    if (!aligned(image, 16) || image_pitch % 16 || !aligned(target, target_align) || target_pitch % target_align ||
        (grad_image && (!aligned(grad_image, 16) || grad_pitch % 16)) || !aligned(result, sizeof(double)))
        return bad("misaligned pointer or row pitch");
    const uint32_t tiles_x = (width + LT_W - 1) / LT_W, tiles_y = (height + LT_H - 1) / LT_H;
    if ((uint64_t)tiles_x * tiles_y > 0x7fffffffu) return bad("frame too large");
    const uint32_t tiles = tiles_x * tiles_y;
    const uint64_t pixels = (uint64_t)width * height;
    CK(cudaSetDevice(ctx->device));
    // context-owned scratch: grown with the frame size, never shrunk, freed with the context
    CK(ctx->loss_partials.grow((uint64_t)tiles * 3));
    if (grad_image) CK(ctx->loss_abc.grow(pixels * 9));
    LossParams P{};
    P.image = reinterpret_cast<const float4*>(image);
    P.image_pitch = image_pitch;
    P.target = target;
    P.target_pitch = target_pitch;
    P.target_u8 = target_fmt == GSB_FORMAT_RGBA8;
    P.width = width;
    P.height = height;
    P.tiles_x = tiles_x;
    P.abc = grad_image ? ctx->loss_abc.p : nullptr;
    P.plane = pixels;
    P.partials = ctx->loss_partials;
    P.num_tiles = tiles;
    P.grad = reinterpret_cast<float4*>(grad_image);
    P.grad_pitch = grad_pitch;
    const double n = 3.0 * (double)pixels;
    P.k_l1 = (float)((1.0 - (double)lambda_dssim) / n);
    P.k_ssim = (float)((double)lambda_dssim / n);
    cudaStream_t s = stream_or_own(ctx, stream);
    k_loss_forward<<<tiles, L_THREADS, 0, s>>>(P);
    CK(cudaGetLastError());
    if (grad_image) {
        k_loss_backward<<<tiles, L_THREADS, 0, s>>>(P);
        CK(cudaGetLastError());
    }
    k_loss_reduce<<<1, LR_THREADS, 0, s>>>(ctx->loss_partials, tiles, 1.0 / n, (double)lambda_dssim, result);
    CK(cudaGetLastError());
    return GSB_OK;
}
