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
//   k_loss_backward  one CTA per tile (gradient only): stages A, B, C and x, y with a halo of 5, blurs A, B, x B, C and y C
//                    with the same window and stores d loss / d x = (1 - lambda)/N sign(x - y) - lambda/N d S / d x as
//                    float4(r, g, b, 0).
//   k_loss_reduce    one CTA: sums the per-tile rows in a fixed order in fp64 and writes loss, L1, SSIM, MSE.
//
// The window passes and everything per pixel run in fp64: sigma^2 = E[x^2] - mu^2 cancels completely over a flat window,
// and in fp32 the residue (~1e-7 x^2, of one sign over a whole flat region) divided by C2 = 9e-4 biased S by up to 6e-5 on
// sky, backgrounds and saturated areas.  A, B and C are stored as fp32.  No atomics: every output word is a function of
// the inputs alone.  Compiled with -fmad=false like the rest of the library; fused ops are spelled fma / fmaf.
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
constexpr double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
constexpr unsigned FULL = 0xffffffffu;

// g[i] = exp(-(i - 5)^2 / 4.5) / sum in float64
__constant__ double c_win[L_K] = {0.00102838008447911, 0.007598758135239185, 0.03600077212843083, 0.10936068950970002,
                                  0.2130055377112537,  0.26601172486179436,  0.2130055377112537,  0.10936068950970002,
                                  0.03600077212843083, 0.007598758135239185, 0.00102838008447911};

// dynamic shared memory of the two tile kernels (more than the 48 KB of static shared memory)
struct ForwardSmem {
    double h[5][LH_N];                 // horizontal pass: x, y, x^2, y^2, x y
    float x[3][LS_N], y[3][LS_N];      // 0 outside the frame
    double warp[L_THREADS / 32];
};
struct BackwardSmem {
    double h[5][LH_N];                 // horizontal pass: A, B, x B, C, y C
    float x[3][LS_N], y[3][LS_N];      // 0 outside the frame
    float t[3][LS_N];                  // A, B, C of one channel, 0 outside the frame
};

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
    double k_l1, k_ssim;      // (1 - lambda) / N, lambda / N
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

// Stages the tile's x and y with a halo of L_R (0 outside the frame) as three planes each.
__device__ __forceinline__ void stage_xy(const LossParams& P, int x0, int y0, float (*s_x)[LS_N], float (*s_y)[LS_N]) {
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
}

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
    extern __shared__ __align__(16) unsigned char l_smem[];
    ForwardSmem& S = *reinterpret_cast<ForwardSmem*>(l_smem);
    const uint32_t tx = blockIdx.x % P.tiles_x, ty = blockIdx.x / P.tiles_x;
    stage_xy(P, (int)(tx * LT_W) - L_R, (int)(ty * LT_H) - L_R, S.x, S.y);
    const int col = threadIdx.x & 31, row0 = threadIdx.x >> 5;
    double sum_abs = 0.0, sum_sq = 0.0, sum_s = 0.0;
    for (int c = 0; c < 3; c++) {
        __syncthreads();  // staging done / the previous channel's vertical pass has read S.h
        for (int i = threadIdx.x; i < LH_N; i += L_THREADS) {
            const int r = i / LT_W, cc = i % LT_W;
            const float* px = &S.x[c][r * LS_W + cc];
            const float* py = &S.y[c][r * LS_W + cc];
            double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0, m4 = 0.0;
#pragma unroll
            for (int k = 0; k < L_K; k++) {
                const double w = c_win[k], a = px[k], b = py[k];
                const double wa = w * a, wb = w * b;
                m0 += wa;
                m1 += wb;
                m2 = fma(wa, a, m2);
                m3 = fma(wb, b, m3);
                m4 = fma(wa, b, m4);
            }
            S.h[0][i] = m0; S.h[1][i] = m1; S.h[2][i] = m2; S.h[3][i] = m3; S.h[4][i] = m4;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < L_PIX; j++) {
            const int r = row0 + j * (L_THREADS / 32);
            const uint32_t gx = tx * LT_W + col, gy = ty * LT_H + r;
            if (gx >= P.width || gy >= P.height) continue;
            double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
            for (int k = 0; k < L_K; k++) {
                const double w = c_win[k];
#pragma unroll
                for (int q = 0; q < 5; q++) m[q] = fma(w, S.h[q][(r + k) * LT_W + col], m[q]);
            }
            const double ux = m[0], uy = m[1];
            const double vx = fma(-ux, ux, m[2]), vy = fma(-uy, uy, m[3]), cxy = fma(-ux, uy, m[4]);
            const double a1 = fma(2.0 * ux, uy, C1), a2 = fma(2.0, cxy, C2);
            const double b1 = fma(ux, ux, fma(uy, uy, C1)), b2 = vx + vy + C2;
            const double r1 = 1.0 / b1, r2 = 1.0 / b2;
            const double s = a1 * a2 * (r1 * r2);
            const int si = (r + L_R) * LS_W + col + L_R;
            const float xv = S.x[c][si], yv = S.y[c][si], d = xv - yv;
            sum_abs += (double)fabsf(d);
            sum_sq += (double)d * (double)d;
            sum_s += s;
            if (P.abc) {
                const double dmx = 2.0 * uy * a2 * (r1 * r2) - 2.0 * ux * s * r1;  // dS / d mu_x
                const double B = -s * r2;                                           // dS / d sigma_x^2
                const double Cc = 2.0 * a1 * (r1 * r2);                             // dS / d sigma_xy
                // A relative to the pixel's own values: small where the window is flat (section 11)
                const double A = dmx - 2.0 * (ux - (double)xv) * B - (uy - (double)yv) * Cc;
                const size_t p = (size_t)gy * P.width + gx;
                P.abc[(3 * c + 0) * P.plane + p] = (float)A;
                P.abc[(3 * c + 1) * P.plane + p] = (float)B;
                P.abc[(3 * c + 2) * P.plane + p] = (float)Cc;
            }
        }
    }
    const double t0 = cta_sum(sum_abs, S.warp), t1 = cta_sum(sum_sq, S.warp), t2 = cta_sum(sum_s, S.warp);
    if (threadIdx.x == 0) {
        P.partials[blockIdx.x] = t0;
        P.partials[P.num_tiles + blockIdx.x] = t1;
        P.partials[2 * (size_t)P.num_tiles + blockIdx.x] = t2;
    }
}

// d S / d x_q = sum_p w(q - p) (A_p + 2 (x_q - x_p) B_p + (y_q - y_p) C_p), gathered as
// w*A + 2 (x_q (w*B) - w*(x B)) + (y_q (w*C) - w*(y C)) in fp64: the two differences cancel where the window is flat, and
// the rounding of B and C to fp32 is common to both of their terms.
__global__ void __launch_bounds__(L_THREADS) k_loss_backward(const __grid_constant__ LossParams P) {
    extern __shared__ __align__(16) unsigned char l_smem[];
    BackwardSmem& S = *reinterpret_cast<BackwardSmem*>(l_smem);
    const uint32_t tx = blockIdx.x % P.tiles_x, ty = blockIdx.x / P.tiles_x;
    const int x0 = (int)(tx * LT_W) - L_R, y0 = (int)(ty * LT_H) - L_R;
    const int col = threadIdx.x & 31, row0 = threadIdx.x >> 5;
    stage_xy(P, x0, y0, S.x, S.y);
    float4 out[L_PIX];
    for (int c = 0; c < 3; c++) {
        if (c) __syncthreads();  // the previous channel's passes have read S.t and S.h
        for (int i = threadIdx.x; i < LS_N; i += L_THREADS) {
            const int gx = x0 + i % LS_W, gy = y0 + i / LS_W;
            const bool in = gx >= 0 && gy >= 0 && gx < (int)P.width && gy < (int)P.height;
            const size_t p = in ? (size_t)gy * P.width + gx : 0;
#pragma unroll
            for (int q = 0; q < 3; q++) S.t[q][i] = in ? P.abc[(3 * c + q) * P.plane + p] : 0.0f;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < LH_N; i += L_THREADS) {
            const int r = i / LT_W, cc = i % LT_W, o = r * LS_W + cc;
            double hA = 0.0, hB = 0.0, hxB = 0.0, hC = 0.0, hyC = 0.0;
#pragma unroll
            for (int k = 0; k < L_K; k++) {
                const double w = c_win[k];
                const double wb = w * S.t[1][o + k], wc = w * S.t[2][o + k];
                hA = fma(w, (double)S.t[0][o + k], hA);
                hB += wb;
                hxB = fma(wb, (double)S.x[c][o + k], hxB);
                hC += wc;
                hyC = fma(wc, (double)S.y[c][o + k], hyC);
            }
            S.h[0][i] = hA; S.h[1][i] = hB; S.h[2][i] = hxB; S.h[3][i] = hC; S.h[4][i] = hyC;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < L_PIX; j++) {
            const int r = row0 + j * (L_THREADS / 32);
            double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
            for (int k = 0; k < L_K; k++) {
                const double w = c_win[k];
#pragma unroll
                for (int q = 0; q < 5; q++) m[q] = fma(w, S.h[q][(r + k) * LT_W + col], m[q]);
            }
            const int si = (r + L_R) * LS_W + col + L_R;
            const float xv = S.x[c][si], yv = S.y[c][si];
            const double g = m[0] + 2.0 * fma((double)xv, m[1], -m[2]) + fma((double)yv, m[3], -m[4]);
            const double sgn = xv > yv ? 1.0 : (xv < yv ? -1.0 : 0.0);
            const float v = (float)(P.k_l1 * sgn - P.k_ssim * g);
            if (c == 0) out[j].x = v;
            else if (c == 1) out[j].y = v;
            else out[j].z = v;
        }
    }
#pragma unroll
    for (int j = 0; j < L_PIX; j++) {
        const uint32_t gx = tx * LT_W + col, gy = ty * LT_H + row0 + j * (L_THREADS / 32);
        if (gx < P.width && gy < P.height)
            reinterpret_cast<float4*>(reinterpret_cast<unsigned char*>(P.grad) + (size_t)gy * P.grad_pitch)[gx] =
                make_float4(out[j].x, out[j].y, out[j].z, 0.0f);
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
    P.k_l1 = (1.0 - (double)lambda_dssim) / n;
    P.k_ssim = (double)lambda_dssim / n;
    CK(cudaFuncSetAttribute(k_loss_forward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ForwardSmem)));
    CK(cudaFuncSetAttribute(k_loss_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BackwardSmem)));
    cudaStream_t s = stream_or_own(ctx, stream);
    k_loss_forward<<<tiles, L_THREADS, sizeof(ForwardSmem), s>>>(P);
    CK(cudaGetLastError());
    if (grad_image) {
        k_loss_backward<<<tiles, L_THREADS, sizeof(BackwardSmem), s>>>(P);
        CK(cudaGetLastError());
    }
    k_loss_reduce<<<1, LR_THREADS, 0, s>>>(ctx->loss_partials, tiles, 1.0 / n, (double)lambda_dssim, result);
    CK(cudaGetLastError());
    return GSB_OK;
}
