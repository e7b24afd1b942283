// gsb_bilagrid.cu -- gsb_bilagrid_apply / gsb_bilagrid_backward: per-image bilateral-grid colour correction for training
// (Wang et al. 2024, "Bilateral Guided Radiance Field Processing"; gsplat's BilateralGrid).  A grid is 12 x L x Y x X fp32 in
// the order [k][l][y][x]; coefficient k = 4 c + j is row c, column j of the 3 x 4 affine matrix A = [M | t] sliced at the
// pixel's (x, y) and at the luma of its colour (DESIGN.md section 17).
//
// The frame is cut into blocks that never straddle a grid cell: the columns whose clamped cell floor(ix) is cx form one
// contiguous range, and so do the rows of a cell cy.  A block is up to 32 columns x 32 rows of one (cx, cy) cell, so all of
// its pixels read the same 2 x 2 (x, y) nodes and only the L z-nodes: 48 L floats, staged into shared memory as [l][corner][k].
//
//   k_bilagrid_apply     one CTA per block: out = A(p) (r, g, b, 1), A copied.  16 B read and 16 B written per pixel.
//   k_bilagrid_backward  one CTA per block: d image in the same pass and, for d grid, the block's 4 L 12 sums.  A thread's
//                        four pixels (one column, rows w, w + 8, ...) are summed per z-level in fp32, the 32 lanes by a shuffle
//                        tree, the 8 warps in order in fp64 into the block's partial row.
//   k_bilagrid_reduce    one thread per grid word: the partial rows of the <= 4 cells around its node, in a fixed order, in
//                        fp64, rounded once.
// No atomics: every output word is a function of the inputs alone.  Compiled with -fmad=false like the rest of the library;
// fused ops are spelled fmaf.
#include <climits>

#include "gsb_ctx.cuh"

namespace gsb {
namespace {

constexpr int BG_W = 32, BG_ROWS = 4, BG_WARPS = 8;  // a block: 32 columns x (8 warps x 4 rows)
constexpr int BG_H = BG_WARPS * BG_ROWS;
constexpr int BG_THREADS = 32 * BG_WARPS;
constexpr int BG_MAX = 64;   // largest grid dimension
constexpr int BG_NODE = 48;  // floats per z-level of a block: 4 corners x 12 coefficients
constexpr int BG_RTHREADS = 256;
constexpr unsigned FULL = 0xffffffffu;

struct BilagridParams {
    const float4* image;
    size_t image_pitch;
    const float* grid;
    uint32_t gx, gy, gl;
    float4* out;                // apply
    size_t out_pitch;
    const float4* grad_out;     // backward
    size_t grad_out_pitch;
    float4* grad_image;         // null: no image gradient
    size_t grad_image_pitch;
    double* partials;           // null: no grid gradient; otherwise [blocks][gl][4][12]
    uint32_t width, height;
    uint32_t chunks_x, chunks_y;          // blocks per cell along x and y
    uint32_t xb[BG_MAX], yb[BG_MAX];      // first column (row) of each cell; xb[gx - 1] = width, yb[gy - 1] = height
};

// The clamped cell of pixel coordinate p and its fraction: i = ((p + 0.5) / n) (g - 1), i0 = min(floor(i), g - 2).  The host
// evaluates the same fp32 operations to cut the frame into blocks.
__host__ __device__ __forceinline__ int cell_of(uint32_t p, uint32_t n, uint32_t g, float* frac) {
    const float i = (((float)p + 0.5f) / (float)n) * (float)(g - 1);
    int i0 = (int)floorf(i);
    if (i0 > (int)g - 2) i0 = (int)g - 2;
    *frac = i - (float)i0;
    return i0;
}

__device__ __forceinline__ float lerp(float f, float lo, float hi) { return fmaf(f, hi - lo, lo); }

// Stages the block's 4 L 12 grid words as s[l][corner][k], corner = dx + 2 dy.
__device__ __forceinline__ void stage_grid(const BilagridParams& P, uint32_t cx, uint32_t cy, float* s) {
    const uint32_t n = BG_NODE * P.gl;
    for (uint32_t i = threadIdx.x; i < n; i += BG_THREADS) {
        const uint32_t k = i % 12, c = (i / 12) % 4, l = i / BG_NODE;
        s[i] = P.grid[(((size_t)k * P.gl + l) * P.gy + cy + (c >> 1)) * P.gx + cx + (c & 1)];
    }
}

struct Block {
    uint32_t cx, cy, x, x_end, y, y_end;
};

__device__ __forceinline__ Block block_of(const BilagridParams& P) {
    Block b;
    b.cx = blockIdx.x / P.chunks_x;
    b.cy = blockIdx.y / P.chunks_y;
    b.x = P.xb[b.cx] + (blockIdx.x % P.chunks_x) * BG_W;
    b.y = P.yb[b.cy] + (blockIdx.y % P.chunks_y) * BG_H;
    b.x_end = min(P.xb[b.cx + 1], b.x + BG_W);
    b.y_end = min(P.yb[b.cy + 1], b.y + BG_H);
    return b;
}

// One pixel's slice: A (12 coefficients) and, when wanted, dA/d iz, from the staged block.
struct Slice {
    float fx, fy, fz;
    int z0;
    bool inside;  // 0 < gray < 1: iz is not clamped
};

__device__ __forceinline__ Slice slice_at(const BilagridParams& P, uint32_t px, uint32_t py, float4 v) {
    Slice s;
    cell_of(px, P.width, P.gx, &s.fx);
    cell_of(py, P.height, P.gy, &s.fy);
    const float gray = (0.299f * v.x + 0.587f * v.y) + 0.114f * v.z;
    const float iz = fminf(fmaxf(gray, 0.0f), 1.0f) * (float)(P.gl - 1);
    s.z0 = min((int)floorf(iz), (int)P.gl - 2);
    s.fz = iz - (float)s.z0;
    s.inside = gray > 0.0f && gray < 1.0f;
    return s;
}

// A = trilinear slice in lerp form (x, then y, then z); dA = the z-difference of the two xy-interpolated planes.
template <bool DERIV>
__device__ __forceinline__ void interpolate(const float* sg, const Slice& s, float* A, float* dA) {
    const float4* lo = reinterpret_cast<const float4*>(sg + s.z0 * BG_NODE);
    const float4* hi = reinterpret_cast<const float4*>(sg + (s.z0 + 1) * BG_NODE);
#pragma unroll
    for (int q = 0; q < 3; q++) {
        float a[2][4];
#pragma unroll
        for (int z = 0; z < 2; z++) {
            const float4* n = z ? hi : lo;
            const float4 c00 = n[q], c01 = n[3 + q], c10 = n[6 + q], c11 = n[9 + q];
            a[z][0] = lerp(s.fy, lerp(s.fx, c00.x, c01.x), lerp(s.fx, c10.x, c11.x));
            a[z][1] = lerp(s.fy, lerp(s.fx, c00.y, c01.y), lerp(s.fx, c10.y, c11.y));
            a[z][2] = lerp(s.fy, lerp(s.fx, c00.z, c01.z), lerp(s.fx, c10.z, c11.z));
            a[z][3] = lerp(s.fy, lerp(s.fx, c00.w, c01.w), lerp(s.fx, c10.w, c11.w));
        }
#pragma unroll
        for (int e = 0; e < 4; e++) {
            A[4 * q + e] = lerp(s.fz, a[0][e], a[1][e]);
            if (DERIV) dA[4 * q + e] = a[1][e] - a[0][e];
        }
    }
}

__device__ __forceinline__ float affine(const float* A, int c, float4 v) {
    return ((A[4 * c] * v.x + A[4 * c + 1] * v.y) + A[4 * c + 2] * v.z) + A[4 * c + 3];
}

__device__ __forceinline__ const float4* pixel(const float4* base, size_t pitch, uint32_t x, uint32_t y) {
    return reinterpret_cast<const float4*>(reinterpret_cast<const unsigned char*>(base) + (size_t)y * pitch) + x;
}
__device__ __forceinline__ float4* pixel(float4* base, size_t pitch, uint32_t x, uint32_t y) {
    return reinterpret_cast<float4*>(reinterpret_cast<unsigned char*>(base) + (size_t)y * pitch) + x;
}

__global__ void __launch_bounds__(BG_THREADS) k_bilagrid_apply(const __grid_constant__ BilagridParams P) {
    __shared__ __align__(16) float s_grid[BG_NODE * BG_MAX];
    const Block b = block_of(P);
    if (b.x >= b.x_end || b.y >= b.y_end) return;  // an empty cell (CTA-uniform)
    stage_grid(P, b.cx, b.cy, s_grid);
    __syncthreads();
    const uint32_t px = b.x + (threadIdx.x & 31);
    if (px >= b.x_end) return;
#pragma unroll
    for (int r = 0; r < BG_ROWS; r++) {
        const uint32_t py = b.y + (threadIdx.x >> 5) + r * BG_WARPS;
        if (py >= b.y_end) break;
        const float4 v = *pixel(P.image, P.image_pitch, px, py);
        const Slice s = slice_at(P, px, py, v);
        float A[12];
        interpolate<false>(s_grid, s, A, nullptr);
        *pixel(P.out, P.out_pitch, px, py) = make_float4(affine(A, 0, v), affine(A, 1, v), affine(A, 2, v), v.w);
    }
}

// dynamic shared memory: the staged grid, then [warp][l][48] per-warp sums of the grid gradient
__global__ void __launch_bounds__(BG_THREADS) k_bilagrid_backward(const __grid_constant__ BilagridParams P) {
    extern __shared__ __align__(16) float bg_smem[];
    float* s_grid = bg_smem;
    float* s_warp = bg_smem + BG_NODE * P.gl;
    const Block b = block_of(P);
    const bool empty = b.x >= b.x_end || b.y >= b.y_end;  // CTA-uniform
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t row_words = BG_NODE * P.gl;
    if (P.partials)
        for (uint32_t i = threadIdx.x; i < BG_WARPS * row_words; i += BG_THREADS) s_warp[i] = 0.0f;
    if (!empty) stage_grid(P, b.cx, b.cy, s_grid);
    __syncthreads();

    // per pixel: what the grid gradient needs later (in, g, fy, fz, z0); fx is the column's
    float4 in[BG_ROWS], gr[BG_ROWS];
    float fy[BG_ROWS], fz[BG_ROWS], fx = 0.0f;
    int z0[BG_ROWS];
    int zmin = INT_MAX, zmax = -1;
    const uint32_t px = b.x + lane;
#pragma unroll
    for (int r = 0; r < BG_ROWS; r++) {
        const uint32_t py = b.y + warp + r * BG_WARPS;
        z0[r] = -2;  // no pixel: matches no level
        fy[r] = fz[r] = 0.0f;
        in[r] = gr[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (empty || px >= b.x_end || py >= b.y_end) continue;
        const float4 v = *pixel(P.image, P.image_pitch, px, py);
        const float4 g = *pixel(P.grad_out, P.grad_out_pitch, px, py);
        const Slice s = slice_at(P, px, py, v);
        if (P.grad_image) {
            float A[12], dA[12];
            interpolate<true>(s_grid, s, A, dA);
            float d0 = (A[0] * g.x + A[4] * g.y) + A[8] * g.z;
            float d1 = (A[1] * g.x + A[5] * g.y) + A[9] * g.z;
            float d2 = (A[2] * g.x + A[6] * g.y) + A[10] * g.z;
            if (s.inside) {  // the luma guidance: d out / d iz chained through iz = gray (L - 1)
                const float t = ((g.x * affine(dA, 0, v) + g.y * affine(dA, 1, v)) + g.z * affine(dA, 2, v)) * (float)(P.gl - 1);
                d0 += 0.299f * t;
                d1 += 0.587f * t;
                d2 += 0.114f * t;
            }
            *pixel(P.grad_image, P.grad_image_pitch, px, py) = make_float4(d0, d1, d2, 0.0f);
        }
        in[r] = v;
        gr[r] = g;
        fx = s.fx;
        fy[r] = s.fy;
        fz[r] = s.fz;
        z0[r] = s.z0;
        zmin = min(zmin, s.z0);
        zmax = max(zmax, s.z0);
    }
    if (!P.partials) return;

    // the z-levels this warp's pixels reach: [lo, hi + 1]
    const int lo = __reduce_min_sync(FULL, zmin), hi = __reduce_max_sync(FULL, zmax);
    for (int l = lo; l <= hi + 1 && hi >= 0; l++) {
        float acc[BG_NODE];
#pragma unroll
        for (int i = 0; i < BG_NODE; i++) acc[i] = 0.0f;
#pragma unroll
        for (int r = 0; r < BG_ROWS; r++) {
            if (z0[r] != l && z0[r] + 1 != l) continue;
            const float wz = z0[r] == l ? 1.0f - fz[r] : fz[r];
            const float wy0 = wz * (1.0f - fy[r]), wy1 = wz * fy[r];
            const float w[4] = {wy0 * (1.0f - fx), wy0 * fx, wy1 * (1.0f - fx), wy1 * fx};
            const float g[3] = {gr[r].x, gr[r].y, gr[r].z};
            const float v[4] = {in[r].x, in[r].y, in[r].z, 1.0f};
#pragma unroll
            for (int c = 0; c < 3; c++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const float q = g[c] * v[j];
#pragma unroll
                    for (int n = 0; n < 4; n++) acc[n * 12 + 4 * c + j] = fmaf(w[n], q, acc[n * 12 + 4 * c + j]);
                }
        }
#pragma unroll
        for (int i = 0; i < BG_NODE; i++) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(FULL, acc[i], o);
        }
        if (lane == 0)
#pragma unroll
            for (int i = 0; i < BG_NODE; i++) s_warp[(warp * P.gl + l) * BG_NODE + i] = acc[i];
    }
    __syncthreads();
    double* row = P.partials + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * row_words;
    for (uint32_t i = threadIdx.x; i < row_words; i += BG_THREADS) {
        double a = 0.0;
#pragma unroll
        for (int w = 0; w < BG_WARPS; w++) a += (double)s_warp[w * row_words + i];
        row[i] = a;
    }
}

// grad_grid[k][l][y][x]: the partial rows of the cells (cx, cy) in {x - 1, x} x {y - 1, y}, each cell's blocks in order.
__global__ void __launch_bounds__(BG_RTHREADS) k_bilagrid_reduce(const __grid_constant__ BilagridParams P, float* __restrict__ grad_grid) {
    const uint32_t words = 12 * P.gl * P.gy * P.gx;
    const uint32_t row_words = BG_NODE * P.gl, blocks_x = (P.gx - 1) * P.chunks_x;
    for (uint32_t i = blockIdx.x * BG_RTHREADS + threadIdx.x; i < words; i += gridDim.x * BG_RTHREADS) {
        const uint32_t x = i % P.gx, y = (i / P.gx) % P.gy, l = (i / (P.gx * P.gy)) % P.gl, k = i / (P.gx * P.gy * P.gl);
        double a = 0.0;
        for (int dy = 1; dy >= 0; dy--) {
            const int cy = (int)y - dy;
            if (cy < 0 || cy > (int)P.gy - 2) continue;
            for (int dx = 1; dx >= 0; dx--) {
                const int cx = (int)x - dx;
                if (cx < 0 || cx > (int)P.gx - 2) continue;
                const uint32_t o = l * BG_NODE + (dx + 2 * dy) * 12 + k;
                for (uint32_t jy = 0; jy < P.chunks_y; jy++)
                    for (uint32_t jx = 0; jx < P.chunks_x; jx++) {
                        const size_t blk = (size_t)(cy * P.chunks_y + jy) * blocks_x + cx * P.chunks_x + jx;
                        a += P.partials[blk * row_words + o];
                    }
            }
        }
        grad_grid[i] = (float)a;
    }
}

bool aligned(const void* p, size_t a) { return reinterpret_cast<uintptr_t>(p) % a == 0; }

// Fills the frame-and-grid part of P (the cell boundaries and blocks) and validates the arguments common to both entries.
const char* prepare(BilagridParams& P, uint32_t width, uint32_t height, const float* image, size_t image_pitch,
                    const float* grid, uint32_t gx, uint32_t gy, uint32_t gl, dim3* blocks) {
    if (width == 0 || height == 0) return "bad image size";
    if (gx < 2 || gy < 2 || gl < 2 || gx > BG_MAX || gy > BG_MAX || gl > BG_MAX) return "grid dimension outside [2, 64]";
    if (image_pitch < (size_t)width * 16) return "row pitch below the row size";
    if (!aligned(image, 16) || image_pitch % 16 || !aligned(grid, 4)) return "misaligned pointer or row pitch";
    P.image = reinterpret_cast<const float4*>(image);
    P.image_pitch = image_pitch;
    P.grid = grid;
    P.gx = gx;
    P.gy = gy;
    P.gl = gl;
    P.width = width;
    P.height = height;
    uint32_t max_len[2] = {0, 0};
    for (int axis = 0; axis < 2; axis++) {
        const uint32_t n = axis ? height : width, g = axis ? gy : gx;
        uint32_t* b = axis ? P.yb : P.xb;
        // cells are monotone in the pixel coordinate: b[c] is the first pixel whose cell is >= c
        uint32_t p = 0;
        for (uint32_t c = 0; c + 1 < g; c++) {
            float f;
            while (p < n && cell_of(p, n, g, &f) < (int)c) p++;
            b[c] = p;
        }
        b[g - 1] = n;
        for (uint32_t c = 0; c + 1 < g; c++) max_len[axis] = std::max(max_len[axis], b[c + 1] - b[c]);
    }
    P.chunks_x = (max_len[0] + BG_W - 1) / BG_W;
    P.chunks_y = (max_len[1] + BG_H - 1) / BG_H;
    const uint64_t bx = (uint64_t)(gx - 1) * P.chunks_x, by = (uint64_t)(gy - 1) * P.chunks_y;
    if (bx > 0x7fffffffu || by > 65535) return "frame too large";
    *blocks = dim3((uint32_t)bx, (uint32_t)by);
    return nullptr;
}

}  // namespace
}  // namespace gsb

extern "C" int gsb_bilagrid_apply(gsb_ctx* ctx, uint32_t width, uint32_t height, const float* image, size_t image_pitch,
                                  const float* grid, uint32_t grid_x, uint32_t grid_y, uint32_t grid_l, float* out,
                                  size_t out_pitch, void* stream) {
    using namespace gsb;
    if (!ctx) return GSB_ERR_INVALID;
    auto bad = [&](const char* what) { return fail(ctx, GSB_ERR_INVALID, (std::string("gsb_bilagrid_apply: ") + what).c_str()); };
    if (!image || !grid || !out) return bad("null argument");
    BilagridParams P{};
    dim3 blocks;
    if (const char* e = prepare(P, width, height, image, image_pitch, grid, grid_x, grid_y, grid_l, &blocks)) return bad(e);
    if (out_pitch < (size_t)width * 16) return bad("row pitch below the row size");
    if (!aligned(out, 16) || out_pitch % 16) return bad("misaligned pointer or row pitch");
    P.out = reinterpret_cast<float4*>(out);
    P.out_pitch = out_pitch;
    CK(cudaSetDevice(ctx->device));
    k_bilagrid_apply<<<blocks, BG_THREADS, 0, stream_or_own(ctx, stream)>>>(P);
    CK(cudaGetLastError());
    return GSB_OK;
}

extern "C" int gsb_bilagrid_backward(gsb_ctx* ctx, uint32_t width, uint32_t height, const float* image, size_t image_pitch,
                                     const float* grid, uint32_t grid_x, uint32_t grid_y, uint32_t grid_l, const float* grad_out,
                                     size_t grad_out_pitch, float* grad_image, size_t grad_image_pitch, float* grad_grid,
                                     void* stream) {
    using namespace gsb;
    if (!ctx) return GSB_ERR_INVALID;
    auto bad = [&](const char* what) { return fail(ctx, GSB_ERR_INVALID, (std::string("gsb_bilagrid_backward: ") + what).c_str()); };
    if (!image || !grid || !grad_out) return bad("null argument");
    if (!grad_image && !grad_grid) return bad("neither gradient requested");
    BilagridParams P{};
    dim3 blocks;
    if (const char* e = prepare(P, width, height, image, image_pitch, grid, grid_x, grid_y, grid_l, &blocks)) return bad(e);
    const size_t row = (size_t)width * 16;
    if (grad_out_pitch < row || (grad_image && grad_image_pitch < row)) return bad("row pitch below the row size");
    if (!aligned(grad_out, 16) || grad_out_pitch % 16 || (grad_image && (!aligned(grad_image, 16) || grad_image_pitch % 16)) ||
        (grad_grid && !aligned(grad_grid, 4)))
        return bad("misaligned pointer or row pitch");
    P.grad_out = reinterpret_cast<const float4*>(grad_out);
    P.grad_out_pitch = grad_out_pitch;
    P.grad_image = reinterpret_cast<float4*>(grad_image);
    P.grad_image_pitch = grad_image_pitch;
    const uint64_t row_words = (uint64_t)BG_NODE * grid_l;
    CK(cudaSetDevice(ctx->device));
    if (grad_grid) {
        // context-owned scratch: grown with the number of blocks and the grid's depth, never shrunk, freed with the context
        CK(ctx->bilagrid_partials.grow((uint64_t)blocks.x * blocks.y * row_words));
        P.partials = ctx->bilagrid_partials;
    }
    const size_t smem = (size_t)(BG_NODE + (P.partials ? BG_WARPS * BG_NODE : 0)) * grid_l * sizeof(float);
    CK(cudaFuncSetAttribute(k_bilagrid_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BG_NODE * (1 + BG_WARPS) * BG_MAX * sizeof(float))));
    cudaStream_t s = stream_or_own(ctx, stream);
    k_bilagrid_backward<<<blocks, BG_THREADS, smem, s>>>(P);
    CK(cudaGetLastError());
    if (grad_grid) {
        const uint32_t words = 12 * grid_l * grid_y * grid_x;
        k_bilagrid_reduce<<<std::min<uint32_t>((words + BG_RTHREADS - 1) / BG_RTHREADS, 4 * ctx->num_sms), BG_RTHREADS, 0, s>>>(P, grad_grid);
        CK(cudaGetLastError());
    }
    return GSB_OK;
}
