// gsb_init.cu -- gsb_init_from_points: activated records of a point cloud (Kerbl et al. 2023's initialisation from SfM
// points), each point an isotropic Gaussian whose scale is sqrt(mean squared distance to its three nearest neighbours)
// (DESIGN.md section 13).  The 3-nearest-neighbour search is exact in fp32:
//
//   k_init_bbox / k_init_bbox_final  bounding box and non-finite flag (per-CTA partials, reduced by one thread in CTA order)
//   k_init_morton                    63-bit Morton code of each point over the box (21 bits per axis), payload = index
//   Onesweep (k_sort_hist, k_onesweep_pass<u64>)  the (code, index) pairs, private control and look-back words
//   k_init_gather                    sorted points as float4 (x, y, z, bits(index))
//   k_init_leaf_boxes / k_init_node_boxes  fp32 AABBs of 32 consecutive sorted points (leaves) and, level by level, of 32
//                                    consecutive nodes: an implicit 32-ary tree, at most 6 levels for n < 2^30
//   k_init_knn                       one warp per leaf, one lane per point: three smallest d in sorted registers, seeded from
//                                    the leaf's other 31 points, then a descent from the root that visits a node when some
//                                    lane's lower bound is strictly below that lane's third value; writes the scale by index
//   k_init_records                   the n x 60 records, one thread per float4 of a row (coalesced stores)
//
// The bound of a box is the distance formula applied to the point clamped into the box.  Every IEEE operation is monotone
// (and rounding is symmetric in sign), so it is <= the computed d of every point inside: a skipped node holds no point whose
// d is below the lane's third value, hence nothing that changes the multiset of the three smallest.  The result does not
// depend on the Morton resolution, the sort or the visiting order.  No floating-point atomics.
// Compiled with -fmad=false: every fp32 operation is one IEEE operation.
#include <algorithm>

#include "gsb_ctx.cuh"
#include "gsb_geom.cuh"

namespace gsb {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int BB_THREADS = 256;
constexpr int KNN_THREADS = 256;  // 8 warps = 8 leaves per CTA
constexpr int MAX_LEVELS = 7;     // leaves + up to 6 levels above them (n < 2^30: 2^25 leaves)

struct BBox {
    float lo[3], hi[3];
    uint32_t nonfinite;
    uint32_t pad;
};

__device__ __forceinline__ float sq_dist(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = bx - ax, dy = by - ay, dz = bz - az;  // x_j - x_i
    return (dx * dx + dy * dy) + dz * dz;
}

__device__ __forceinline__ uint64_t umin64(uint64_t a, uint64_t b) { return a < b ? a : b; }

// the three smallest values seen, b0 <= b1 <= b2: an insertion network (a value >= b2 leaves them unchanged)
__device__ __forceinline__ void insert3(float d, float& b0, float& b1, float& b2) {
    b2 = fminf(b2, fmaxf(b1, d));
    b1 = fminf(b1, fmaxf(b0, d));
    b0 = fminf(b0, d);
}

template <typename T, typename F>
__device__ __forceinline__ T warp_reduce(T v, F op) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(FULL, v, o));
    return v;
}

// per-CTA bounding box of the finite coordinates and the OR of "a coordinate is not finite"
__global__ void __launch_bounds__(BB_THREADS) k_init_bbox(const float* __restrict__ xyz, uint64_t n, BBox* __restrict__ partial) {
    __shared__ float s[BB_THREADS / 32][6];
    __shared__ uint32_t s_bad[BB_THREADS / 32];
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    uint32_t bad = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * BB_THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * BB_THREADS) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float v = __ldg(xyz + i * 3 + a);
            if (isfinite(v)) {
                lo[a] = fminf(lo[a], v);
                hi[a] = fmaxf(hi[a], v);
            } else {
                bad = 1;
            }
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        lo[a] = warp_reduce(lo[a], [](float x, float y) { return fminf(x, y); });
        hi[a] = warp_reduce(hi[a], [](float x, float y) { return fmaxf(x, y); });
    }
    bad = __any_sync(FULL, bad) ? 1u : 0u;
    if (lane == 0) {
        for (int a = 0; a < 3; a++) s[warp][a] = lo[a], s[warp][3 + a] = hi[a];
        s_bad[warp] = bad;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        BBox b;
        for (int a = 0; a < 3; a++) b.lo[a] = INFINITY, b.hi[a] = -INFINITY;
        b.nonfinite = 0;
        b.pad = 0;
        for (int w = 0; w < BB_THREADS / 32; w++) {
            for (int a = 0; a < 3; a++) b.lo[a] = fminf(b.lo[a], s[w][a]), b.hi[a] = fmaxf(b.hi[a], s[w][3 + a]);
            b.nonfinite |= s_bad[w];
        }
        partial[blockIdx.x] = b;
    }
}

// one thread: the partials in order; also stores the element count the sort reads from device memory
__global__ void k_init_bbox_final(const BBox* __restrict__ partial, int count, BBox* __restrict__ out, uint32_t* d_m, uint32_t n) {
    BBox b = partial[0];
    for (int k = 1; k < count; k++) {
        const BBox p = partial[k];
        for (int a = 0; a < 3; a++) b.lo[a] = fminf(b.lo[a], p.lo[a]), b.hi[a] = fmaxf(b.hi[a], p.hi[a]);
        b.nonfinite |= p.nonfinite;
    }
    *out = b;
    *d_m = n;
}

// 21 bits -> every third bit of 63
__device__ __forceinline__ unsigned long long spread21(uint32_t v) {
    unsigned long long x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

struct MortonGrid {
    float lo[3], scale[3];  // cell = (v - lo) * scale, clamped to [0, 2^21 - 1]
};

__global__ void __launch_bounds__(256) k_init_morton(const float* __restrict__ xyz, uint64_t n, const MortonGrid g,
                                                    unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        unsigned long long code = 0;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float c = fminf(fmaxf((__ldg(xyz + i * 3 + a) - g.lo[a]) * g.scale[a], 0.0f), 2097151.0f);
            code |= spread21((uint32_t)c) << a;
        }
        keys[i] = code;
        vals[i] = (uint32_t)i;
    }
}

__global__ void __launch_bounds__(256) k_init_gather(const float* __restrict__ xyz, uint64_t n, const uint32_t* __restrict__ order,
                                                    float4* __restrict__ pts) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t j = order[i];
        pts[i] = make_float4(__ldg(xyz + (uint64_t)j * 3), __ldg(xyz + (uint64_t)j * 3 + 1), __ldg(xyz + (uint64_t)j * 3 + 2),
                             __uint_as_float(j));
    }
}

// warp w: the AABB of leaf w's points (lanes past n contribute the empty box)
__global__ void __launch_bounds__(256) k_init_leaf_boxes(const float4* __restrict__ pts, uint64_t n, uint32_t leaves,
                                                        float4* __restrict__ lo, float4* __restrict__ hi) {
    const uint32_t leaf = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (leaf >= leaves) return;  // whole warps
    const uint64_t i = (uint64_t)leaf * 32 + (threadIdx.x & 31);
    float4 p = i < n ? pts[i] : make_float4(NAN, NAN, NAN, 0.0f);  // fminf / fmaxf ignore NaN
    const auto mn = [](float x, float y) { return fminf(x, y); };
    const auto mx = [](float x, float y) { return fmaxf(x, y); };
    const float ax = warp_reduce(p.x, mn), ay = warp_reduce(p.y, mn), az = warp_reduce(p.z, mn);
    const float bx = warp_reduce(p.x, mx), by = warp_reduce(p.y, mx), bz = warp_reduce(p.z, mx);
    if ((threadIdx.x & 31) == 0) {
        lo[leaf] = make_float4(ax, ay, az, 0.0f);
        hi[leaf] = make_float4(bx, by, bz, 0.0f);
    }
}

// warp w: the AABB of nodes 32 w .. 32 w + 31 of the level below (`below` of them)
__global__ void __launch_bounds__(256) k_init_node_boxes(const float4* __restrict__ lo_in, const float4* __restrict__ hi_in, uint32_t below,
                                                        uint32_t count, float4* __restrict__ lo, float4* __restrict__ hi) {
    const uint32_t node = (uint32_t)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (node >= count) return;
    const uint32_t c = node * 32 + (threadIdx.x & 31);
    const float4 a = c < below ? lo_in[c] : make_float4(NAN, NAN, NAN, 0.0f);
    const float4 b = c < below ? hi_in[c] : make_float4(NAN, NAN, NAN, 0.0f);
    const auto mn = [](float x, float y) { return fminf(x, y); };
    const auto mx = [](float x, float y) { return fmaxf(x, y); };
    const float ax = warp_reduce(a.x, mn), ay = warp_reduce(a.y, mn), az = warp_reduce(a.z, mn);
    const float bx = warp_reduce(b.x, mx), by = warp_reduce(b.y, mx), bz = warp_reduce(b.z, mx);
    if ((threadIdx.x & 31) == 0) {
        lo[node] = make_float4(ax, ay, az, 0.0f);
        hi[node] = make_float4(bx, by, bz, 0.0f);
    }
}

struct Tree {
    const float4* lo;  // node boxes of every level, level l at off[l]
    const float4* hi;
    uint32_t off[MAX_LEVELS];
    uint32_t cnt[MAX_LEVELS];
    int top;           // the root's level (cnt[top] == 1); 0: a single leaf
};

// lane c < nchild holds child c's box; bit c of the result: some active lane's bound is strictly below its b2
__device__ __forceinline__ uint32_t test_children(const Tree& T, int level, uint32_t first, uint32_t nchild, int lane, bool active,
                                                  float px, float py, float pz, float b2) {
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
    if ((uint32_t)lane < nchild) {
        lo = T.lo[T.off[level] + first + lane];
        hi = T.hi[T.off[level] + first + lane];
    }
    uint32_t mask = 0;
    for (uint32_t c = 0; c < nchild; c++) {
        const float lx = __shfl_sync(FULL, lo.x, c), ly = __shfl_sync(FULL, lo.y, c), lz = __shfl_sync(FULL, lo.z, c);
        const float hx = __shfl_sync(FULL, hi.x, c), hy = __shfl_sync(FULL, hi.y, c), hz = __shfl_sync(FULL, hi.z, c);
        const float bound = sq_dist(px, py, pz, fminf(fmaxf(px, lx), hx), fminf(fmaxf(py, ly), hy), fminf(fmaxf(pz, lz), hz));
        if (__any_sync(FULL, active && bound < b2)) mask |= 1u << c;
    }
    return mask;
}

__global__ void __launch_bounds__(KNN_THREADS) k_init_knn(const float4* __restrict__ pts, uint64_t n, const __grid_constant__ Tree T,
                                                         float* __restrict__ scale) {
    const uint32_t leaf = (uint32_t)(((uint64_t)blockIdx.x * KNN_THREADS + threadIdx.x) >> 5);
    if (leaf >= T.cnt[0]) return;  // whole warps
    const int lane = threadIdx.x & 31;
    const uint64_t i = (uint64_t)leaf * 32 + lane;
    const bool active = i < n;
    const float4 p = active ? pts[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const uint32_t valid = (uint32_t)umin64(32, n - (uint64_t)leaf * 32);
    float b0 = INFINITY, b1 = INFINITY, b2 = INFINITY;
    // seed: the leaf's other points
    for (uint32_t k = 1; k < 32; k++) {
        const uint32_t src = (lane + k) & 31;
        const float qx = __shfl_sync(FULL, p.x, src), qy = __shfl_sync(FULL, p.y, src), qz = __shfl_sync(FULL, p.z, src);
        if (src < valid) insert3(sq_dist(p.x, p.y, p.z, qx, qy, qz), b0, b1, b2);
    }
    // descent: lane l keeps the mask of children still to visit at level l (warp-uniform values, a stack in registers)
    if (T.top > 0) {
        int level = T.top;
        uint32_t node = 0;  // index within its level
        uint32_t stack = 0;
        {
            const uint32_t m = test_children(T, level - 1, 0, T.cnt[level - 1], lane, active, p.x, p.y, p.z, b2);
            if (lane == level) stack = m;
        }
        while (true) {
            uint32_t m = __shfl_sync(FULL, stack, level);
            if (m == 0) {
                if (level == T.top) break;
                level++;
                node >>= 5;
                continue;
            }
            // the child on this warp's own path first, then the following ones cyclically (near in Morton order)
            const uint32_t a = (leaf >> (5 * (level - 1))) & 31;
            const uint32_t r = __funnelshift_r(m, m, a);
            const uint32_t c = (a + (uint32_t)(__ffs(r) - 1)) & 31;
            m &= ~(1u << c);
            if (lane == level) stack = m;
            const uint32_t child = node * 32 + c;
            if (level == 1) {  // a leaf: every one of its points against every lane
                if (child == leaf) continue;  // seeded above: a neighbour must enter once only
                const uint64_t j = (uint64_t)child * 32 + lane;
                const uint32_t cnt = (uint32_t)umin64(32, n - (uint64_t)child * 32);
                const float4 q = j < n ? pts[j] : make_float4(0.f, 0.f, 0.f, 0.f);
                for (uint32_t k = 0; k < cnt; k++) {
                    const float qx = __shfl_sync(FULL, q.x, k), qy = __shfl_sync(FULL, q.y, k), qz = __shfl_sync(FULL, q.z, k);
                    insert3(sq_dist(p.x, p.y, p.z, qx, qy, qz), b0, b1, b2);
                }
            } else {
                level--;
                node = child;
                const uint32_t nchild = min(32u, T.cnt[level - 1] - child * 32);
                const uint32_t mm = test_children(T, level - 1, child * 32, nchild, lane, active, p.x, p.y, p.z, b2);
                if (lane == level) stack = mm;
            }
        }
    }
    if (!active) return;
    // D over the m = min(3, n - 1) smallest, summed in ascending order
    float D;
    if (n >= 4) D = ((b0 + b1) + b2) / 3.0f;
    else if (n == 3) D = (b0 + b1) / 2.0f;
    else if (n == 2) D = b0 / 1.0f;
    else D = 0.0f;
    scale[__float_as_uint(p.w)] = sqrtf(fmaxf(D, 1e-7f));
}

// thread (row, k): float4 k of the row.  Records: (x, y, z, 1), (s, s, s, opacity), (1, 0, 0, 0), SH with
// sh[c] = (rgb[c] - 0.5) / SH_C0 for c < 3 and 0 elsewhere.
template <bool VEC>
__global__ void __launch_bounds__(256) k_init_records(const float* __restrict__ xyz, const float* __restrict__ rgb, const float* __restrict__ scale,
                                                     uint64_t n, float opacity, float* __restrict__ out) {
    const uint64_t total = n * 15;
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t row = t / 15;
        const uint32_t k = (uint32_t)(t - row * 15);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k == 0) {
            v = make_float4(__ldg(xyz + row * 3), __ldg(xyz + row * 3 + 1), __ldg(xyz + row * 3 + 2), 1.0f);
        } else if (k == 1) {
            const float s = __ldg(scale + row);
            v = make_float4(s, s, s, opacity);
        } else if (k == 2) {
            v.x = 1.0f;
        } else if (k == 3) {
            v.x = (__ldg(rgb + row * 3) - 0.5f) / SH_C0;
            v.y = (__ldg(rgb + row * 3 + 1) - 0.5f) / SH_C0;
            v.z = (__ldg(rgb + row * 3 + 2) - 0.5f) / SH_C0;
        }
        if constexpr (VEC) {
            reinterpret_cast<float4*>(out)[t] = v;
        } else {
            float* o = out + t * 4;
            o[0] = v.x, o[1] = v.y, o[2] = v.z, o[3] = v.w;
        }
    }
}

template <typename T>
T* carve(unsigned char*& at, uint64_t count) {
    T* p = reinterpret_cast<T*>(at);
    at += (count * sizeof(T) + 255) & ~(uint64_t)255;
    return p;
}

unsigned grid_for(uint64_t items, unsigned threads, int num_sms) {
    const uint64_t blocks = (items + threads - 1) / threads;
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks, (uint64_t)num_sms * 16));
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" int gsb_init_from_points(gsb_ctx* ctx, const float* xyz, const float* rgb, uint64_t n, float opacity, float* vertices,
                                    void* stream) {
    if (!ctx) return GSB_ERR_INVALID;
    auto bad = [&](const char* what) { return fail(ctx, GSB_ERR_INVALID, (std::string("gsb_init_from_points: ") + what).c_str()); };
    if (n == 0) return GSB_OK;
    if (!xyz || !rgb || !vertices) return bad("null argument");
    for (const void* p : {(const void*)xyz, (const void*)rgb, (const void*)vertices})
        if (reinterpret_cast<uintptr_t>(p) % 4) return bad("array not aligned to 4 B");
    if (n >= (1ull << 30)) return bad("limited to 2^30 - 1 points");
    if (!(opacity > 0.0f && opacity < 1.0f)) return bad("opacity outside (0, 1) or NaN");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = stream_or_own(ctx, stream);

    // the implicit tree: level 0 = leaves of 32 sorted points, level l + 1 groups 32 nodes of level l
    Tree T{};
    uint64_t nodes = 0;
    {
        uint64_t c = (n + 31) / 32;
        int l = 0;
        while (true) {
            T.off[l] = (uint32_t)nodes;
            T.cnt[l] = (uint32_t)c;
            nodes += c;
            if (c == 1) break;
            c = (c + 31) / 32;
            l++;
        }
        T.top = l;
    }
    const int bb_blocks = (int)grid_for(n, BB_THREADS, ctx->num_sms);
    const uint32_t sort_tiles = (uint32_t)((n + sort_tile_items() - 1) / sort_tile_items());
    // scratch, one allocation freed before returning
    uint64_t bytes = 0;
    const auto add = [&](uint64_t b) { bytes += (b + 255) & ~(uint64_t)255; };
    add(sizeof(BBox) * bb_blocks);
    add(sizeof(BBox));
    add(sizeof(SortCtl));
    add(4);
    add((uint64_t)sort_tiles * 256 * 8);
    add(8 * n), add(8 * n), add(4 * n), add(4 * n);
    add(16 * n);
    add(4 * n);
    add(16 * nodes), add(16 * nodes);
    unsigned char* base = nullptr;
    CK(dev_alloc(&base, bytes));
    unsigned char* at = base;
    BBox* partial = carve<BBox>(at, bb_blocks);
    BBox* box = carve<BBox>(at, 1);
    SortCtl* sc = carve<SortCtl>(at, 1);
    uint32_t* d_m = carve<uint32_t>(at, 1);
    unsigned long long* status = carve<unsigned long long>(at, (uint64_t)sort_tiles * 256);
    unsigned long long* keys[2] = {carve<unsigned long long>(at, n), carve<unsigned long long>(at, n)};
    uint32_t* vals[2] = {carve<uint32_t>(at, n), carve<uint32_t>(at, n)};
    float4* pts = carve<float4>(at, n);
    float* scale = carve<float>(at, n);
    float4* lo = carve<float4>(at, nodes);
    float4* hi = carve<float4>(at, nodes);
    T.lo = lo;
    T.hi = hi;

    int rc = GSB_OK;
    cudaError_t e = cudaSuccess;
    const auto run = [&]() -> cudaError_t {
        k_init_bbox<<<bb_blocks, BB_THREADS, 0, s>>>(xyz, n, partial);
        k_init_bbox_final<<<1, 1, 0, s>>>(partial, bb_blocks, box, d_m, (uint32_t)n);
        cudaError_t err = cudaGetLastError();
        if (err != cudaSuccess) return err;
        BBox hb;
        if ((err = cudaMemcpyAsync(&hb, box, sizeof hb, cudaMemcpyDeviceToHost, s)) != cudaSuccess) return err;
        if ((err = cudaStreamSynchronize(s)) != cudaSuccess) return err;
        if (hb.nonfinite) {
            rc = bad("a coordinate is not finite");
            return cudaSuccess;
        }
        MortonGrid g;
        for (int a = 0; a < 3; a++) {  // the resolution affects the speed only, never the result
            const double ext = (double)hb.hi[a] - (double)hb.lo[a];
            g.lo[a] = hb.lo[a];
            g.scale[a] = ext > 0.0 ? (float)(2097151.0 / ext) : 0.0f;
        }
        const unsigned grid = grid_for(n, 256, ctx->num_sms);
        k_init_morton<<<grid, 256, 0, s>>>(xyz, n, g, keys[0], vals[0]);
        if ((err = cudaGetLastError()) != cudaSuccess) return err;
        // private sort control and look-back words: the context's control block is left alone
        if ((err = cudaMemsetAsync(sc, 0, sizeof(SortCtl), s)) != cudaSuccess) return err;
        if ((err = cudaMemsetAsync(status, 0, (size_t)sort_tiles * 256 * 8, s)) != cudaSuccess) return err;
        SortParams sp;
        sp.keys[0] = keys[0];
        sp.keys[1] = keys[1];
        sp.key_bytes = 8;
        sp.vals[0] = vals[0];
        sp.vals[1] = vals[1];
        sp.d_m = d_m;
        sp.m_hint = (uint32_t)n;
        sp.key_bits = 63;
        sp.status = status;
        sp.status_tiles = sort_tiles;
        sp.epoch_base = 1;  // zeroed words: epoch 0 = not published
        sp.sc = sc;
        sp.num_sms = ctx->num_sms;
        sp.discard_sorted_keys = true;
        uint32_t passes = 0;
        if ((err = launch_sort(sp, &passes, s)) != cudaSuccess) return err;
        k_init_gather<<<grid, 256, 0, s>>>(xyz, n, vals[passes & 1], pts);
        const uint32_t leaves = T.cnt[0];
        k_init_leaf_boxes<<<(unsigned)(((uint64_t)leaves * 32 + 255) / 256), 256, 0, s>>>(pts, n, leaves, lo, hi);
        if ((err = cudaGetLastError()) != cudaSuccess) return err;
        for (int l = 1; l <= T.top; l++) {
            k_init_node_boxes<<<(unsigned)(((uint64_t)T.cnt[l] * 32 + 255) / 256), 256, 0, s>>>(lo + T.off[l - 1], hi + T.off[l - 1],
                                                                                            T.cnt[l - 1], T.cnt[l], lo + T.off[l],
                                                                                            hi + T.off[l]);
            if ((err = cudaGetLastError()) != cudaSuccess) return err;
        }
        k_init_knn<<<(unsigned)(((uint64_t)leaves * 32 + KNN_THREADS - 1) / KNN_THREADS), KNN_THREADS, 0, s>>>(pts, n, T, scale);
        if ((err = cudaGetLastError()) != cudaSuccess) return err;
        const unsigned rgrid = grid_for(n * 15, 256, ctx->num_sms);
        if (reinterpret_cast<uintptr_t>(vertices) % 16 == 0)
            k_init_records<true><<<rgrid, 256, 0, s>>>(xyz, rgb, scale, n, opacity, vertices);
        else
            k_init_records<false><<<rgrid, 256, 0, s>>>(xyz, rgb, scale, n, opacity, vertices);
        if ((err = cudaGetLastError()) != cudaSuccess) return err;
        return cudaStreamSynchronize(s);  // the records are written and the scratch is free to go
    };
    e = run();
    if (e != cudaSuccess) cudaStreamSynchronize(s);
    cudaFree(base);
    if (e != cudaSuccess) return fail(ctx, e == cudaErrorMemoryAllocation ? GSB_ERR_OOM : GSB_ERR_CUDA, "gsb_init_from_points", e);
    return rc;
}
