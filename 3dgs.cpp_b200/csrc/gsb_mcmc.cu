// gsb_mcmc.cu -- the two scene updates of 3D Gaussian Splatting as Markov Chain Monte Carlo (Kheradmand et al. 2024;
// DESIGN.md section 16), on the resident scene: gsb_mcmc_noise adds the SGLD position noise to every row, gsb_mcmc_relocate
// turns rows into copies of others with the closed-form opacity and scale correction.  Both write params, the activated
// records and the context's scene words in place, as k_adam_step does, so the next frame needs no upload.
//
// k_mcmc_noise: one thread per row, grid-stride; its random numbers are a function of (seed, step, row) alone (counter-based
// Philox), so there is no RNG state and no atomics.  Relocation: a counting pass (atomic increments into a per-call n x u32
// scratch, whose totals do not depend on the order), a check, then the source rows from their old records and, in a
// launch of its own, the copies from the new source rows.
// Compiled with -fmad=false: every fp32 and fp64 operation is one IEEE operation.
#include <math.h>

#include <initializer_list>
#include <string>

#include "gsb_ctx.cuh"
#include "gsb_geom.cuh"

namespace gsb {
namespace {

constexpr int MC_THREADS = 256;

// Philox4x32-10 (Salmon et al. 2011), Random123's philox4x32_10: ten rounds, the key bumped by the Weyl constants
// between rounds.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        if (r) k0 += 0x9E3779B9u, k1 += 0xBB67AE85u;
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// ((float)x + 0.5f) * 2^-32, in (0, 1]
__device__ __forceinline__ float uniform01(uint32_t x) { return ((float)x + 0.5f) * 2.3283064365386963e-10f; }

struct NoiseParams {
    float4* params;      // n x 15 float4: column 0-2 updated, column 3 rewritten as read
    float* vertices;     // n x 60: columns 0-2 updated
    float4* pos_op;      // xyz updated, opacity read
    const float4* cov_a;
    const float2* cov_b;
    uint64_t n;
    float scale;
    uint32_t key0, key1, step_lo, step_hi;
};

__global__ void __launch_bounds__(MC_THREADS) k_mcmc_noise(const NoiseParams P) {
    for (uint64_t i = (uint64_t)blockIdx.x * MC_THREADS + threadIdx.x; i < P.n; i += (uint64_t)gridDim.x * MC_THREADS) {
        const uint4 x = philox4x32_10(make_uint4((uint32_t)i, P.step_lo, P.step_hi, 0u), P.key0, P.key1);
        const float u0 = uniform01(x.x), u1 = uniform01(x.y), u2 = uniform01(x.z), u3 = uniform01(x.w);
        const float rho = sqrtf(-2.0f * logf(u0));  // Box-Muller
        const float e0 = rho * cospif(2.0f * u1), e1 = rho * sinpif(2.0f * u1);
        const float e2 = sqrtf(-2.0f * logf(u2)) * cospif(2.0f * u3);
        const float4 po = P.pos_op[i];
        // sigma(-k((1 - o) - 0.995)) with k = 100; 0 once expf overflows
        const float gate = 1.0f / (1.0f + expf(100.0f * (po.w - 0.005f)));
        const float gs = gate * P.scale;
        const float a = e0 * gs, b = e1 * gs, c = e2 * gs;
        const float4 ca = P.cov_a[i];  // Sigma rows (S00 S01 S02), (S01 S11 S12), (S02 S12 S22)
        const float2 cb = P.cov_b[i];
        float4 p = P.params[i * 15];
        p.x = p.x + ((ca.x * a + ca.y * b) + ca.z * c);
        p.y = p.y + ((ca.y * a + ca.w * b) + cb.x * c);
        p.z = p.z + ((ca.z * a + cb.x * b) + cb.y * c);
        P.params[i * 15] = p;
        float* v = P.vertices + i * 60;
        v[0] = p.x, v[1] = p.y, v[2] = p.z;
        P.pos_op[i] = make_float4(p.x, p.y, p.z, po.w);
    }
}

struct RelocParams {
    float4* params;  // n x 15 float4 each
    float4* exp_avg;
    float4* exp_avg_sq;
    float4* vertices;
    float4* pos_op;
    float4* cov_a;
    float2* cov_b;
    float4* sh;      // n x 12 float4
    const uint32_t* dst;
    const uint32_t* src;
    uint64_t k, n;
    uint32_t* count;      // n: occurrences of the row in src
    uint32_t* dst_count;  // n: occurrences of the row in dst
    uint32_t* bad;        // 1: a precondition does not hold
    float min_opacity;
};

__global__ void __launch_bounds__(MC_THREADS) k_reloc_count(const RelocParams P) {
    for (uint64_t j = (uint64_t)blockIdx.x * MC_THREADS + threadIdx.x; j < P.k; j += (uint64_t)gridDim.x * MC_THREADS) {
        const uint32_t s = P.src[j], d = P.dst[j];
        if (s >= P.n || d >= P.n) {
            *P.bad = 1u;
            continue;
        }
        atomicAdd(P.count + s, 1u);
        atomicAdd(P.dst_count + d, 1u);
    }
}

// every destination appears once in dst and never in src
__global__ void __launch_bounds__(MC_THREADS) k_reloc_check(const RelocParams P) {
    for (uint64_t j = (uint64_t)blockIdx.x * MC_THREADS + threadIdx.x; j < P.k; j += (uint64_t)gridDim.x * MC_THREADS) {
        const uint32_t d = P.dst[j];
        if (d < P.n && (P.dst_count[d] != 1u || P.count[d] != 0u)) *P.bad = 1u;
    }
}

// The new values of every source row, from its old record and its count (r = 1 + count): opacity, scale, their raw
// parameters, zero moments and the scene words.
__global__ void __launch_bounds__(MC_THREADS) k_reloc_sources(const RelocParams P) {
    for (uint64_t i = (uint64_t)blockIdx.x * MC_THREADS + threadIdx.x; i < P.n; i += (uint64_t)gridDim.x * MC_THREADS) {
        const uint32_t c = P.count[i];
        if (c == 0u) continue;
        const uint64_t w = i * 15;
        const float4 so = P.vertices[w + 1];
        const double r = (double)c + 1.0, alpha = (double)so.w;
        const double x = 1.0 - pow(1.0 - alpha, 1.0 / r);
        // sum_{j=1..r} (-1)^(j-1) C(r, j) x^j / sqrt(j), t_j = C(r, j) x^j by t_j = t_(j-1) (r - j + 1) / j x
        double denom = 0.0, t = 1.0;
        for (uint32_t j = 1; j <= c + 1u; j++) {
            t = t * (r - (double)j + 1.0) / (double)j * x;
            const double term = t / sqrt((double)j);
            denom = (j & 1u) ? denom + term : denom - term;
        }
        const double coeff = alpha / denom;
        const float o = (float)fmin(fmax(x, (double)P.min_opacity), 1.0 - 0x1p-23);
        const float4 s = make_float4((float)((double)so.x * coeff), (float)((double)so.y * coeff), (float)((double)so.z * coeff), o);
        P.vertices[w + 1] = s;
        const double od = (double)o;
        P.params[w + 1] = make_float4((float)log((double)s.x), (float)log((double)s.y), (float)log((double)s.z),
                                      (float)log(od / (1.0 - od)));
        const float4 zero = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll
        for (int q = 0; q < 15; q++) P.exp_avg[w + q] = zero, P.exp_avg_sq[w + q] = zero;
        store_cov3d(P.vertices[w], s, P.vertices[w + 2], i, P.pos_op, P.cov_a, P.cov_b, 1.0f);  // gsb_scene_upload's words
    }
}

// Pair j: row dst[j] becomes the new row src[j], one thread per float4 of the row (launched after k_reloc_sources).
__global__ void __launch_bounds__(MC_THREADS) k_reloc_copy(const RelocParams P) {
    const uint64_t total = P.k * 15;
    for (uint64_t t = (uint64_t)blockIdx.x * MC_THREADS + threadIdx.x; t < total; t += (uint64_t)gridDim.x * MC_THREADS) {
        const uint64_t j = t / 15;
        const uint32_t q = (uint32_t)(t - j * 15);
        const uint64_t s = P.src[j], d = P.dst[j];
        P.params[d * 15 + q] = P.params[s * 15 + q];
        P.vertices[d * 15 + q] = P.vertices[s * 15 + q];
        const float4 zero = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        P.exp_avg[d * 15 + q] = zero;
        P.exp_avg_sq[d * 15 + q] = zero;
        if (q >= 3) {
            P.sh[d * 12 + (q - 3)] = P.sh[s * 12 + (q - 3)];
        } else if (q == 0) {
            P.pos_op[d] = P.pos_op[s];
            P.cov_a[d] = P.cov_a[s];
            P.cov_b[d] = P.cov_b[s];
        }
    }
}

unsigned grid_for(uint64_t items, int num_sms) {  // one wave at most: 8 CTAs of 256 threads per SM
    const uint64_t blocks = (items + MC_THREADS - 1) / MC_THREADS;
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks, (uint64_t)num_sms * 8));
}

// The checks both entries share with gsb_adam_step; `fn` starts every message.
int check_training_call(gsb_ctx* ctx, const char* fn, std::initializer_list<const void*> arrays) {
    auto bad = [&](const char* what) { return fail(ctx, GSB_ERR_INVALID, (std::string(fn) + ": " + what).c_str()); };
    if (ctx->shard) return bad("sharded contexts have no training step");
    if (!ctx->pos_op) return fail(ctx, GSB_ERR_NO_SCENE, (std::string(fn) + ": no scene uploaded").c_str());
    if (ctx->scene_sh_half) return bad("fp16 SH storage has no training step");
    for (const void* p : arrays)
        if (!p) return bad("null argument");
    for (const void* p : arrays)
        if (reinterpret_cast<uintptr_t>(p) % 16) return bad("array not aligned to 16 B");
    return GSB_OK;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" int gsb_mcmc_noise(gsb_ctx* ctx, float* params, float* vertices, float scale, uint64_t seed, uint64_t step, void* stream) {
    if (!ctx) return GSB_ERR_INVALID;
    const char* fn = "gsb_mcmc_noise";
    int rc = check_training_call(ctx, fn, {params, vertices});
    if (rc != GSB_OK) return rc;
    if (!(scale >= 0.0f && scale <= 3.4028234663852886e38f)) return fail(ctx, GSB_ERR_INVALID, "gsb_mcmc_noise: scale below 0 or not finite");
    CK(cudaSetDevice(ctx->device));
    NoiseParams P{};
    P.params = reinterpret_cast<float4*>(params);
    P.vertices = vertices;
    P.pos_op = ctx->pos_op;
    P.cov_a = ctx->cov_a;
    P.cov_b = ctx->cov_b;
    P.n = ctx->n;
    P.scale = scale;
    P.key0 = (uint32_t)seed, P.key1 = (uint32_t)(seed >> 32);
    P.step_lo = (uint32_t)step, P.step_hi = (uint32_t)(step >> 32);
    // the scene changes in place: the last frame no longer describes it; graphs, arena and hints stay (as gsb_adam_step)
    ctx->scene_gen++;
    if (P.n == 0) return GSB_OK;
    k_mcmc_noise<<<grid_for(P.n, ctx->num_sms), MC_THREADS, 0, stream_or_own(ctx, stream)>>>(P);
    CK(cudaGetLastError());
    return GSB_OK;
}

extern "C" int gsb_mcmc_relocate(gsb_ctx* ctx, float* params, float* exp_avg, float* exp_avg_sq, float* vertices, const uint32_t* dst,
                                 const uint32_t* src, uint64_t k, float min_opacity, void* stream) {
    if (!ctx) return GSB_ERR_INVALID;
    const char* fn = "gsb_mcmc_relocate";
    auto bad = [&](const char* what) { return fail(ctx, GSB_ERR_INVALID, (std::string(fn) + ": " + what).c_str()); };
    int rc = check_training_call(ctx, fn, {params, exp_avg, exp_avg_sq, vertices});
    if (rc != GSB_OK) return rc;
    if (!(min_opacity >= 0.0f && min_opacity < 1.0f)) return bad("min_opacity outside [0, 1) or NaN");
    if (k == 0) return GSB_OK;
    if (!dst || !src) return bad("null argument");
    if (reinterpret_cast<uintptr_t>(dst) % 4 || reinterpret_cast<uintptr_t>(src) % 4) return bad("index array not aligned to 4 B");
    const uint64_t n = ctx->n;
    if (k >= n) return bad("k must be below n (the destinations are distinct rows that are not sources)");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = stream_or_own(ctx, stream);
    uint32_t* scratch = nullptr;  // count[n], dst_count[n], bad
    CK(dev_alloc(&scratch, 2 * n + 1));
    RelocParams P{};
    P.params = reinterpret_cast<float4*>(params);
    P.exp_avg = reinterpret_cast<float4*>(exp_avg);
    P.exp_avg_sq = reinterpret_cast<float4*>(exp_avg_sq);
    P.vertices = reinterpret_cast<float4*>(vertices);
    P.pos_op = ctx->pos_op;
    P.cov_a = ctx->cov_a;
    P.cov_b = ctx->cov_b;
    P.sh = reinterpret_cast<float4*>(ctx->sh.p);
    P.dst = dst;
    P.src = src;
    P.k = k;
    P.n = n;
    P.count = scratch;
    P.dst_count = scratch + n;
    P.bad = scratch + 2 * n;
    P.min_opacity = min_opacity;
    uint32_t violated = 0;
    const auto run = [&]() -> cudaError_t {
        cudaError_t e = cudaMemsetAsync(scratch, 0, (2 * n + 1) * sizeof(uint32_t), s);
        if (e != cudaSuccess) return e;
        k_reloc_count<<<grid_for(k, ctx->num_sms), MC_THREADS, 0, s>>>(P);
        k_reloc_check<<<grid_for(k, ctx->num_sms), MC_THREADS, 0, s>>>(P);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if ((e = cudaMemcpyAsync(&violated, P.bad, sizeof violated, cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
        if (violated) return cudaSuccess;  // nothing written
        ctx->scene_gen++;  // the scene changes in place, as after gsb_adam_step
        k_reloc_sources<<<grid_for(n, ctx->num_sms), MC_THREADS, 0, s>>>(P);
        k_reloc_copy<<<grid_for(k * 15, ctx->num_sms), MC_THREADS, 0, s>>>(P);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        return cudaStreamSynchronize(s);  // the rows are written and the scratch is free to go
    };
    const cudaError_t e = run();
    if (e != cudaSuccess) cudaStreamSynchronize(s);
    cudaFree(scratch);
    if (e != cudaSuccess) return fail(ctx, e == cudaErrorMemoryAllocation ? GSB_ERR_OOM : GSB_ERR_CUDA, fn, e);
    if (violated) return bad("an index >= n, a repeated destination, or a destination that is also a source");
    return GSB_OK;
}
