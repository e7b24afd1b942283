// gsb_blend.cu -- per-16x16-tile front-to-back alpha blending.
// Replaces render.comp:30-99 (dispatch src/Renderer.cpp:654-677).  The reference makes every
// pixel thread gather idx + uv + conic + colour from global memory for every Gaussian of the
// tile's run (render.comp:62-65,87; README.md:87 lists staging as a TODO).  Here one CTA of 128
// threads owns one tile; warp w owns the 8x8 pixel block at (8 (w & 1), 8 (w >> 1)) and each lane
// two pixels of one column of it.  The CTA
//   * stages the run in batches of 256 compact 48-B records into shared memory once;
//   * while staging, each thread classifies its Gaussians against the four 8x8 blocks of the tile:
//     a block whose best-case exponent is below the shader's own alpha < 1/255 cut (with an fp32
//     error margin) can never contribute, so that warp never touches the record (bit-identical
//     result: those pairs hit `continue` in render.comp:78);
//   * each warp compacts the batch with one ballot per 32 records and walks only its survivors,
//     reading each record as a shared-memory broadcast; the walk is branch-free per lane (the
//     shader's `continue`s and `break` are predicates on the state updates).
// With coarse bins (gsb_set_tile_cull level 2) the tile's run is filtered out of its block's list,
// which is fetched in segments by TMA bulk copies.  The per-pixel `break` (render.comp:83-85)
// becomes T == 0 + warp / block votes.
//
// EXACT mode: -fmad=false, ops in render.comp's order, exp = the fixed IEEE sequence of gsb_exp.cuh
// (bit-identical to oracle exp-mode 1).  FAST mode: explicit FMA + ex2.approx.
#include "gsb_cull.cuh"
#include "gsb_exp.cuh"
#include "gsb_internal.cuh"
#include "gsb_tma.cuh"

namespace gsb {

namespace {

constexpr unsigned FULL = 0xffffffffu;

// shared-memory loads by 32-bit shared-window address (one LDS each, immediate offsets, no generic-pointer arithmetic)
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

__device__ __forceinline__ uint32_t unorm8(float v) {
    v = fminf(fmaxf(v, 0.0f), 1.0f);  // NaN -> 0
    return __float2uint_rn(v * 255.0f);
}

// ------------------------------------------------------------------------------------------------------------------
// k_blend -- two pixels per thread.
//
// Lane (lx = lane & 7, ly = lane >> 3) of warp w owns the two pixels (lx, ly) and (lx, ly + 4) of the warp's 8x8 block.
// The two pixels share a column, so one staged record (three LDS.128) serves both, and the terms of render.comp:64-66
// that depend on dx only are computed once per record instead of once per pixel; everything else is two independent
// scalar chains (ILP for the issue-bound walk).  Every step is a single correctly rounded IEEE operation (-fmad=false:
// no contraction), so EXACT mode stays bit-identical to the oracle.
// ------------------------------------------------------------------------------------------------------------------
#ifndef GSB_BLEND_BATCH
#define GSB_BLEND_BATCH 256  // records staged per batch (2 per thread)
#endif
#ifndef GSB_BLEND_MIN_BLOCKS
#define GSB_BLEND_MIN_BLOCKS 8
#endif
#ifndef GSB_BLEND_CHECK
#define GSB_BLEND_CHECK 8  // records walked between two "is the whole warp done" votes
#endif
constexpr int BLEND_THREADS = 128;
constexpr int BLEND_SEG = 4 * BLEND_THREADS;  // list entries scanned per batch at most
constexpr int BLEND_BATCH = GSB_BLEND_BATCH;
constexpr int BLEND_WARPS = BLEND_THREADS / 32;

struct __align__(16) StagedRec {  // 48 B: three 16-B slots = three LDS.128 per visited record
    float4 q0;  // ux uy -A/2 -B       (exact power-of-two / sign scalings of the conic: render.comp:66 becomes
    float4 q1;  // -C/2 opacity r g     ((-A/2 dx) dx + (-C/2 dy) dy) + ((-B) dx) dy, bit for bit)
    float4 q2;  // b power_cut bits(index in batch) -
};

// Bit w set <=> warp w's 8x8 pixel block may receive a contribution from this Gaussian (gsb_cull.cuh).
__device__ __forceinline__ uint32_t block_mask(float ux, float uy, float A, float B, float C, float cut, float tile_x0, float tile_y0) {
    if (!(A > 0.0f) || !(C > 0.0f)) return 0xfu;  // not positive definite / NaN: never cull
    const float inv_a = __frcp_rn(A), inv_c = __frcp_rn(C);
    uint32_t mask = 0;
#pragma unroll
    for (int w = 0; w < BLEND_WARPS; w++) {
        const float x0 = tile_x0 + (float)((w & 1) * 8), y0 = tile_y0 + (float)((w >> 1) * 8);
        if (rect_may_contribute(ux, uy, A, B, C, inv_a, inv_c, x0, y0, 8.0f, 8.0f, cut)) mask |= 1u << w;
    }
    return mask;
}

// Per-pixel state of gsb_set_backward frames (k_blend<..., RECORD = true>): for each of the thread's two pixels, the
// transmittance after its last contributor and that contributor's list position + 1 (0 = none).  Empty otherwise, so the
// plain instantiations carry no trace of it.
template <bool ON>
struct BlendRecord {
    float t0 = 1.0f, t1 = 1.0f;
    uint32_t last0 = 0, last1 = 0;
    __device__ __forceinline__ void note(bool ok0, bool ok1, float tt0, float tt1, uint32_t pos1) {
        if (ok0) {
            t0 = tt0;
            last0 = pos1;
        }
        if (ok1) {
            t1 = tt1;
            last1 = pos1;
        }
    }
    __device__ __forceinline__ void store(const BlendParams& P, bool in0, bool in1, uint32_t px, uint32_t py0, uint32_t py1) const {
        if (in0) P.record[(size_t)py0 * P.width + px] = make_uint2(__float_as_uint(t0), last0);
        if (in1) P.record[(size_t)py1 * P.width + px] = make_uint2(__float_as_uint(t1), last1);
    }
};
template <>
struct BlendRecord<false> {
    __device__ __forceinline__ void note(bool, bool, float, float, uint32_t) {}
    __device__ __forceinline__ void store(const BlendParams&, bool, bool, uint32_t, uint32_t, uint32_t) const {}
};

// COARSE (gsb_set_tile_cull level 2): the list is that of a block of 2^cs x 2^cs tiles and every entry's key carries the mask
// of the block's tiles inside the Gaussian's tile AABB.  Staging becomes a stream compaction: the CTA scans the list 128
// entries at a time (keys + payloads only, coalesced), keeps the entries whose mask has this tile's bit -- in list order, so
// the tile's own (depth, index) order is preserved -- and gathers records only for those, until the batch holds up to
// BLEND_BATCH of them.  The walk is unchanged.
// RECORD (gsb_set_backward, per-tile lists only): each pixel also stores its final transmittance (the product of 1 - alpha
// over its contributors: the T the shader holds at its break or at the end of the list) and the list position + 1 of its
// last contributor into P.record -- what gsb_backward.cu needs to walk the list back to front.  The image is unchanged.
template <int MODE, bool STATS, bool COARSE, bool RECORD = false>
__global__ void __launch_bounds__(BLEND_THREADS, GSB_BLEND_MIN_BLOCKS) k_blend(const __grid_constant__ BlendParams P) {
    static_assert(!(RECORD && COARSE), "the backward state is recorded on per-tile lists only");
    __shared__ StagedRec s_rec[BLEND_BATCH];
    __shared__ uint8_t s_mask[BLEND_BATCH];
    __shared__ uint32_t s_wc[BLEND_WARPS];
    // COARSE: the next segment of the block's (key, payload) run, fetched by TMA (cp.async.bulk) while the current batch is
    // gathered and walked: BASELINE north_star's "TMA bulk staging of per-tile Gaussian runs into shared memory"
    __shared__ alignas(16) uint32_t s_seg[COARSE ? 2 : 1][COARSE ? BLEND_SEG + 4 : 4];
    __shared__ unsigned long long s_bar;
    __shared__ alignas(16) uint16_t s_list[BLEND_WARPS][BLEND_BATCH];  // per warp: shared-window addresses of the records it must visit
    // COARSE: compact id and list position of the batch's entries.  They live in the same 2 KB as the per-warp lists: written
    // by the fill, read by the record gather, and only then (a barrier later) do the warps build their lists; the barrier at
    // the end of the batch separates the walk from the next fill.  (27 KB instead of 29 KB per CTA = 8 instead of 7 per SM.)
    static_assert(sizeof(uint16_t) * BLEND_WARPS * BLEND_BATCH >= 2 * sizeof(uint32_t) * BLEND_BATCH, "s_cid + s_eidx alias s_list");
    uint32_t* const s_cid = reinterpret_cast<uint32_t*>(&s_list[0][0]);
    uint32_t* const s_eidx = s_cid + BLEND_BATCH;
    __shared__ uint32_t s_used, s_walked, s_hits;
    static_assert(sizeof(StagedRec) * BLEND_BATCH < 65536, "u16 list entries hold shared-window addresses");

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tx = blockIdx.x % P.tiles_x;
    const uint32_t ty = P.tile_row_begin + blockIdx.x / P.tiles_x;
    // render.comp:43-44; stored as (start, ~end), empty = all ones.  With coarse bins (gsb_set_tile_cull level 2) the list is
    // that of the 2^cs x 2^cs tile block holding this tile: still in (depth, index) order, and the staging below keeps exactly
    // the records whose tile AABB holds (tx, ty) = the tile's own list in the reference.
    const uint32_t cs = P.coarse_shift;
    uint2 range = P.ranges[(ty >> cs) * P.bins_x + (tx >> cs)];
    range.y = ~range.y;
    const uint32_t px = tx * GSB_TILE + (warp & 1) * 8 + (lane & 7);
    const uint32_t py0 = ty * GSB_TILE + (warp >> 1) * 8 + (lane >> 3), py1 = py0 + 4;
    const bool in0 = px < P.width && py0 < P.height, in1 = px < P.width && py1 < P.height;  // :37-39
    const float fx = (float)px, fy0 = (float)py0, fy1 = (float)py1;
    const float tile_x0 = (float)(tx * GSB_TILE), tile_y0 = (float)(ty * GSB_TILE);
    if (tid == 0) {
        s_used = 0;
        s_walked = 0;
        s_hits = 0;
    }
    __syncthreads();

    // transmittance (0 = finished or outside the image) and colour a/b/c of pixel 0/1
    float T0 = in0 ? 1.0f : 0.0f, T1 = in1 ? 1.0f : 0.0f, ca0 = 0.f, ca1 = 0.f, cb0 = 0.f, cb1 = 0.f, cc0 = 0.f, cc1 = 0.f;
#define BLEND_DONE (T0 == 0.0f && T1 == 0.0f)
    uint32_t used = 0, walked = 0, hits = 0, staged = 0;
    BlendRecord<RECORD> brec;
    const uint32_t rec_sh = (uint32_t)__cvta_generic_to_shared(&s_rec[0]);
    const uint32_t list_sh = (uint32_t)__cvta_generic_to_shared(&s_list[warp][0]);

    const uint32_t tbit = 16u + (((ty & ((1u << cs) - 1u)) << cs) | (tx & ((1u << cs) - 1u)));  // this tile's bit in a coarse key
    uint32_t cursor = range.x;  // COARSE: next list entry to scan
    uint32_t seg_a = range.x & ~3u, seg_parity = 0u;
    bool seg_pending = COARSE && range.x < range.y;  // a bulk copy into s_seg is in flight
    if (COARSE) {
        if (tid == 0) {
            mbar_init(&s_bar, 1);
            mbar_fence_init();
            if (range.x < range.y) {
                const uint32_t bytes = (((min(range.y, range.x + (uint32_t)BLEND_SEG) - seg_a) + 3u) & ~3u) * 4u;
                mbar_expect_tx(&s_bar, 2u * bytes);
                tma_load(s_seg[0], P.keys + seg_a, bytes, &s_bar);
                tma_load(s_seg[1], P.vals + seg_a, bytes, &s_bar);
            }
        }
        __syncthreads();  // the barrier object is initialised before anyone waits on it
    }
    for (uint32_t base = range.x; COARSE ? (cursor < range.y) : (base < range.y); base += BLEND_BATCH) {
        uint32_t cnt;
        if constexpr (COARSE) {
            // ---- fill: scan up to 4 x 128 entries (loads issued together), compact this tile's entries in list order ----
            constexpr int STEPS = 4;
            uint32_t kk[STEPS], vv[STEPS];
            // the segment that starts at `cursor` (16-B aligned start seg_a <= cursor).  One warp polls the mbarrier, the others
            // sleep on the hardware barrier: 128 threads spinning on try_wait cost issue slots the other CTAs' walks need
            if (warp == 0) mbar_wait(&s_bar, seg_parity);
            __syncthreads();
            seg_parity ^= 1u;
            seg_pending = false;
#pragma unroll
            for (int j = 0; j < STEPS; j++) {
                const uint32_t e = cursor + (uint32_t)(j * BLEND_THREADS + tid);
                kk[j] = 0u;
                vv[j] = 0u;
                if (e < range.y) {
                    kk[j] = s_seg[0][e - seg_a];
                    vv[j] = s_seg[1][e - seg_a];
                }
            }
            uint32_t nfill = 0, steps = 0;
#pragma unroll
            for (int j = 0; j < STEPS; j++) {
                if (cursor + (uint32_t)(j * BLEND_THREADS) >= range.y || nfill > (uint32_t)(BLEND_BATCH - BLEND_THREADS)) break;  // uniform
                const bool match = (kk[j] >> tbit) & 1u;
                const unsigned bits = __ballot_sync(FULL, match);
                if (lane == 0) s_wc[warp] = __popc(bits);
                __syncthreads();
                uint32_t off = nfill + __popc(bits & ((1u << lane) - 1u)), tot = 0;
#pragma unroll
                for (int w = 0; w < BLEND_WARPS; w++) {
                    const uint32_t c = s_wc[w];
                    if (w < warp) off += c;
                    tot += c;
                }
                if (match) {
                    s_cid[off] = vv[j];
                    s_eidx[off] = cursor - range.x + (uint32_t)(j * BLEND_THREADS + tid);
                }
                nfill += tot;
                steps++;
                __syncthreads();  // s_wc is reused by the next step; s_cid / s_eidx are read below
            }
            cursor = min(range.y, cursor + steps * (uint32_t)BLEND_THREADS);
            cnt = nfill;
            // every thread has read its entries (the barriers of the steps above): fetch the next segment now, it lands while
            // this batch's records are gathered and walked
            if (cursor < range.y) {
                seg_a = cursor & ~3u;
                seg_pending = true;
                if (tid == 0) {
                    const uint32_t bytes = (((min(range.y, cursor + (uint32_t)BLEND_SEG) - seg_a) + 3u) & ~3u) * 4u;
                    fence_proxy_async();
                    mbar_expect_tx(&s_bar, 2u * bytes);
                    tma_load(s_seg[0], P.keys + seg_a, bytes, &s_bar);
                    tma_load(s_seg[1], P.vals + seg_a, bytes, &s_bar);
                }
            }
        } else {
            cnt = min((uint32_t)BLEND_BATCH, range.y - base);
        }
        if (STATS) staged += cnt;
#pragma unroll
        for (int j = 0; j < BLEND_BATCH / BLEND_THREADS; j++) {
            const uint32_t li = (uint32_t)(j * BLEND_THREADS + tid);
            if (li < cnt) {
                const uint32_t cid = COARSE ? s_cid[li] : __ldg(P.vals + base + li);
                const float4* rec = P.recs + (size_t)cid * GSB_REC_F4;
                const float4 a = __ldg(rec), col = __ldg(rec + 2);
                const float2 b = __ldg(reinterpret_cast<const float2*>(rec + 1));  // conic.z, opacity
                const float cut = power_cut(b.y);
                const uint32_t m = block_mask(a.x, a.y, a.z, a.w, b.x, cut, tile_x0, tile_y0);
                if (m) {
                    s_rec[li].q0 = make_float4(a.x, a.y, -0.5f * a.z, -a.w);
                    s_rec[li].q1 = make_float4(-0.5f * b.x, b.y, col.x, col.y);
                    // q2.z: position in the list relative to the batch's base offset (the consumed-entries statistic)
                    s_rec[li].q2 = make_float4(col.z, cut, __uint_as_float(COARSE ? s_eidx[li] : li), 0.f);
                }
                s_mask[li] = (uint8_t)m;
            }
        }
        __syncthreads();
        if (!__all_sync(FULL, BLEND_DONE)) {
            uint32_t n = 0;
            for (uint32_t c = 0; c < cnt; c += 32) {  // one ballot per 32 records
                const bool mine = (c + lane < cnt) && ((s_mask[c + lane] >> warp) & 1u);
                const unsigned bits = __ballot_sync(FULL, mine);
                if (mine) s_list[warp][n + __popc(bits & ((1u << lane) - 1u))] = (uint16_t)(rec_sh + (c + lane) * sizeof(StagedRec));
                n += __popc(bits);
            }
            __syncwarp();
            const uint32_t base_off = COARSE ? 0u : base - range.x;
            uint32_t k0 = 0;
            for (; k0 < n; k0 += GSB_BLEND_CHECK) {
                if (__all_sync(FULL, BLEND_DONE)) break;
                const uint32_t k1 = min(n, k0 + (uint32_t)GSB_BLEND_CHECK);
                for (uint32_t k = k0; k < k1; k++) {
                    const uint32_t addr = lds_u16(list_sh + 2u * k);
                    const float4 q0 = lds_f4(addr), q1 = lds_f4(addr + 16u), q2 = lds_f4(addr + 32u);
                    const float cut = q2.y;
                    const float dx = q0.x - fx, dy0 = q0.y - fy0, dy1 = q0.y - fy1;  // :64 (one column: dx is shared)
                    float pw0, pw1, al0, al1;
                    if (MODE == GSB_MODE_EXACT) {
                        // :66 with the pre-scaled conic: ((A' dx) dx + (C' dy) dy) + (B' dx) dy
                        const float adx = (q0.z * dx) * dx, bdx = q0.w * dx;
                        pw0 = (adx + (q1.x * dy0) * dy0) + bdx * dy0;
                        pw1 = (adx + (q1.x * dy1) * dy1) + bdx * dy1;
                        al0 = fminf(0.99f, q1.y * exp_shared_inrange(pw0));  // :77
                        al1 = fminf(0.99f, q1.y * exp_shared_inrange(pw1));
                    } else {
                        const float ad = q0.z * dx, bdx = q0.w * dx;
                        pw0 = fmaf(ad, dx, fmaf(q1.x * dy0, dy0, bdx * dy0));
                        pw1 = fmaf(ad, dx, fmaf(q1.x * dy1, dy1, bdx * dy1));
                        al0 = fminf(0.99f, q1.y * __expf(pw0));
                        al1 = fminf(0.99f, q1.y * __expf(pw1));
                    }
                    // A finished (or out-of-image) pixel carries T == 0 (a live one has T >= 1e-4): its test_T is 0, so it
                    // "finishes" again at every record it would touch, never accumulates, and needs no separate flag.
                    // in0 / in1: :68-70 and, below the Gaussian's cut, alpha < 1/255 (:78); a NaN power passes like in the shader
                    const bool in0k = !(pw0 > 0.0f || pw0 < cut) && !(al0 < 1.0f / 255.0f);  // :78-80
                    const bool in1k = !(pw1 > 0.0f || pw1 < cut) && !(al1 < 1.0f / 255.0f);
                    const float tt0 = T0 * (1.0f - al0), tt1 = T1 * (1.0f - al1);  // :82
                    const bool ok0 = in0k && !(tt0 < 0.0001f), ok1 = in1k && !(tt1 < 0.0001f);  // :83-85 (the break)
                    if (STATS) {
                        const uint32_t u = base_off + __float_as_uint(q2.z) + 1u;
                        used = ((in0k && !ok0 && T0 != 0.0f) || (in1k && !ok1 && T1 != 0.0f)) ? max(used, u) : used;
                        if (P.stats > 1) hits += (in0k && T0 != 0.0f ? 1u : 0u) + (in1k && T1 != 0.0f ? 1u : 0u);  // debug frames only
                    }
                    // the products are computed unconditionally, only the accumulates and the transmittance are predicated
                    float w0a, w1a, w0b, w1b, w0c, w1c;
                    if (MODE == GSB_MODE_EXACT) {
                        w0a = (q1.z * al0) * T0;  // :87
                        w1a = (q1.z * al1) * T1;
                        w0b = (q1.w * al0) * T0;
                        w1b = (q1.w * al1) * T1;
                        w0c = (q2.x * al0) * T0;
                        w1c = (q2.x * al1) * T1;
                    } else {
                        const float w0 = al0 * T0, w1 = al1 * T1;
                        w0a = q1.z * w0;
                        w1a = q1.z * w1;
                        w0b = q1.w * w0;
                        w1b = q1.w * w1;
                        w0c = q2.x * w0;
                        w1c = q2.x * w1;
                    }
                    if (ok0) {
                        ca0 = __fadd_rn(ca0, w0a);
                        cb0 = __fadd_rn(cb0, w0b);
                        cc0 = __fadd_rn(cc0, w0c);
                    }
                    if (ok1) {
                        ca1 = __fadd_rn(ca1, w1a);
                        cb1 = __fadd_rn(cb1, w1b);
                        cc1 = __fadd_rn(cc1, w1c);
                    }
                    if constexpr (RECORD) brec.note(ok0, ok1, tt0, tt1, base_off + __float_as_uint(q2.z) + 1u);
                    if (in0k) T0 = ok0 ? tt0 : 0.0f;  // :88, or the break
                    if (in1k) T1 = ok1 ? tt1 : 0.0f;
                }
            }
            if (STATS) {
                walked += min(k0, n);
                if (!BLEND_DONE) used = COARSE ? cursor - range.x : base_off + cnt;  // a live pixel read the whole batch
            }
        }
        if (__syncthreads_and(BLEND_DONE)) break;
    }
#undef BLEND_DONE
    if (COARSE && seg_pending) mbar_wait(&s_bar, seg_parity);  // never leave with a bulk copy still writing this CTA's shared memory
    if constexpr (RECORD) brec.store(P, in0, in1, px, py0, py1);

    if (STATS) {
        if (in0 || in1) atomicMax(&s_used, used);
        if (lane == 0 && walked) atomicAdd(&s_walked, walked);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(FULL, hits, o);
        if (lane == 0 && hits) atomicAdd(&s_hits, hits);
    }
    // Destinations: the caller's buffer, or -- frame sharding -- the whole-frame buffer of EVERY rank (peer memory over
    // NVLink; posted stores, so the framebuffer exchange rides under the blend instead of following it as a collective).
    const int ndst = P.num_peers > 0 ? P.num_peers : 1;
    const uint32_t row0 = py0 - P.out_first_row;
    if (P.format == GSB_FORMAT_RGBA32F) {
        for (int d = 0; d < ndst; d++) {
            unsigned char* band = static_cast<unsigned char*>(P.num_peers > 0 ? P.peer_frames[d] : P.out);
            if (in0) reinterpret_cast<float4*>(band + (size_t)row0 * P.row_pitch_bytes)[px] = make_float4(ca0, cb0, cc0, 1.0f);  // :98 vec4(c, 1)
            if (in1) reinterpret_cast<float4*>(band + (size_t)(row0 + 4) * P.row_pitch_bytes)[px] = make_float4(ca1, cb1, cc1, 1.0f);
        }
    } else {
        // 8-bit formats: transpose the tile through shared memory so that every warp store covers whole 64-B tile rows
        // (also what lets gsb_render write a pinned host frame directly at a good PCIe payload size)
        __syncthreads();  // everyone is out of the batch loop: s_rec can be reused
        uint32_t* s_tile = reinterpret_cast<uint32_t*>(&s_rec[0]);  // [16][16]
        const bool bgra = P.format == GSB_FORMAT_BGRA8;
        {
            const uint32_t r0 = unorm8(ca0), g0 = unorm8(cb0), b0 = unorm8(cc0), r1 = unorm8(ca1), g1 = unorm8(cb1), b1 = unorm8(cc1);
            const uint32_t lx = (warp & 1) * 8 + (lane & 7), ly = (warp >> 1) * 8 + (lane >> 3);
            s_tile[ly * 16 + lx] = bgra ? (b0 | (g0 << 8) | (r0 << 16) | 0xff000000u) : (r0 | (g0 << 8) | (b0 << 16) | 0xff000000u);
            s_tile[(ly + 4) * 16 + lx] = bgra ? (b1 | (g1 << 8) | (r1 << 16) | 0xff000000u) : (r1 | (g1 << 8) | (b1 << 16) | 0xff000000u);
        }
        __syncthreads();
        if (tid < 64) {  // thread -> (row = tid / 4, 4 pixels at x = 4 (tid % 4)): 4 consecutive threads = one 64-B tile row
            const uint32_t ry = (uint32_t)tid >> 2, rx = ((uint32_t)tid & 3u) * 4u;
            const uint32_t gy = ty * GSB_TILE + ry, gx = tx * GSB_TILE + rx;
            if (gy < P.height && gx < P.width) {
                const uint4 v = *reinterpret_cast<const uint4*>(&s_tile[ry * 16 + rx]);
                for (int d = 0; d < ndst; d++) {
                    unsigned char* band = static_cast<unsigned char*>(P.num_peers > 0 ? P.peer_frames[d] : P.out);
                    uint32_t* dst = reinterpret_cast<uint32_t*>(band + (size_t)(gy - P.out_first_row) * P.row_pitch_bytes) + gx;
                    if (gx + 3 < P.width && (reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
                        *reinterpret_cast<uint4*>(dst) = v;
                    } else {  // ragged right edge (W not a multiple of 4) or an unaligned pitch
                        const uint32_t e[4] = {v.x, v.y, v.z, v.w};
                        for (uint32_t q = 0; q < 4 && gx + q < P.width; q++) dst[q] = e[q];
                    }
                }
            }
        }
    }
    if (STATS) {
        __syncthreads();
        if (tid == 0) {
            if (s_used) atomicAdd(&P.ctl->blend_consumed, (unsigned long long)s_used);
            if (s_walked) atomicAdd(&P.ctl->blend_walked, (unsigned long long)s_walked);
            if (s_hits) atomicAdd(&P.ctl->blend_hits, (unsigned long long)s_hits);
            if (staged) atomicAdd(&P.ctl->blend_staged, (unsigned long long)staged);
        }
    }
}

}  // namespace

cudaError_t launch_blend(const BlendParams& p, cudaStream_t s) {
    const uint32_t rows = p.tile_row_end - p.tile_row_begin;
    const uint32_t blocks = rows * p.tiles_x;
    if (blocks == 0) return cudaSuccess;
    if (p.coarse_shift) {
        if (p.stats) {
            if (p.mode == GSB_MODE_EXACT) k_blend<GSB_MODE_EXACT, true, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
            else k_blend<GSB_MODE_FAST, true, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
        } else {
            if (p.mode == GSB_MODE_EXACT) k_blend<GSB_MODE_EXACT, false, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
            else k_blend<GSB_MODE_FAST, false, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
        }
    } else if (p.record) {  // gsb_set_backward
        if (p.stats) {
            if (p.mode == GSB_MODE_EXACT) k_blend<GSB_MODE_EXACT, true, false, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
            else k_blend<GSB_MODE_FAST, true, false, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
        } else {
            if (p.mode == GSB_MODE_EXACT) k_blend<GSB_MODE_EXACT, false, false, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
            else k_blend<GSB_MODE_FAST, false, false, true><<<blocks, BLEND_THREADS, 0, s>>>(p);
        }
    } else if (p.stats) {
        if (p.mode == GSB_MODE_EXACT) k_blend<GSB_MODE_EXACT, true, false><<<blocks, BLEND_THREADS, 0, s>>>(p);
        else k_blend<GSB_MODE_FAST, true, false><<<blocks, BLEND_THREADS, 0, s>>>(p);
    } else {
        if (p.mode == GSB_MODE_EXACT) k_blend<GSB_MODE_EXACT, false, false><<<blocks, BLEND_THREADS, 0, s>>>(p);
        else k_blend<GSB_MODE_FAST, false, false><<<blocks, BLEND_THREADS, 0, s>>>(p);
    }
    return cudaGetLastError();
}

}  // namespace gsb
