// gsb_sort.cu -- device-wide Onesweep LSD radix sort of (key, u32 payload) pairs, keys u32 or u64.
// Replaces the reference's 8 x (sort/hist.comp:69-94 + sort/sort.comp:99-213) dispatch loop
// (src/Renderer.cpp:598-629).  Same contract: stable, ascending by key, 8-bit digits; but
//   * ONE histogram kernel reads the keys once and produces the digit histograms of all passes,
//   * each pass is ONE kernel: per-tile ranking + chained-scan decoupled look-back over tiles
//     (no O(workgroups^2) histogram re-reads as in sort.comp:112) + shared-memory staged,
//     coalesced scatter of key and payload,
//   * only P = ceil(key_bits / 8) passes run (the reference always runs 8 over 64 bits), and the
//     element count is read from device memory (no host round trip).
// The frame uses it twice (DESIGN.md "two-level LSD"): 32-bit depth keys over the N_v visible
// Gaussians, then 32-bit tile-id keys over the M instances; gsb_sort_pairs exposes the u64 form.
// No tensor cores: integer/byte work, HBM- and latency-bound.
#include "gsb_internal.cuh"
#include "gsb_tma.cuh"

namespace gsb {

namespace {

#ifndef GSB_SORT_MATCH_ATOMIC
#define GSB_SORT_MATCH_ATOMIC 1  // 1: match equal digits with shared-memory atomicOr lane masks; 0: 8 ballots per digit
#endif
constexpr int SORT_IPT = 16;  // pairs per thread
#ifndef GSB_SORT_THREADS
#define GSB_SORT_THREADS 256  // 256 threads x 16 = 4096-pair tiles, TWO persistent CTAs per SM: finer tiles balance the SMs better on the small depth sort
#endif
constexpr int SORT_THREADS = GSB_SORT_THREADS;
constexpr int SORT_TILE = SORT_THREADS * SORT_IPT;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int RADIX = 256;
constexpr unsigned FULL = 0xffffffffu;

#ifndef GSB_HIST_CTAS
#define GSB_HIST_CTAS 3  // k_sort_hist CTAs per SM
#endif
constexpr int HIST_THREADS = 512;
constexpr int HIST_IPT = 8;
constexpr int HIST_TILE = HIST_THREADS * HIST_IPT;

// look-back word: [63:32] epoch, [31:30] flag, [29:0] count.  Epoch tagging means the status
// array never needs clearing between passes or frames.
constexpr uint32_t LB_AGG = 1u << 30;
constexpr uint32_t LB_PREFIX = 2u << 30;
constexpr uint32_t LB_COUNT = (1u << 30) - 1u;
#ifndef GSB_LB_WINDOW
#define GSB_LB_WINDOW 8
#endif
constexpr int LB_WINDOW = GSB_LB_WINDOW;  // predecessors inspected per look-back step (loads in flight)

__device__ __forceinline__ unsigned long long ld_volatile(const unsigned long long* p) {
    return *reinterpret_cast<const volatile unsigned long long*>(p);
}
__device__ __forceinline__ void st_volatile(unsigned long long* p, unsigned long long v) {
    *reinterpret_cast<volatile unsigned long long*>(p) = v;
}

template <typename KeyT>
__device__ __forceinline__ KeyT key_max();
template <>
__device__ __forceinline__ uint32_t key_max<uint32_t>() {
    return 0xffffffffu;
}
template <>
__device__ __forceinline__ unsigned long long key_max<unsigned long long>() {
    return ~0ull;
}

// ------------------------------------------------------------------------------------------
// Histogram of every digit in one read of the keys (replaces hist.comp, run once not 8x).
// ------------------------------------------------------------------------------------------
template <typename KeyT, int P>
__global__ void __launch_bounds__(HIST_THREADS) k_sort_hist(const KeyT* __restrict__ keys, const uint32_t* __restrict__ d_m,
                                                            SortCtl* sc) {
    __shared__ uint32_t s_hist[P][RADIX];
    const int tid = threadIdx.x;
    for (int k = tid; k < P * RADIX; k += HIST_THREADS) (&s_hist[0][0])[k] = 0;
    __syncthreads();
    const uint32_t m = *d_m;
    const uint32_t num_tiles = (m + HIST_TILE - 1) / HIST_TILE;
    for (uint32_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const uint32_t base = tile * HIST_TILE;
        KeyT k[HIST_IPT];
#pragma unroll
        for (int it = 0; it < HIST_IPT; it++) {
            const uint32_t idx = base + it * HIST_THREADS + tid;
            k[it] = idx < m ? __ldg(keys + idx) : key_max<KeyT>();
        }
#pragma unroll
        for (int it = 0; it < HIST_IPT; it++) {
            const uint32_t idx = base + it * HIST_THREADS + tid;
            const bool valid = idx < m;
#pragma unroll
            for (int p = 0; p < P; p++) {
                const uint32_t d = (uint32_t)(k[it] >> (8 * p)) & 255u;
                // Lanes that share lane 0's digit are counted with one ballot and a single shared atomic instead
                // of up to 32 serialised ones (skewed digits: depth exponent byte, equal depths of one Gaussian).
                const uint32_t d0 = __shfl_sync(FULL, d, 0);
                const unsigned same = __ballot_sync(FULL, valid && d == d0);
                if ((threadIdx.x & 31) == 0) {
                    if (same) atomicAdd(&s_hist[p][d0], (uint32_t)__popc(same));
                } else if (valid && d != d0) {
                    atomicAdd(&s_hist[p][d], 1u);
                }
            }
        }
    }
    __syncthreads();
    for (int k = tid; k < P * RADIX; k += HIST_THREADS) {
        const uint32_t c = (&s_hist[0][0])[k];
        if (c) atomicAdd(&sc->hist[0][0] + k, c);
    }
}

// ------------------------------------------------------------------------------------------
// One Onesweep pass (replaces one hist.comp + sort.comp pair).
//
// Persistent kernel, two 256-thread CTAs per SM, tile = 4096 pairs (GSB_SORT_THREADS).
//  * TMA: the next tile's keys and payloads are fetched by cp.async.bulk (SASS UBLKCP) into the
//    second shared-memory buffer while the current tile is ranked and scattered; completion is an
//    mbarrier transaction count.  No registers are tied up by loads in flight.
//  * ranking: warp-striped.  u32 keys: every lane ORs its lane bit into a per-warp, per-digit mask
//    word in shared memory and reads the word back (= its peers); u64 keys (gsb_sort_pairs, off the
//    frame path): 8 ballots per 8-bit digit.  MATCH.ANY is avoided: its cost grows with the number of
//    distinct digits in the warp.  Per-warp digit counters in smem give the stable rank.
//  * the tile is permuted IN PLACE in shared memory (raw -> digit-sorted), so the global scatter
//    writes runs of consecutive addresses per digit (coalesced key / payload stores).
//  * chained scan: tile aggregate published right after ranking, decoupled look-back per digit
//    with LB_WINDOW predecessors in flight, done after the in-place permutation so the
//    predecessors' latency overlaps local work.
// ------------------------------------------------------------------------------------------
template <typename KeyT>
constexpr bool kMatchAtomic = GSB_SORT_MATCH_ATOMIC && sizeof(KeyT) == 4;
template <typename KeyT>
struct PassSmem {
    KeyT keys[2][SORT_TILE];            // double buffer: current / prefetch
    uint32_t vals[2][SORT_TILE];
    uint32_t whist[SORT_WARPS][RADIX];  // per-warp digit counters -> exclusive offsets across warps
    // per-warp lane masks per digit (atomicOr matching), always left zero; u32 keys only (the frame's instantiation)
    uint32_t match[kMatchAtomic<KeyT> ? SORT_WARPS : 1][RADIX];
    uint32_t bin_start[RADIX];          // exclusive scan of the tile's digit counts
    int32_t out_base[RADIX];            // global index of bin d's first element minus bin_start[d]
    uint32_t gexcl[RADIX];              // exclusive scan of the global histogram of this pass
    uint32_t warp_sums[SORT_WARPS];
    unsigned long long mbar[2];         // TMA completion barriers, one per buffer
    uint32_t tile[2];                   // ticket held by each buffer
};
template <typename KeyT>
constexpr int ctas_per_sm() {
    return SORT_THREADS >= 512 ? 1 : 2;
}

// digit -> counter slot: XOR swizzle so digits that differ by a multiple of 32 do not pile up in one bank
__device__ __forceinline__ uint32_t sw(uint32_t d) { return d ^ (d >> 5); }

// lanes of the warp holding the same 8-bit digit, by 8 ballots
__device__ __forceinline__ unsigned match_digit8(uint32_t d) {
    unsigned m = FULL;
#pragma unroll
    for (int b = 0; b < 8; b++) {
        const bool bit = (d >> b) & 1u;
        const unsigned vote = __ballot_sync(FULL, bit);
        m &= bit ? vote : ~vote;
    }
    return m;
}

// exclusive scan of one value per thread across the block (NW warps)
template <int NW>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* warp_sums) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(FULL, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    uint32_t before = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) {
        const uint32_t s = warp_sums[w];
        if (w < warp) before += s;
    }
    __syncthreads();
    return before + incl - v;
}

template <typename KeyT>
__global__ void __launch_bounds__(SORT_THREADS, ctas_per_sm<KeyT>())
    k_onesweep_pass(const KeyT* __restrict__ kin, const uint32_t* __restrict__ vin, KeyT* __restrict__ kout,
                    uint32_t* __restrict__ vout, const uint32_t* __restrict__ d_m, SortCtl* sc, int pass,
                    unsigned long long* status, uint32_t status_tiles, const uint32_t* __restrict__ d_epoch, uint32_t epoch_off,
                    uint2* __restrict__ ranges, uint32_t range_mask) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    PassSmem<KeyT>& S = *reinterpret_cast<PassSmem<KeyT>*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int shift = 8 * pass;
    const uint32_t m = *d_m;
    uint32_t num_tiles = (m + SORT_TILE - 1) / SORT_TILE;
    if (num_tiles > status_tiles) num_tiles = status_tiles;  // host sizes status for the arena capacity
    // the frame's epoch lives in device memory (bumped by k_frame_init) so a captured CUDA graph replays with fresh tags
    const uint32_t epoch = (d_epoch ? *d_epoch : 0u) + epoch_off;
    const unsigned long long epoch_hi = (unsigned long long)epoch << 32;

    auto fetch = [&](int buf) {  // thread 0: take the next ticket and start its TMA loads into `buf`
        const uint32_t t = atomicAdd(&sc->ticket[pass], 1u);
        S.tile[buf] = t;
        if (t < num_tiles && m - t * SORT_TILE >= (uint32_t)SORT_TILE) {  // full tile: TMA; the ragged last tile is loaded by the threads
            fence_proxy_async();  // generic-proxy accesses to `buf` are done (barrier) -> async proxy may write
            mbar_expect_tx(&S.mbar[buf], SORT_TILE * (sizeof(KeyT) + 4));
            tma_load(S.keys[buf], kin + (size_t)t * SORT_TILE, SORT_TILE * sizeof(KeyT), &S.mbar[buf]);
            tma_load(S.vals[buf], vin + (size_t)t * SORT_TILE, SORT_TILE * 4, &S.mbar[buf]);
        }
    };

    if (tid == 0) {
        mbar_init(&S.mbar[0], 1);
        mbar_init(&S.mbar[1], 1);
        mbar_fence_init();
    }
    // exclusive prefix of the global histogram of this digit (thread d <-> bin d)
    {
        const uint32_t c = tid < RADIX ? sc->hist[pass][tid] : 0u;
        const uint32_t ex = block_excl_scan<SORT_WARPS>(c, S.warp_sums);
        if (tid < RADIX) S.gexcl[tid] = ex;
    }
    if constexpr (kMatchAtomic<KeyT>)
        for (int k = tid; k < SORT_WARPS * RADIX; k += SORT_THREADS) (&S.match[0][0])[k] = 0u;
    if (tid == 0) fetch(0);
    __syncthreads();

    int cur = 0;
    uint32_t parity0 = 0u, parity1 = 0u;
    while (true) {
        const uint32_t tile = S.tile[cur];
        if (tile >= num_tiles) break;
        if (tid == 0) fetch(cur ^ 1);  // buffer cur^1 was released by the barrier that ended the previous iteration
        const uint32_t tile_base = tile * SORT_TILE;
        const uint32_t valid = min((uint32_t)SORT_TILE, m - tile_base);
        KeyT* sk = S.keys[cur];
        uint32_t* sv = S.vals[cur];

        // zero the per-warp counters
#pragma unroll
        for (int k = 0; k < SORT_WARPS * RADIX / SORT_THREADS; k++) (&S.whist[0][0])[k * SORT_THREADS + tid] = 0;
        if (valid == (uint32_t)SORT_TILE) {
            if (cur == 0) {
                mbar_wait(&S.mbar[0], parity0);
                parity0 ^= 1u;
            } else {
                mbar_wait(&S.mbar[1], parity1);
                parity1 ^= 1u;
            }
        } else {  // ragged last tile: plain loads, padded with the maximum key so the padding sorts last
#pragma unroll 4
            for (int it = 0; it < SORT_IPT; it++) {
                const uint32_t li = it * SORT_THREADS + tid;
                const bool ok = li < valid;
                sk[li] = ok ? __ldg(kin + tile_base + li) : key_max<KeyT>();
                sv[li] = ok ? __ldg(vin + tile_base + li) : 0u;
            }
        }
        __syncthreads();

        // ---- rank inside the warp (stable): warp-striped so (warp, round, lane) order == memory order ----
        const uint32_t wbase = warp * (32 * SORT_IPT) + lane;
        uint16_t rank[SORT_IPT];
        {
            uint32_t dg[SORT_IPT];
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) dg[it] = sw((uint32_t)(sk[wbase + it * 32] >> shift) & 255u);
            if constexpr (kMatchAtomic<KeyT>) {
            // Matching by shared-memory atomics: every lane ORs its lane bit into the warp's mask word of its digit,
            // reads the word back (= the lanes holding the same digit) and the lowest such lane clears it again.
            // ~10 instructions per pair instead of ~55 for eight ballots (the ranking was 40 % of the kernel).
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) {
                volatile uint32_t* mm = &S.match[warp][dg[it]];
                atomicOr(const_cast<uint32_t*>(mm), 1u << lane);
                __syncwarp();
                const unsigned peers = *mm;
                __syncwarp();
                const int leader = __ffs(peers) - 1;
                uint32_t prev = 0;
                if (lane == leader) {
                    *mm = 0u;
                    prev = S.whist[warp][dg[it]];
                    S.whist[warp][dg[it]] = prev + __popc(peers);
                }
                prev = __shfl_sync(FULL, prev, leader);
                rank[it] = (uint16_t)(prev + __popc(peers & ((1u << lane) - 1u)));
                __syncwarp();
            }
            } else {
            unsigned peers[SORT_IPT];
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) peers[it] = match_digit8(dg[it]);
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) {  // the counter update is the only serial part
                const int leader = __ffs(peers[it]) - 1;
                uint32_t prev = 0;
                if (lane == leader) {
                    prev = S.whist[warp][dg[it]];
                    S.whist[warp][dg[it]] = prev + __popc(peers[it]);
                }
                prev = __shfl_sync(FULL, prev, leader);
                rank[it] = (uint16_t)(prev + __popc(peers[it] & ((1u << lane) - 1u)));
                __syncwarp();
            }
            }
        }
        __syncthreads();

        // ---- per digit (thread d < 256): exclusive scan across warps, tile count, publish the aggregate ----
        uint32_t count = 0;
        if (tid < RADIX) {
#pragma unroll
            for (int w = 0; w < SORT_WARPS; w++) {
                const uint32_t c = S.whist[w][sw(tid)];
                S.whist[w][sw(tid)] = count;
                count += c;
            }
            // tile 0 has no predecessors: inclusive prefix right away
            st_volatile(status + (size_t)tile * RADIX + tid, epoch_hi | (tile == 0 ? LB_PREFIX : LB_AGG) | count);
        }
        const uint32_t bstart = block_excl_scan<SORT_WARPS>(count, S.warp_sums);  // threads >= 256 contribute 0
        if (tid < RADIX) S.bin_start[sw(tid)] = bstart;
        __syncthreads();

        // ---- permute the tile in place: raw order -> digit-sorted order ----
        {
            KeyT key[SORT_IPT];
            uint32_t val[SORT_IPT];
            uint32_t pos[SORT_IPT];
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) {
                key[it] = sk[wbase + it * 32];
                val[it] = sv[wbase + it * 32];
            }
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) {  // all lookups first (independent LDS), then all stores
                const uint32_t d = sw((uint32_t)(key[it] >> shift) & 255u);
                pos[it] = S.bin_start[d] + S.whist[warp][d] + rank[it];
            }
            __syncthreads();
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) {
                sk[pos[it]] = key[it];
                sv[pos[it]] = val[it];
            }
        }

        // ---- decoupled look-back for digit `tid`, LB_WINDOW predecessors in flight ----
        if (tid < RADIX) {
            uint32_t excl = 0;
            int t = (int)tile - 1;
            bool done = tile == 0;
            while (!done) {
                unsigned long long w[LB_WINDOW];
#pragma unroll
                for (int j = 0; j < LB_WINDOW; j++)
                    w[j] = (t - j >= 0) ? ld_volatile(status + (size_t)(t - j) * RADIX + tid) : (epoch_hi | LB_PREFIX);
#pragma unroll
                for (int j = 0; j < LB_WINDOW; j++) {
                    if (done) break;
                    const uint32_t lo = (uint32_t)w[j];
                    if ((w[j] >> 32) != epoch) break;  // not yet published in this pass: poll again from here
                    excl += lo & LB_COUNT;
                    --t;
                    if (lo & LB_PREFIX) done = true;
                }
            }
            if (tile != 0) st_volatile(status + (size_t)tile * RADIX + tid, epoch_hi | LB_PREFIX | (excl + count));
            S.out_base[sw(tid)] = (int32_t)(S.gexcl[tid] + excl) - (int32_t)bstart;
        }
        __syncthreads();

        // ---- coalesced global scatter: consecutive idx of one digit -> consecutive addresses ----
        {
            KeyT k[SORT_IPT];
            uint32_t v[SORT_IPT];
            int32_t g[SORT_IPT];
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) {
                k[it] = sk[it * SORT_THREADS + tid];
                v[it] = sv[it * SORT_THREADS + tid];
            }
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++)
                g[it] = S.out_base[sw((uint32_t)(k[it] >> shift) & 255u)] + (int32_t)(it * SORT_THREADS + tid);
#pragma unroll
            for (int it = 0; it < SORT_IPT; it++) {
                if ((uint32_t)(it * SORT_THREADS + tid) < valid) {
                    if (kout != nullptr) kout[g[it]] = k[it];  // null: nobody reads the fully sorted keys (last pass)
                    vout[g[it]] = v[it];
                }
            }
            // Tile ranges fused into the LAST pass (tile_boundary.comp:22-50): inside one digit bin the tile keeps its
            // input order, which is sorted by the lower digits, so equal keys are adjacent in the shared-memory
            // buffer and land on consecutive global positions.  Every maximal run reports its first position with
            // atomicMin on ranges[key].x and its end with atomicMin on ranges[key].y = ~end (both fields start at
            // 0xFFFFFFFF); runs split across tiles merge by the min.
            if (ranges != nullptr) {
                if constexpr (sizeof(KeyT) == 4) {
#pragma unroll
                    for (int it = 0; it < SORT_IPT; it++) {
                        const uint32_t idx = (uint32_t)(it * SORT_THREADS + tid);
                        if (idx < valid) {
                            // range_mask: the bits that were sorted (a key may carry a payload above them: coarse bins)
                            const uint32_t key = (uint32_t)k[it] & range_mask;
                            if (idx == 0 || ((uint32_t)sk[idx - 1] & range_mask) != key) atomicMin(&ranges[key].x, (uint32_t)g[it]);
                            if (idx == valid - 1 || ((uint32_t)sk[idx + 1] & range_mask) != key) atomicMin(&ranges[key].y, ~((uint32_t)g[it] + 1u));
                        }
                    }
                }
            }
        }
        __syncthreads();  // buffer `cur` may now be refilled by TMA
        cur ^= 1;
    }
}

template <typename KeyT>
cudaError_t launch_hist(const KeyT* keys, const SortParams& p, uint32_t P, uint32_t blocks, cudaStream_t s) {
    switch (P) {
        case 1: k_sort_hist<KeyT, 1><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
        case 2: k_sort_hist<KeyT, 2><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
        case 3: k_sort_hist<KeyT, 3><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
        case 4: k_sort_hist<KeyT, 4><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
        default:
            if constexpr (sizeof(KeyT) == 8) {
                switch (P) {
                    case 5: k_sort_hist<KeyT, 5><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
                    case 6: k_sort_hist<KeyT, 6><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
                    case 7: k_sort_hist<KeyT, 7><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
                    default: k_sort_hist<KeyT, 8><<<blocks, HIST_THREADS, 0, s>>>(keys, p.d_m, p.sc); break;
                }
            } else {
                return cudaErrorInvalidValue;
            }
    }
    return cudaGetLastError();
}

template <typename KeyT>
cudaError_t launch_sort_t(const SortParams& p, uint32_t P, cudaStream_t s) {
    const uint32_t hint = p.m_hint ? p.m_hint : 1;
    KeyT* keys[2] = {static_cast<KeyT*>(p.keys[0]), static_cast<KeyT*>(p.keys[1])};
    {  // histogram: persistent grid-stride, at most 2 CTAs per SM
        uint32_t blocks = (hint + HIST_TILE - 1) / HIST_TILE;
        const uint32_t cap = (uint32_t)p.num_sms * GSB_HIST_CTAS;
        if (blocks > cap) blocks = cap;
        if (blocks == 0) blocks = 1;
        cudaError_t e = launch_hist<KeyT>(keys[0], p, P, blocks, s);
        if (e != cudaSuccess) return e;
        if (p.events && (e = cudaEventRecord(p.events[0], s)) != cudaSuccess) return e;
    }
    const size_t smem = sizeof(PassSmem<KeyT>);  // opt-in done once by sort_prepare()
    uint32_t blocks = (hint + SORT_TILE - 1) / SORT_TILE;
    const uint32_t cap = (uint32_t)p.num_sms * ctas_per_sm<KeyT>();  // persistent CTAs; ticket loop: any grid size is correct
    if (blocks > cap) blocks = cap;
    if (blocks == 0) blocks = 1;
    for (uint32_t pass = 0; pass < P; pass++) {
        const int src = pass & 1, dst = src ^ 1;
        KeyT* kout = (pass + 1 == P && p.discard_sorted_keys) ? nullptr : keys[dst];
        k_onesweep_pass<KeyT><<<blocks, SORT_THREADS, smem, s>>>(keys[src], p.vals[src], kout, p.vals[dst], p.d_m, p.sc,
                                                                 (int)pass, p.status, p.status_tiles, p.d_epoch, p.epoch_base + pass,
                                                                 pass + 1 == P ? p.ranges : nullptr, p.range_key_mask ? p.range_key_mask : 0xffffffffu);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        if (p.events && (e = cudaEventRecord(p.events[1 + pass], s)) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace

uint32_t sort_tile_items() { return SORT_TILE; }

cudaError_t sort_prepare() {
    cudaError_t e = cudaFuncSetAttribute(k_onesweep_pass<uint32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)sizeof(PassSmem<uint32_t>));
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k_onesweep_pass<unsigned long long>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)sizeof(PassSmem<unsigned long long>));
}

cudaError_t launch_sort(const SortParams& p, uint32_t* passes, cudaStream_t s) {
    const uint32_t P = (p.key_bits + 7) / 8;
    *passes = P;
    if (P == 0) return cudaSuccess;
    if (p.key_bytes == 4 && P <= 4) return launch_sort_t<uint32_t>(p, P, s);
    if (p.key_bytes == 8 && P <= 8) return launch_sort_t<unsigned long long>(p, P, s);
    return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------------
// Tile ranges (replaces fillBuffer(0) + tile_boundary.comp:22-50, Renderer.cpp:633-652).
// Encoding: ranges[t] = (start, ~end), untouched = (0xFFFFFFFF, 0xFFFFFFFF) = empty.  They are produced by the
// last Onesweep pass of the instance sort (see k_onesweep_pass); the 0xFF fill is part of k_frame_init (gsb_api.cu); this file provides the
// degenerate case of a single tile (no tile-id bits to sort, hence no pass).
// ------------------------------------------------------------------------------------------
namespace {
__global__ void k_ranges_single_tile(const uint32_t* __restrict__ d_m, uint2* __restrict__ ranges) {
    const uint32_t m = *d_m;
    if (m) ranges[0] = make_uint2(0u, ~m);
}
}  // namespace

cudaError_t launch_ranges_single_tile(const uint32_t* d_m, uint2* ranges, cudaStream_t s) {
    k_ranges_single_tile<<<1, 1, 0, s>>>(d_m, ranges);
    return cudaGetLastError();
}

}  // namespace gsb
