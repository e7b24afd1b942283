// gsb_shard.cu -- one frame sharded over the GPUs of an NVSwitch domain (SURVEY 8e; no reference counterpart: the
// reference is single-GPU).
//
// Sharding is two-dimensional:
//   * the SCENE is sharded by Gaussian index: rank r holds slice [r S, (r + 1) S), S = ceil(N / G), and projects only
//     that slice (k_project is the frame's bandwidth-heaviest kernel; replicating it caps the speed-up at ~2x);
//   * the FRAME is sharded by tile rows: rank d blends band d (equal-height bands of R = ceil(tiles_y / G) tile rows).
// Between the two sits ONE exchange over peer memory, fused into the kernels on either side instead of a collective:
//   k_project (ROUTED, gsb_preprocess.cu) every cull survivor of the local slice is delivered straight from the projection's
//             registers -- its 64-B record with the AABB clipped to the band, and its depth key -- into the exchange buffers
//             of every rank whose band its AABB touches, by plain stores into peer-mapped memory (NVLink).  Slots are
//             deterministic: rank d's buffer is divided into G regions of S slots, region s receives rank s's survivors in
//             Gaussian-index order (G simultaneous decoupled look-back scans on the source), so the band's survivor list is
//             in global index order exactly like k_project's compaction on one GPU, and the band's pixels are bit-identical
//             to the single-GPU frame, without a separate routing pass over the compacted records.
//   k_blend   stores its band straight into the whole-frame buffer of EVERY rank (the all-gather of the framebuffer,
//             done by the producer's stores; GSB_SHARD_GATHER=nccl replaces it by one in-place ncclAllGather).
// Cross-GPU ordering uses mailbox words in peer memory: `routed` (+ counts: a rank's records for my band have landed) and
// `framed` (+ overflow flag: its band of the framebuffer has landed).  A signal is a one-warp kernel after the producing kernel, a wait a one-warp kernel that
// spins on acquire loads (bounded: a dead peer raises an error instead of hanging the GPU).  Exchange and frame
// buffers are double-buffered by frame parity; no "may I overwrite your buffers" handshake is needed: a rank writes into
// buffers of parity f & 1 in frame f, their last readers ran in frame f - 2, and every rank waited for every rank's
// `framed` of frame f - 2 (which follows that rank's last read) before it left frame f - 2.
//
// Two ways to form the group, same kernels:
//   gsb_group_create      one process drives all GPUs (SURVEY 8b `gs_create_sharded(int ndev, ...)`); peers are plain
//                         device pointers (cudaDeviceEnablePeerAccess).  The same device may be listed several times,
//                         which is how the single-GPU test suite exercises the whole protocol.
//   gsb_create_sharded    one process per GPU (torchrun / MPI): NCCL (dlopen'ed, only here) bootstraps the group and
//                         carries the cudaIpc handles of the windows; nothing of the frame path goes through NCCL
//                         unless GSB_SHARD_GATHER=nccl.
#include <dlfcn.h>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <vector>

#include "gsb_ctx.cuh"

using namespace gsb;

namespace gsb {

struct Mailbox {  // in every rank's window; every word has exactly one writer (peer p writes index p)
    uint32_t reserved[GSB_MAX_SHARDS];
    uint32_t routed[GSB_MAX_SHARDS];
    uint32_t framed[GSB_MAX_SHARDS];
    uint32_t count[2][GSB_MAX_SHARDS];     // [parity][source]: records delivered for my band
    uint32_t overflow[2][GSB_MAX_SHARDS];  // [parity][rank]: that rank's instance arena overflowed in this frame
    uint32_t error;                        // set locally: a wait timed out
    uint32_t pad[7];
};
static_assert(sizeof(Mailbox) == 256, "mailbox layout");

struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

struct ShardState {
    int rank = 0, world = 1;
    uint64_t n_total = 0, slice = 0, cap = 0;  // cap = world * slice (slots of an exchange buffer)
    uint32_t frame = 0;
    bool gather_nccl = false;

    // window: everything peers write into.  One allocation, identical layout on every rank.
    unsigned char* window = nullptr;
    size_t window_bytes = 0, off_recs[2] = {}, off_dkeys[2] = {}, off_frame[2] = {};
    size_t frame_bytes = 0;     // one padded whole frame (world * R * 16 rows)
    uint32_t frame_w = 0, frame_h = 0;
    int frame_fmt = -1;
    unsigned char* peer_window[GSB_MAX_SHARDS] = {};  // this rank's view of every rank's window (own included)

    // destination-side dense survivor arrays (the plain context's are the source-side ones)
    DevArray<uint32_t> dkeys_d[2];
    DevArray<uint32_t> dvals_d[2];
    DevArray<unsigned long long> emit_status_d;
    DevArray<uint32_t> route_status;   // [chunks of the slice][GSB_MAX_SHARDS]
    Mailbox* mailbox_host = nullptr;   // pinned copy of the own mailbox (overflow flags, error) at the end of a frame
    uint32_t last_parity = 0;

    // group plumbing
    struct gsb_group* group = nullptr;  // in-process group (owns the contexts), or
    NcclApi nccl;                       // process-per-GPU
    ncclComm_t comm = nullptr;
    bool ipc_open[GSB_MAX_SHARDS] = {};

    Mailbox* mailbox(int p) const { return reinterpret_cast<Mailbox*>(peer_window[p]); }
    float4* recs_x(int p, int par) const { return reinterpret_cast<float4*>(peer_window[p] + off_recs[par]); }
    uint32_t* dkeys_x(int p, int par) const { return reinterpret_cast<uint32_t*>(peer_window[p] + off_dkeys[par]); }
    void* frame_x(int p, int par) const { return peer_window[p] + off_frame[par]; }
};

}  // namespace gsb

struct gsb_group {
    std::vector<gsb_ctx*> ctx;
    std::string err;
};

namespace {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_vol(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }

struct PeerWords {  // one mailbox word per rank
    uint32_t* p[GSB_MAX_SHARDS];
};

// Signal: lane p publishes `value` (and, before it, up to two payload words) into peer p's mailbox.  Launched after the
// kernel whose (remote) writes it announces; the release store orders it after them for the acquiring reader.
__global__ void k_shard_signal(PeerWords flag, uint32_t value, int world, PeerWords payload, const uint32_t* payload_src, int payload_per_peer) {
    const int p = threadIdx.x;
    if (p >= world) return;
    if (payload_src != nullptr) *payload.p[p] = payload_src[payload_per_peer ? p : 0];
    __threadfence_system();
    st_release_sys(flag.p[p], value);
}

// Wait: lane p spins until peer p's word in the OWN mailbox reaches `value` (frame numbers, compared modulo 2^32).
__global__ void k_shard_wait(const uint32_t* words, uint32_t value, int world, uint32_t* error, long long timeout_cycles) {
    const int p = threadIdx.x;
    if (p < world) {
        const long long t0 = clock64();
        while ((int32_t)(ld_acquire_sys(words + p) - value) < 0) {
            if (clock64() - t0 > timeout_cycles) {
                atomicExch(error, 1u + (uint32_t)p);
                break;
            }
            __nanosleep(40);
        }
    }
    __syncwarp();
    __threadfence_system();
}

struct GatherParams {
    const uint32_t* counts;  // own mailbox: count[parity][source]
    const uint32_t* dkeys_x;
    uint32_t slice;
    int world;
    uint32_t* dkeys;
    uint32_t* dvals;
    Control* ctl;
};

// Destination side: the G regions become the dense (depth key, compact id) list of the Gaussian-level sort, in
// (source rank, slot) = global Gaussian-index order; compact id = slot in the (sparse) exchange buffers.
__global__ void k_shard_gather(const __grid_constant__ GatherParams P) {
    uint32_t prefix[GSB_MAX_SHARDS + 1];
    prefix[0] = 0;
#pragma unroll
    for (int p = 0; p < GSB_MAX_SHARDS; p++) prefix[p + 1] = prefix[p] + (p < P.world ? min(ld_vol(P.counts + p), P.slice) : 0u);
    const uint32_t total = prefix[GSB_MAX_SHARDS];
    if (blockIdx.x == 0 && threadIdx.x == 0) P.ctl->num_visible = total;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        int p = 0;
#pragma unroll
        for (int q = 1; q < GSB_MAX_SHARDS; q++)
            if (i >= prefix[q]) p = q;
        const uint32_t cid = (uint32_t)p * P.slice + (i - prefix[p]);
        P.dkeys[i] = P.dkeys_x[cid];
        P.dvals[i] = cid;
    }
}

int group_fail(gsb_group* g, int code, const std::string& what) {
    if (g) g->err = what;
    return code;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// (Re)compute the window layout for the current scene / frame size.  Identical on every rank by construction.
size_t layout_window(ShardState* sh) {
    size_t off = sizeof(Mailbox);
    for (int par = 0; par < 2; par++) {
        off = align_up(off, 256);
        sh->off_recs[par] = off;
        off += sh->cap * GSB_REC_F4 * sizeof(float4);
    }
    for (int par = 0; par < 2; par++) {
        off = align_up(off, 256);
        sh->off_dkeys[par] = off;
        off += sh->cap * sizeof(uint32_t);
    }
    for (int par = 0; par < 2; par++) {
        off = align_up(off, 256);
        sh->off_frame[par] = off;
        off += sh->frame_bytes;
    }
    return align_up(off, 256);
}

void close_peers(gsb_ctx* ctx) {
    ShardState* sh = ctx->shard;
    for (int p = 0; p < sh->world; p++) {
        if (sh->ipc_open[p]) cudaIpcCloseMemHandle(sh->peer_window[p]);
        sh->ipc_open[p] = false;
        sh->peer_window[p] = nullptr;
    }
}

// Free + allocate this rank's window for the current layout (no exchange yet).
int realloc_window(gsb_ctx* ctx) {
    ShardState* sh = ctx->shard;
    if (sh->window) cudaFree(sh->window);
    sh->window = nullptr;
    sh->window_bytes = layout_window(sh);
    CK(cudaMalloc(reinterpret_cast<void**>(&sh->window), sh->window_bytes));
    CK(cudaMemset(sh->window, 0, sizeof(Mailbox)));
    CK(cudaDeviceSynchronize());
    sh->frame = 0;
    ctx->alloc_gen++;
    return GSB_OK;
}

// process-per-GPU: all ranks call this together after realloc_window; NCCL carries the IPC handles
int exchange_windows_ipc(gsb_ctx* ctx) {
    ShardState* sh = ctx->shard;
    cudaIpcMemHandle_t mine;
    CK(cudaIpcGetMemHandle(&mine, sh->window));
    cudaIpcMemHandle_t* d_all = nullptr;
    CK(cudaMalloc(reinterpret_cast<void**>(&d_all), sizeof(cudaIpcMemHandle_t) * sh->world));
    CK(cudaMemcpy(d_all + sh->rank, &mine, sizeof mine, cudaMemcpyHostToDevice));
    ncclResult_t nr = sh->nccl.AllGather(d_all + sh->rank, d_all, sizeof(cudaIpcMemHandle_t), ncclChar, sh->comm, ctx->stream);
    if (nr != ncclSuccess) {
        cudaFree(d_all);
        return fail(ctx, GSB_ERR_CUDA, (std::string("ncclAllGather: ") + sh->nccl.GetErrorString(nr)).c_str());
    }
    CK(cudaStreamSynchronize(ctx->stream));
    std::vector<cudaIpcMemHandle_t> all(sh->world);
    CK(cudaMemcpy(all.data(), d_all, sizeof(cudaIpcMemHandle_t) * sh->world, cudaMemcpyDeviceToHost));
    cudaFree(d_all);
    for (int p = 0; p < sh->world; p++) {
        if (p == sh->rank) {
            sh->peer_window[p] = sh->window;
            continue;
        }
        void* ptr = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&ptr, all[p], cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return fail(ctx, GSB_ERR_CUDA, "cudaIpcOpenMemHandle (peer memory over NVLink is required for frame sharding)", e);
        sh->peer_window[p] = static_cast<unsigned char*>(ptr);
        sh->ipc_open[p] = true;
    }
    return GSB_OK;
}

// a tiny all-gather doubles as the barrier between "everyone stopped using the old windows" and "free them"
int barrier_ipc(gsb_ctx* ctx) {
    ShardState* sh = ctx->shard;
    unsigned char* d = nullptr;
    CK(cudaMalloc(reinterpret_cast<void**>(&d), (size_t)sh->world));
    ncclResult_t nr = sh->nccl.AllGather(d + sh->rank, d, 1, ncclChar, sh->comm, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    cudaFree(d);
    if (nr != ncclSuccess) return fail(ctx, GSB_ERR_CUDA, (std::string("ncclAllGather: ") + sh->nccl.GetErrorString(nr)).c_str());
    if (e != cudaSuccess) return fail(ctx, GSB_ERR_CUDA, "barrier", e);
    return GSB_OK;
}

// Make the windows match (scene, frame size): collective.  In-process groups are handled by the group code.
int ensure_windows_ipc(gsb_ctx* ctx) {
    CK(cudaStreamSynchronize(ctx->stream));
    int rc = barrier_ipc(ctx);
    if (rc != GSB_OK) return rc;
    close_peers(ctx);
    rc = barrier_ipc(ctx);
    if (rc != GSB_OK) return rc;
    rc = realloc_window(ctx);
    if (rc != GSB_OK) return rc;
    return exchange_windows_ipc(ctx);
}

int ensure_windows_group(gsb_group* g) {
    for (gsb_ctx* c : g->ctx) {
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
    }
    for (gsb_ctx* c : g->ctx) {
        cudaSetDevice(c->device);
        int rc = realloc_window(c);
        if (rc != GSB_OK) return group_fail(g, rc, c->err);
    }
    for (gsb_ctx* c : g->ctx)
        for (size_t p = 0; p < g->ctx.size(); p++) c->shard->peer_window[p] = g->ctx[p]->shard->window;
    return GSB_OK;
}

bool frame_layout_changed(ShardState* sh, uint32_t W, uint32_t H, int fmt, size_t* bytes) {
    const uint32_t tiles_y = (H + GSB_TILE - 1) / GSB_TILE;
    const uint32_t R = (tiles_y + sh->world - 1) / sh->world;
    *bytes = align_up((size_t)sh->world * R * GSB_TILE * W * bytes_per_pixel(fmt), 256);
    return sh->window == nullptr || *bytes != sh->frame_bytes || W != sh->frame_w || H != sh->frame_h || fmt != sh->frame_fmt;
}

PeerWords words_of(ShardState* sh, size_t field_offset, int index_is_rank, int par_offset_words) {
    PeerWords w{};
    for (int p = 0; p < sh->world; p++)
        w.p[p] = reinterpret_cast<uint32_t*>(reinterpret_cast<unsigned char*>(sh->mailbox(p)) + field_offset) + par_offset_words +
                 (index_is_rank ? sh->rank : 0);
    return w;
}

constexpr long long WAIT_TIMEOUT_CYCLES = 6000000000ll;  // ~3 s at 1.9 GHz: a dead peer becomes an error, not a hung GPU

// One sharded frame is enqueued in three phases; a phase ends where the stream would next WAIT for the other ranks:
//   1  frame start, k_project over the local slice (its survivors are stored straight into peer memory), signal `routed`
//   2  wait `routed`, gather, depth sort / emission / tile sort, blend (peer stores), signal `framed`
//   3  wait `framed`, mailbox + stats copy, completion event
// A process that drives ONE rank enqueues 1-3 back to back.  A group that drives every rank from one host thread enqueues
// phase k of EVERY rank before phase k + 1 of any: each wait is then enqueued after all the signals it depends on, so a
// host-side call that blocks until another device drains (first-use module loading, cudaMalloc / cudaFree with peer
// mappings) can never sit between a spinning wait and the signal that would release it.  (Enqueuing rank 0's
// whole frame first can leave it spinning in k_shard_wait until the 3 s timeout while rank 1's first launches are stuck
// behind it.)
struct ShardFrame {
    gsb_uniforms ubo;
    int fmt = 0;
    cudaStream_t stream = nullptr;
    uint32_t f = 0, R = 0, tiles_y = 0, rb = 0, re = 0;
    int par = 0;
    FramePlan fp{};
};

int enqueue_sharded_phase(gsb_ctx* ctx, ShardFrame& F, int phase) {
    ShardState* sh = ctx->shard;
    const int G = sh->world, r = sh->rank;
    cudaStream_t stream = F.stream;
    Mailbox* mb = sh->mailbox(r);
    if (phase == 1) {
        const gsb_uniforms* ubo = &F.ubo;
        const uint32_t H = ubo->height;
        F.tiles_y = (H + GSB_TILE - 1) / GSB_TILE;
        F.R = (F.tiles_y + G - 1) / G;
        F.rb = std::min(F.tiles_y, (uint32_t)r * F.R);
        F.re = std::min(F.tiles_y, F.rb + F.R);
        F.f = ++sh->frame;
        F.par = (int)(F.f & 1u);
        sh->last_parity = (uint32_t)F.par;
        // the dense destination-side arrays and the exchange buffers of this parity take the place of the plain context's
        // survivor arrays for the middle of the frame and the blend
        const uint64_t n_local = ctx->n;
        int rc = plan_frame(ctx, ubo, F.rb, F.re, stream, &F.fp);
        if (rc != GSB_OK) return rc;
        F.fp.nv_q = std::min<uint32_t>(quantise_hint(ctx->nv_hint ? ctx->nv_hint : sh->cap), quantise_hint(sh->cap));
        const uint32_t chunks_local = (uint32_t)((n_local + 255) / 256), chunks_cap = (uint32_t)((sh->cap + 255) / 256);
        // project_status covers the local slice, emit_status_d the band's survivor list (up to `cap` slots)
        CK(launch_frame_init(ctx->ctl, ctx->project_status, std::max(chunks_local, 1u), sh->emit_status_d, std::max(chunks_cap, 1u), ctx->ranges,
                             F.fp.T, stream, sh->route_status, std::max(chunks_local, 1u) * GSB_MAX_SHARDS));
        if (ctx->timers) CK(cudaEventRecord(ctx->ev[0], stream));
        // ---- k_project over the local slice (whole frame, no band clip) delivers every survivor straight into the exchange
        // buffers (parity f & 1: last read in frame f - 2, see the header) of the ranks whose band it touches, and announces it ----
        ProjectParams pp = project_params(ctx, F.ubo, 0, F.tiles_y);  // its recs, dkeys and dvals are unused by the routed kernel
        pp.index_base = (uint32_t)((uint64_t)r * sh->slice);
        pp.route_world = G;
        pp.band_rows = std::max(F.R, 1u);
        pp.route_status = sh->route_status;
        for (int d = 0; d < G; d++) {
            pp.route_dst_recs[d] = sh->recs_x(d, F.par) + (size_t)r * sh->slice * GSB_REC_F4;
            pp.route_dst_dkeys[d] = sh->dkeys_x(d, F.par) + (size_t)r * sh->slice;
        }
        CK(launch_project(pp, false, stream));
        k_shard_signal<<<1, 32, 0, stream>>>(words_of(sh, offsetof(Mailbox, routed), 1, 0), F.f, G,
                                             words_of(sh, offsetof(Mailbox, count), 1, F.par * GSB_MAX_SHARDS), ctx->ctl->route_total, 1);
        CK(cudaGetLastError());
        return GSB_OK;
    }
    if (phase == 2) {
        k_shard_wait<<<1, 32, 0, stream>>>(mb->routed, F.f, G, &mb->error, WAIT_TIMEOUT_CYCLES);
        if (ctx->timers) CK(cudaEventRecord(ctx->ev[1], stream));  // "preprocess" = projection + exchange
        GatherParams gp{};
        gp.counts = mb->count[F.par];
        gp.dkeys_x = sh->dkeys_x(r, F.par);
        gp.slice = (uint32_t)sh->slice;
        gp.world = G;
        gp.dkeys = sh->dkeys_d[0];
        gp.dvals = sh->dvals_d[0];
        gp.ctl = ctx->ctl;
        k_shard_gather<<<std::min<uint32_t>((F.fp.nv_q + 255) / 256, (uint32_t)ctx->num_sms * 8u), 256, 0, stream>>>(gp);
        CK(cudaGetLastError());

        // ---- the middle of the frame and the blend run on the band's survivors: this parity's exchange buffers and the
        // destination-side arrays ----
        const Survivors sv{sh->recs_x(r, F.par), {sh->dkeys_d[0], sh->dkeys_d[1]}, {sh->dvals_d[0], sh->dvals_d[1]}, sh->emit_status_d};
        int rc;
        if (ctx->use_graph && !ctx->timers && !ctx->debug) rc = launch_middle_graph(ctx, F.fp, sv, stream);
        else rc = enqueue_middle(ctx, F.fp, sv, stream, ctx->timers);
        if (rc != GSB_OK) return rc;

        const size_t pitch = (size_t)F.ubo.width * bytes_per_pixel(F.fmt);
        void* frames[GSB_MAX_SHARDS];
        for (int p = 0; p < G; p++) frames[p] = sh->frame_x(p, F.par);
        if (F.rb < F.re) {
            if (sh->gather_nccl) rc = enqueue_blend(ctx, F.fp, sv, F.rb, F.re, nullptr, pitch, F.fmt, stream, &frames[r], 1);
            else rc = enqueue_blend(ctx, F.fp, sv, F.rb, F.re, nullptr, pitch, F.fmt, stream, frames, G);
            if (rc != GSB_OK) return rc;
        }
        if (sh->gather_nccl && sh->comm) {  // the baseline: one in-place all-gather of the equal-height bands
            const size_t band_bytes = (size_t)F.R * GSB_TILE * pitch;
            unsigned char* fb = static_cast<unsigned char*>(frames[r]);
            ncclResult_t nr = sh->nccl.AllGather(fb + (size_t)r * band_bytes, fb, band_bytes, ncclChar, sh->comm, stream);
            if (nr != ncclSuccess) return fail(ctx, GSB_ERR_CUDA, (std::string("ncclAllGather: ") + sh->nccl.GetErrorString(nr)).c_str());
        }
        if (ctx->timers) CK(cudaEventRecord(ctx->ev[7], stream));  // end of this rank's own blend (gsb_stats::shard_blend_ms)
        // S3: my band (and my overflow flag) has landed everywhere
        k_shard_signal<<<1, 32, 0, stream>>>(words_of(sh, offsetof(Mailbox, framed), 1, 0), F.f, G,
                                             words_of(sh, offsetof(Mailbox, overflow), 1, F.par * GSB_MAX_SHARDS), &ctx->ctl->overflow, 0);
        CK(cudaGetLastError());
        return GSB_OK;
    }
    // phase 3: wait for everyone's band
    k_shard_wait<<<1, 32, 0, stream>>>(mb->framed, F.f, G, &mb->error, WAIT_TIMEOUT_CYCLES);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(sh->mailbox_host, mb, sizeof(Mailbox), cudaMemcpyDeviceToHost, stream));
    return enqueue_tail(ctx, F.fp, F.ubo, stream);
}

// Enqueue one sharded frame of ONE rank on `stream`.  Collective: every rank enqueues the same frame; never blocks the host.
int enqueue_sharded(gsb_ctx* ctx, const gsb_uniforms* ubo, int fmt, cudaStream_t stream) {
    ShardFrame F;
    F.ubo = *ubo;
    F.fmt = fmt;
    F.stream = stream;
    for (int phase = 1; phase <= 3; phase++) {
        int rc = enqueue_sharded_phase(ctx, F, phase);
        if (rc != GSB_OK) return rc;
    }
    return GSB_OK;
}

// after wait_frame(): peer timeout? any rank's arena overflowed (every rank sees the same flags -> same decision)?
int sharded_frame_status(gsb_ctx* ctx, bool* any_overflow) {
    ShardState* sh = ctx->shard;
    *any_overflow = false;
    if (sh->mailbox_host->error) {
        char msg[96];
        snprintf(msg, sizeof msg, "frame sharding: rank %u did not arrive within the timeout", sh->mailbox_host->error - 1u);
        cudaMemsetAsync(&sh->mailbox(sh->rank)->error, 0, sizeof(uint32_t), ctx->stream);
        cudaStreamSynchronize(ctx->stream);
        return fail(ctx, GSB_ERR_CUDA, msg);
    }
    for (int p = 0; p < sh->world; p++)
        if (sh->mailbox_host->overflow[sh->last_parity][p]) *any_overflow = true;
    return GSB_OK;
}

int copy_frame_out(gsb_ctx* ctx, const gsb_uniforms* ubo, void* out, size_t pitch, gsb_memory out_mem, int fmt, cudaStream_t s) {
    ShardState* sh = ctx->shard;
    const size_t tight = (size_t)ubo->width * bytes_per_pixel(fmt);
    if (pitch == 0) pitch = tight;
    CK(cudaMemcpy2DAsync(out, pitch, sh->frame_x(sh->rank, (int)sh->last_parity), tight, tight, ubo->height,
                         out_mem == GSB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, s));
    if (out_mem == GSB_MEM_HOST) CK(cudaStreamSynchronize(s));
    return GSB_OK;
}

int attach_shard(gsb_ctx* ctx, int rank, int world) {
    ShardState* sh = new (std::nothrow) ShardState();
    if (!sh) return GSB_ERR_OOM;
    sh->rank = rank;
    sh->world = world;
    if (const char* v = getenv("GSB_SHARD_GATHER")) sh->gather_nccl = strcmp(v, "nccl") == 0;
    ctx->shard = sh;
    CK(cudaMallocHost(reinterpret_cast<void**>(&sh->mailbox_host), sizeof(Mailbox)));
    memset(sh->mailbox_host, 0, sizeof(Mailbox));
    return GSB_OK;
}

// slice upload + destination-side arrays.  `vertices` = this rank's slice.
int upload_slice(gsb_ctx* ctx, const float* vertices, uint64_t n_total, gsb_memory mem) {
    ShardState* sh = ctx->shard;
    if (n_total >= (1ull << 30)) return fail(ctx, GSB_ERR_INVALID, "scene limited to 2^30 - 1 Gaussians");
    sh->n_total = n_total;
    sh->slice = std::max<uint64_t>((n_total + sh->world - 1) / sh->world, 1);
    sh->cap = sh->slice * sh->world;
    const uint64_t first = std::min(n_total, (uint64_t)sh->rank * sh->slice), count = std::min(sh->slice, n_total - first);
    int rc = gsb_scene_upload(ctx, count ? vertices : nullptr, count, mem);
    if (rc != GSB_OK) return rc;
    CK(sh->dkeys_d[0].grow(sh->cap));
    CK(sh->dkeys_d[1].grow(sh->cap));
    CK(sh->dvals_d[0].grow(sh->cap));
    CK(sh->dvals_d[1].grow(sh->cap));
    CK(sh->emit_status_d.grow((sh->cap + 255) / 256));
    CK(sh->route_status.grow(((sh->slice + 255) / 256) * GSB_MAX_SHARDS));
    ctx->alloc_gen++;
    rc = ensure_sort_status(ctx, std::max<uint64_t>(sh->cap, ctx->capacity));
    if (rc != GSB_OK) return rc;
    if (ctx->capacity < sh->slice * 2) rc = ensure_arena(ctx, std::max<uint64_t>(sh->slice * 2, 1024));
    sh->frame_bytes = 0;  // forces a window (re)allocation at the next render
    sh->frame_w = sh->frame_h = 0;
    if (sh->window) cudaFree(sh->window);
    sh->window = nullptr;
    return rc;
}

int check_sharded_args(gsb_ctx* ctx, const gsb_uniforms* ubo, int fmt) {
    if (!ctx) return GSB_ERR_INVALID;
    if (!ctx->shard) return fail(ctx, GSB_ERR_INVALID, "not a sharded context (gsb_create_sharded / gsb_group_create)");
    if (!ubo) return fail(ctx, GSB_ERR_INVALID, "null argument");
    if (!ctx->shard->n_total || !ctx->pos_op) return fail(ctx, GSB_ERR_NO_SCENE, "no scene uploaded");
    const int rc = check_image(ctx, ubo, fmt);
    if (rc != GSB_OK) return rc;
    if (ctx->debug) return fail(ctx, GSB_ERR_INVALID, "gsb_set_debug is not available on a sharded context");
    return GSB_OK;
}

bool load_nccl(NcclApi* a, std::string* why) {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
        a->lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
        if (a->lib) break;
    }
    if (!a->lib) {
        *why = std::string("libnccl.so.2 not found: ") + dlerror();
        return false;
    }
    a->GetUniqueId = reinterpret_cast<decltype(a->GetUniqueId)>(dlsym(a->lib, "ncclGetUniqueId"));
    a->CommInitRank = reinterpret_cast<decltype(a->CommInitRank)>(dlsym(a->lib, "ncclCommInitRank"));
    a->CommDestroy = reinterpret_cast<decltype(a->CommDestroy)>(dlsym(a->lib, "ncclCommDestroy"));
    a->AllGather = reinterpret_cast<decltype(a->AllGather)>(dlsym(a->lib, "ncclAllGather"));
    a->GetErrorString = reinterpret_cast<decltype(a->GetErrorString)>(dlsym(a->lib, "ncclGetErrorString"));
    if (!a->GetUniqueId || !a->CommInitRank || !a->CommDestroy || !a->AllGather || !a->GetErrorString) {
        *why = "libnccl.so.2 lacks a required symbol";
        return false;
    }
    return true;
}

thread_local std::string g_shard_error;

}  // namespace

namespace gsb {

void shard_destroy(gsb_ctx* ctx) {
    ShardState* sh = ctx->shard;
    if (!sh) return;
    close_peers(ctx);
    if (sh->window) cudaFree(sh->window);
    if (sh->mailbox_host) cudaFreeHost(sh->mailbox_host);
    if (sh->comm) sh->nccl.CommDestroy(sh->comm);
    delete sh;  // frees the device arrays
    ctx->shard = nullptr;
}

}  // namespace gsb

extern "C" {

// ------------------------------------------------------------------------------------------ process per GPU
int gsb_shard_unique_id(gsb_shard_id* out) {
    if (!out) return GSB_ERR_INVALID;
    static_assert(sizeof(gsb_shard_id) >= sizeof(ncclUniqueId), "id size");
    NcclApi api;
    std::string why;
    if (!load_nccl(&api, &why)) {
        g_shard_error = why;
        return GSB_ERR_CUDA;
    }
    ncclUniqueId id;
    if (api.GetUniqueId(&id) != ncclSuccess) {
        g_shard_error = "ncclGetUniqueId failed";
        return GSB_ERR_CUDA;
    }
    memset(out, 0, sizeof *out);
    memcpy(out, &id, sizeof id);
    return GSB_OK;
}

const char* gsb_shard_last_error(void) { return g_shard_error.c_str(); }

int gsb_create_sharded(int device, int rank, int world, const gsb_shard_id* id, gsb_ctx** out) {
    if (!out || !id || world < 1 || world > GSB_MAX_SHARDS || rank < 0 || rank >= world) return GSB_ERR_INVALID;
    int rc = gsb_create(device, out);
    if (rc != GSB_OK) return rc;
    gsb_ctx* ctx = *out;
    auto bail = [&](int code, const std::string& what) {
        g_shard_error = what;
        gsb_destroy(ctx);
        *out = nullptr;
        return code;
    };
    rc = attach_shard(ctx, rank, world);
    if (rc != GSB_OK) return bail(rc, ctx->err);
    ShardState* sh = ctx->shard;
    std::string why;
    if (!load_nccl(&sh->nccl, &why)) return bail(GSB_ERR_CUDA, why);
    ncclUniqueId nid;
    memcpy(&nid, id, sizeof nid);
    ncclResult_t nr = sh->nccl.CommInitRank(&sh->comm, world, nid, rank);
    if (nr != ncclSuccess) {
        sh->comm = nullptr;
        return bail(GSB_ERR_CUDA, std::string("ncclCommInitRank: ") + sh->nccl.GetErrorString(nr));
    }
    return GSB_OK;
}

int gsb_shard_rank(const gsb_ctx* ctx) { return ctx && ctx->shard ? ctx->shard->rank : -1; }
int gsb_shard_world(const gsb_ctx* ctx) { return ctx && ctx->shard ? ctx->shard->world : 0; }

int gsb_shard_slice(uint64_t n_total, int rank, int world, uint64_t* first, uint64_t* count) {
    if (world < 1 || rank < 0 || rank >= world || !first || !count) return GSB_ERR_INVALID;
    const uint64_t slice = std::max<uint64_t>((n_total + world - 1) / world, 1);
    *first = std::min(n_total, (uint64_t)rank * slice);
    *count = std::min(slice, n_total - *first);
    return GSB_OK;
}

int gsb_shard_band(const gsb_ctx* ctx, uint32_t height, uint32_t* row_begin, uint32_t* row_end) {
    if (!ctx || !ctx->shard || !row_begin || !row_end) return GSB_ERR_INVALID;
    const uint32_t tiles_y = (height + GSB_TILE - 1) / GSB_TILE, R = (tiles_y + ctx->shard->world - 1) / ctx->shard->world;
    *row_begin = std::min(tiles_y, (uint32_t)ctx->shard->rank * R);
    *row_end = std::min(tiles_y, *row_begin + R);
    return GSB_OK;
}

int gsb_scene_upload_sharded(gsb_ctx* ctx, const float* slice_vertices, uint64_t n_total, gsb_memory mem) {
    if (!ctx) return GSB_ERR_INVALID;
    if (!ctx->shard || ctx->shard->group) return fail(ctx, GSB_ERR_INVALID, "not a gsb_create_sharded context");
    CK(cudaSetDevice(ctx->device));
    return upload_slice(ctx, slice_vertices, n_total, mem);
}

static int ensure_frame_ipc(gsb_ctx* ctx, const gsb_uniforms* ubo, int fmt) {
    ShardState* sh = ctx->shard;
    size_t bytes = 0;
    if (!frame_layout_changed(sh, ubo->width, ubo->height, fmt, &bytes)) return GSB_OK;
    int rc = wait_frame(ctx);
    if (rc != GSB_OK) return rc;
    sh->frame_bytes = bytes;
    sh->frame_w = ubo->width;
    sh->frame_h = ubo->height;
    sh->frame_fmt = fmt;
    return ensure_windows_ipc(ctx);
}

int gsb_render_sharded_async(gsb_ctx* ctx, const gsb_uniforms* ubo, gsb_format fmt, void* stream) {
    int rc = check_sharded_args(ctx, ubo, fmt);
    if (rc != GSB_OK) return rc;
    if (ctx->shard->group) return fail(ctx, GSB_ERR_INVALID, "use gsb_group_render on a group context");
    CK(cudaSetDevice(ctx->device));
    rc = ensure_frame_ipc(ctx, ubo, fmt);
    if (rc != GSB_OK) return rc;
    poll_frame(ctx);
    return enqueue_sharded(ctx, ubo, fmt, stream_or_own(ctx, stream));
}

int gsb_render_sharded(gsb_ctx* ctx, const gsb_uniforms* ubo, void* out, size_t pitch, gsb_memory out_mem, gsb_format fmt, void* stream) {
    int rc = check_sharded_args(ctx, ubo, fmt);
    if (rc != GSB_OK) return rc;
    if (ctx->shard->group) return fail(ctx, GSB_ERR_INVALID, "use gsb_group_render on a group context");
    CK(cudaSetDevice(ctx->device));
    rc = ensure_frame_ipc(ctx, ubo, fmt);
    if (rc != GSB_OK) return rc;
    cudaStream_t s = stream_or_own(ctx, stream);
    for (int attempt = 0;; attempt++) {
        rc = enqueue_sharded(ctx, ubo, fmt, s);
        if (rc != GSB_OK) return rc;
        rc = wait_frame(ctx);
        if (rc != GSB_OK) return rc;
        bool any = false;
        rc = sharded_frame_status(ctx, &any);
        if (rc != GSB_OK) return rc;
        if (!any) break;
        // some rank's arena overflowed: every rank sees the same flags, so all of them re-render together
        if (attempt >= 3) return fail(ctx, GSB_ERR_OVERFLOW, "instance arena overflow persists after regrow");
        rc = regrow_after_overflow(ctx, ctx->stream);
        if (rc != GSB_OK) return rc;
    }
    if (out) return copy_frame_out(ctx, ubo, out, pitch, out_mem, fmt, s);
    return GSB_OK;
}

const void* gsb_shard_frame(const gsb_ctx* ctx) {
    if (!ctx || !ctx->shard || !ctx->shard->window) return nullptr;
    return ctx->shard->frame_x(ctx->shard->rank, (int)ctx->shard->last_parity);
}

// ------------------------------------------------------------------------------------------ one process, several GPUs
int gsb_group_create(int ndev, const int* devices, gsb_group** out) {
    if (!out || ndev < 1 || ndev > GSB_MAX_SHARDS) return GSB_ERR_INVALID;
    *out = nullptr;
    gsb_group* g = new (std::nothrow) gsb_group();
    if (!g) return GSB_ERR_OOM;
    for (int i = 0; i < ndev; i++) {
        gsb_ctx* c = nullptr;
        int rc = gsb_create(devices ? devices[i] : i, &c);
        if (rc == GSB_OK) {
            rc = attach_shard(c, i, ndev);
            if (rc != GSB_OK) gsb_destroy(c);
        }
        if (rc != GSB_OK) {
            g_shard_error = gsb_last_error(nullptr);
            gsb_group_destroy(g);
            return rc;
        }
        c->shard->group = g;
        g->ctx.push_back(c);
    }
    for (gsb_ctx* a : g->ctx)  // peers are plain pointers: enable access between distinct devices
        for (gsb_ctx* b : g->ctx)
            if (a->device != b->device) {
                cudaSetDevice(a->device);
                cudaError_t e = cudaDeviceEnablePeerAccess(b->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                    g_shard_error = std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e);
                    gsb_group_destroy(g);
                    return GSB_ERR_CUDA;
                }
                cudaGetLastError();
            }
    *out = g;
    return GSB_OK;
}

void gsb_group_destroy(gsb_group* g) {
    if (!g) return;
    for (gsb_ctx* c : g->ctx) {
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
    }
    for (gsb_ctx* c : g->ctx) gsb_destroy(c);
    delete g;
}

int gsb_group_size(const gsb_group* g) { return g ? (int)g->ctx.size() : 0; }
gsb_ctx* gsb_group_context(gsb_group* g, int rank) { return g && rank >= 0 && rank < (int)g->ctx.size() ? g->ctx[rank] : nullptr; }
const char* gsb_group_last_error(const gsb_group* g) { return g ? g->err.c_str() : g_shard_error.c_str(); }

int gsb_group_scene_upload(gsb_group* g, const float* vertices, uint64_t n, gsb_memory mem) {
    if (!g) return GSB_ERR_INVALID;
    if (n && !vertices) return group_fail(g, GSB_ERR_INVALID, "null vertices");
    const int G = (int)g->ctx.size();
    for (int r = 0; r < G; r++) {
        gsb_ctx* c = g->ctx[r];
        uint64_t first = 0, count = 0;
        gsb_shard_slice(n, r, G, &first, &count);
        cudaSetDevice(c->device);
        int rc = upload_slice(c, vertices + first * 60, n, mem);
        if (rc != GSB_OK) return group_fail(g, rc, c->err);
    }
    return GSB_OK;
}

static int group_enqueue(gsb_group* g, const gsb_uniforms* ubo, int fmt) {
    for (gsb_ctx* c : g->ctx) {
        int rc = check_sharded_args(c, ubo, fmt);
        if (rc != GSB_OK) return group_fail(g, rc, c->err);
    }
    size_t bytes = 0;
    if (frame_layout_changed(g->ctx[0]->shard, ubo->width, ubo->height, fmt, &bytes)) {
        for (gsb_ctx* c : g->ctx) {
            cudaSetDevice(c->device);
            int rc = wait_frame(c);
            if (rc != GSB_OK) return group_fail(g, rc, c->err);
            c->shard->frame_bytes = bytes;
            c->shard->frame_w = ubo->width;
            c->shard->frame_h = ubo->height;
            c->shard->frame_fmt = fmt;
        }
        int rc = ensure_windows_group(g);
        if (rc != GSB_OK) return rc;
    }
    for (gsb_ctx* c : g->ctx) {  // every allocation of every rank first (see ensure_ranges)
        cudaSetDevice(c->device);
        int rc = ensure_ranges(c, ubo->width, ubo->height);
        if (rc != GSB_OK) return group_fail(g, rc, c->err);
    }
    std::vector<ShardFrame> F(g->ctx.size());
    for (size_t i = 0; i < g->ctx.size(); i++) {
        gsb_ctx* c = g->ctx[i];
        cudaSetDevice(c->device);
        poll_frame(c);
        F[i].ubo = *ubo;
        F[i].fmt = fmt;
        F[i].stream = c->stream;
    }
    // one host thread enqueues every rank's frame, phase by phase (see enqueue_sharded_phase); the ranks meet on the device
    for (int phase = 1; phase <= 3; phase++)
        for (size_t i = 0; i < g->ctx.size(); i++) {
            gsb_ctx* c = g->ctx[i];
            cudaSetDevice(c->device);
            int rc = enqueue_sharded_phase(c, F[i], phase);
            if (rc != GSB_OK) return group_fail(g, rc, c->err);
        }
    return GSB_OK;
}

int gsb_group_render_async(gsb_group* g, const gsb_uniforms* ubo, gsb_format fmt) {
    if (!g || !ubo) return GSB_ERR_INVALID;
    return group_enqueue(g, ubo, fmt);
}

int gsb_group_render(gsb_group* g, const gsb_uniforms* ubo, void* out, size_t pitch, gsb_memory out_mem, gsb_format fmt) {
    if (!g || !ubo) return GSB_ERR_INVALID;
    for (int attempt = 0;; attempt++) {
        int rc = group_enqueue(g, ubo, fmt);
        if (rc != GSB_OK) return rc;
        bool any = false;
        for (gsb_ctx* c : g->ctx) {
            cudaSetDevice(c->device);
            rc = wait_frame(c);
            bool a = false;
            if (rc == GSB_OK) rc = sharded_frame_status(c, &a);
            if (rc != GSB_OK) return group_fail(g, rc, c->err);
            any = any || a;
        }
        if (!any) break;
        if (attempt >= 3) return group_fail(g, GSB_ERR_OVERFLOW, "instance arena overflow persists after regrow");
        for (gsb_ctx* c : g->ctx) {
            cudaSetDevice(c->device);
            rc = regrow_after_overflow(c, c->stream);
            if (rc != GSB_OK) return group_fail(g, rc, c->err);
        }
    }
    if (out) {
        gsb_ctx* c = g->ctx[0];
        cudaSetDevice(c->device);
        int rc = copy_frame_out(c, ubo, out, pitch, out_mem, fmt, c->stream);
        if (rc != GSB_OK) return group_fail(g, rc, c->err);
        if (out_mem != GSB_MEM_HOST && cudaStreamSynchronize(c->stream) != cudaSuccess) return group_fail(g, GSB_ERR_CUDA, "frame copy");
    }
    return GSB_OK;
}

}  // extern "C"
