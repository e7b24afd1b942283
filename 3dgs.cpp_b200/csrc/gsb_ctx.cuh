// gsb_ctx.cuh -- the context object behind the C ABI and the frame-orchestration helpers shared by gsb_api.cu (single
// GPU) and gsb_shard.cu (frame sharded over several GPUs).  Not part of the public ABI.
#pragma once
#include <algorithm>
#include <string>
#include <utility>

#include "gsb_internal.cuh"

namespace gsb {
struct ShardState;  // gsb_shard.cu

template <typename T>
cudaError_t dev_alloc(T** p, size_t count) {
    return cudaMalloc(reinterpret_cast<void**>(p), std::max<size_t>(count, 1) * sizeof(T));
}

// A device array owned by a context: freed with it or by reset(), and grown, never shrunk, by grow().  Memory is given back
// only then: a smaller scene upload, for one, keeps the larger buffers.  Moving an array (`group = {}` frees a struct of
// them) leaves the source empty.
template <typename T>
struct DevArray {
    T* p = nullptr;
    uint64_t count = 0;  // elements asked for by the last grow() that allocated

    DevArray() = default;
    DevArray(const DevArray&) = delete;
    DevArray& operator=(DevArray&& o) noexcept {
        if (this != &o) {
            reset();
            p = std::exchange(o.p, nullptr);
            count = std::exchange(o.count, 0);
        }
        return *this;
    }
    ~DevArray() { reset(); }
    operator T*() const { return p; }

    // cudaFree waits for all work on the device
    void reset() {
        if (p) cudaFree(p);
        p = nullptr;
        count = 0;
    }
    // Room for n elements: unless that many are allocated, frees, then allocates max(n, 1).  A failed allocation leaves the
    // array empty (count 0), so that the next call tries again.
    cudaError_t grow(uint64_t n) {
        if (p && n <= count) return cudaSuccess;
        reset();
        const cudaError_t e = dev_alloc(&p, n);
        if (e != cudaSuccess) p = nullptr;
        else count = n;
        return e;
    }
};

// The survivor arrays the middle of a frame and the blend read: the context's own, or on a sharded context the band's
// (the exchange buffers of the frame's parity and the destination-side sort arrays of ShardState).
struct Survivors {
    const float4* recs;
    uint32_t* dkeys[2];  // Gaussian-level sort: depth bits
    uint32_t* dvals[2];  //                       compact ids
    unsigned long long* emit_status;  // k_emit look-back words
    bool operator==(const Survivors& o) const {
        return recs == o.recs && dkeys[0] == o.dkeys[0] && dkeys[1] == o.dkeys[1] && dvals[0] == o.dvals[0] && dvals[1] == o.dvals[1] &&
               emit_status == o.emit_status;
    }
};

// gsb_set_backward_deterministic: the buffers behind DetBackward, allocated on first deterministic use, grown with the arena
// and the scene, and freed with bw_record.
struct DetBuffers {
    DevArray<double> slots;  // 11 fp64 per arena entry (the blend's per-(tile, entry) partials), 12 once a depth backward ran,
                             // 24 once a feature backward of more than 4 channels ran
    DevArray<uint32_t> keys[2];
    DevArray<uint32_t> pos[2];
    DevArray<unsigned long long> status;
    DevArray<SortCtl> sc;
    DevArray<uint2> runs;    // n (start, ~end) runs, one per possible survivor
};

struct FramePlan {
    uint32_t W, H, tiles_x, tiles_y, T, rb, re;
    uint32_t cs, bins_x, bins;  // instance-sort bins: 2^cs x 2^cs tile blocks (cs = 0: the tiles themselves, bins == T)
    uint32_t nv_q, m_q, depth_passes, passes;
    int fin;
};

// The last frame enqueued on a context, plain or sharded: what gsb_get_stats, gsb_debug_size / _download, the backward pass
// and the selective gsb_adam_step read about it.  Filled by enqueue_tail only; what ends part of its use (a new frame's
// enqueue, an arena regrow, gsb_set_backward(0), a scene upload) clears `recorded` or `exists`.
struct LastFrame {
    FramePlan plan{};
    gsb_uniforms ubo{};      // its camera
    int mode = GSB_MODE_EXACT;
    bool antialiased = false;  // gsb_set_antialiased when enqueued: its opacities carry the compensation
    float background[3] = {};  // gsb_set_background when enqueued: the colour its pixels were composited over
    gsb_camera_model camera{};  // gsb_set_camera_model when enqueued (kind 0: pinhole)
    int sh_degree = 3;       // gsb_set_sh_degree when enqueued: the SH bands its colours summed (its backward pass follows it)
    uint64_t scene_gen = 0;  // gsb_ctx::scene_gen when enqueued; 0: no frame yet (a frame needs an upload, which bumps it)
    bool pending = false;    // its completion event and stats copy have not been waited for (wait_frame)
    bool exists = false;     // its stats and debug buffers may be read (a scene upload clears it)
    bool debug = false;      // ran with gsb_set_debug on (its debug buffers and sorted keys exist)
    bool timers = false;     // recorded the stage events (gsb_get_stats may read them)
    bool recorded = false;   // its backward state is stored: per-pixel record and per-tile lists (gsb_set_backward, cs == 0)
    bool band = false;       // a band of tile rows, not the whole frame
    bool depth = false;      // rendered by gsb_render_depth (gsb_render_backward_depth needs such a frame)
};
}  // namespace gsb
using gsb::Control;
using gsb::DevArray;

// Captured CUDA graph of the "middle" of a frame (depth sort, key emission, tile sort: 9-10 kernels whose arguments do
// not depend on the camera).  Replaces recordRenderCommandBuffer's pre-recorded command buffer (src/Renderer.cpp:532-717).
struct MiddleKey {
    uint32_t tiles_x = 0, num_tiles = 0, nv_q = 0, m_q = 0, cull = 0, cs = 0;
    uint64_t alloc_gen = 0;
    gsb::Survivors sv{};  // the survivor arrays the graph reads (on a sharded context they depend on the frame's parity)
    bool operator==(const MiddleKey& o) const {
        return tiles_x == o.tiles_x && num_tiles == o.num_tiles && nv_q == o.nv_q && m_q == o.m_q && cull == o.cull && cs == o.cs &&
               alloc_gen == o.alloc_gen && sv == o.sv;
    }
};
struct MiddleGraph {
    MiddleKey key;
    cudaGraphExec_t exec = nullptr;
    uint64_t last_use = 0;
};


struct gsb_ctx {
    int device = 0;
    int num_sms = 132;  // H100 SXM; gsb_create reads the device's own count
    cudaStream_t stream = nullptr;
    std::string err;

    // scene
    uint64_t n = 0;
    DevArray<float4> pos_op;
    DevArray<float4> cov_a;
    DevArray<float2> cov_b;
    DevArray<float> sh;         // [n][48] fp32, or [n][48] fp16 when sh_half
    bool sh_half = false;       // gsb_set_sh_storage(1): takes effect at the next gsb_scene_upload
    bool scene_sh_half = false; // storage of the uploaded scene

    // frame state
    Control* ctl = nullptr;
    Control* ctl_host = nullptr;  // pinned mirror, filled at the end of each frame
    DevArray<uint32_t> project_status;        // k_project look-back words (one per 256-Gaussian chunk)
    DevArray<unsigned long long> emit_status;  // k_emit look-back words
    DevArray<float4> recs;
    DevArray<uint32_t> dkeys[2];  // Gaussian-level sort: depth bits
    DevArray<uint32_t> dvals[2];  //                       compact ids
    uint64_t capacity = 0;
    DevArray<uint32_t> keys[2];   // instance-level sort: tile ids (capacity + 16 entries)
    DevArray<uint32_t> vals[2];   //                      compact ids
    DevArray<unsigned long long> sort_status;  // [tiles][256] look-back words of the frame's sorts
    DevArray<uint2> ranges;
    DevArray<unsigned char> fb;   // staging frame of gsb_render to pageable host memory
    DevArray<unsigned char> depth_fb;  // staging (D, A) band of gsb_render_depth to pageable host memory

    int mode = GSB_MODE_EXACT;
    bool debug = false;
    bool timers = true;
    bool antialiased = false;   // gsb_set_antialiased: k_project scales opacities by the dilation's compensation
    float background[3] = {};   // gsb_set_background: k_blend composites every pixel over this colour (zeros: no term)
    gsb_camera_model camera{};  // gsb_set_camera_model: k_project's lens (kind 0: the UBO's pinhole camera)
    int sh_degree = 3;          // gsb_set_sh_degree: k_project sums the SH coefficients of bands <= sh_degree
    int tile_cull = 0;          // gsb_set_tile_cull level: 0 reference-equivalent lists, 1 exact per-tile culling, 2 coarse bins
    uint32_t coarse_shift = 2;  // level 2 bins are 2^shift x 2^shift tiles (GSB_COARSE_SHIFT)
    cudaEvent_t ev[8] = {};
    cudaEvent_t ev_sort[9] = {};  // instance sort: after hist, after each pass
    cudaEvent_t ev_done = nullptr;
    gsb::LastFrame frame;
    bool host_direct = true;    // gsb_render to page-locked host memory: blend straight into it (GSB_HOST_DIRECT=0: always stage)
    bool use_graph = true;      // replay the sorts + key emission from a captured CUDA graph when timers and debug are off
    uint64_t alloc_gen = 0;     // bumped by every (re)allocation a captured graph could point into
    uint64_t graph_clock = 0;
    uint32_t frames_since_epoch_clear = 0;
    MiddleGraph graphs[4] = {};
    uint32_t m_hint = 0;
    uint32_t nv_hint = 0;
    uint32_t regrow_count = 0;

    // debug copies
    DevArray<uint32_t> dbg_tiles;
    DevArray<uint4> dbg_aabb;
    DevArray<uint32_t> dbg_keys_unsorted;
    DevArray<uint32_t> dbg_vals_unsorted;
    DevArray<unsigned long long> dbg_offsets;  // N: k_emit's exclusive scan value per depth-sorted survivor

    // reverse mode (gsb_set_backward / gsb_render_backward)
    bool backward = false;          // frames record the per-pixel state the backward needs
    DevArray<uint2> bw_record;      // W x H (bits(final T), last contributor position + 1) of the last recorded frame
    DevArray<double> bw_scratch;    // n x 9 per-survivor fp64 accumulators of the blend backward (kept zero between calls)
    DevArray<double> bw_cam_partials;  // [4 * num_sms][GSB_UBO_WORDS] per-CTA fp64 partial sums of gsb_render_backward_camera
    DevArray<double> bw_abs;        // n x 2 per-survivor fp64 sums of |d u|, |d v| of gsb_render_backward_density (kept zero)
    DevArray<double> bw_depth;      // n x 1 per-survivor fp64 dL/d depth of gsb_render_backward_depth (kept zero)
    DevArray<double> bw_feat;       // n x 16 per-survivor fp64 dL/d features of gsb_render_backward_features' atomic path (kept zero)
    bool bw_deterministic = false;  // gsb_set_backward_deterministic
    gsb::DetBuffers bw_det;
    DevArray<double> bg_partials;   // [background_grad_rows(H)][3] per-CTA fp64 partial sums of gsb_background_gradient
    uint64_t scene_gen = 0;        // bumped by every gsb_scene_upload, gsb_adam_step, gsb_mcmc_noise and gsb_mcmc_relocate

    // gsb_image_loss (gsb_loss.cu): allocated on first use, grown with the frame size
    DevArray<float> loss_abc;        // 9 x W x H: the gather terms A, B, C of each RGB channel (only for a gradient)
    DevArray<double> loss_partials;  // 3 x tiles: per-tile fp64 sums of |x - y|, (x - y)^2 and the SSIM map

    // gsb_bilagrid_backward (gsb_bilagrid.cu): allocated on first use, grown with the frame and grid size
    DevArray<double> bilagrid_partials;  // [blocks][L][4][12] per-block fp64 sums of the grid gradient

    // frame sharding over several GPUs (gsb_shard.cu); null for a plain context
    gsb::ShardState* shard = nullptr;
};


namespace gsb {

int fail(gsb_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess);

#define CK(call)                                                       \
    do {                                                               \
        cudaError_t e_ = (call);                                       \
        if (e_ != cudaSuccess) return gsb::fail(ctx, e_ == cudaErrorMemoryAllocation ? GSB_ERR_OOM : GSB_ERR_CUDA, #call, e_); \
    } while (0)

// the caller's stream of an entry point, or the context's own for NULL
inline cudaStream_t stream_or_own(const gsb_ctx* ctx, void* s) { return s ? static_cast<cudaStream_t>(s) : ctx->stream; }

void drop_graphs(gsb_ctx* ctx);
int ensure_sort_status(gsb_ctx* ctx, uint64_t items);
int ensure_arena(gsb_ctx* ctx, uint64_t capacity);
uint32_t bits_for(uint32_t count);
uint32_t quantise_hint(uint64_t hint);
size_t bytes_per_pixel(int fmt);
int wait_frame(gsb_ctx* ctx);
void poll_frame(gsb_ctx* ctx);
int regrow_after_overflow(gsb_ctx* ctx, cudaStream_t stream);
int ensure_ranges(gsb_ctx* ctx, uint32_t W, uint32_t H);
// fills the size-derived fields of a plan, (re)allocates the tile ranges and handles the look-back epoch wrap
int plan_frame(gsb_ctx* ctx, const gsb_uniforms* ubo, uint32_t rb, uint32_t re, cudaStream_t stream, FramePlan* out);
ProjectParams project_params(const gsb_ctx* ctx, const gsb_uniforms& ubo, uint32_t rb, uint32_t re);
int enqueue_middle(gsb_ctx* ctx, const FramePlan& fp, const Survivors& sv, cudaStream_t stream, bool events);
int launch_middle_graph(gsb_ctx* ctx, const FramePlan& fp, const Survivors& sv, cudaStream_t stream);
// depth_out (gsb_render_depth): the band's (D, A) buffer, depth_pitch bytes per row, laid out like band_out; null for none
int enqueue_blend(gsb_ctx* ctx, const FramePlan& fp, const Survivors& sv, uint32_t b0, uint32_t b1, void* band_out, size_t pitch,
                  int fmt, cudaStream_t stream, void* const* peer_frames = nullptr, int num_peer_frames = 0, void* depth_out = nullptr,
                  size_t depth_pitch = 0);
int enqueue_tail(gsb_ctx* ctx, const FramePlan& fp, const gsb_uniforms& ubo, cudaStream_t stream);
int check_image(gsb_ctx* ctx, const gsb_uniforms* ubo, int fmt);
int check_render_args(gsb_ctx* ctx, const gsb_uniforms* ubo, uint32_t& rb, uint32_t& re, const void* out, size_t& pitch, int fmt);

// gsb_shard.cu
void shard_destroy(gsb_ctx* ctx);

}  // namespace gsb
