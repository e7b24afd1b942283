// gsb_internal.cuh -- shared declarations of libgsb200 (not part of the public ABI).
//
// Device data layout (HBM), all fp32:
//   scene   pos_op[N]  float4 (x, y, z, opacity)            16 B  coalesced LDG.128
//           cov_a[N]   float4 (S00, S01, S02, S11)          16 B
//           cov_b[N]   float2 (S12, S22)                     8 B
//           sh[N][48]  RGB-interleaved degree-3 SH         192 B  read by cull survivors only
//   frame   recs[Nv][4] float4  compacted per-survivor record, 64 B, 64-B aligned (GSB_REC_F4 float4):
//               q0 = (uv.x, uv.y, conic.x, conic.y)                  \ first 32-B sector: all k_emit reads
//               q1 = (conic.z, opacity, bits(x0 | y0 << 16), bits(w | h << 16))  / (tile AABB, band-clipped)
//               q2 = (color.r, color.g, color.b, depth)              the blend reads q0, q1.xy, q2.xyz
//               q3 = (radius, bits(original index), -, -)            debug downloads only
//           dkeys[2][Nv] u32 bits(depth), dvals[2][Nv] u32 compact id      -- Gaussian-level sort
//           keys[2][cap] u32 tile id,     vals[2][cap] u32 compact id      -- instance-level sort
//           ranges[T] uint2 (start, ~end) per tile; (0xFFFFFFFF, 0xFFFFFFFF) = empty
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "gs_b200.h"

#define GSB_TILE 16
#define GSB_REC_F4 4  // float4 per survivor record
#define GSB_MAX_SHARDS 8  // GPUs of one NVSwitch domain a frame can be sharded over

namespace gsb {

// control words of one Onesweep sort (device memory, zeroed at frame start)
struct SortCtl {
    uint32_t ticket[8];     // tile tickets, one per radix pass
    uint32_t hist[8][256];  // global digit histograms
};

// ---- per-frame control block (device memory, zeroed by k_frame_init at frame start, except overflow_sticky) ----
struct Control {
    uint32_t project_ticket;   // chunk tickets of k_project
    uint32_t emit_ticket;      // chunk tickets of k_emit
    uint32_t num_visible;      // N_v
    uint32_t num_instances;    // M clamped to the arena capacity
    uint32_t overflow;         // 1 if M_total > capacity in THIS frame
    uint32_t overflow_sticky;  // OR of `overflow` over every frame since it was last reported; survives k_frame_init
    uint32_t epoch;            // look-back epoch of this frame's sorts: += 16 per frame by k_frame_init, never zeroed
    uint32_t pad0;
    unsigned long long instances_total;  // unclamped M
    unsigned long long blend_consumed;
    unsigned long long candidates_total;  // AABB instances before tile culling (the reference's M)
    unsigned long long blend_walked;      // (warp, record) visits of the blend's inner loop (k_blend with stats on)
    unsigned long long blend_hits;        // (pixel, Gaussian) pairs of those visits that passed the shader's tests
    unsigned long long blend_staged;      // records gathered into shared memory by the blend
    SortCtl sort_depth;        // Gaussian-level sort (32-bit depth keys)
    SortCtl sort_tile;         // instance-level sort (tile-id keys)
    // frame sharding (gsb_shard.cu): per-destination-band survivor totals of the routed k_project
    uint32_t route_total[GSB_MAX_SHARDS];
};

struct ProjectParams {
    const float4* pos_op;
    const float4* cov_a;
    const float2* cov_b;
    const float* sh;
    int sh_half;          // sh holds 48 fp16 per Gaussian (gsb_set_sh_storage; non-parity)
    uint32_t n;
    uint32_t index_base;  // global index of this context's first Gaussian (frame sharding: the rank's slice; else 0)
    gsb_uniforms ubo;
    uint32_t tile_row_begin, tile_row_end;  // band clip (multi-GPU); [0, tiles_y) = whole frame
    // outputs (compacted by survivor rank)
    float4* recs;
    uint32_t* dkeys;
    uint32_t* dvals;
    uint32_t* status;  // decoupled look-back words, one per 256-Gaussian chunk
    Control* ctl;
    // debug outputs (may be null)
    uint32_t* dbg_tiles;  // N
    uint4* dbg_aabb;      // N
    // frame sharding (route_world > 0): instead of compacting into recs / dkeys, every survivor is delivered -- its 64-B record
    // with the tile AABB clipped to the band, and its depth key -- into the exchange buffers of each rank whose band (band_rows
    // tile rows per rank) its AABB touches; route_dst_* point at THIS source's region inside rank d's buffers (peer memory)
    int route_world;
    uint32_t band_rows;
    uint32_t* route_status;  // [chunks][GSB_MAX_SHARDS] look-back words, one column per destination
    float4* route_dst_recs[GSB_MAX_SHARDS];
    uint32_t* route_dst_dkeys[GSB_MAX_SHARDS];
    // A variant of k_project appends its fields here, after all the others, so that the fields every other instantiation
    // reads keep their offsets and those instantiations keep their code.  launch_project picks the instantiation from these
    // fields; the routed kernel of a sharded frame has none of the variants.
    gsb_camera_model camera;  // gsb_set_camera_model: kind 0 = the UBO's pinhole camera
    float tan2_max;           // OPENCV: tan^2(camera.max_theta), computed in double and rounded to fp32 once by launch_project
    int sh_degree;            // gsb_set_sh_degree: 3, or 0..2 for the SHDEG instantiations
    int antialiased;          // gsb_set_antialiased: the AA instantiations
};

struct EmitParams {
    const uint32_t* sorted_cid;  // survivors in (depth, index) order
    uint32_t nv_hint;            // host estimate of N_v (sizes the grid only)
    uint32_t tiles_x;
    uint32_t* keys;              // tile ids
    uint32_t* vals;              // compact ids
    uint32_t capacity;
    unsigned long long* status;  // decoupled look-back words, one per 256-survivor chunk
    Control* ctl;
    int num_sms;
    const float4* recs;          // survivor records: tile AABB (+ centre, conic, opacity for the optional instance culling)
    int cull;                    // gsb_set_tile_cull level 1: exact per-tile instance culling (k_emit<true>)
    uint32_t coarse_shift;       // gsb_set_tile_cull level 2: bin by 2^shift x 2^shift tile blocks (tiles_x = bins per row); 0 = by tile
    unsigned long long* dbg_offsets;  // debug (may be null): exclusive instance offset of each depth-sorted survivor
};

cudaError_t launch_cov3d(const float* vtx_aos, uint64_t count, uint64_t dst_offset, float4* pos_op,
                         float4* cov_a, float2* cov_b, float* sh, float scale_factor, cudaStream_t s, bool sh_half = false);
cudaError_t launch_project(const ProjectParams& p, bool debug, cudaStream_t s);
cudaError_t launch_emit(const EmitParams& p, cudaStream_t s);

struct SortParams {  // host-side arguments of launch_sort
    void* keys[2] = {};        // u32 or u64 keys (key_bytes)
    uint32_t* vals[2] = {};
    int key_bytes = 4;         // 4 or 8
    const uint32_t* d_m = nullptr;  // device pointer to the element count
    uint32_t m_hint = 0;       // host estimate of the count (sizes the grids only; any value is correct)
    uint32_t key_bits = 0;
    unsigned long long* status = nullptr;  // epoch-tagged look-back words [tiles][256]
    uint32_t status_tiles = 0;  // capacity of status in tiles
    const uint32_t* d_epoch = nullptr;  // device word added to the epoch (the frame counter of Control; null = 0)
    uint32_t epoch_base = 0;   // pass p tags its look-back words with *d_epoch + epoch_base + p: unique per (frame, sort, pass)
    SortCtl* sc = nullptr;     // must be zero on entry
    int num_sms = 0;
    cudaEvent_t* events = nullptr;  // optional: events[0] after the histogram, events[1 + p] after pass p
    uint2* ranges = nullptr;   // optional (u32 keys): the last pass also produces the tile ranges (start, ~end)
    uint32_t range_key_mask = 0;  // bits of a key that index `ranges` (0 = all; coarse bins keep a tile mask above bit 15)
    bool discard_sorted_keys = false;  // the last pass writes payloads only (the caller never reads the sorted keys)
};
// Returns the number of passes P via *passes; sorted data ends in keys[P & 1].
cudaError_t launch_sort(const SortParams& p, uint32_t* passes, cudaStream_t s);
uint32_t sort_tile_items();

// One kernel instead of four memsets: zeroes the control block (keeping overflow_sticky) and the look-back words of
// k_project / k_emit (and, on a sharded context, the route_words look-back words of the routed k_project), and fills the
// tile ranges with (0xFFFFFFFF, 0xFFFFFFFF) = empty.
cudaError_t launch_frame_init(Control* ctl, uint32_t* project_status, uint32_t project_chunks, unsigned long long* emit_status,
                              uint32_t emit_chunks, uint2* ranges, uint32_t num_tiles, cudaStream_t s, uint32_t* route_status = nullptr,
                              uint32_t route_words = 0);
cudaError_t sort_prepare();  // one-time function attributes (dynamic shared memory opt-in) of the Onesweep kernels
cudaError_t launch_ranges_single_tile(const uint32_t* d_m, uint2* ranges, cudaStream_t s);

struct BlendParams {
    const float4* recs;
    const uint32_t* vals;
    const uint32_t* keys;   // coarse bins only: the sorted keys (block id | tile mask << 16)
    const uint2* ranges;
    uint32_t width, height, tiles_x;
    uint32_t coarse_shift, bins_x;  // the sorted lists and `ranges` are per 2^shift x 2^shift tile block (0: per tile), bins_x blocks per row
    uint32_t tile_row_begin, tile_row_end;
    void* out;              // pixel row `out_first_row` of the frame lives at out + 0
    uint32_t out_first_row; // 16 * tile_row_begin for a band buffer, 0 for a whole-frame buffer
    int num_peers;          // > 0: store the band into these whole-frame buffers instead of `out` (one per rank, peer memory)
    void* peer_frames[GSB_MAX_SHARDS];
    size_t row_pitch_bytes;
    int format;             // gsb_format
    int mode;               // gsb_mode
    int stats;              // 1: count blend_consumed / blend_walked (~4 instructions per record); 2: blend_hits as well
    Control* ctl;
    // gsb_set_backward (per-tile lists only): per pixel of the W x H frame, (bits(final transmittance), list position + 1 of the
    // last contributing entry, 0 = none).  Null: a plain frame.  Appended last so the other fields keep their offsets.
    uint2* record;
    // gsb_set_background: every pixel is stored as c + T_final * background (all zeros: the default kernels, no term).
    // Appended last so the other fields keep their offsets.
    float background[3];
    // gsb_render_depth: per pixel of the band, (D, A) as a float2, depth_pitch_bytes apart, pixel row `out_first_row` at
    // depth_alpha + 0 (never with num_peers).  Null: no depth output (the default kernels).  Appended last so the other fields
    // keep their offsets.
    void* depth_alpha;
    size_t depth_pitch_bytes;
};
cudaError_t launch_blend(const BlendParams& p, cudaStream_t s);

// A background of zeros (either sign) adds nothing: such frames and backward passes run the default instantiations.
inline bool has_background(const float bg[3]) { return bg[0] != 0.0f || bg[1] != 0.0f || bg[2] != 0.0f; }

// gsb_backward.cu: the reverse pass of one whole frame recorded by k_blend<..., RECORD = true>.  BackwardParams below is the
// argument of every backward kernel, and these are its first fields.  They are a base of it rather than the head of one flat
// struct because the code NVVM makes depends on that nesting, not only on the offsets: with the same fields flat, eight lens
// instantiations of k_preprocess_backward (fisheye and OpenCV, without the camera gradient, with AA, depth or a degree below
// 3) load the camera model in another order and get other register counts.
struct BackwardCore {
    // forward state of the frame
    const float4* recs;       // survivor records (compact id order)
    const uint32_t* vals;     // sorted per-tile lists (compact ids)
    const uint2* ranges;      // (start, ~end) per tile
    const uint2* record;      // per pixel: (bits(final T), last contributor position + 1)
    const Control* ctl;       // num_visible
    uint32_t width, height, tiles_x, num_tiles;
    int mode;                 // gsb_mode of the frame
    gsb_uniforms ubo;         // the frame's camera
    // scene
    const float* vertices;    // n x 60: the records last uploaded (scale, rotation, SH, position)
    const float4* cov_a;      // the uploaded Sigma (what k_project read)
    const float2* cov_b;
    // upstream gradient and outputs
    const float* grad_image;  // H x W float4, row_pitch_bytes apart
    size_t row_pitch_bytes;
    double* scratch;          // n x 9 per survivor: d uv (2), d conic (3), d opacity, d colour (3); zero on entry, zero again on exit
    float* grad_vertices;     // n x 60, zeroed by the caller; may be null when grad_ubo is set (frozen scene)
    int num_sms;
    // gsb_render_backward_camera (null otherwise).  Appended last so the other fields keep their offsets.
    double* cam_partials;     // [num_sms * 4][GSB_UBO_WORDS] per-CTA partial sums of dL/d(UBO), fully overwritten
    gsb_uniforms* grad_ubo;   // fp32 dL/d(UBO), fully overwritten
    // gsb_render_backward_density (null otherwise).  Appended last so the other fields keep their offsets.
    double* abs_scratch;      // n x 2 per survivor: sum over pixels of |d u|, |d v|; zero on entry, zero again on exit
    float* density;           // n x 4 per Gaussian: |d uv|, |abs d uv| (NDC units), views, max radius; accumulated into
    // gsb_set_backward_deterministic (null otherwise).  Appended last so the other fields keep their offsets.
    double* det_slots;        // per list position: that tile's fp64 partial sums of the entry (9 columns, 11 with density)
};
struct BackwardParams : BackwardCore {
    // A variant of the backward kernels appends its fields here, after all the others, so that the fields every other
    // instantiation reads keep their offsets and those instantiations keep their code.  launch_backward picks the
    // instantiations from these fields.
    float background[3];      // the frame's gsb_set_background, behind every pixel's last contributor (all zeros: no term)
    // gsb_render_backward_depth (null otherwise): the upstream dL/d(D, A) per pixel (grad_image may then be null) and its
    // per-survivor scratch
    const float2* grad_depth; // H x W (dL/dD, dL/dA), depth_pitch bytes apart
    size_t depth_pitch;
    double* depth_scratch;    // n x 1 fp64 dL/df per survivor: zero on entry, zero again on exit
    gsb_camera_model camera;  // the frame's gsb_set_camera_model: kind 0 = pinhole, else a lens frame (fisheye, OpenCV, orthographic)
    // gsb_render_backward_fisheye (null otherwise): a lens frame's dL/d(lens), fully overwritten; with cam_partials set
    gsb_camera_model* grad_lens;
    int sh_degree;            // the frame's gsb_set_sh_degree: below 3 the SH columns of the dropped bands are not written
                              // (the caller zeroed them) and the view direction takes the live coefficients only
    int antialiased;          // the frame ran with gsb_set_antialiased on (its opacities carry the compensation)
};
#define GSB_UBO_WORDS 40  // 4-byte words of gsb_uniforms; the camera gradient is reduced in this layout

// gsb_set_backward_deterministic: the buffers that group the per-(tile, entry) slots by survivor without atomics.  All
// M-sized arrays hold the arena capacity; every one is fully rewritten (or zeroed) by each call.
struct DetBackward {
    uint32_t* keys[2];             // the sort's keys: compact id of each list position (a copy: the frame's lists stay intact)
    uint32_t* pos[2];              // its payloads: the list position
    uint2* runs;                   // per survivor: (start, ~end) of its run in the sorted positions; all ones = no entry
    SortCtl* sc;                   // private sort control words, zeroed per call
    unsigned long long* status;    // private look-back words, zeroed per call
    uint32_t status_tiles;
    uint32_t m_hint;               // sizes the sort's grids only
    uint32_t key_bits;             // bits of the largest compact id
};
// gsb_features.cu: feature maps of the last recorded frame (gsb_render_features) and their backward pass.  The frame's fields
// and the caller's arrays are filled in by gsb_api.cu; launch_backward fills the scratch and deterministic ones.
struct FeatureParams {
    const float4* recs;
    const uint32_t* vals;
    const uint2* ranges;
    const uint2* record;
    const Control* ctl;
    uint32_t width, height, tiles_x, num_tiles;
    int mode;
    int num_sms;
    const float* features;  // n x channels, tight
    uint32_t channels;
    uint32_t c0;            // first channel of the chunk being launched
    float* map;             // gsb_render_features: H x W x channels, map_pitch bytes per row
    size_t map_pitch;
    const float* grad_map;  // backward: dL/d map, H x W x channels, grad_pitch bytes per row
    size_t grad_pitch;
    float* grad_features;   // n x channels, written for the survivors (zeroed by the caller); null: none
    double* scratch;        // the colour pass's n x 9 per-survivor sums: columns 0-5 gain the feature terms; null: no geometry
    double* abs_scratch;    // n x 2 |d u|, |d v| sums of gsb_render_backward_density; null: no density statistics
    double* feat_scratch;   // atomic path: n x 16 fp64 per-survivor feature sums, zero on entry and on exit
    double* det_slots;      // deterministic path: (8 + chunk width) fp64 per arena entry
    const uint32_t* pos;    // deterministic path: the colour pass's sorted list positions and per-survivor runs
    const uint2* runs;
};
uint32_t feature_chunk(uint32_t channels);  // channels per pass: 4 or 16
cudaError_t launch_render_features(FeatureParams p, cudaStream_t s);
cudaError_t launch_feature_backward(FeatureParams p, bool det, cudaStream_t s);

// features: gsb_render_backward_features' feature arguments (null for the other entries).  Its pass runs after the colour
// pass's sums (which are skipped when there is neither an image nor a depth gradient) and before k_density_accumulate and
// k_preprocess_backward; with neither grad_vertices nor grad_ubo only the feature gradient is formed.
// det: gsb_set_backward_deterministic's buffers (null: the atomic reduction).  A grad_lens on a pinhole frame is
// cudaErrorInvalidValue.
cudaError_t launch_backward(const BackwardParams& p, const DetBackward* det, const FeatureParams* features, cudaStream_t s);
// gsb_background_gradient: out[c] = sum over the W x H pixels of T_final(p) grad_image(p)[c], from the recorded frame's
// (bits(T), last) words.  fp64 products and sums in an order fixed by W and H (background_grad_rows(H) per-CTA partials,
// then one CTA), no atomics.  partials holds 3 doubles per row of background_grad_rows(H).
uint32_t background_grad_rows(uint32_t height);
cudaError_t launch_background_grad(const uint2* record, const float* grad_image, size_t row_pitch_bytes, uint32_t width,
                                   uint32_t height, double* partials, float* out, cudaStream_t s);

// gsb_optim.cu: one Adam step over the scene's rows (gsb_adam_step).  Every per-row array is n x 60 floats = 15 float4 per row.
struct AdamParams {
    float4* params;            // raw parameters: position, -, log scale, opacity logit, quaternion wxyz, SH
    float4* exp_avg;
    float4* exp_avg_sq;
    const float4* grad;        // dL/d(activated record), as gsb_render_backward writes it
    float4* vertices;          // OUT: the activated records
    float4* pos_op;            // OUT: the scene words k_ingest_cov3d would store for them
    float4* cov_a;
    float2* cov_b;
    float4* sh;
    uint64_t n;
    const float4* recs;        // selective: the last frame's survivor records (index in q3.y); null: every row
    const Control* ctl;        // selective: num_visible
    float lr[6];               // position, scale, opacity, rotation, SH DC, SH rest
    float beta1, beta2, eps, bias_correction1, bias_correction2_sqrt;
    // gsb_adam_step_filter3d: n per-row variances of the 3D smoothing filter (k_adam_step<true>); null: the plain step
    // (k_adam_step<false>).  Appended last so the other fields keep their offsets.
    const float* variance;
};
cudaError_t launch_adam(const AdamParams& p, int num_sms, cudaStream_t s);

// gsb_features.cu: gsb_adam_step_features, n x channels raw features and their moments (rows of the last frame's survivors
// when recs is set).
struct FeatureAdamParams {
    float* features;
    float* exp_avg;
    float* exp_avg_sq;
    const float* grad;
    uint64_t n;
    uint32_t channels;
    const float4* recs;  // selective: the last frame's survivor records (index in q3.y); null: every row
    const Control* ctl;  // selective: num_visible
    float lr, beta1, beta2, eps, bias_correction1, bias_correction2_sqrt;
};
cudaError_t launch_adam_features(const FeatureAdamParams& p, int num_sms, cudaStream_t s);

// gsb_filter3d.cu: gsb_filter3d_variance.  cams: k device copies of gsb_uniforms; focal = the largest focal_x of the k;
// dmax: one zeroed word (the largest seen depth's bits).  variance: n floats, overwritten.
cudaError_t launch_filter3d(const float4* vertices, uint64_t n, const gsb_uniforms* cams, uint32_t k, float focal,
                            uint32_t* dmax, float* variance, int num_sms, cudaStream_t s);
// gsb_filter3d_variance_lens.  models: k device copies of the cameras' lens models, an OPENCV one with max_theta replaced by
// tan^2(max_theta) rounded to fp32 once (k_project's tan2_max); smax: one zeroed word (the largest seen
// scale's bits).  variance: n floats, overwritten.
cudaError_t launch_filter3d_lens(const float4* vertices, uint64_t n, const gsb_uniforms* cams, const gsb_camera_model* models,
                                 uint32_t k, uint32_t* smax, float* variance, int num_sms, cudaStream_t s);

}  // namespace gsb
