/*
 * gs_b200.h -- C ABI of libgsb200.so: the H100 (sm_90a) CUDA replacement for the per-frame
 * compute path of shg8/3DGS.cpp (project+SH -> bin -> sort -> blend).
 *
 * The reference has no plugin/FFI seam for this path; the seam is compile-time inside
 * Renderer/GSScene (SURVEY.md 8b).  Every entry point below therefore names the reference
 * code it replaces (paths relative to /root/reference).  A maintainer swaps the Vulkan
 * dispatch for these calls as shown in INTEGRATION.md.
 *
 * Conventions: plain pointers and sizes, no C++/torch types; every function returns
 * GSB_OK (0) or a negative gsb_status and never throws; gsb_last_error() gives the text.
 * A context is single-owner: one CUDA device, calls from one thread at a time (the reference
 * is single-threaded with FRAMES_IN_FLIGHT = 1, src/vulkan/VulkanContext.h:6).
 * There is NO CPU fallback: without a CUDA device gsb_create() fails with GSB_ERR_NO_DEVICE.
 */
#ifndef GS_B200_H
#define GS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSB_ABI_VERSION 3

typedef struct gsb_ctx gsb_ctx;

typedef enum gsb_status {
    GSB_OK = 0,
    GSB_ERR_INVALID = -1,   /* bad argument */
    GSB_ERR_NO_DEVICE = -2, /* no usable CUDA device (the product has no CPU path) */
    GSB_ERR_CUDA = -3,      /* CUDA runtime error, see gsb_last_error */
    GSB_ERR_NO_SCENE = -4,  /* render before gsb_scene_upload */
    GSB_ERR_OOM = -5,       /* device allocation failed */
    GSB_ERR_OVERFLOW = -6   /* instance arena could not be grown enough */
} gsb_status;

/* Renderer::UniformBuffer -- src/Renderer.h:21-29 == preprocess.comp:16-24 (std140, 160 bytes,
 * column-major mat4).  Produced on the host by Renderer::updateUniforms (src/Renderer.cpp:719-754). */
typedef struct gsb_uniforms {
    float camera_position[4];
    float proj_mat[16];
    float view_mat[16];
    uint32_t width;
    uint32_t height;
    float tan_fovx;
    float tan_fovy;
} gsb_uniforms;

/* VertexAttribute -- src/shaders/common.glsl:42-49 == Renderer.h:31-38; only used by
 * gsb_debug_download(GSB_BUF_ATTR) so intermediates can be diffed against the reference layout. */
typedef struct gsb_vertex_attribute {
    float conic_opacity[4];
    float color_radii[4];
    uint32_t aabb[4];
    float uv[2];
    float depth;
    uint32_t magic;
} gsb_vertex_attribute;

/* Output image formats.  The reference stores vec4(c,1) into a B8G8R8A8_UNORM swapchain image
 * (render.comp:98, src/vulkan/Swapchain.cpp:24); RGBA32F is the un-quantised value of that store. */
typedef enum gsb_format {
    GSB_FORMAT_RGBA32F = 0, /* float4 per pixel, 16 B */
    GSB_FORMAT_RGBA8 = 1,   /* UNORM8, R,G,B,A byte order */
    GSB_FORMAT_BGRA8 = 2    /* UNORM8, B,G,R,A byte order (the reference swapchain format) */
} gsb_format;

/* Arithmetic mode of the blend stage.
 * EXACT: every fp32 op is a single IEEE operation in render.comp's order and exp() is the fixed
 *        operation sequence documented in DESIGN.md; bit-identical to oracle exp-mode 1.
 * FAST : FMA contraction + ex2.approx; same algorithm, results within ~1e-6 of EXACT except at
 *        the shader's own step functions. */
typedef enum gsb_mode { GSB_MODE_EXACT = 0, GSB_MODE_FAST = 1 } gsb_mode;

typedef enum gsb_memory { GSB_MEM_HOST = 0, GSB_MEM_DEVICE = 1 } gsb_memory;

/* Buffers retrievable with gsb_debug_download, in the REFERENCE's layouts (SURVEY Appendix B). */
typedef enum gsb_buffer {
    GSB_BUF_COV3D = 0,         /* scene->cov3DBuffer: N * 6 float                 (GSScene.cpp:158) */
    GSB_BUF_ATTR = 1,          /* vertexAttributeBuffer: N * gsb_vertex_attribute (Renderer.cpp:169); culled entries zero */
    GSB_BUF_TILES_OVERLAP = 2, /* tileOverlapBuffer: N * u32                      (Renderer.cpp:170) */
    GSB_BUF_PREFIX_SUM = 3,    /* inclusive scan in Gaussian-index order: N * u32 (Renderer.cpp:215); derived on the
                                  host from TILES_OVERLAP -- the device scans in depth order inside k_emit */
    GSB_BUF_KEYS_UNSORTED = 4, /* sortKBuffer after the reference's radix pass 3 (bits 0-31 = depth sorted, tile
                                  bits not yet): M * u64.  Equals preprocess_sort's output stably sorted by depth;
                                  this implementation emits the instances directly in that order (DESIGN.md) */
    GSB_BUF_VALS_UNSORTED = 5, /* the payloads (Gaussian indices) that go with KEYS_UNSORTED: M * u32 */
    GSB_BUF_KEYS_SORTED = 6,   /* sortKBufferEven after the 8 passes: M * u64 */
    GSB_BUF_VALS_SORTED = 7,   /* sortVBufferEven after the 8 passes: M * u32 (Gaussian indices) */
    GSB_BUF_TILE_BOUNDARY = 8, /* tileBoundaryBuffer: T * 2 u32                   (Renderer.cpp:321) */
    /* No reference counterpart: the two device results the two-level sort adds (DESIGN.md section 3), exposed so the
     * device scan and the Gaussian-level sort are pinned directly and not only through the key placement. */
    GSB_BUF_DEPTH_ORDER = 9,   /* N_v * u32: Gaussian indices of the cull survivors in (depth bits, index) order */
    GSB_BUF_EMIT_OFFSETS = 10  /* N_v * u64: k_emit's exclusive scan of the tile counts in that order = the slot of each
                                  survivor's first instance (prefix_sum.comp's job, in depth order) */
} gsb_buffer;

/* The reference's six timestamp pairs (src/Renderer.cpp:484-699) + its "instances" text metric
 * (:540).  Mapping: preprocess_ms = k_project; preprocess_sort_ms = k_emit (tile-count scan + key
 * emission, so prefix_sum_ms is 0); sort_ms = Gaussian-level depth sort + instance-level tile sort. */
typedef struct gsb_stats {
    uint64_t num_gaussians;     /* N */
    uint64_t num_visible;       /* N_v: survivors of the three culls */
    uint64_t num_instances;     /* M: (Gaussian, tile) instances emitted and sorted this frame */
    uint64_t num_instances_aabb; /* AABB instances = the reference's "instances" (Renderer.cpp:540); equals
                                   num_instances unless gsb_set_tile_cull is on */
    uint64_t blend_consumed;    /* sum over tiles of run entries read before the tile terminated */
    uint64_t instance_capacity; /* current arena capacity in instances */
    uint32_t sort_passes;       /* radix passes of the instance-level (tile id) sort = ceil(log2(T) / 8) */
    uint32_t regrow_count;      /* times the arena was regrown and the frame re-rendered so far */
    float preprocess_ms, prefix_sum_ms, preprocess_sort_ms, sort_ms, tile_boundary_ms, render_ms;
    float frame_ms;         /* first kernel to last kernel of the frame */
    float sort_depth_ms;    /* Onesweep over the N_v visible Gaussians, 32-bit depth keys (histogram + passes) */
    float sort_tile_ms;     /* Onesweep over the M instances, tile-id keys (histogram + passes) */
    float sort_hist_ms;     /* the histogram kernel of the instance sort */
    float sort_pass_ms[8];  /* each pass kernel of the instance sort (first sort_passes entries) */
    uint32_t sort_depth_passes; /* passes of the Gaussian-level sort (4) */
    uint32_t pad_;
    uint64_t blend_warp_visits; /* (warp, record) visits of the blend's inner loop = evaluated pixel-pair x Gaussian work / 64
                                   (each visit evaluates 64 pixels); counted only while timers or debug are on */
    uint64_t blend_pixel_hits;  /* (pixel, Gaussian) pairs of those visits that passed render.comp:68-80 (power <= 0 and
                                   alpha >= 1/255): hits / (64 * visits) = SIMT lane utilisation of the blend's walk; counted on
                                   gsb_set_debug frames only (0 otherwise) */
    uint64_t blend_staged;      /* records gathered into shared memory by the blend (with coarse bins: this tile's entries among the
                                   blend_consumed list entries it scanned; otherwise equal to the entries read) */
    float shard_blend_ms;       /* frame sharding only: this rank's blend kernel alone (render_ms also holds the wait below) */
    float shard_wait_ms;        /* frame sharding only: from the end of this rank's blend until every rank's band has landed */
} gsb_stats;

/* ---- lifetime: replaces Renderer::initializeVulkan + create*Pipeline (Renderer.cpp:119-155,166-364) ---- */
int gsb_abi_version(void);
int gsb_device_count(void);
int gsb_create(int device, gsb_ctx **out);
void gsb_destroy(gsb_ctx *ctx);
/* Text of the last error on ctx (ctx == NULL: last gsb_create error on this thread). */
const char *gsb_last_error(const gsb_ctx *ctx);

/* ---- scene: replaces vertexBuffer->uploadFrom + GSScene::precomputeCov3D (GSScene.cpp:61,157-184) ----
 * vertices: n records of GSScene::Vertex (src/GSScene.h:41-46): 60 floats =
 * position(xyz,1) scale_opacity(exp(s),sigmoid(o)) rotation(w,x,y,z normalised) sh[48] (RGB-interleaved),
 * i.e. exactly what GSScene::load (GSScene.cpp:36-59) stages.  mem says where `vertices` lives.
 * Precomputes cov3D on the device (precomp_cov3d.comp:25-48, scale_factor 1.0 as GSScene.cpp:176). */
int gsb_scene_upload(gsb_ctx *ctx, const float *vertices, uint64_t n, gsb_memory mem);
uint64_t gsb_scene_size(const gsb_ctx *ctx);

/* Storage of the 48 SH coefficients, chosen BEFORE gsb_scene_upload (default 0 = fp32, 192 B per Gaussian).  1 = fp16 (96 B):
 * NOT a parity mode -- colours come from coefficients rounded to half precision (relative 2^-11), so pixels differ from the
 * reference / oracle by up to ~1e-3; geometry, culling, instance lists and sort order are unaffected.  It halves the
 * dominant term of k_project's HBM traffic (SURVEY 8f row 2 "optional fp16 SH storage mode (non-parity)"). */
int gsb_set_sh_storage(gsb_ctx *ctx, int half_precision);

/* ---- configuration ---- */
int gsb_set_mode(gsb_ctx *ctx, gsb_mode mode);
/* debug != 0: keep every intermediate so gsb_debug_download works (extra HBM traffic). */
int gsb_set_debug(gsb_ctx *ctx, int debug);
/* How the per-tile lists are produced (default 0).  The IMAGE is bit-identical at every level.
 *   0  reference-equivalent: one (Gaussian, tile) instance per tile of the AABB (preprocess_sort.comp:47-58); M, keys,
 *      payloads and tile ranges equal the reference's.
 *   1  exact instance culling: an instance is dropped at key emission if the Gaussian provably stays below the shader's
 *      own alpha < 1/255 cut on every pixel of the tile; M and the key / payload / tile-range buffers are an ordered
 *      subset of the reference's.  Trades a per-candidate test for fewer instances to sort.
 *   2  coarse bins: the instance sort runs over blocks of 4 x 4 tiles (one entry per (Gaussian, block), the key carrying
 *      the mask of the block's tiles inside the Gaussian's tile AABB); every tile then walks its block's depth-ordered
 *      list and keeps the entries whose mask has its bit -- exactly the tile's own list of level 0, in the same order.
 *      ~3x fewer instances to emit and sort.  num_instances then counts (Gaussian, block) entries; num_instances_aabb
 *      stays the reference's count.  Unavailable (falls back to 1) with gsb_set_debug, whose downloads are per tile,
 *      and for frames of more than 65536 blocks. */
int gsb_set_tile_cull(gsb_ctx *ctx, int level);
/* Anti-aliased rendering (default 0; no reference counterpart).  preprocess.comp:63-65 dilates the screen-space covariance
 * by 0.3 px^2 and keeps the opacity, so a Gaussian smaller than a pixel is drawn as a blob of at least 0.3 px^2 at full
 * opacity, and thin structure thickens and brightens when a scene is rendered farther away or at a lower resolution than
 * it was trained at.  While on, every Gaussian that passes the det > 0 test keeps the dilated covariance for its conic,
 * radius and tiles and has its opacity scaled, in fp32 in this order (the rule of gsplat's rasterize_mode="antialiased"):
 *     det0 = c00 * c11 - c10 * c01            the undilated cov2d, in the product order of the dilated det
 *     comp = sqrt(max(0, det0 / det))         det = the dilated determinant; a NaN ratio gives 0
 *     opacity = opacity * comp
 * so opacity * sqrt(det) -- a Gaussian's integrated weight -- is that of the undilated footprint.  The blend, tile-cull
 * levels 1 and 2 and the backward pass see the compensated opacity, which is what GSB_BUF_ATTR's conic_opacity[3] holds;
 * conic, radius, tile AABB, depth, colour and the survivor set are those of the default mode.  Takes effect at the next
 * frame; the backward entries and the selective gsb_adam_step follow the setting the last frame was rendered with and
 * differentiate through comp.  NULL ctx or a sharded context (gsb_create_sharded, a gsb_group rank): GSB_ERR_INVALID. */
int gsb_set_antialiased(gsb_ctx *ctx, int enabled);
/* Background colour (default black; no reference counterpart).  rgb: 3 host floats, NULL = (0, 0, 0).  render.comp:98 stores
 * vec4(c, 1), the colour composited over black; with a background every colour channel of every pixel is stored as
 *     out = c + T_final * bg          (one fp32 multiply, then one add, each rounded; EXACT and FAST alike)
 * T_final being the transmittance after the pixel's last contributor (at the T' < 1e-4 break, the T before the breaking
 * Gaussian).  A pixel no Gaussian reaches is bg exactly.  8-bit formats quantise out as before; A stays 1 (255).  All zeros
 * (either sign) is the default frame, bit for bit.  Any finite values (a learned colour may leave [0, 1]); NaN or +-inf:
 * GSB_ERR_INVALID.  Takes effect at the next frame; the frame records it and the backward entries follow the frame's value.
 * Every context accepts it, sharded ones and gsb_group ranks included; changing it drops no captured graph. */
int gsb_set_background(gsb_ctx *ctx, const float *rgb);
/* Camera model of the frames (default PINHOLE: the UBO's proj_mat / tan_fov, the reference's camera, bit for bit).
 * FISHEYE is COLMAP's OPENCV_FISHEYE (Kannala-Brandt) lens: k_project reads only view_mat, camera_position, width and height
 * of the UBO, and with t = (x, y, z) the view-space position (x right, y down, z forward), r = |(x, y)|, d = |t|,
 * theta = atan2(r, z) and rho = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8):
 *   culled unless d > 0.2 and theta <= max_theta (NaN culled);  uv = (fx (rho / r) x + cx, fy (rho / r) y + cy), (cx, cy) at r = 0;
 *   cov2d = J W Sigma W^T J^T + 0.3 I with J = d uv / d t exact (no tan_fov clamp);  depth key d (sorts lenses past 180 deg).
 * The conic, culls, radius, tile AABB, opacity (and its anti-aliased compensation) and SH colour follow from it as for a
 * pinhole frame.  Pixel (i, j) is sampled at (i, j): COLMAP's principal point is (cx - 0.5, cy - 0.5) here.
 * The frame records the model; gsb_render_backward and gsb_render_backward_density follow the frame's, and for a fisheye frame
 * gsb_render_backward_camera and gsb_render_backward_density with a non-NULL grad_uniforms return GSB_ERR_INVALID (no pose
 * gradient through the lens).  m NULL or kind PINHOLE: the default.  GSB_ERR_INVALID, the setting unchanged, for a NULL ctx,
 * a sharded context or gsb_group rank, an unknown kind, fx or fy not positive and finite, any other field not finite,
 * max_theta outside (0, pi), or d theta_d / d theta <= 0 anywhere on [0, max_theta] (checked on the host in double).
 * Takes effect at the next frame; changing it drops no captured graph. */
typedef enum gsb_camera_kind { GSB_CAMERA_PINHOLE = 0, GSB_CAMERA_FISHEYE = 1 } gsb_camera_kind;
typedef struct gsb_camera_model {
    uint32_t kind;        /* gsb_camera_kind */
    float fx, fy, cx, cy; /* pixels; pixel (i, j) is sampled at (i, j), as the blend does (COLMAP's cx - 0.5) */
    float k[4];           /* Kannala-Brandt / OpenCV fisheye: theta_d = theta (1 + k1 t^2 + k2 t^4 + k3 t^6 + k4 t^8), t = theta */
    float max_theta;      /* radians, in (0, pi): rays farther off the axis are culled */
} gsb_camera_model;
int gsb_set_camera_model(gsb_ctx *ctx, const gsb_camera_model *m);
/* per-stage cudaEvent timers (the QueryManager analogue, Renderer.cpp:85-100). Default on. */
int gsb_set_timers(gsb_ctx *ctx, int enabled);
/* Replay the camera-independent middle of the frame (both sorts + key emission) from a captured CUDA graph instead of
 * ~10 separate launches -- the analogue of the reference's pre-recorded renderCommandBuffer (Renderer.cpp:532-717).
 * Default on; only used while timers and debug are off (both need per-kernel host calls). */
int gsb_set_graph(gsb_ctx *ctx, int enabled);
/* Page-locked host memory for frames / vertex data handed to gsb_render / gsb_scene_upload: copies to and from it are
 * asynchronous DMA (the reference's host-visible staging buffers, Buffer::staging, src/vulkan/Buffer.cpp). */
int gsb_host_alloc(void **out, size_t bytes);
void gsb_host_free(void *p);
/* Pre-size the (tile,depth) instance arena (the reference's sortBufferSizeMultiplier,
 * Renderer.cpp:541-563, grows N*k on overflow; this does the same between frames). */
int gsb_reserve_instances(gsb_ctx *ctx, uint64_t capacity);

/* ---- the frame: replaces Renderer::draw()'s two submits (Renderer.cpp:388-405), i.e.
 * preprocess.comp -> prefix_sum.comp x(log2N+1) -> preprocess_sort.comp -> 8x(hist.comp, sort.comp)
 * -> tile_boundary.comp -> render.comp, without the mid-frame fence + host read of M (:391,:538).
 *
 * Renders tile rows [tile_row_begin, tile_row_end) of the (ubo->width x ubo->height) frame
 * (pass 0, UINT32_MAX for the whole frame; a sub-range is the multi-GPU band of SURVEY 8e).
 * `out` receives pixel rows [16*tile_row_begin, min(H, 16*tile_row_end)) densely, row-major,
 * `row_pitch_bytes` apart (0 = tight).  out_mem says whether `out` is host or device memory.
 * `stream` is a cudaStream_t (NULL = the context's own stream).  The call returns when the frame
 * (and, for host output, the copy) has completed.  If the instance arena overflows, the arena is
 * regrown and the frame re-rendered transparently (the reference's retry, Renderer.cpp:397-399). */
int gsb_render(gsb_ctx *ctx, const gsb_uniforms *ubo, uint32_t tile_row_begin, uint32_t tile_row_end,
               void *out, size_t row_pitch_bytes, gsb_memory out_mem, gsb_format fmt, void *stream);

/* Enqueue-only variant for pipelined callers (bench e2e): never synchronises, never regrows;
 * overflow is reported by the next gsb_get_stats()/gsb_render().  out must be device memory. */
int gsb_render_async(gsb_ctx *ctx, const gsb_uniforms *ubo, uint32_t tile_row_begin,
                     uint32_t tile_row_end, void *out_device, size_t row_pitch_bytes, gsb_format fmt,
                     void *stream);

/* Waits for the last frame and fills stats (the retrieveTimestamps analogue, Renderer.cpp:85-100). */
int gsb_get_stats(gsb_ctx *ctx, gsb_stats *out);

/* ---- reverse mode: gradient of one rendered frame with respect to the scene and the camera (no reference counterpart) ----
 * Keep what the next frames need for gsb_render_backward (default 0).  The image is unchanged.  Set before gsb_render.
 * While on, tile-cull level 2 falls back to 1, as under gsb_set_debug; every frame also stores 8 B per pixel (its final
 * transmittance and the list position of its last contributing Gaussian).  Sharded contexts: GSB_ERR_INVALID. */
int gsb_set_backward(gsb_ctx *ctx, int enabled);

/* Deterministic reverse mode (default 0).  While on, gsb_render_backward, gsb_render_backward_camera and
 * gsb_render_backward_density use no floating-point atomics: every output word is a function of the frame, the
 * vertices and grad_image alone, bit for bit -- the same on every call, on any stream, whatever the arena capacity,
 * and the same at tile-cull levels 0 and 1.  Takes effect at the next backward call; the forward is unchanged.
 * The first deterministic call allocates about 105 B per arena entry (gsb_reserve_instances) and 8 B per Gaussian, freed by
 * gsb_set_backward(ctx, 0); GSB_ERR_OOM if that fails.  NULL ctx or a sharded context: GSB_ERR_INVALID. */
int gsb_set_backward_deterministic(gsb_ctx *ctx, int enabled);

/* Gradient of the last frame.  All pointers are device memory, enqueued on `stream` (NULL = the context's stream).
 *   vertices      n x 60 floats: the records last passed to gsb_scene_upload (scale and rotation are read from here)
 *   grad_image    H x W float4 (RGBA32F layout, row_pitch_bytes apart, 0 = tight); the A channel is ignored (the output is 1)
 *   grad_vertices n x 60 floats, OVERWRITTEN: d/d position xyz, scale xyz, opacity, rotation wxyz (as stored, no
 *                 normalisation), sh[48]; zero for position.w, for culled Gaussians and for Gaussians outside every list used
 * The parameters are the activated ones gsb_scene_upload receives (exp(s), sigmoid(o), the normalised quaternion); a caller
 * chains through its own activations.  By default gradients are accumulated with (fp64) atomics, so they are not guaranteed to
 * be bitwise reproducible from run to run; gsb_set_backward_deterministic makes them so.  GSB_ERR_NO_SCENE before any upload or frame; GSB_ERR_INVALID if the last frame was rendered with
 * gsb_set_backward off, was a band rather than the whole frame, or overflowed the instance arena (gsb_render_async), if
 * the scene was uploaded again or stepped (gsb_adam_step) or the arena grew (gsb_reserve_instances) after it, if the scene
 * stores fp16 SH, or on a sharded context. */
int gsb_render_backward(gsb_ctx *ctx, const float *vertices, const float *grad_image, size_t row_pitch_bytes,
                        float *grad_vertices, void *stream);

/* gsb_render_backward plus the gradient with respect to the last frame's camera: the same arguments, preconditions and error
 * codes, and also GSB_ERR_INVALID for a NULL grad_uniforms.
 *   grad_vertices  may be NULL (a frozen scene: only the camera is differentiated, no n x 60 store or memset); otherwise it
 *                  receives exactly what gsb_render_backward writes
 *   grad_uniforms  device memory, OVERWRITTEN with dL/d(each float field of the frame's gsb_uniforms), in fp32.  Non-zero only
 *                  in camera_position[0..2], proj_mat rows 0, 1 and 3 (elements [c*4 + r], r != 2), view_mat rows 0-2
 *                  ([c*4 + r], r != 3), tan_fovx and tan_fovy; every other word (camera_position[3], proj_mat row 2, view_mat
 *                  row 3, width, height) is 0.  Depth order, culls, radii and tile AABBs are step functions of the camera.
 * The gradient treats the UBO's fields as independent inputs: proj_mat already contains view_mat, and tan_fov enters the EWA
 * Jacobian separately from proj_mat, so a caller chains it through its own camera model (gs_b200.uniforms_torch does so
 * for Renderer::makeUniforms).  The camera gradient is reduced without global atomics, per CTA then in one fixed-order pass. */
int gsb_render_backward_camera(gsb_ctx *ctx, const float *vertices, const float *grad_image, size_t row_pitch_bytes,
                               float *grad_vertices, gsb_uniforms *grad_uniforms, void *stream);

/* The backward pass plus the per-Gaussian statistics of adaptive density control (clone / split / prune): the same arguments,
 * preconditions and error codes as gsb_render_backward, and also GSB_ERR_INVALID for a NULL density or when grad_vertices and
 * grad_uniforms are both NULL.
 *   grad_vertices  may be NULL; otherwise it receives exactly what gsb_render_backward writes
 *   grad_uniforms  may be NULL; otherwise it receives exactly what gsb_render_backward_camera writes
 *   density        device memory, n x 4 floats indexed by Gaussian (the upload's row order), ACCUMULATED INTO (the caller zeroes
 *                  it when resetting its statistics).  For every Gaussian that survived the last frame's culls:
 *                  [0] += |(dL/du W/2, dL/dv H/2)|, the screen-space gradient in NDC units (u = ((ndc + 1) W - 1) / 2);
 *                  [1] += |(sum_p |dL_p/du| W/2, sum_p |dL_p/dv| H/2)|, the absolute gradient (absolute value per pixel and
 *                         component before the sum over pixels);
 *                  [2] += 1, zero gradient or not (the number of views);
 *                  [3] = max([3], the frame's pixel radius ceil(3 sqrt(lambda_max))).
 *                  Culled Gaussians' rows are not touched. */
int gsb_render_backward_density(gsb_ctx *ctx, const float *vertices, const float *grad_image, size_t row_pitch_bytes,
                                float *grad_vertices, gsb_uniforms *grad_uniforms, float *density, void *stream);

/* dL/d(background) of the last frame (gsb_set_background): grad_background (device, 3 floats) is OVERWRITTEN with
 * sum over the W x H pixels p of T_final(p) g(p), g from grad_image (as for gsb_render_backward: H x W float4,
 * row_pitch_bytes apart, 0 = tight, A ignored).  It does not depend on the background's value, so it is defined for a frame
 * rendered over black too.  The products are formed exactly and summed in fp64 in an order that depends only on W and H,
 * without atomics, then rounded once: the words are a function of the recorded frame and grad_image alone, whatever the
 * stream, tile-cull level, deterministic switch or arena.  Enqueued on `stream` (NULL = the context's), never synchronises;
 * runs for an empty scene as well.  The same last-frame preconditions and error codes as gsb_render_backward (fp16 SH storage
 * excepted: T_final does not depend on it); GSB_ERR_INVALID for a NULL pointer, a bad pitch or a sharded context. */
int gsb_background_gradient(gsb_ctx *ctx, const float *grad_image, size_t row_pitch_bytes, float *grad_background,
                            void *stream);

/* Photometric loss of a frame against a target, and its gradient (no reference counterpart): the loss of 3DGS training,
 * loss = (1 - lambda) L1 + lambda (1 - SSIM), with SSIM over an 11 x 11 Gaussian window (sigma 1.5) applied with zero
 * padding, C1 = 0.01^2, C2 = 0.03^2 (DESIGN.md section 11).  All pointers are device memory, enqueued on `stream` (NULL = the
 * context's stream); never synchronises.
 *   image        H x W float4, RGBA32F layout (render_torch's / gsb_render's float output), image_pitch apart (0 = tight)
 *   target       H x W in target_fmt: GSB_FORMAT_RGBA32F or GSB_FORMAT_RGBA8 (UNORM8, read as v / 255.0f); A is ignored
 *   lambda_dssim in [0, 1]
 *   grad_image   may be NULL (metrics only); otherwise OVERWRITTEN with d loss / d image, A = 0 -- exactly the grad_image
 *                gsb_render_backward takes
 *   result       4 doubles, OVERWRITTEN: loss, L1, SSIM, MSE (means over the 3 W H RGB values)
 * Needs no scene and leaves the last frame's backward state alone.  No atomics: the result and the gradient are bitwise
 * reproducible for the same inputs, whatever the stream or the pitches.  The context keeps a scratch of 24 B per 32 x 16 tile
 * and, with a gradient, 36 B per pixel, grown with the frame size and freed with the context; calls on different streams
 * share it, so the caller orders them.  GSB_ERR_INVALID for a NULL ctx, image, target or result, W or H of 0, lambda outside
 * [0, 1] or NaN, any other target format, a pitch below the row size, or a pointer or pitch not aligned to 16 B (float4
 * buffers) or 4 B (an RGBA8 target). */
int gsb_image_loss(gsb_ctx *ctx, uint32_t width, uint32_t height, const float *image, size_t image_pitch,
                   const void *target, size_t target_pitch, gsb_format target_fmt, float lambda_dssim,
                   float *grad_image, size_t grad_pitch, double *result, void *stream);

/* Bilateral-grid colour correction of a frame (Wang et al. 2024; gsplat's BilateralGrid; DESIGN.md section 17): the per-image
 * appearance model of training, applied to the rendered frame before the loss.  All pointers are device memory, enqueued on
 * `stream` (NULL = the context's stream); never synchronises.  Needs no scene and leaves the scene and the last frame's
 * backward state alone.
 *   image  H x W float4 (r, g, b, a), RGBA32F layout, image_pitch bytes apart
 *   grid   12 x L x Y x X floats (grid_l, grid_y, grid_x, each in [2, 64]), contiguous in the order [k][l][y][x]: one row of a
 *          torch (N, 12, L, Y, X) parameter.  Coefficient k = 4 c + j is row c (output R, G, B), column j of A = [M | t].
 *          The identity is A = [I | 0] at every node.
 * Per pixel (px, py), every step an fp32 IEEE operation:
 *   ix = ((px + 0.5) / W) (X - 1), iy = ((py + 0.5) / H) (Y - 1), gray = (0.299 r + 0.587 g) + 0.114 b,
 *   iz = clamp(gray, 0, 1) (L - 1) (border padding, align_corners = True in F.grid_sample's terms);
 *   x0 = min(floor(ix), X - 2), fx = ix - x0, and likewise for y and z;
 *   A = the trilinear interpolation of each coefficient over the 8 nodes in lerp form, fmaf(f, hi - lo, lo), along x, then
 *   y, then z (constant nodes give their value exactly);
 *   out_c = ((A_c0 r + A_c1 g) + A_c2 b) + A_c3, out.a = a.
 * An identity grid returns the image's RGB bit for bit for finite inputs (a -0 may become +0).
 * GSB_ERR_INVALID for a NULL ctx, image, grid or out, W or H of 0, a grid dimension outside [2, 64], a pitch below 16 W, a
 * float4 buffer or pitch not 16-B aligned or a grid not 4-B aligned. */
int gsb_bilagrid_apply(gsb_ctx *ctx, uint32_t width, uint32_t height, const float *image, size_t image_pitch,
                       const float *grid, uint32_t grid_x, uint32_t grid_y, uint32_t grid_l,
                       float *out, size_t out_pitch, void *stream);

/* Gradients of gsb_bilagrid_apply from g = d loss / d out (H x W float4, grad_out_pitch apart; its A channel is ignored):
 *   grad_image  H x W float4, OVERWRITTEN with d image_j = sum_c A_cj g_c + w_j (L - 1) sum_c g_c sum_k (dA_ck / d iz) in_k,
 *               in = (r, g, b, 1), w = (0.299, 0.587, 0.114); the luma term is 0 where iz is clamped (gray <= 0 or
 *               gray >= 1), and at an integer iz it uses the cell z0 above.  A = 0: the grad_image gsb_render_backward takes.
 *   grad_grid   12 L Y X floats, OVERWRITTEN with d grid[4 c + j][node] = sum_p w_node(p) g_c(p) in_j(p), w_node the pixel's
 *               trilinear weight of that node.
 * Either may be NULL, not both; each is the same words whether or not the other is requested.  No atomics: the grid gradient
 * is summed in fp64 in an order that depends only on W, H and the grid's shape and rounded once, so every output word is a
 * function of the inputs alone, on any stream and in any context.  With grad_grid the context keeps a scratch of 384 L B per
 * block of up to 32 x 32 pixels within one grid cell, grown with the frame and grid size and freed with the context; calls on
 * different streams share it, so the caller orders them.  The error codes of gsb_bilagrid_apply, with grad_out for out, and
 * GSB_ERR_INVALID also for both gradients NULL or a misaligned grad_image, its pitch or grad_grid. */
int gsb_bilagrid_backward(gsb_ctx *ctx, uint32_t width, uint32_t height, const float *image, size_t image_pitch,
                          const float *grid, uint32_t grid_x, uint32_t grid_y, uint32_t grid_l,
                          const float *grad_out, size_t grad_out_pitch,
                          float *grad_image, size_t grad_image_pitch, float *grad_grid, void *stream);

/* ---- training: one fused Adam step of the resident scene (no reference counterpart; DESIGN.md section 12) ---- */
typedef struct gsb_adam_config {
    float lr[6];                  /* position, scale, opacity, rotation, sh dc (columns 12-14), sh rest (15-59); >= 0 */
    float beta1, beta2, eps;      /* beta in [0, 1), eps >= 0 */
    float bias_correction1;       /* 1 - beta1^t, computed in double and rounded; in (0, 1] */
    float bias_correction2_sqrt;  /* sqrt(1 - beta2^t), likewise */
    uint32_t selective;           /* 0: all n rows; 1: the last frame's survivors only */
} gsb_adam_config;

/* One torch.optim.Adam step (no weight decay) of the scene's raw parameters, which also writes the activated records and
 * the scene words the next frame reads, so no gsb_scene_upload follows it.  All arrays are device memory of n =
 * gsb_scene_size rows of 60 floats in the column layout of the records; enqueued on `stream` (NULL = the context's stream);
 * never synchronises.
 *   params        raw parameters, UPDATED: position (0-2), log scale (4-6), opacity logit (7), quaternion wxyz (8-11, any
 *                 norm), SH (12-59); column 3 is neither read as a parameter nor written
 *   exp_avg, exp_avg_sq  Adam's moments in the same layout, UPDATED (column 3 untouched)
 *   grad_vertices dL/d(activated record) as gsb_render_backward writes it; the step chains it through exp, sigmoid and
 *                 q / |q| of the parameters before the update (a sum of several frames' gradients is fine in dense mode)
 *   vertices      OVERWRITTEN with the activated records of the updated parameters: (p, 1), exp(log s), sigmoid(logit),
 *                 q / |q|, SH -- what the next gsb_render_backward takes
 * The scene words (position, opacity, Sigma, SH) of each updated row become bit-identical to what gsb_scene_upload of that
 * `vertices` row stores.  selective = 0 updates all n rows (torch's semantics: zero-gradient rows decay their moments and
 * move); selective = 1 only the survivors of the last frame, read on the device, and leaves every other row of all five
 * arrays and of the scene untouched; it needs what gsb_render_backward needs of the last frame (recorded, whole, of this
 * scene, not overflowed) and waits for that frame if it is still pending.  No atomics: every output word is a function of
 * the inputs.  The step changes the scene, so the last frame no longer describes it: gsb_render_backward and a second
 * selective step return GSB_ERR_INVALID until the next frame.  Keeps the captured graphs, the instance arena and the grid
 * hints.  GSB_ERR_NO_SCENE before any upload; GSB_ERR_INVALID for a NULL ctx, array or cfg, a sharded context, fp16 SH
 * storage, a learning rate below 0 or NaN, a beta outside [0, 1), eps < 0 or NaN, or a bias correction outside (0, 1]. */
int gsb_adam_step(gsb_ctx *ctx, float *params, float *exp_avg, float *exp_avg_sq, const float *grad_vertices,
                  float *vertices, const gsb_adam_config *cfg, void *stream);

/* ---- training: Mip-Splatting's 3D smoothing filter (Yu et al. 2024; no reference counterpart; DESIGN.md section 18) ---- */
/* The per-Gaussian variance of the filter from the k >= 1 training cameras (Mip-Splatting's compute_3D_filter in this
 * renderer's camera convention).  vertices: n x 60 floats of device memory, 16-B aligned, of which only the positions in
 * columns 0-2 are read; cameras: k gsb_uniforms in host memory; variance: n floats of device memory, OVERWRITTEN.  Per
 * Gaussian i and camera c, in fp32 with the frame's own arithmetic (clip_view of preprocess.comp, then ndc2Pix
 * u = ((ndcx + 1) W - 1) / 2, likewise v, whose half-pixel offset is kept): i is seen by c iff vz > 0.2f,
 * -0.15f W <= u <= 1.15f W and -0.15f H <= v <= 1.15f H (NaN is never seen).  d_i = the least vz over the cameras that see
 * i; rows no camera sees take the largest d of the seen rows; f = the largest focal_x = (float)W / (2.0f tan_fovx) over all
 * k cameras; variance_i = (t t) 0.2f with t = d_i / f.  If no row is seen every variance is 0.  Min and max are exact, so
 * every output word is a function of the inputs: bitwise reproducible on any stream, in any context, on any grid.
 * Enqueued on `stream` (NULL = the context's stream); returns when the variances are written.  Needs no scene and leaves
 * the context's scene and frame state alone, as gsb_init_from_points does; scratch (160 B per camera) is allocated and
 * freed inside the call.  GSB_ERR_INVALID for a NULL ctx, a sharded context, NULL cameras, k == 0, a camera of width or
 * height 0 or whose tan_fovx or tan_fovy is not positive and finite; then, for n > 0, a NULL vertices or variance,
 * vertices not 16-B aligned or variance not 4-B aligned.  n == 0 returns GSB_OK and writes nothing. */
int gsb_filter3d_variance(gsb_ctx *ctx, const float *vertices, uint64_t n, const gsb_uniforms *cameras, uint32_t k,
                          float *variance, void *stream);

/* gsb_adam_step with every updated row's scale and opacity passed through the 3D smoothing filter of its variance v
 * (variance: n floats of device memory, 4-B aligned, finite and >= 0, e.g. from gsb_filter3d_variance; not checked here).
 * With x the raw parameters, in fp32, each operation one IEEE op in this order, for k = 0, 1, 2:
 *   s_k = expf(x_k), q_k = s_k s_k, d_k = q_k + v, e_k = sqrtf(d_k), r_k = q_k / d_k
 *   c = sqrtf((r_0 r_1) r_2), o = sigmoid(x_w), o_f = o c
 * the record's scale is (e_0, e_1, e_2) and its opacity o_f (Mip-Splatting's get_scaling_with_3D_filter and
 * get_opacity_with_3D_filter; the product of per-axis ratios does not underflow as prod s^2 / prod (s^2 + v) does); position,
 * rotation and SH are activated as by gsb_adam_step.  With g the record's gradient and v held constant, the chain rule is
 *   d logit = ((g_w c) o) (1 - o),   d log s_k = (g_k s_k) (s_k / e_k) + (g_w o_f) (v / d_k)
 * A zero variance gives gsb_adam_step's words (a -0 may become +0).  Everything else -- preconditions, selective mode, the
 * scene words (those of gsb_scene_upload of the filtered `vertices`), the error codes, with GSB_ERR_INVALID also for a NULL
 * or misaligned variance -- is gsb_adam_step's. */
int gsb_adam_step_filter3d(gsb_ctx *ctx, float *params, float *exp_avg, float *exp_avg_sq, const float *grad_vertices,
                           float *vertices, const float *variance, const gsb_adam_config *cfg, void *stream);

/* ---- training: a scene initialised from a point cloud (no reference counterpart; DESIGN.md section 13) ---- */
/* Kerbl et al. 2023's initialisation from SfM points: every point becomes an isotropic Gaussian.  All pointers are device
 * memory: xyz and rgb are n x 3 floats, tightly packed; vertices (n x 60 floats) is OVERWRITTEN with activated
 * GSScene::Vertex records, what gsb_scene_upload takes.  Row i:
 *   position    (x, y, z, 1), copied bit for bit
 *   scale       columns 4-6 all hold s = sqrtf(fmaxf(D, 1e-7f)); column 7 is `opacity`
 *   rotation    (1, 0, 0, 0)
 *   SH          sh[c] = (rgb[c] - 0.5f) / SH_C0 for c = 0, 1, 2 (two IEEE operations, rgb not clamped); sh[3..47] = 0
 * D: with d = (dx*dx + dy*dy) + dz*dz, dx = x_j - x_i (likewise y, z), one IEEE fp32 operation each in this order, over the
 * other rows j != i (by index: a duplicate point counts, at distance 0), m = min(3, n - 1) and d_1 <= ... <= d_m the m
 * smallest values of d: D = ((d_1 + d_2) + d_3) / 3.0f, summed in ascending order (for m < 3 the same sum over m terms
 * divided by (float)m); D = 0 for n = 1.  The multiset of the m smallest values is unique, so every output word is a
 * function of the inputs alone: bitwise reproducible on any stream, in any context, on any grid.
 * Enqueued on `stream` (NULL = the context's stream); returns when the records are written.  Needs no scene and leaves the
 * context's scene and frame state alone (control block, arena, captured graphs, backward recording): a gsb_render_backward
 * of the last frame still works after it and gives the same words.  Scratch is allocated and freed inside the call.
 * n == 0 returns GSB_OK and writes nothing.  GSB_ERR_INVALID for a NULL ctx, a NULL pointer, a pointer not aligned to 4 B,
 * n >= 2^30, an opacity outside (0, 1) or NaN, and a coordinate that is not finite (found on the device; nothing is written
 * then). */
int gsb_init_from_points(gsb_ctx *ctx, const float *xyz, const float *rgb, uint64_t n, float opacity, float *vertices,
                         void *stream);

/* ---- training: 3D Gaussian Splatting as Markov Chain Monte Carlo (Kheradmand et al. 2024; no reference counterpart;
 * DESIGN.md section 16) ----
 * Both entries update the resident scene in place, as gsb_adam_step does: params, vertices (and for relocation exp_avg,
 * exp_avg_sq) are device memory of n = gsb_scene_size rows of 60 floats in the column layout of the records, 16-B aligned;
 * every changed row's scene words become bit-identical to what gsb_scene_upload of its `vertices` row stores; the last frame
 * no longer describes the scene (gsb_render_backward and a selective gsb_adam_step return GSB_ERR_INVALID until the next
 * frame) and the captured graphs, the instance arena and the grid hints are kept.  GSB_ERR_NO_SCENE before any upload;
 * GSB_ERR_INVALID for a NULL ctx or array, a misaligned array, a sharded context or fp16 SH storage.
 *
 * SGLD position noise on every row i, enqueued on `stream` (NULL = the context's stream), never synchronises:
 *   x0..x3  Philox4x32-10 (Random123's philox4x32_10) of counter (i, lo32(step), hi32(step), 0), key (lo32(seed), hi32(seed))
 *   u_k     ((float)x_k + 0.5f) * 2^-32, in (0, 1]
 *   eps     eps0 = sqrtf(-2 logf(u0)) cospif(2 u1), eps1 = sqrtf(-2 logf(u0)) sinpif(2 u1), eps2 = sqrtf(-2 logf(u2)) cospif(2 u3)
 *   gate    1.0f / (1.0f + expf(100.0f * (o - 0.005f))), o the scene's opacity word (0 once expf overflows, o >~ 0.892)
 *   d       Sigma e with e_k = eps_k * (gate * scale), each row summed ((S_r0 e0 + S_r1 e1) + S_r2 e2), Sigma the scene's words
 * and p' = params[i, 0:3] + d is written to params columns 0-2, vertices columns 0-2 and the scene's position; nothing else
 * changes.  The noise is a function of (seed, step, row) alone: bitwise reproducible on any grid or stream.  scale is the
 * caller's position learning rate times noise_lr (5e5 in the paper); GSB_ERR_INVALID also for a scale below 0 or not finite. */
int gsb_mcmc_noise(gsb_ctx *ctx, float *params, float *vertices, float scale, uint64_t seed, uint64_t step, void *stream);

/* Relocation: pair j makes row dst[j] (device, k u32) a copy of row src[j] (device, k u32), after the source's opacity and
 * scale are corrected so that the r = 1 + #{j : src[j] = s} copies of a source s render as it did.  In fp64, alpha =
 * vertices[s, 7] and the scales vertices[s, 4..6]:
 *   x      = 1 - (1 - alpha)^(1 / r)
 *   denom  = sum_{j=1..r} (-1)^(j-1) C(r, j) x^j / sqrt(j), with t_j = C(r, j) x^j as t_j = t_(j-1) (r - j + 1) / j x
 *   coeff  = alpha / denom                                          (r is not clamped)
 * each value rounded once to fp32: the source's record gets opacity clamp(x, min_opacity, 1 - 2^-23) and scale s * coeff,
 * its params the logit log(o / (1 - o)) and log scale log(s), in fp64 of those fp32 values; every dst row of the five arrays
 * and of the scene becomes the source's new row; exp_avg and exp_avg_sq are zero on source and dst rows; every other row
 * is untouched.  Each output word is a function of the inputs, whatever the scheduling.  Preconditions, checked on the
 * device before anything is written: every index < n, the dst rows distinct, no dst row also a src row (src may repeat);
 * a violation returns GSB_ERR_INVALID with nothing written.  Enqueued on `stream`; returns once the rows are written (the
 * scratch, n x 8 B, is allocated and freed inside the call).  k == 0 returns GSB_OK and writes nothing (dst and src may then
 * be NULL).  GSB_ERR_INVALID also for k >= n, a NULL or not 4-B aligned dst or src, and min_opacity outside [0, 1) or NaN. */
int gsb_mcmc_relocate(gsb_ctx *ctx, float *params, float *exp_avg, float *exp_avg_sq, float *vertices, const uint32_t *dst,
                      const uint32_t *src, uint64_t k, float min_opacity, void *stream);

/* Size in bytes of a debug buffer for the last frame (0 if unavailable), and its download. */
size_t gsb_debug_size(gsb_ctx *ctx, gsb_buffer which);
int gsb_debug_download(gsb_ctx *ctx, gsb_buffer which, void *dst, size_t bytes);

/* ---- standalone stage entry points (device pointers), used by tests/bench to pin each kernel ---- */
/* Onesweep LSD radix sort of (u64 key, u32 value) pairs over the low `key_bits` bits; stable.
 * Replaces the 8x(hist.comp + sort.comp) loop (Renderer.cpp:598-629).  Sorted data ends in
 * keys/vals (the "Even" buffers, Renderer.cpp:641); keys_tmp/vals_tmp are the "Odd" buffers.
 * Needs no scene and leaves the context's scene and frame state alone (control block, arena, captured graphs, backward
 * recording): a gsb_render_backward of the last frame still works after it and gives the same words.  Its look-back and
 * control words and the pair count are scratch allocated and freed inside the call. */
int gsb_sort_pairs(gsb_ctx *ctx, uint64_t *keys, uint32_t *vals, uint64_t *keys_tmp, uint32_t *vals_tmp,
                   uint64_t m, uint32_t key_bits, void *stream);
/* The same operator over u32 keys (key_bits <= 32): the instantiation the frame itself runs twice -- depth
 * bits over the visible Gaussians, tile ids over the instances (the reference's passes 0-3 and 4-7 of the same
 * loop, Renderer.cpp:598-629).  Leaves the frame state alone like gsb_sort_pairs. */
int gsb_sort_pairs32(gsb_ctx *ctx, uint32_t *keys, uint32_t *vals, uint32_t *keys_tmp, uint32_t *vals_tmp,
                     uint64_t m, uint32_t key_bits, void *stream);

/* ---- one frame over several GPUs of an NVSwitch domain (SURVEY 8b `gs_create_sharded`, 8e) ----
 * No reference counterpart (the reference is single-GPU).  The scene is sharded by Gaussian index (rank r holds and
 * projects slice r), the frame by tile rows (rank d sorts and blends band d); survivors travel from their slice's rank
 * to their band's rank(s) and the blended bands to every rank's whole-frame buffer by stores into peer-mapped memory
 * (NVLink), ordered by mailbox words -- no collective call in the frame.  Every rank ends the frame holding the whole
 * framebuffer, bit-identical to a single-GPU gsb_render of the same scene and camera.
 *
 * (a) one process drives all GPUs.  `devices` = ndev CUDA device ids (NULL: 0 .. ndev-1); an id may repeat (several
 *     ranks on one GPU -- how the single-GPU tests cover the protocol).  vertices = all n GSScene::Vertex records. */
typedef struct gsb_group gsb_group;
int gsb_group_create(int ndev, const int *devices, gsb_group **out);
void gsb_group_destroy(gsb_group *g);
int gsb_group_size(const gsb_group *g);
gsb_ctx *gsb_group_context(gsb_group *g, int rank); /* per-rank context: gsb_set_mode / _tile_cull / _timers, gsb_get_stats */
const char *gsb_group_last_error(const gsb_group *g);
int gsb_group_scene_upload(gsb_group *g, const float *vertices, uint64_t n, gsb_memory mem);
/* Renders the frame on all GPUs and waits; grows instance arenas and re-renders on overflow like gsb_render.  `out` (may be
 * NULL) receives the whole frame from rank 0's copy; gsb_shard_frame(gsb_group_context(g, r)) is rank r's device copy. */
int gsb_group_render(gsb_group *g, const gsb_uniforms *ubo, void *out, size_t row_pitch_bytes, gsb_memory out_mem, gsb_format fmt);
int gsb_group_render_async(gsb_group *g, const gsb_uniforms *ubo, gsb_format fmt); /* enqueue only, never synchronises */

/* (b) one process per GPU (torchrun / MPI).  Rank 0 calls gsb_shard_unique_id and the host program distributes the 128
 *     bytes by any means; NCCL (dlopen'ed libnccl.so.2, used only here) bootstraps the group and carries the cudaIpc handles
 *     of the exchange windows.  GSB_SHARD_GATHER=nccl reassembles the framebuffer with one in-place ncclAllGather instead
 *     of the blend's peer stores (the baseline the fused path is measured against). */
typedef struct gsb_shard_id { unsigned char bytes[128]; } gsb_shard_id;
int gsb_shard_unique_id(gsb_shard_id *out);
const char *gsb_shard_last_error(void); /* text of the last gsb_shard_unique_id / gsb_create_sharded / gsb_group_create error */
int gsb_create_sharded(int device, int rank, int world, const gsb_shard_id *id, gsb_ctx **out); /* gsb_destroy frees it */
int gsb_shard_rank(const gsb_ctx *ctx);
int gsb_shard_world(const gsb_ctx *ctx);
/* Slice of rank `rank`: Gaussians [first, first + count) with S = ceil(n_total / world), first = rank * S. */
int gsb_shard_slice(uint64_t n_total, int rank, int world, uint64_t *first, uint64_t *count);
/* Tile rows [begin, end) of the frame this rank blends at image height `height` (equal-height bands). */
int gsb_shard_band(const gsb_ctx *ctx, uint32_t height, uint32_t *row_begin, uint32_t *row_end);
/* slice_vertices = this rank's slice only (gsb_shard_slice), n_total = size of the whole scene. */
int gsb_scene_upload_sharded(gsb_ctx *ctx, const float *slice_vertices, uint64_t n_total, gsb_memory mem);
/* Collective: every rank calls it with the same ubo / fmt.  Waits for the frame; `out` (may be NULL) receives this rank's
 * copy of the WHOLE frame.  The first call at a new frame size (re)allocates and re-exchanges the windows. */
int gsb_render_sharded(gsb_ctx *ctx, const gsb_uniforms *ubo, void *out, size_t row_pitch_bytes, gsb_memory out_mem,
                       gsb_format fmt, void *stream);
int gsb_render_sharded_async(gsb_ctx *ctx, const gsb_uniforms *ubo, gsb_format fmt, void *stream);
/* This rank's device copy of the last whole frame (tight pitch); valid until the second-next render call. */
const void *gsb_shard_frame(const gsb_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* GS_B200_H */
