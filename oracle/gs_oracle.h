/*
 * gs_oracle.h -- CPU oracle for the 3DGS.cpp per-frame compute path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load it, and only as the checker (or as the timed CPU baseline).
 *
 * PARITY: the reference (shg8/3DGS.cpp @ f614d66) ships no tests, golden vectors or
 * fixtures for this path (SURVEY.md section 4 / 8c) and needs Vulkan to run.  This file
 * is a restatement "by formula" of the cited shader / host lines, in fp32 with no FMA
 * contraction (-ffp-contract=off).
 *   PINNED: the shader stages (A1, A3-A8) are compared bit for bit with the reference's
 *   own shader source run on the CPU (ref_driver.cpp, tests/test_ref_shaders.py), except
 *   the arithmetic GLSL leaves to the implementation (glsl_shim.hpp, DESIGN.md section 2).
 *   UNPINNED: the host math (A0 gso_load_records / gso_load_ply, A2
 *   gso_uniforms_from_camera / gso_camera_translate) comes from glm 1.0.0
 *   (CMakeLists.txt:31-36, not vendored) and stays a restatement of glm's formulas.
 *
 * All matrices are column-major like GLSL/glm: m[col*R + row].
 */
#ifndef GS_ORACLE_H
#define GS_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Renderer::UniformBuffer, src/Renderer.h:21-29 == preprocess.comp:16-24 (std140, 160 B). */
typedef struct gso_uniforms {
    float camera_position[4];
    float proj_mat[16];
    float view_mat[16];
    uint32_t width;
    uint32_t height;
    float tan_fovx;
    float tan_fovy;
} gso_uniforms;

/* VertexAttribute, src/shaders/common.glsl:42-49 == Renderer.h:31-38 (64 B). */
typedef struct gso_attr {
    float conic_opacity[4];
    float color_radii[4];
    uint32_t aabb[4];
    float uv[2];
    float depth;
    uint32_t magic;
} gso_attr;

#define GSO_VERTEX_FLOATS 60  /* GSScene::Vertex, src/GSScene.h:41-46: pos4, scale_opacity4, rot4, sh48 */
#define GSO_RECORD_FLOATS 62  /* VertexStorage, src/GSScene.cpp:17-24 */
#define GSO_MAGIC 0x4d415449u /* common.glsl:14 */

/* exp() flavour used by the blend stage:
 *   0 = libm expf (default; the plain restatement of GLSL exp, render.comp:77)
 *   1 = "shared-definition" exp: a fixed sequence of correctly-rounded IEEE ops
 *       (Cody-Waite reduction + degree-5 Horner with fmaf) that the CUDA kernel
 *       reproduces bit for bit (the kernel's per-Gaussian early skip only drops pairs
 *       whose alpha is < 1/255 under this same exp, so it is not part of the definition).
 *       GLSL leaves exp precision implementation-defined, so both are valid
 *       readings of the reference; tests check 0-vs-1 agree to 1e-4. */
typedef struct gso_synth_params { /* same fields as the product's gsh_synth_params (host/gs_b200_host.h) */
    float center[3], half_extent[3];
    float log_scale_min, log_scale_max, opacity_min, opacity_max, sh_dc_range, sh_rest_sigma;
} gso_synth_params;
void gso_synth_records(uint64_t seed, uint64_t first, uint64_t n, const gso_synth_params *p, float *records);
void gso_set_num_threads(int n);
/* tests only: mask = H*W bytes (caller-zeroed) or NULL to switch the probe off; see gs_oracle.c */
void gso_set_step_probe(uint8_t *mask, float rel_delta);
void gso_set_exp_mode(int mode);
int gso_get_exp_mode(void);
float gso_exp_shared(float x);

/* A0: GSScene::load record activation, src/GSScene.cpp:36-59. rec: n*62 floats, vtx: n*60 floats. */
void gso_load_records(const float *rec, uint64_t n, float *vtx);
/* PLY header parse + load, src/GSScene.cpp:26-68,99-149. Returns malloc'd n*60 floats (caller frees
 * with gso_free) or NULL. */
float *gso_load_ply(const char *path, uint64_t *n_out);
void gso_free(void *p);

/* A1: precomp_cov3d.comp:25-48 with scale_factor (GSScene.cpp:176 passes 1.0). cov: n*6 floats. */
void gso_cov3d(const float *vtx, uint64_t n, float scale_factor, float *cov);

/* A2: Renderer::updateUniforms, src/Renderer.cpp:719-754. quat is (w,x,y,z). */
void gso_uniforms_from_camera(const float pos[3], const float quat_wxyz[4], float fov_deg,
                              float near_plane, float far_plane, uint32_t width, uint32_t height,
                              gso_uniforms *out);
/* Renderer::Camera::translate, src/Renderer.h:47-49 (glm quat * vec3). */
void gso_camera_translate(float pos[3], const float quat_wxyz[4], const float t[3]);

/* A3: preprocess.comp:115-182.  attr: n entries; tiles: n u32.  Culled entries are zeroed
 * (the reference leaves stale data there; only color_radii.w = 0 and tiles = 0 are defined).
 * tile_row_begin/end clip the AABB's y range to a band of tile rows before counting
 * (NOT in the reference: the multi-GPU sharding of SURVEY 8e; pass 0, UINT32_MAX for the
 * reference behaviour). */
void gso_preprocess(const float *vtx, const float *cov, uint64_t n, const gso_uniforms *u,
                    uint32_t tile_row_begin, uint32_t tile_row_end, gso_attr *attr, uint32_t *tiles);

/* A4: prefix_sum.comp:32-58 + Renderer.cpp:497-526: inclusive scan; returns M = scan[n-1]. */
uint64_t gso_scan_inclusive(const uint32_t *tiles, uint64_t n, uint32_t *scan);

/* A5: preprocess_sort.comp:31-60. keys/vals have M entries. tileX = ceil(W/16). */
void gso_emit_keys(const gso_attr *attr, const uint32_t *scan, uint64_t n, uint32_t tileX,
                   uint64_t *keys, uint32_t *vals);

/* A6: sort/hist.comp + sort/sort.comp, Renderer.cpp:598-629: stable LSD radix, 8 passes x 8 bits,
 * result back in the input ("Even") buffers. */
void gso_sort(uint64_t *keys, uint32_t *vals, uint64_t m);

/* A7: tile_boundary.comp:22-50 after fillBuffer(0) (Renderer.cpp:633). ranges: 2*T u32. */
void gso_tile_ranges(const uint64_t *keys, uint64_t m, uint32_t num_tiles, uint32_t *ranges);

/* A8: render.comp:30-99. rgba: H*W*4 floats (row-major, alpha = 1). Only pixel rows inside
 * tile rows [tile_row_begin, tile_row_end) are written.  consumed (may be NULL): per-tile
 * count of run entries read before every pixel of the tile had terminated (for the
 * algorithmic-bytes figure of SURVEY 8d). */
void gso_blend(const gso_attr *attr, const uint32_t *vals, const uint32_t *ranges, uint32_t width,
               uint32_t height, uint32_t tile_row_begin, uint32_t tile_row_end, float *rgba,
               uint32_t *consumed);

/* Swapchain image conversion: vec4 -> B8G8R8A8_UNORM (src/vulkan/Swapchain.cpp:24): clamp to [0,1],
 * *255, round to nearest even.  bgra != 0 gives BGRA byte order, else RGBA. */
void gso_pack_unorm8(const float *rgba, uint64_t npix, int bgra, uint8_t *out);

typedef struct gso_frame {
    uint64_t n, m;
    uint32_t width, height, tiles_x, tiles_y;
    gso_attr *attr;     /* n */
    uint32_t *tiles;    /* n */
    uint32_t *scan;     /* n */
    uint64_t *keys;     /* m, sorted */
    uint32_t *vals;     /* m, sorted */
    uint64_t *keys_unsorted; /* m */
    uint32_t *vals_unsorted; /* m */
    uint32_t *ranges;   /* 2*T */
    uint32_t *consumed; /* T */
    float *rgba;        /* H*W*4 */
    double t_stage[6];  /* seconds: preprocess, prefix_sum, preprocess_sort, sort, tile_boundary, render */
} gso_frame;

/* The whole frame, Renderer::draw() order (src/Renderer.cpp:366-426). Returns 0 on success. */
int gso_render_frame(const float *vtx, const float *cov, uint64_t n, const gso_uniforms *u,
                     uint32_t tile_row_begin, uint32_t tile_row_end, gso_frame *out);
void gso_frame_free(gso_frame *f);

int gso_num_threads(void);

#ifdef __cplusplus
}
#endif
#endif
