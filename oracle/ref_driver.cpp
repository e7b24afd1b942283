/*
 * ref_driver.cpp -- runs the reference renderer's own compute shaders on the CPU, translated by glsl_to_cpp.py onto
 * glsl_shim.hpp, dispatch by dispatch as the reference's host code records them (src/Renderer.cpp of shg8/3DGS.cpp
 * @ f614d66).  TEST INFRASTRUCTURE ONLY: it pins the oracle (gs_oracle.c) to the shaders' code rather than to a reading
 * of it (tests/test_ref_shaders.py), and the CUDA frame to both (tests/test_gpu_ref_shaders.py).
 *
 * Built by `make -C oracle ref` into oracle/_ref/libgsref.so when the reference tree is present.  One C entry per stage,
 * plus a whole frame in Renderer::draw() order.  Buffers are the caller's memory, bound with the sizes Renderer.cpp
 * gives them, so `.length()` in a shader is what it is on the device.
 */
#include "glsl_shim.hpp"

#include "gs_oracle.h"

#include "precomp_cov3d.inc"
#include "preprocess.inc"
#include "prefix_sum.inc"
#include "preprocess_sort.inc"
#include "hist.inc"
#include "sort.inc"
#include "tile_boundary.inc"
#include "render.inc"

using namespace glsl;

static_assert(sizeof(sh_preprocess::Vertex) == 240, "Vertex is 240 B in std430 (gso: 60 floats)");
static_assert(sizeof(sh_preprocess::VertexAttribute) == 64, "VertexAttribute is 64 B in std430 (gso_attr)");
static_assert(sizeof(sh_preprocess::VertexAttribute) == sizeof(gso_attr), "VertexAttribute matches gso_attr");

namespace {

/* vkCmdDispatch(gx, gy, 1) of one translated shader */
void dispatch(void (*entry)(), uvec3 local, uint gx, uint gy, bool cooperative) {
    for (uint y = 0; y < gy; y++)
        for (uint x = 0; x < gx; x++) run_workgroup(entry, uvec3(x, y, 0), uvec3(gx, gy, 1), local, cooperative);
}

uint groups_256(uint64_t n) { return (uint)((n + 255) / 256); } /* Renderer.cpp:477 numGroups */

/* Renderer.cpp:137 numRadixSortBlocksPerWorkgroup (every platform but Apple) */
constexpr uint kSortBlocksPerWorkgroup = 32;

mat4 mat4_of(const float *m) {
    mat4 o;
    for (int c = 0; c < 4; c++) o[c] = vec4(m[c * 4 + 0], m[c * 4 + 1], m[c * 4 + 2], m[c * 4 + 3]);
    return o;
}

} // namespace

extern "C" {

void gsr_set_exp_mode(int mode) { g_exp_mode = mode; }

/* precomp_cov3d.comp, dispatched as GSScene.cpp:174-180 does: ceil(N / 256) groups, push constant scale_factor. */
void gsr_cov3d(const float *vtx, uint64_t n, float scale_factor, float *cov) {
    namespace S = sh_precomp_cov3d;
    S::vertices.bind((void *)vtx, n);
    S::cov3ds.bind(cov, n * 6);
    S::scale_factor = scale_factor;
    dispatch(S::glsl_main, S::LOCAL_SIZE, groups_256(n), 1, false);
}

/* preprocess.comp, Renderer.cpp:483-486.  attr and tiles are the caller's buffers and are not cleared first: a row the
 * shader returns from early keeps whatever the caller put in the fields it does not write. */
void gsr_preprocess(const float *vtx, const float *cov, uint64_t n, const gso_uniforms *u, gso_attr *attr,
                    uint32_t *tiles) {
    namespace S = sh_preprocess;
    S::vertices.bind((void *)vtx, n);
    S::cov3ds.bind((void *)cov, n * 6);
    S::attr.bind(attr, n);
    S::tiles_overlap.bind(tiles, n);
    S::camera_position = vec4(u->camera_position[0], u->camera_position[1], u->camera_position[2],
                              u->camera_position[3]);
    S::proj_mat = mat4_of(u->proj_mat);
    S::view_mat = mat4_of(u->view_mat);
    S::width = u->width;
    S::height = u->height;
    S::tan_fovx = u->tan_fovx;
    S::tan_fovy = u->tan_fovy;
    dispatch(S::glsl_main, S::LOCAL_SIZE, groups_256(n), 1, false);
}

/* The prefix sum of Renderer.cpp:489-523: copy tiles into Ping, then ceil(log2(N)) + 1 Hillis-Steele dispatches that
 * alternate Ping -> Pong and Pong -> Ping.  `scan` receives the buffer Renderer.cpp reads the total from and binds to
 * preprocess_sort (:517-523, :579): Ping if iters is even, else Pong.  Returns scan[N - 1], numInstances (:538). */
uint32_t gsr_scan(const uint32_t *tiles, uint64_t n, uint32_t *scan) {
    namespace S = sh_prefix_sum;
    if (n == 0) return 0;
    std::vector<uint32_t> ping(tiles, tiles + n), pong(n, 0);
    S::src.bind(ping.data(), n);
    S::dst.bind(pong.data(), n);
    const auto iters = static_cast<uint32_t>(std::ceil(std::log2(static_cast<float>(n)))); /* :500 */
    for (uint32_t timestep = 0; timestep <= iters; timestep++) {                             /* :501-514 */
        S::timestep = timestep;
        dispatch(S::glsl_main, S::LOCAL_SIZE, groups_256(n), 1, false);
    }
    const std::vector<uint32_t> &out = iters % 2 == 0 ? ping : pong;
    std::memcpy(scan, out.data(), n * 4);
    return out[n - 1];
}

/* preprocess_sort.comp, Renderer.cpp:577-587: keys and payloads into the Even buffers, push constant tileX. */
void gsr_emit_keys(const gso_attr *attr, const uint32_t *scan, uint64_t n, uint32_t tile_x, uint64_t m,
                   uint64_t *keys, uint32_t *vals) {
    namespace S = sh_preprocess_sort;
    S::attr.bind((void *)attr, n);
    S::prefixSum.bind((void *)scan, n);
    S::keys.bind(keys, m);
    S::payloads.bind(vals, m);
    S::tileX = tile_x;
    dispatch(S::glsl_main, S::LOCAL_SIZE, groups_256(n), 1, false);
}

/* The 8 hist.comp + sort.comp passes of Renderer.cpp:598-629: pass i reads Even and writes Odd when i is even, the
 * reverse when odd, so the sorted pairs end in the caller's (Even) buffers (:641).  Each workgroup covers
 * kSortBlocksPerWorkgroup blocks of 256 keys (:600-601). */
void gsr_sort(uint64_t *keys, uint32_t *vals, uint64_t m) {
    namespace H = sh_hist;
    namespace R = sh_sort;
    if (m == 0) return;
    uint invocation_size = (uint)((m + kSortBlocksPerWorkgroup - 1) / kSortBlocksPerWorkgroup);
    invocation_size = (invocation_size + 255) / 256;
    std::vector<uint64_t> keys_odd(m);
    std::vector<uint32_t> vals_odd(m);
    std::vector<uint32_t> hist((size_t)invocation_size * 256);
    for (int i = 0; i < 8; i++) {
        uint64_t *kin = i % 2 == 0 ? keys : keys_odd.data(), *kout = i % 2 == 0 ? keys_odd.data() : keys;
        uint32_t *vin = i % 2 == 0 ? vals : vals_odd.data(), *vout = i % 2 == 0 ? vals_odd.data() : vals;
        H::g_num_elements = R::g_num_elements = (uint)m; /* :603-607 */
        H::g_num_blocks_per_workgroup = R::g_num_blocks_per_workgroup = kSortBlocksPerWorkgroup;
        H::g_shift = R::g_shift = (uint)(i * 8);
        H::g_num_workgroups = R::g_num_workgroups = invocation_size;
        H::g_elements_in.bind(kin, m);
        H::g_histograms.bind(hist.data(), hist.size());
        dispatch(H::glsl_main, H::LOCAL_SIZE, invocation_size, 1, true); /* :612 */
        R::g_elements_in.bind(kin, m);
        R::g_elements_out.bind(kout, m);
        R::g_payload_in.bind(vin, m);
        R::g_payload_out.bind(vout, m);
        R::g_histograms.bind(hist.data(), hist.size());
        dispatch(R::glsl_main, R::LOCAL_SIZE, invocation_size, 1, true); /* :620 */
    }
}

/* fillBuffer(0) then tile_boundary.comp, Renderer.cpp:633-648. */
void gsr_tile_ranges(const uint64_t *keys, uint64_t m, uint32_t num_tiles, uint32_t *ranges) {
    namespace S = sh_tile_boundary;
    std::memset(ranges, 0, (size_t)num_tiles * 8);
    S::keys.bind((void *)keys, m);
    S::boundaries.bind(ranges, (uint64_t)num_tiles * 2);
    S::numInstances = (uint)m;
    dispatch(S::glsl_main, S::LOCAL_SIZE, groups_256(m), 1, false);
}

/* render.comp, Renderer.cpp:654-677: one 16x16 workgroup per tile, push constants width and height, into an RGBA32F
 * image of width x height texels. */
void gsr_blend(const gso_attr *attr, uint64_t n, const uint32_t *vals, uint64_t m, const uint32_t *ranges,
               uint32_t width, uint32_t height, float *rgba) {
    namespace S = sh_render;
    const uint tiles_x = (width + 15) / 16, tiles_y = (height + 15) / 16;
    S::attr.bind((void *)attr, n);
    S::boundaries.bind((void *)ranges, (uint64_t)tiles_x * tiles_y * 2);
    S::sorted_vertices.bind((void *)vals, m);
    S::output_image.data = rgba;
    S::output_image.width = (int)width;
    S::output_image.height = (int)height;
    S::width = width;
    S::height = height;
    dispatch(S::glsl_main, S::LOCAL_SIZE, tiles_x, tiles_y, false);
}

/* The whole frame: precomp_cov3d (GSScene::load, scale factor 1), then Renderer::draw()'s stages.  Fills a gso_frame
 * (oracle/gs_oracle.h) the caller releases with gsr_frame_free; rgba is zero where nothing is stored. */
int gsr_render_frame(const float *vtx, uint64_t n, const gso_uniforms *u, gso_frame *f) {
    std::memset(f, 0, sizeof *f);
    f->n = n;
    f->width = u->width;
    f->height = u->height;
    f->tiles_x = (u->width + 15) / 16;
    f->tiles_y = (u->height + 15) / 16;
    const size_t T = (size_t)f->tiles_x * f->tiles_y, nn = n ? n : 1;
    float *cov = (float *)std::calloc(nn * 6, 4);
    f->attr = (gso_attr *)std::calloc(nn, sizeof(gso_attr));
    f->tiles = (uint32_t *)std::calloc(nn, 4);
    f->scan = (uint32_t *)std::calloc(nn, 4);
    f->ranges = (uint32_t *)std::calloc(T ? T * 2 : 2, 4);
    f->consumed = (uint32_t *)std::calloc(T ? T : 1, 4);
    f->rgba = (float *)std::calloc((size_t)u->width * u->height * 4 + 4, sizeof(float));
    if (!cov || !f->attr || !f->tiles || !f->scan || !f->ranges || !f->consumed || !f->rgba) {
        std::free(cov);
        return -1;
    }
    gsr_cov3d(vtx, n, 1.0f, cov);
    gsr_preprocess(vtx, cov, n, u, f->attr, f->tiles);
    f->m = gsr_scan(f->tiles, n, f->scan);
    const size_t mm = f->m ? f->m : 1;
    f->keys = (uint64_t *)std::calloc(mm, 8);
    f->vals = (uint32_t *)std::calloc(mm, 4);
    f->keys_unsorted = (uint64_t *)std::calloc(mm, 8);
    f->vals_unsorted = (uint32_t *)std::calloc(mm, 4);
    if (!f->keys || !f->vals || !f->keys_unsorted || !f->vals_unsorted) {
        std::free(cov);
        return -1;
    }
    gsr_emit_keys(f->attr, f->scan, n, f->tiles_x, f->m, f->keys, f->vals);
    std::memcpy(f->keys_unsorted, f->keys, f->m * 8);
    std::memcpy(f->vals_unsorted, f->vals, f->m * 4);
    gsr_sort(f->keys, f->vals, f->m);
    gsr_tile_ranges(f->keys, f->m, (uint32_t)T, f->ranges);
    gsr_blend(f->attr, n, f->vals, f->m, f->ranges, u->width, u->height, f->rgba);
    std::free(cov);
    return 0;
}

void gsr_frame_free(gso_frame *f) {
    std::free(f->attr);
    std::free(f->tiles);
    std::free(f->scan);
    std::free(f->keys);
    std::free(f->vals);
    std::free(f->keys_unsorted);
    std::free(f->vals_unsorted);
    std::free(f->ranges);
    std::free(f->consumed);
    std::free(f->rgba);
    std::memset(f, 0, sizeof *f);
}

} // extern "C"
