// gs_viewer_headless -- the reference viewer's command line (apps/viewer/main.cpp:12-98) without a window:
//   gs_viewer_headless [-d DEVICE] [-w WIDTH] [-h HEIGHT] [-v] [--frames N] [--camera x,y,z[,qw,qx,qy,qz]]
//                      [--fov DEG] [--camera-path poses.txt] [--mode exact|fast] [--cull [LEVEL]] [--antialiased]
//                      [--sh-degree N] [--background r,g,b] [--fisheye fx,fy,cx,cy[,k1,k2,k3,k4[,max_theta_deg]]]
//                      [--opencv fx,fy,cx,cy[,k1,k2,p1,p2[,max_theta_deg]]] [--ortho fx,fy,cx,cy] [--out image.ppm]
//                      [--float-out image.pfm] scene.ply
// --antialiased: gsb_set_antialiased (opacity compensated for the 0.3 px dilation, as scenes trained that way expect).
// --sh-degree N: gsb_set_sh_degree (0..3; the colour sums the SH bands <= N only, e.g. for a scene trained at a lower degree).
// --background r,g,b: gsb_set_background (e.g. 1,1,1 for an object scene trained over white; default black).
// --fisheye fx,fy,cx,cy[,k1,k2,k3,k4[,max_theta_deg]]: gsb_set_camera_model with an OpenCV-fisheye lens (pixel (i, j) sampled at
// (i, j): COLMAP's cx - 0.5); without max_theta_deg, the largest angle up to 175 deg at which theta_d still increases.
// --opencv fx,fy,cx,cy[,k1,k2,p1,p2[,max_theta_deg]]: the same with COLMAP's OPENCV (radial-tangential) lens; without
// max_theta_deg, the largest angle up to 80 deg at which r R(r^2) still increases (python's opencv_camera default).
// --ortho fx,fy,cx,cy: gsb_set_camera_model with the orthographic camera, fx and fy in pixels per world unit (e.g. a top-down
// orthophoto of an aerial scene).
// --camera-path: one pose per line `x y z qw qx qy qz [fov]` (# comments); `--frames` frames are rendered at each pose
// and one JSON line is printed per pose (SURVEY 8d: record M for every timed camera).
// Loads the .ply through GSScene, renders N frames through Renderer::draw() (B8G8R8A8 like the swapchain),
// prints the six per-stage timers + `instances` (Renderer.cpp:85-100,540) as one JSON line per run and
// optionally writes the last frame as a binary PPM (8-bit, what the swapchain would show) and / or as a PFM (float32 RGB, the
// unquantised blend render.comp:98 stores: what the 1e-4 parity tolerance is defined on).  The first JSON line also carries
// the load times (file read + activation, upload + cov3D ingest).  Environment: VKGS_PHYSICAL_DEVICE like the viewer.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "Renderer.h"

static void usage() {
    std::puts("usage: gs_viewer_headless [-d device] [-w width] [-h height] [-v] [--frames n] [--camera x,y,z[,qw,qx,qy,qz]]\n"
              "                          [--fov deg] [--camera-path poses.txt] [--mode exact|fast] [--cull [0|1|2]] [--antialiased]\n"
              "                          [--sh-degree 0|1|2|3] [--background r,g,b] [--fisheye fx,fy,cx,cy[,k1,k2,k3,k4[,max_theta_deg]]]\n"
              "                          [--opencv fx,fy,cx,cy[,k1,k2,p1,p2[,max_theta_deg]]] [--ortho fx,fy,cx,cy]\n"
              "                          [--out image.ppm] [--float-out image.pfm] scene.ply");
}

int main(int argc, char** argv) {
    Renderer::Configuration cfg;
    std::string out_path, float_path, scene, path_file;
    int cull_level = 0, sh_degree = 3;
    uint32_t frames = 1;
    bool verbose = false, cull = false, antialiased = false, background = false;
    float bg[3] = {0, 0, 0};
    uint32_t lens_kind = GSB_CAMERA_PINHOLE;  // --fisheye, --opencv or --ortho
    float lens[9] = {0, 0, 0, 0, 0, 0, 0, 0, -1.0f};  // fx fy cx cy k[0..3] max_theta_deg (< 0: the default)
    float cam[7] = {0, 0, 0, 1, 0, 0, 0};
    float fov = 45.0f;
    if (const char* env = std::getenv("VKGS_PHYSICAL_DEVICE")) cfg.physicalDeviceId = static_cast<uint8_t>(std::atoi(env));
    for (int i = 1; i < argc; i++) {
        const std::string a = argv[i];
        auto next = [&]() -> const char* {
            if (i + 1 >= argc) {
                usage();
                std::exit(1);
            }
            return argv[++i];
        };
        if (a == "-d" || a == "--device") cfg.physicalDeviceId = static_cast<uint8_t>(std::atoi(next()));
        else if (a == "-w" || a == "--width") cfg.width = static_cast<uint32_t>(std::atoi(next()));
        else if (a == "-h" || a == "--height") cfg.height = static_cast<uint32_t>(std::atoi(next()));
        else if (a == "-v" || a == "--verbose") verbose = true;
        else if (a == "--frames") frames = static_cast<uint32_t>(std::atoi(next()));
        else if (a == "--fov") fov = static_cast<float>(std::atof(next()));
        else if (a == "--mode") cfg.mode = std::string(next()) == "fast" ? GSB_MODE_FAST : GSB_MODE_EXACT;
        else if (a == "--cull") {
            cull = true;
            cull_level = 1;
            if (i + 1 < argc && std::strlen(argv[i + 1]) == 1 && argv[i + 1][0] >= '0' && argv[i + 1][0] <= '2') cull_level = argv[++i][0] - '0';
        } else if (a == "--antialiased") antialiased = true;
        else if (a == "--sh-degree") {
            const std::string d = next();
            if (d.size() != 1 || d[0] < '0' || d[0] > '3') {
                usage();
                return 1;
            }
            sh_degree = d[0] - '0';
        }
        else if (a == "--background") {
            background = true;
            int k = 0;
            for (char* tok = std::strtok(const_cast<char*>(next()), ","); tok && k < 3; tok = std::strtok(nullptr, ",")) bg[k++] = static_cast<float>(std::atof(tok));
        }
        else if (a == "--fisheye" || a == "--opencv" || a == "--ortho") {
            lens_kind = a == "--fisheye" ? GSB_CAMERA_FISHEYE : a == "--opencv" ? GSB_CAMERA_OPENCV : GSB_CAMERA_ORTHO;
            int k = 0;
            for (char* tok = std::strtok(const_cast<char*>(next()), ","); tok && k < 9; tok = std::strtok(nullptr, ",")) lens[k++] = static_cast<float>(std::atof(tok));
            if (k < 4) {
                usage();
                return 1;
            }
        }
        else if (a == "--float-out") float_path = next();
        else if (a == "--out") out_path = next();
        else if (a == "--camera-path") path_file = next();
        else if (a == "--camera") {
            int k = 0;
            for (char* tok = std::strtok(const_cast<char*>(next()), ","); tok && k < 7; tok = std::strtok(nullptr, ",")) cam[k++] = static_cast<float>(std::atof(tok));
        } else if (a == "--help") {
            usage();
            return 0;
        } else scene = a;
    }
    if (scene.empty()) {
        usage();
        return 1;
    }
    cfg.scene = scene;
    try {  // the viewer catches at top level and logs (main.cpp:94-105)
        Renderer renderer(cfg);
        const auto t0 = std::chrono::steady_clock::now();
        renderer.initialize();
        const double load_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (cull && gsb_set_tile_cull(renderer.context(), cull_level) != GSB_OK) throw std::runtime_error("gsb_set_tile_cull failed");
        if (antialiased && gsb_set_antialiased(renderer.context(), 1) != GSB_OK) throw std::runtime_error("gsb_set_antialiased failed");
        if (sh_degree != 3 && gsb_set_sh_degree(renderer.context(), sh_degree) != GSB_OK) throw std::runtime_error("gsb_set_sh_degree failed");
        if (background && gsb_set_background(renderer.context(), bg) != GSB_OK) throw std::runtime_error("gsb_set_background failed");
        if (lens_kind != GSB_CAMERA_PINHOLE) {
            gsb_camera_model m{};
            m.kind = lens_kind;
            m.fx = lens[0], m.fy = lens[1], m.cx = lens[2], m.cy = lens[3];
            for (int k = 0; k < 4; k++) m.k[k] = lens[4 + k];
            if (lens[8] >= 0.0f) {
                m.max_theta = lens[8] * static_cast<float>(M_PI / 180.0);
            } else if (lens_kind == GSB_CAMERA_ORTHO) {  // no field-of-view cull: the setter names any extra word it refuses
                m.max_theta = 0.0f;
            } else if (lens_kind == GSB_CAMERA_OPENCV) {  // the smallest positive root u0 of 1 + 3 k1 u + 5 k2 u^2, less 1e-4
                const double k1 = m.k[0], k2 = m.k[1], cap = 80.0 * M_PI / 180.0;
                double u0 = INFINITY;
                if (k2 == 0.0) {
                    if (k1 < 0.0) u0 = -1.0 / (3.0 * k1);
                } else if (9.0 * k1 * k1 - 20.0 * k2 >= 0.0) {
                    const double sq = std::sqrt(9.0 * k1 * k1 - 20.0 * k2);
                    for (double d : {3.0 * k1 + sq, 3.0 * k1 - sq})
                        if (d != 0.0 && -2.0 / d > 0.0) u0 = std::fmin(u0, -2.0 / d);
                }
                m.max_theta = static_cast<float>(std::isfinite(u0) ? std::fmin(cap, std::atan(std::sqrt(u0 * (1.0 - 1e-4)))) : cap);
            } else {  // walk out in 0.1 mrad steps while d theta_d / d theta stays positive
                const double cap = 175.0 * M_PI / 180.0;
                double t = 0.0;
                for (; t + 1e-4 <= cap; t += 1e-4) {
                    const double u = (t + 1e-4) * (t + 1e-4);
                    if (!(1.0 + u * (3.0 * m.k[0] + u * (5.0 * m.k[1] + u * (7.0 * m.k[2] + u * 9.0 * m.k[3]))) > 0.0)) break;
                }
                m.max_theta = static_cast<float>(t);
            }
            if (gsb_set_camera_model(renderer.context(), &m) != GSB_OK) throw std::runtime_error(gsb_last_error(renderer.context()));
        }
        struct Pose {
            float v[7];
            float fov;
        };
        std::vector<Pose> poses;
        if (path_file.empty()) {
            poses.push_back(Pose{{cam[0], cam[1], cam[2], cam[3], cam[4], cam[5], cam[6]}, fov});
        } else {
            std::ifstream pf(path_file);
            if (!pf) throw std::runtime_error("cannot open camera path: " + path_file);
            std::string line;
            while (std::getline(pf, line)) {
                if (line.empty() || line[0] == '#') continue;
                Pose p{{0, 0, 0, 1, 0, 0, 0}, fov};
                const int got = std::sscanf(line.c_str(), "%f %f %f %f %f %f %f %f", &p.v[0], &p.v[1], &p.v[2], &p.v[3], &p.v[4], &p.v[5], &p.v[6], &p.fov);
                if (got < 7) throw std::runtime_error("bad camera path line: " + line);
                poses.push_back(p);
            }
            if (poses.empty()) throw std::runtime_error("camera path is empty: " + path_file);
        }
        if (verbose) std::fprintf(stderr, "loaded %llu Gaussians in %.1f ms\n", (unsigned long long)renderer.getScene()->getNumVertices(), load_ms);
        for (size_t pi = 0; pi < poses.size(); pi++) {
            const Pose& po = poses[pi];
            renderer.camera.position = {po.v[0], po.v[1], po.v[2]};
            renderer.camera.rotation = {po.v[3], po.v[4], po.v[5], po.v[6]};
            renderer.camera.fov = po.fov;
            const auto t1 = std::chrono::steady_clock::now();
            renderer.run(frames);
            const double wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
            const gsb_stats s = renderer.retrieveTimestamps();
            std::printf("{\"scene\": \"%s\", \"pose\": %zu, \"gaussians\": %llu, \"load_ms\": %.1f, \"read_activate_ms\": %.1f, \"upload_ms\": %.1f, "
                        "\"width\": %u, \"height\": %u, \"frames\": %u, \"fps_wall\": %.2f, "
                        "\"instances\": %llu, \"instances_aabb\": %llu, \"visible\": %llu, \"preprocess_ms\": %.4f, \"prefix_sum_ms\": %.4f, "
                        "\"preprocess_sort_ms\": %.4f, \"sort_ms\": %.4f, \"tile_boundary_ms\": %.4f, \"render_ms\": %.4f, \"frame_ms\": %.4f}\n",
                        scene.c_str(), pi, (unsigned long long)s.num_gaussians, load_ms, renderer.getScene()->lastReadMs,
                        renderer.getScene()->lastUploadMs, cfg.width, cfg.height, frames, 1000.0 * frames / wall_ms,
                        (unsigned long long)s.num_instances, (unsigned long long)s.num_instances_aabb, (unsigned long long)s.num_visible,
                        s.preprocess_ms, s.prefix_sum_ms, s.preprocess_sort_ms, s.sort_ms, s.tile_boundary_ms, s.render_ms, s.frame_ms);
        }
        if (!out_path.empty()) {
            const auto& px = renderer.frame();  // B8G8R8A8
            std::ofstream f(out_path, std::ios::binary);
            f << "P6\n" << cfg.width << " " << cfg.height << "\n255\n";
            std::vector<unsigned char> rgb(static_cast<size_t>(cfg.width) * cfg.height * 3);
            for (size_t p = 0; p < static_cast<size_t>(cfg.width) * cfg.height; p++) {
                rgb[p * 3 + 0] = px[p * 4 + 2];
                rgb[p * 3 + 1] = px[p * 4 + 1];
                rgb[p * 3 + 2] = px[p * 4 + 0];
            }
            f.write(reinterpret_cast<const char*>(rgb.data()), static_cast<std::streamsize>(rgb.size()));
        }
        if (!float_path.empty()) {  // PFM: "PF", width height, -1.0 (little endian), rows bottom to top, float32 RGB
            const float* px = static_cast<const float*>(renderer.render(cfg.width, cfg.height, GSB_FORMAT_RGBA32F));
            std::ofstream f(float_path, std::ios::binary);
            f << "PF\n" << cfg.width << " " << cfg.height << "\n-1.0\n";
            std::vector<float> row(static_cast<size_t>(cfg.width) * 3);
            for (uint32_t y = cfg.height; y-- > 0;) {
                for (uint32_t x = 0; x < cfg.width; x++)
                    for (int c = 0; c < 3; c++) row[x * 3 + c] = px[(static_cast<size_t>(y) * cfg.width + x) * 4 + c];
                f.write(reinterpret_cast<const char*>(row.data()), static_cast<std::streamsize>(row.size() * sizeof(float)));
            }
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "critical: %s\n", e.what());
        return 2;
    }
    return 0;
}
