"""gs_b200 -- thin ctypes binding over the C ABI of libgsb200.so (include/gs_b200.h) and the
C bridge of the C++ host library libgsb200_host.so (host/gs_b200_host.h).

This is plumbing for tests and bench.py only: the product is the CUDA library + the C++ host.
There is NO fallback: if libgsb200.so is missing this module raises at import, and without a
CUDA device `Context()` raises (gsb_create -> GSB_ERR_NO_DEVICE).  Nothing here touches oracle/.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

PKG_ROOT = Path(__file__).resolve().parents[2]  # .../3dgs.cpp_b200
LIB_PATH = Path(os.environ.get("GSB200_LIB", PKG_ROOT / "libgsb200.so"))  # override only for A/B experiments
HOST_LIB_PATH = PKG_ROOT / "libgsb200_host.so"

if not LIB_PATH.exists():
    raise ImportError(f"{LIB_PATH} not built: run `python __graft_entry__.py build` (nvcc, sm_90a)")
if not HOST_LIB_PATH.exists():
    raise ImportError(f"{HOST_LIB_PATH} not built: run `python __graft_entry__.py build`")

lib = C.CDLL(str(LIB_PATH), mode=os.RTLD_GLOBAL)
host = C.CDLL(str(HOST_LIB_PATH))

# ---- enums (gs_b200.h) ----
OK = 0
ERR_INVALID, ERR_NO_DEVICE, ERR_CUDA, ERR_NO_SCENE, ERR_OOM, ERR_OVERFLOW = -1, -2, -3, -4, -5, -6
FORMAT_RGBA32F, FORMAT_RGBA8, FORMAT_BGRA8 = 0, 1, 2
MODE_EXACT, MODE_FAST = 0, 1
MEM_HOST, MEM_DEVICE = 0, 1
CAMERA_PINHOLE, CAMERA_FISHEYE, CAMERA_OPENCV, CAMERA_ORTHO = 0, 1, 2, 3
(BUF_COV3D, BUF_ATTR, BUF_TILES_OVERLAP, BUF_PREFIX_SUM, BUF_KEYS_UNSORTED, BUF_VALS_UNSORTED,
 BUF_KEYS_SORTED, BUF_VALS_SORTED, BUF_TILE_BOUNDARY, BUF_DEPTH_ORDER, BUF_EMIT_OFFSETS) = range(11)
ALL_ROWS = 0xFFFFFFFF

EXPORTED_SYMBOLS = [  # every symbol include/gs_b200.h declares
    "gsb_abi_version", "gsb_device_count", "gsb_create", "gsb_destroy", "gsb_last_error",
    "gsb_scene_upload", "gsb_scene_size", "gsb_set_mode", "gsb_set_debug", "gsb_set_timers", "gsb_set_tile_cull", "gsb_set_sh_storage",
    "gsb_set_antialiased", "gsb_set_background", "gsb_set_camera_model", "gsb_set_sh_degree",
    "gsb_reserve_instances", "gsb_render", "gsb_render_async", "gsb_get_stats", "gsb_debug_size",
    "gsb_debug_download", "gsb_sort_pairs", "gsb_sort_pairs32", "gsb_set_graph", "gsb_host_alloc", "gsb_host_free",
    # reverse mode
    "gsb_set_backward", "gsb_render_backward", "gsb_render_backward_camera", "gsb_render_backward_density",
    "gsb_set_backward_deterministic", "gsb_background_gradient",
    # rendered depth and alpha with their gradients
    "gsb_render_depth", "gsb_render_backward_depth",
    # rendered feature maps with their gradients
    "gsb_render_features", "gsb_render_backward_features", "gsb_adam_step_features",
    # camera and lens gradients through a lens (fisheye, OpenCV or orthographic)
    "gsb_render_backward_fisheye",
    # training loss, optimizer step and initialisation from a point cloud
    "gsb_image_loss", "gsb_adam_step", "gsb_init_from_points",
    # Mip-Splatting's 3D smoothing filter
    "gsb_filter3d_variance", "gsb_adam_step_filter3d", "gsb_filter3d_variance_lens",
    # bilateral-grid appearance correction
    "gsb_bilagrid_apply", "gsb_bilagrid_backward",
    # 3DGS-MCMC: position noise and relocation
    "gsb_mcmc_noise", "gsb_mcmc_relocate",
    # frame sharding over several GPUs
    "gsb_group_create", "gsb_group_destroy", "gsb_group_size", "gsb_group_context", "gsb_group_last_error",
    "gsb_group_scene_upload", "gsb_group_render", "gsb_group_render_async",
    "gsb_shard_unique_id", "gsb_shard_last_error", "gsb_create_sharded", "gsb_shard_rank", "gsb_shard_world", "gsb_shard_slice",
    "gsb_shard_band", "gsb_scene_upload_sharded", "gsb_render_sharded", "gsb_render_sharded_async", "gsb_shard_frame",
]
HOST_EXPORTED_SYMBOLS = [  # host/gs_b200_host.h
    "gsh_last_error", "gsh_initialize", "gsh_draw", "gsh_pan_translation", "gsh_movement", "gsh_cleanup",
    "gsh_set_camera", "gsh_get_camera", "gsh_key_input", "gsh_render", "gsh_frame", "gsh_stats",
    "gsh_num_vertices", "gsh_context", "gsh_uniforms_from_camera", "gsh_camera_translate",
    "gsh_activate_records", "gsh_load_ply", "gsh_free", "gsh_write_ply", "gsh_synth_default_params",
    "gsh_synth_records",
]


class Uniforms(C.Structure):
    """gsb_uniforms == Renderer::UniformBuffer (src/Renderer.h:21-29), 160 bytes."""
    _fields_ = [("camera_position", C.c_float * 4), ("proj_mat", C.c_float * 16), ("view_mat", C.c_float * 16),
                ("width", C.c_uint32), ("height", C.c_uint32), ("tan_fovx", C.c_float), ("tan_fovy", C.c_float)]


assert C.sizeof(Uniforms) == 160

# The float fields of gsb_uniforms in ABI order: camera_position[4], proj_mat[16], view_mat[16], tan_fovx, tan_fovy -- the
# 4-byte words of the struct without width and height (words 36 and 37).
UBO_FLOATS = 38
UBO_FLOAT_WORDS = list(range(36)) + [38, 39]


def pack_uniforms(u: Uniforms) -> np.ndarray:
    """The UBO_FLOATS float fields of u, in ABI order, as a float32 array."""
    return np.frombuffer(bytes(u), np.float32)[UBO_FLOAT_WORDS].copy()


def unpack_uniforms(floats, width, height) -> Uniforms:
    """The Uniforms whose float fields are `floats` (UBO_FLOATS values in ABI order) and whose size is width x height."""
    f = _f32(floats, UBO_FLOATS)
    words = np.zeros(40, np.float32)
    words[UBO_FLOAT_WORDS] = f
    words[36:38] = np.array([width, height], np.uint32).view(np.float32)
    return Uniforms.from_buffer_copy(words.tobytes())


class Stats(C.Structure):
    _fields_ = [("num_gaussians", C.c_uint64), ("num_visible", C.c_uint64), ("num_instances", C.c_uint64), ("num_instances_aabb", C.c_uint64),
                ("blend_consumed", C.c_uint64), ("instance_capacity", C.c_uint64), ("sort_passes", C.c_uint32),
                ("regrow_count", C.c_uint32), ("preprocess_ms", C.c_float), ("prefix_sum_ms", C.c_float),
                ("preprocess_sort_ms", C.c_float), ("sort_ms", C.c_float), ("tile_boundary_ms", C.c_float),
                ("render_ms", C.c_float), ("frame_ms", C.c_float), ("sort_depth_ms", C.c_float),
                ("sort_tile_ms", C.c_float), ("sort_hist_ms", C.c_float), ("sort_pass_ms", C.c_float * 8),
                ("sort_depth_passes", C.c_uint32), ("pad_", C.c_uint32), ("blend_warp_visits", C.c_uint64), ("blend_pixel_hits", C.c_uint64), ("blend_staged", C.c_uint64), ("shard_blend_ms", C.c_float), ("shard_wait_ms", C.c_float)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["sort_pass_ms"] = list(self.sort_pass_ms)[:self.sort_passes]
        return d


class SynthParams(C.Structure):
    _fields_ = [("center", C.c_float * 3), ("half_extent", C.c_float * 3), ("log_scale_min", C.c_float),
                ("log_scale_max", C.c_float), ("opacity_min", C.c_float), ("opacity_max", C.c_float),
                ("sh_dc_range", C.c_float), ("sh_rest_sigma", C.c_float)]


class CameraModel(C.Structure):
    """gsb_camera_model: the lens of gsb_set_camera_model (fisheye_camera, fisheye_from_colmap, opencv_camera,
    opencv_from_colmap and camera_from_colmap make one)."""
    _fields_ = [("kind", C.c_uint32), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("k", C.c_float * 4), ("max_theta", C.c_float)]


FISHEYE_MAX_THETA_CAP = 175.0 * np.pi / 180.0  # fisheye_camera's default max_theta never exceeds this (175 deg)


def fisheye_camera(fx, fy, cx, cy, k=(0.0, 0.0, 0.0, 0.0), max_theta=None) -> CameraModel:
    """An OpenCV-fisheye (Kannala-Brandt) lens for Context.set_camera_model: theta_d = theta (1 + k1 theta^2 + k2 theta^4 +
    k3 theta^6 + k4 theta^8), pixel (i, j) sampled at (i, j) (so cx, cy are COLMAP's plus 0.5; see fisheye_from_colmap).
    max_theta (radians) culls rays farther off the axis; None = the largest angle up to FISHEYE_MAX_THETA_CAP at which
    theta_d is still increasing (found on a 0.1 mrad grid, as gs_viewer_headless --fisheye does)."""
    k = [float(x) for x in k]
    if len(k) != 4:
        raise ValueError("fisheye_camera: k must hold 4 coefficients")
    if max_theta is None:
        t = np.arange(1, int(FISHEYE_MAX_THETA_CAP / 1e-4) + 1) * 1e-4
        u = t * t
        dq = 1.0 + u * (3.0 * k[0] + u * (5.0 * k[1] + u * (7.0 * k[2] + u * 9.0 * k[3])))
        bad = np.nonzero(~(dq > 0.0))[0]
        max_theta = float(t[-1] if bad.size == 0 else (t[bad[0] - 1] if bad[0] > 0 else 0.0))
    return CameraModel(CAMERA_FISHEYE, float(fx), float(fy), float(cx), float(cy), (C.c_float * 4)(*k), float(max_theta))


# opencv_camera's default max_theta never exceeds this (80 deg).  A choice, not a measured optimum: a phone or DSLR lens
# calibrated as OPENCV rarely sees farther off the axis, and past it the polynomial is an extrapolation of the calibration.
OPENCV_MAX_THETA_CAP = 80.0 * np.pi / 180.0


def opencv_monotone_limit(k1, k2) -> float:
    """The largest r^2 up to which the radial map r R(r^2), R = 1 + k1 r^2 + k2 r^4, is strictly increasing: the smallest
    positive root of 1 + 3 k1 u + 5 k2 u^2 (inf if there is none), in closed form."""
    k1, k2 = float(k1), float(k2)
    if k2 == 0.0:
        return -1.0 / (3.0 * k1) if k1 < 0.0 else np.inf
    disc = 9.0 * k1 * k1 - 20.0 * k2
    if disc < 0.0:
        return np.inf
    sq = np.sqrt(disc)
    # the two roots as -2 / (3 k1 +- sq) (the stable form of (-3 k1 -+ sq) / (10 k2)); only a positive one bounds the map
    roots = [-2.0 / d for d in (3.0 * k1 + sq, 3.0 * k1 - sq) if d != 0.0]
    positive = [r for r in roots if r > 0.0]
    return min(positive) if positive else np.inf


def opencv_camera(fx, fy, cx, cy, k=(0.0, 0.0, 0.0, 0.0), max_theta=None) -> CameraModel:
    """An OpenCV (Brown-Conrady radial-tangential) lens for Context.set_camera_model, k = (k1, k2, p1, p2) in COLMAP's OPENCV
    order: xn = x / z, yn = y / z, r^2 = xn^2 + yn^2, R = 1 + k1 r^2 + k2 r^4, xd = xn R + 2 p1 xn yn + p2 (r^2 + 2 xn^2),
    yd = yn R + p1 (r^2 + 2 yn^2) + 2 p2 xn yn, uv = (fx xd + cx, fy yd + cy), pixel (i, j) sampled at (i, j) (so cx, cy are
    COLMAP's minus 0.5; see opencv_from_colmap).  max_theta (radians, in (0, pi/2)) culls rays farther off the axis; None =
    the largest angle up to OPENCV_MAX_THETA_CAP at which r R(r^2) is still increasing (opencv_monotone_limit, less 1e-4 of
    it in r^2 so that gsb_set_camera_model's strict test passes)."""
    k = [float(x) for x in k]
    if len(k) != 4:
        raise ValueError("opencv_camera: k must hold 4 coefficients (k1, k2, p1, p2)")
    if max_theta is None:
        u0 = opencv_monotone_limit(k[0], k[1])
        max_theta = OPENCV_MAX_THETA_CAP if not np.isfinite(u0) else min(OPENCV_MAX_THETA_CAP, float(np.arctan(np.sqrt(u0 * (1.0 - 1e-4)))))
    return CameraModel(CAMERA_OPENCV, float(fx), float(fy), float(cx), float(cy), (C.c_float * 4)(*k), float(max_theta))


def opencv_from_colmap(fx, fy, cx, cy, k1, k2, p1, p2) -> CameraModel:
    """COLMAP's OPENCV parameters (fx, fy, cx, cy, k1, k2, p1, p2) as an opencv_camera.  COLMAP puts pixel centres at i + 0.5,
    this renderer samples pixel (i, j) at (i, j): the principal point moves by half a pixel."""
    return opencv_camera(fx, fy, float(cx) - 0.5, float(cy) - 0.5, (k1, k2, p1, p2))


def camera_from_colmap(model: str, params) -> CameraModel:
    """The CameraModel of a COLMAP camera (its model name and params, as cameras.txt lists them).  SIMPLE_PINHOLE (f, cx, cy),
    PINHOLE (fx, fy, cx, cy), SIMPLE_RADIAL (f, cx, cy, k), RADIAL (f, cx, cy, k1, k2) and OPENCV (fx, fy, cx, cy, k1, k2, p1,
    p2) become opencv_from_colmap with 0 for the coefficients a model lacks; OPENCV_FISHEYE (fx, fy, cx, cy, k1..k4) becomes
    fisheye_from_colmap.  Any other model (FULL_OPENCV, THIN_PRISM_FISHEYE, ...) raises ValueError."""
    p = [float(x) for x in params]
    counts = {"SIMPLE_PINHOLE": 3, "PINHOLE": 4, "SIMPLE_RADIAL": 4, "RADIAL": 5, "OPENCV": 8, "OPENCV_FISHEYE": 8}
    if model not in counts:
        raise ValueError(f"camera_from_colmap: unsupported COLMAP camera model {model!r}")
    if len(p) != counts[model]:
        raise ValueError(f"camera_from_colmap: {model} takes {counts[model]} parameters, got {len(p)}")
    if model == "OPENCV_FISHEYE":
        return fisheye_from_colmap(*p)
    if model == "OPENCV":
        return opencv_from_colmap(*p)
    if model == "PINHOLE":
        return opencv_from_colmap(*p, 0.0, 0.0, 0.0, 0.0)
    f, cx, cy, ks = p[0], p[1], p[2], p[3:]
    k1, k2 = (ks + [0.0, 0.0])[:2]
    return opencv_from_colmap(f, f, cx, cy, k1, k2, 0.0, 0.0)


def ortho_camera(fx, fy, cx, cy) -> CameraModel:
    """An orthographic (parallel-projection) camera for Context.set_camera_model: fx, fy in pixels per world unit, cx, cy in
    pixels, and with t = (x, y, z) the view-space position, uv = (fx x + cx, fy y + cy), culled unless z > 0.2; pixel (i, j)
    is sampled at (i, j) (gsplat's principal point is (cx - 0.5, cy - 0.5) here).  The frame reads only the UBO's view matrix
    and size; its depth is z, and the SH colour is seen along the camera's forward axis (view row 2) for every Gaussian."""
    return CameraModel(CAMERA_ORTHO, float(fx), float(fy), float(cx), float(cy), (C.c_float * 4)(0.0, 0.0, 0.0, 0.0), 0.0)


LENS_WORDS = 8  # (fx, fy, cx, cy, k[0..3]): lens_tensor's layout and gsb_render_backward_fisheye's grad_lens words 1-8


def lens_tensor(cam: CameraModel, device=None):
    """The (8,) float32 tensor (fx, fy, cx, cy, k[0..3]) of a fisheye, OpenCV or orthographic CameraModel (k1..k4 for a
    fisheye, k1, k2, p1, p2 for OpenCV, 0 for an orthographic camera), for render_torch(..., lens=): a lens a torch
    optimizer can refine.  lens_camera turns it back into the same CameraModel, bit for bit."""
    import torch

    return torch.tensor(np.array([cam.fx, cam.fy, cam.cx, cam.cy, *cam.k], np.float32), device=device)


def lens_camera(lens, max_theta, kind=CAMERA_FISHEYE) -> CameraModel:
    """The CameraModel of kind `kind` (CAMERA_FISHEYE, the default, CAMERA_OPENCV or CAMERA_ORTHO) of an (8,) lens tensor
    (lens_tensor's layout) culled at max_theta (radians; 0 for CAMERA_ORTHO, whose k words are 0 too), bit for bit."""
    import torch

    w = lens.detach().to("cpu", torch.float32).reshape(-1).numpy() if isinstance(lens, torch.Tensor) else np.asarray(lens, np.float32)
    if w.shape != (LENS_WORDS,):
        raise ValueError(f"lens_camera: the lens must hold {LENS_WORDS} values (fx, fy, cx, cy, k[0..3])")
    if kind not in (CAMERA_FISHEYE, CAMERA_OPENCV, CAMERA_ORTHO):
        raise ValueError("lens_camera: kind must be CAMERA_FISHEYE, CAMERA_OPENCV or CAMERA_ORTHO")
    return CameraModel(kind, *(float(x) for x in w[:4]), (C.c_float * 4)(*(float(x) for x in w[4:])), float(max_theta))


def fisheye_from_colmap(fx, fy, cx, cy, k1, k2, k3, k4) -> CameraModel:
    """COLMAP's OPENCV_FISHEYE parameters (fx, fy, cx, cy, k1, k2, k3, k4) as a fisheye_camera.  COLMAP puts pixel centres at
    i + 0.5, this renderer samples pixel (i, j) at (i, j): the principal point moves by half a pixel."""
    return fisheye_camera(fx, fy, float(cx) - 0.5, float(cy) - 0.5, (k1, k2, k3, k4))


class AdamConfig(C.Structure):
    """gsb_adam_config."""
    _fields_ = [("lr", C.c_float * 6), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("bias_correction1", C.c_float), ("bias_correction2_sqrt", C.c_float), ("selective", C.c_uint32)]


# the learning-rate groups of gsb_adam_config.lr, in order: columns 0-2, 4-6, 7, 8-11, 12-14 and 15-59 of the record
ADAM_GROUPS = ("position", "scale", "opacity", "rotation", "sh_dc", "sh_rest")


def adam_config(lr, betas=(0.9, 0.999), eps=1e-15, step=1, selective=False) -> AdamConfig:
    """The gsb_adam_config of Adam's step number `step` (1 for the first): lr is six learning rates in ADAM_GROUPS order;
    the bias corrections 1 - beta1^step and sqrt(1 - beta2^step) are computed in double, as torch.optim.Adam does."""
    lr = [float(x) for x in lr]
    if len(lr) != 6:
        raise ValueError(f"adam_config: lr must hold 6 learning rates ({', '.join(ADAM_GROUPS)}), got {len(lr)}")
    beta1, beta2 = (float(b) for b in betas)
    return AdamConfig((C.c_float * 6)(*lr), beta1, beta2, float(eps), 1 - beta1 ** step, (1 - beta2 ** step) ** 0.5,
                      int(bool(selective)))


ATTR_DTYPE = np.dtype([("conic_opacity", "<f4", 4), ("color_radii", "<f4", 4), ("aabb", "<u4", 4),
                       ("uv", "<f4", 2), ("depth", "<f4"), ("magic", "<u4")])
assert ATTR_DTYPE.itemsize == 64

_vp = C.c_void_p
lib.gsb_abi_version.restype = C.c_int
lib.gsb_device_count.restype = C.c_int
lib.gsb_create.argtypes = [C.c_int, C.POINTER(_vp)]
lib.gsb_destroy.argtypes = [_vp]
lib.gsb_destroy.restype = None
lib.gsb_last_error.argtypes = [_vp]
lib.gsb_last_error.restype = C.c_char_p
lib.gsb_scene_upload.argtypes = [_vp, _vp, C.c_uint64, C.c_int]
lib.gsb_scene_size.argtypes = [_vp]
lib.gsb_scene_size.restype = C.c_uint64
lib.gsb_set_mode.argtypes = [_vp, C.c_int]
lib.gsb_set_debug.argtypes = [_vp, C.c_int]
lib.gsb_set_timers.argtypes = [_vp, C.c_int]
lib.gsb_set_tile_cull.argtypes = [_vp, C.c_int]
lib.gsb_set_antialiased.argtypes = [_vp, C.c_int]
lib.gsb_set_sh_degree.argtypes = [_vp, C.c_int]
lib.gsb_set_background.argtypes = [_vp, C.POINTER(C.c_float)]
lib.gsb_set_camera_model.argtypes = [_vp, C.POINTER(CameraModel)]
lib.gsb_set_sh_storage.argtypes = [_vp, C.c_int]
lib.gsb_set_graph.argtypes = [_vp, C.c_int]
lib.gsb_host_alloc.argtypes = [C.POINTER(_vp), C.c_size_t]
lib.gsb_host_free.argtypes = [_vp]
lib.gsb_host_free.restype = None
lib.gsb_reserve_instances.argtypes = [_vp, C.c_uint64]
lib.gsb_render.argtypes = [_vp, C.POINTER(Uniforms), C.c_uint32, C.c_uint32, _vp, C.c_size_t, C.c_int, C.c_int, _vp]
lib.gsb_render_async.argtypes = [_vp, C.POINTER(Uniforms), C.c_uint32, C.c_uint32, _vp, C.c_size_t, C.c_int, _vp]
lib.gsb_get_stats.argtypes = [_vp, C.POINTER(Stats)]
lib.gsb_debug_size.argtypes = [_vp, C.c_int]
lib.gsb_debug_size.restype = C.c_size_t
lib.gsb_debug_download.argtypes = [_vp, C.c_int, _vp, C.c_size_t]
lib.gsb_sort_pairs.argtypes = [_vp, _vp, _vp, _vp, _vp, C.c_uint64, C.c_uint32, _vp]
lib.gsb_sort_pairs32.argtypes = [_vp, _vp, _vp, _vp, _vp, C.c_uint64, C.c_uint32, _vp]
lib.gsb_set_backward.argtypes = [_vp, C.c_int]
lib.gsb_set_backward_deterministic.argtypes = [_vp, C.c_int]
lib.gsb_render_backward.argtypes = [_vp, _vp, _vp, C.c_size_t, _vp, _vp]
lib.gsb_render_backward_camera.argtypes = [_vp, _vp, _vp, C.c_size_t, _vp, _vp, _vp]
lib.gsb_render_backward_density.argtypes = [_vp, _vp, _vp, C.c_size_t, _vp, _vp, _vp, _vp]
lib.gsb_background_gradient.argtypes = [_vp, _vp, C.c_size_t, _vp, _vp]
lib.gsb_render_depth.argtypes = [_vp, C.POINTER(Uniforms), C.c_uint32, C.c_uint32, _vp, C.c_size_t, C.c_int, C.c_int, _vp,
                                 C.c_size_t, _vp]
lib.gsb_render_backward_depth.argtypes = [_vp, _vp, _vp, C.c_size_t, _vp, C.c_size_t, _vp, _vp, _vp, _vp]
lib.gsb_render_features.argtypes = [_vp, _vp, C.c_uint32, _vp, C.c_size_t, _vp]
lib.gsb_render_backward_features.argtypes = [_vp, _vp, _vp, C.c_size_t, _vp, C.c_size_t, _vp, C.c_uint32, _vp, C.c_size_t, _vp, _vp,
                                             _vp, _vp, _vp]
lib.gsb_render_backward_fisheye.argtypes = [_vp, _vp, _vp, C.c_size_t, _vp, C.c_size_t, _vp, C.c_uint32, _vp, C.c_size_t, _vp, _vp,
                                            _vp, _vp, _vp, _vp]
lib.gsb_adam_step_features.argtypes = [_vp, _vp, _vp, _vp, _vp, C.c_uint32, C.c_float, C.POINTER(AdamConfig), _vp]
lib.gsb_image_loss.argtypes = [_vp, C.c_uint32, C.c_uint32, _vp, C.c_size_t, _vp, C.c_size_t, C.c_int, C.c_float, _vp,
                               C.c_size_t, _vp, _vp]
lib.gsb_bilagrid_apply.argtypes = [_vp, C.c_uint32, C.c_uint32, _vp, C.c_size_t, _vp, C.c_uint32, C.c_uint32, C.c_uint32,
                                   _vp, C.c_size_t, _vp]
lib.gsb_bilagrid_backward.argtypes = [_vp, C.c_uint32, C.c_uint32, _vp, C.c_size_t, _vp, C.c_uint32, C.c_uint32, C.c_uint32,
                                      _vp, C.c_size_t, _vp, C.c_size_t, _vp, _vp]
lib.gsb_adam_step.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(AdamConfig), _vp]
lib.gsb_filter3d_variance.argtypes = [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, _vp]
lib.gsb_filter3d_variance_lens.argtypes = [_vp, _vp, C.c_uint64, _vp, _vp, C.c_uint32, _vp, _vp]
lib.gsb_adam_step_filter3d.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(AdamConfig), _vp]
lib.gsb_init_from_points.argtypes = [_vp, _vp, _vp, C.c_uint64, C.c_float, _vp, _vp]
lib.gsb_mcmc_noise.argtypes = [_vp, _vp, _vp, C.c_float, C.c_uint64, C.c_uint64, _vp]
lib.gsb_mcmc_relocate.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_uint64, C.c_float, _vp]

lib.gsb_group_create.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(_vp)]
lib.gsb_group_destroy.argtypes = [_vp]
lib.gsb_group_destroy.restype = None
lib.gsb_group_size.argtypes = [_vp]
lib.gsb_group_context.argtypes = [_vp, C.c_int]
lib.gsb_group_context.restype = _vp
lib.gsb_group_last_error.argtypes = [_vp]
lib.gsb_group_last_error.restype = C.c_char_p
lib.gsb_group_scene_upload.argtypes = [_vp, _vp, C.c_uint64, C.c_int]
lib.gsb_group_render.argtypes = [_vp, C.POINTER(Uniforms), _vp, C.c_size_t, C.c_int, C.c_int]
lib.gsb_group_render_async.argtypes = [_vp, C.POINTER(Uniforms), C.c_int]
lib.gsb_shard_unique_id.argtypes = [_vp]
lib.gsb_shard_last_error.restype = C.c_char_p
lib.gsb_create_sharded.argtypes = [C.c_int, C.c_int, C.c_int, _vp, C.POINTER(_vp)]
lib.gsb_shard_rank.argtypes = [_vp]
lib.gsb_shard_world.argtypes = [_vp]
lib.gsb_shard_slice.argtypes = [C.c_uint64, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
lib.gsb_shard_band.argtypes = [_vp, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
lib.gsb_scene_upload_sharded.argtypes = [_vp, _vp, C.c_uint64, C.c_int]
lib.gsb_render_sharded.argtypes = [_vp, C.POINTER(Uniforms), _vp, C.c_size_t, C.c_int, C.c_int, _vp]
lib.gsb_render_sharded_async.argtypes = [_vp, C.POINTER(Uniforms), C.c_int, _vp]
lib.gsb_shard_frame.argtypes = [_vp]
lib.gsb_shard_frame.restype = _vp

host.gsh_last_error.restype = C.c_char_p
host.gsh_initialize.argtypes = [C.c_char_p, C.c_int, C.c_uint32, C.c_uint32, C.c_int, C.c_int]
host.gsh_initialize.restype = _vp
host.gsh_draw.argtypes = [_vp]
host.gsh_pan_translation.argtypes = [_vp, C.c_float, C.c_float]
host.gsh_movement.argtypes = [_vp, C.c_float, C.c_float, C.c_float]
host.gsh_key_input.argtypes = [_vp, C.POINTER(C.c_int)]
host.gsh_cleanup.argtypes = [_vp]
host.gsh_cleanup.restype = None
host.gsh_set_camera.argtypes = [_vp, _vp, _vp, C.c_float, C.c_float, C.c_float]
host.gsh_get_camera.argtypes = [_vp, _vp, _vp, C.POINTER(C.c_float)]
host.gsh_render.argtypes = [_vp, C.c_uint32, C.c_uint32, C.c_int, _vp, C.c_size_t]
host.gsh_frame.argtypes = [_vp, C.POINTER(C.c_size_t)]
host.gsh_frame.restype = _vp
host.gsh_stats.argtypes = [_vp, C.POINTER(Stats)]
host.gsh_num_vertices.argtypes = [_vp]
host.gsh_num_vertices.restype = C.c_uint64
host.gsh_context.argtypes = [_vp]
host.gsh_context.restype = _vp
host.gsh_uniforms_from_camera.argtypes = [_vp, _vp, C.c_float, C.c_float, C.c_float, C.c_uint32, C.c_uint32,
                                          C.POINTER(Uniforms)]
host.gsh_uniforms_from_camera.restype = None
host.gsh_camera_translate.argtypes = [_vp, _vp, _vp]
host.gsh_camera_translate.restype = None
host.gsh_activate_records.argtypes = [_vp, C.c_uint64, _vp]
host.gsh_activate_records.restype = None
host.gsh_load_ply.argtypes = [C.c_char_p, C.POINTER(C.c_uint64)]
host.gsh_load_ply.restype = C.POINTER(C.c_float)
host.gsh_free.argtypes = [_vp]
host.gsh_free.restype = None
host.gsh_write_ply.argtypes = [C.c_char_p, _vp, C.c_uint64]
host.gsh_synth_default_params.argtypes = [C.POINTER(SynthParams)]
host.gsh_synth_default_params.restype = None
host.gsh_synth_records.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(SynthParams), _vp]
host.gsh_synth_records.restype = None


class GsbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"gsb error {code}: {msg}")
        self.code = code


def _f32(a, n=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if n is not None:
        assert a.size == n
    return a


# ---------------------------------------------------------------- host-only helpers (no GPU)
def uniforms_from_camera(pos, quat_wxyz, fov_deg, near, far, width, height) -> Uniforms:
    """Renderer::updateUniforms via the C++ host (src/Renderer.cpp:719-754)."""
    u = Uniforms()
    p, q = _f32(pos, 3), _f32(quat_wxyz, 4)
    host.gsh_uniforms_from_camera(p.ctypes.data, q.ctypes.data, fov_deg, near, far, width, height, C.byref(u))
    return u


def camera_translate(pos, quat_wxyz, t):
    p, q, tt = _f32(pos, 3).copy(), _f32(quat_wxyz, 4), _f32(t, 3)
    host.gsh_camera_translate(p.ctypes.data, q.ctypes.data, tt.ctypes.data)
    return p


def activate_records(records: np.ndarray) -> np.ndarray:
    rec = _f32(records).reshape(-1, 62)
    out = np.empty((rec.shape[0], 60), np.float32)
    host.gsh_activate_records(rec.ctypes.data, rec.shape[0], out.ctypes.data)
    return out


def load_ply(path) -> np.ndarray:
    n = C.c_uint64(0)
    p = host.gsh_load_ply(str(path).encode(), C.byref(n))
    if not p:
        raise RuntimeError(host.gsh_last_error().decode())
    try:
        return np.ctypeslib.as_array(p, shape=(n.value, 60)).copy() if n.value else np.empty((0, 60), np.float32)
    finally:
        host.gsh_free(p)


def write_ply(path, records: np.ndarray):
    rec = _f32(records).reshape(-1, 62)
    if host.gsh_write_ply(str(path).encode(), rec.ctypes.data, rec.shape[0]) != 0:
        raise RuntimeError(host.gsh_last_error().decode())


def ply_records(params) -> np.ndarray:
    """The (n, 62) float32 PLY records write_ply takes, of raw parameters in the record's column layout (SceneAdam.params:
    position 0-2, column 3 ignored, log scale 4-6, opacity logit 7, quaternion wxyz 8-11, SH 12-59 RGB-interleaved): x, y, z,
    zero normals, f_dc = sh[0..2], f_rest[15 c + j - 1] = sh[3 j + c] (channel-major), opacity, scale_0..2, rot_0..3, copied
    without any activation -- the exact inverse of the loader's layout.  params is a numpy array or a tensor (copied to the
    host).  A trained scene is saved with write_ply(path, ply_records(opt.params))."""
    if not isinstance(params, np.ndarray):
        params = params.detach().cpu().numpy()
    p = _f32(params).reshape(-1, 60)
    out = np.zeros((p.shape[0], 62), np.float32)
    out[:, 0:3] = p[:, 0:3]
    out[:, 6:9] = p[:, 12:15]
    sh_rest = p[:, 15:60].reshape(-1, 15, 3)  # [row, j - 1, c] = sh[3 j + c]
    out[:, 9:54] = sh_rest.transpose(0, 2, 1).reshape(-1, 45)  # [row, 15 c + j - 1]
    out[:, 54] = p[:, 7]
    out[:, 55:58] = p[:, 4:7]
    out[:, 58:62] = p[:, 8:12]
    return out


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def load_points_ply(path):
    """(xyz, rgb) of a point-cloud PLY as Inria's storePly writes it (COLMAP's points3D as x, y, z, nx, ny, nz, red, green,
    blue): binary little-endian, a single `vertex` element of scalar properties.  x, y, z (float or double) become float32,
    red, green, blue (uchar) float32 / 255; other properties are skipped.  Both are (n, 3) float32 numpy arrays.  ascii or
    big-endian files, list properties, other elements and a missing coordinate or colour raise ValueError."""
    data = Path(path).read_bytes()
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError(f"{path}: not a PLY file")
    body = data.index(b"\n", end) + 1
    fmt, elements = None, []
    for line in data[:body].decode("ascii", "replace").splitlines()[1:]:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info", "end_header"):
            continue
        if tok[0] == "format":
            fmt = tok[1] if len(tok) > 1 else None
        elif tok[0] == "element":
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property":
            if not elements:
                raise ValueError(f"{path}: property before any element")
            if tok[1] == "list":
                raise ValueError(f"{path}: list property '{tok[-1]}' (scalar properties only)")
            if tok[1] not in _PLY_TYPES:
                raise ValueError(f"{path}: unknown property type '{tok[1]}'")
            elements[-1][2].append((tok[2], "<" + _PLY_TYPES[tok[1]]))
        else:
            raise ValueError(f"{path}: unexpected header line '{line}'")
    if fmt != "binary_little_endian":
        raise ValueError(f"{path}: format '{fmt}' (binary_little_endian only)")
    if len(elements) != 1 or elements[0][0] != "vertex":
        raise ValueError(f"{path}: elements {[e[0] for e in elements]} (a single 'vertex' element only)")
    _, n, props = elements[0]
    dtype = np.dtype(props)
    names = dict(props)
    for k in ("x", "y", "z"):
        if names.get(k) not in ("<f4", "<f8"):
            raise ValueError(f"{path}: property '{k}' missing or not float / double")
    for k in ("red", "green", "blue"):
        if names.get(k) != "<u1":
            raise ValueError(f"{path}: property '{k}' missing or not uchar")
    if len(data) - body < n * dtype.itemsize:
        raise ValueError(f"{path}: truncated ({len(data) - body} bytes of vertex data, {n * dtype.itemsize} expected)")
    v = np.frombuffer(data, dtype, count=n, offset=body)
    xyz = np.stack([v[k].astype(np.float32) for k in ("x", "y", "z")], 1)
    rgb = np.stack([v[k].astype(np.float32) for k in ("red", "green", "blue")], 1) / np.float32(255)
    return xyz, rgb


def synth_params(**kw) -> SynthParams:
    p = SynthParams()
    host.gsh_synth_default_params(C.byref(p))
    for k, v in kw.items():
        if k in ("center", "half_extent"):
            getattr(p, k)[:] = list(v)
        else:
            setattr(p, k, v)
    return p


def synth_records(seed: int, n: int, params: SynthParams | None = None, first: int = 0) -> np.ndarray:
    """Deterministic synthetic PLY records (n x 62 float32), SURVEY 8d."""
    params = params or synth_params()
    out = np.empty((n, 62), np.float32)
    host.gsh_synth_records(seed, first, n, C.byref(params), out.ctypes.data)
    return out


def band_for_rank(height: int, rank: int, world: int):
    """Tile-row band [begin, end) of `rank` for frame sharding (SURVEY 8e): equal-height bands of
    R = ceil(ceil(H/16) / world) tile rows (NCCL all-gather needs equal counts); trailing ranks may be
    short or empty.  Returns (begin, end, rows_per_rank)."""
    tiles_y = (height + 15) // 16
    rows_per = (tiles_y + world - 1) // world
    begin = min(tiles_y, rank * rows_per)
    return begin, min(tiles_y, begin + rows_per), rows_per


def stream_ptr(stream=None):
    """cudaStream_t of a torch stream (or None -> the context's own stream)."""
    return None if stream is None else C.c_void_p(stream.cuda_stream)


# ---------------------------------------------------------------- the C ABI context
class Context:
    """gsb_ctx wrapper.  All compute happens in libgsb200's CUDA kernels."""

    def __init__(self, device: int = 0, handle=None):
        self._own = handle is None
        if handle is None:
            h = _vp()
            rc = lib.gsb_create(device, C.byref(h))
            if rc != OK:
                raise GsbError(rc, lib.gsb_last_error(None).decode())
            handle = h
        self.h = handle
        self.device = device
        self.frames = 0  # frames rendered through this wrapper (render_torch checks it between forward and backward)
        self._frame_hw = (0, 0, -1)  # (H, W, frames) of the last frame rendered through this wrapper
        self._depth_frame_id = -1  # the value of `frames` after the last gsb_render_depth frame
        self._background = None  # the last set_background colour (render_torch restores it after a frame of its own)
        self.camera = None  # the last set_camera_model lens (None: pinhole)
        self.sh_degree = 3  # the last set_sh_degree degree (render_torch restores it after a frame of its own)

    def close(self):
        if self.h and self._own:
            lib.gsb_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != OK:
            raise GsbError(rc, lib.gsb_last_error(self.h).decode())

    def upload(self, vertices):
        """vertices: (n, 60) float32 numpy array (host) or torch CUDA tensor (device)."""
        if isinstance(vertices, np.ndarray):
            v = _f32(vertices).reshape(-1, 60)
            self._ck(lib.gsb_scene_upload(self.h, v.ctypes.data, v.shape[0], MEM_HOST))
        else:  # torch tensor on this device
            assert vertices.is_cuda and vertices.is_contiguous() and vertices.dtype.itemsize == 4
            self._ck(lib.gsb_scene_upload(self.h, vertices.data_ptr(), vertices.numel() // 60, MEM_DEVICE))
        self.frames += 1  # a new scene invalidates the last frame as well

    @property
    def num_gaussians(self):
        return lib.gsb_scene_size(self.h)

    def set_mode(self, mode):
        self._ck(lib.gsb_set_mode(self.h, mode))

    def set_debug(self, on=True):
        self._ck(lib.gsb_set_debug(self.h, int(on)))

    def set_tile_cull(self, level=1):
        """gsb_set_tile_cull: 0 reference lists, 1 (True) exact per-tile instance culling, 2 coarse 4x4-tile bins."""
        self._ck(lib.gsb_set_tile_cull(self.h, int(level)))

    def set_antialiased(self, on=True):
        """gsb_set_antialiased: from the next frame, opacities are scaled by sqrt(det(cov2d) / det(cov2d + 0.3 I)), the
        compensation for the 0.3 px dilation (gsplat's antialiased mode).  render_torch, SceneAdam, image_metrics and the
        backward pass follow it (the backward uses the setting of the frame it differentiates)."""
        self._ck(lib.gsb_set_antialiased(self.h, int(on)))

    def set_sh_degree(self, d=3):
        """gsb_set_sh_degree: from the next frame, the colour sums the spherical-harmonics coefficients of bands <= d only
        (d in 0..3, 3 the default; the scene keeps all 16).  The frame equals the degree-3 frame of the scene with the higher
        bands zeroed.  render_torch, SceneAdam and the backward pass follow it (the backward uses the degree of the frame it
        differentiates, and leaves the gradient of every higher band at 0).  ValueError for d outside 0..3."""
        if isinstance(d, bool) or not isinstance(d, (int, np.integer)) or not 0 <= d <= 3:
            raise ValueError(f"set_sh_degree: the degree must be an integer in 0..3, not {d!r}")
        self._ck(lib.gsb_set_sh_degree(self.h, int(d)))
        self.sh_degree = int(d)

    def set_background(self, rgb=None):
        """gsb_set_background: from the next frame, every pixel is composited over the colour rgb (3 finite floats; None =
        black, the default): out = c + T_final * rgb.  The backward pass follows the colour of the frame it differentiates."""
        self._ck(lib.gsb_set_background(self.h, None if rgb is None else (C.c_float * 3)(*(float(x) for x in rgb))))
        self._background = None if rgb is None else [float(x) for x in rgb]

    def set_camera_model(self, cam=None):
        """gsb_set_camera_model: from the next frame, project through the lens `cam` (a CameraModel from fisheye_camera,
        fisheye_from_colmap, opencv_camera, opencv_from_colmap, camera_from_colmap or ortho_camera; None or kind CAMERA_PINHOLE = the UBO's
        pinhole camera, the default).  A lens frame (fisheye, OpenCV or orthographic) reads only the UBO's view matrix, camera
        position and size (an orthographic frame not even the camera position).  Frames, render_torch, SceneAdam and the backward pass follow it (the backward uses the model of the frame it
        differentiates).  The camera and lens gradients of a lens frame come from gsb_render_backward_fisheye
        (Context._backward_fisheye, render_torch(..., lens=), SceneAdam.step)."""
        self._ck(lib.gsb_set_camera_model(self.h, None if cam is None else C.byref(cam)))
        self.camera = None if cam is None or cam.kind == CAMERA_PINHOLE else cam

    def background_gradient(self, grad_image, stream=None):
        """gsb_background_gradient of the last (recorded, whole) frame: dL/d(background) = sum_p T_final(p) grad_image(p) as a
        (3,) float32 CUDA tensor, enqueued on `stream` (a torch stream; default torch's current stream).  grad_image is an
        (H, W, 4) float32 CUDA tensor (A ignored).  Bitwise reproducible; does not wait on the host."""
        import torch

        g = grad_image.detach()
        if g.dtype != torch.float32 or g.dim() != 3 or g.shape[2] != 4 or not g.is_cuda or g.stride(2) != 1 or g.stride(1) != 4:
            raise ValueError("background_gradient: grad_image must be an (H, W, 4) float32 CUDA tensor with dense pixels")
        out = torch.empty(3, dtype=torch.float32, device=g.device)
        s = torch.cuda.current_stream(g.device) if stream is None else stream
        self._ck(lib.gsb_background_gradient(self.h, g.data_ptr(), g.stride(0) * 4, out.data_ptr(), _torch_stream_arg(s)))
        return out

    def set_sh_storage(self, half=True):
        """gsb_set_sh_storage: fp16 SH coefficients from the next upload on (NOT a parity mode)."""
        self._ck(lib.gsb_set_sh_storage(self.h, int(half)))

    def set_timers(self, on=True):
        self._ck(lib.gsb_set_timers(self.h, int(on)))

    def set_graph(self, on=True):
        self._ck(lib.gsb_set_graph(self.h, int(on)))

    def reserve(self, capacity):
        self._ck(lib.gsb_reserve_instances(self.h, capacity))

    @staticmethod
    def band_rows(u: Uniforms, rows):
        tiles_y = (u.height + 15) // 16
        rb, re = (0, tiles_y) if rows is None else rows
        re = min(re, tiles_y)
        return rb, re, min(u.height, re * 16) - rb * 16

    def render(self, u: Uniforms, fmt=FORMAT_RGBA32F, rows=None) -> np.ndarray:
        """Render to a HOST numpy array through gsb_render (band = tile rows [rb, re))."""
        rb, re, nrows = self.band_rows(u, rows)
        out = np.empty((nrows, u.width, 4), np.float32 if fmt == FORMAT_RGBA32F else np.uint8)
        self.frames += 1
        self._frame_hw = (u.height, u.width, self.frames)
        self._ck(lib.gsb_render(self.h, C.byref(u), rb, re, out.ctypes.data, 0, MEM_HOST, fmt, None))
        return out

    def render_depth(self, u: Uniforms, fmt=FORMAT_RGBA32F, rows=None):
        """gsb_render_depth to HOST numpy arrays: (image, depth_alpha), the image as render() gives it and depth_alpha an
        (rows, W, 2) float32 array of (D, A) per pixel: D = sum f alpha T (f the view-space z, or the distance for a fisheye
        camera; z for an OpenCV camera) and A = 1 - T_final.  Expected depth is D / A."""
        rb, re, nrows = self.band_rows(u, rows)
        out = np.empty((nrows, u.width, 4), np.float32 if fmt == FORMAT_RGBA32F else np.uint8)
        da = np.empty((nrows, u.width, 2), np.float32)
        self.frames += 1
        self._frame_hw = (u.height, u.width, self.frames)
        self._ck(lib.gsb_render_depth(self.h, C.byref(u), rb, re, out.ctypes.data, 0, MEM_HOST, fmt, da.ctypes.data, 0, None))
        self._depth_frame_id = self.frames
        return out, da

    @property
    def _depth_frame(self):
        """The last frame rendered through this wrapper came from gsb_render_depth, and nothing changed since."""
        return self._depth_frame_id == self.frames

    def render_features(self, features, out=None, stream=None):
        """gsb_render_features: the (H, W, C) float32 feature map of the last frame (recorded with set_backward, whole) from
        features, an (n, C) float32 CUDA tensor in the upload's row order, C <= 128.  F_c = sum f_ic alpha_i T_i over the frame's
        contributors, 0 where none.  Into `out` (a new tensor if None; rows may be padded) on `stream` (a torch stream; None =
        torch's current stream)."""
        import torch

        f = _check_features("Context.render_features", features, features.device)
        h, w = self._frame_size("Context.render_features")
        if out is None:
            out = torch.empty((h, w, f.shape[1]), dtype=torch.float32, device=f.device)
        if out.dtype != torch.float32 or tuple(out.shape) != (h, w, f.shape[1]) or out.stride()[1:] != (f.shape[1], 1):
            raise ValueError(f"Context.render_features: out must be an ({h}, {w}, {f.shape[1]}) float32 tensor with dense pixels")
        s = _torch_stream_arg(torch.cuda.current_stream(f.device) if stream is None else stream)
        self._ck(lib.gsb_render_features(self.h, f.data_ptr(), f.shape[1], out.data_ptr(), out.stride()[0] * 4, s))
        return out

    def render_backward_features(self, vertices_ptr, features, grad_feature_map, grad_vertices_ptr=None, grad_features_ptr=None,
                                 grad_image_ptr=None, grad_depth_alpha_ptr=None, grad_uniforms_ptr=None, density_ptr=None,
                                 stream=None):
        """gsb_render_backward_features: one backward pass of the image (grad_image_ptr, may be None), depth / alpha
        (grad_depth_alpha_ptr, a render_depth frame only) and the feature map (grad_feature_map, an (H, W, C) float32 CUDA
        tensor, dense pixels) of the last frame.  features: the (n, C) tensor the map was rendered from.  grad_features_ptr
        (n x C floats) is overwritten; grad_vertices_ptr, grad_uniforms_ptr and grad_features_ptr may each be None, not all."""
        import torch

        f = _check_features("Context.render_backward_features", features, features.device)
        _check_feature_map("Context.render_backward_features", grad_feature_map, self._frame_size("Context.render_backward_features"),
                           f)
        s = _torch_stream_arg(torch.cuda.current_stream(features.device) if stream is None else stream)
        self._backward(vertices_ptr, grad_image_ptr, grad_vertices_ptr, s, grad_uniforms_ptr=grad_uniforms_ptr, density_ptr=density_ptr,
                       grad_depth_alpha_ptr=grad_depth_alpha_ptr, features=features, grad_feature_map=grad_feature_map,
                       grad_features_ptr=grad_features_ptr)

    def _frame_size(self, caller):
        """(H, W) of the last frame, which must have been rendered through this wrapper with nothing rendered, uploaded or
        stepped after it: the C entries see only the feature map's row pitch, so its height is checked here."""
        h, w, frame = self._frame_hw
        if frame != self.frames:
            raise ValueError(f"{caller}: the last frame was not rendered through this Context, or the scene changed after it")
        return h, w

    def adam_step_features(self, features, exp_avg, exp_avg_sq, grad_features, lr, cfg: AdamConfig, stream=None):
        """gsb_adam_step_features: torch.optim.Adam (no weight decay) of the (n, C) float32 CUDA tensor `features` in place,
        with its moments, at learning rate lr and cfg's betas, eps, bias corrections and selective (cfg.lr is not read).
        It does not change the scene: the last frame stays valid (a selective step must precede adam_step)."""
        import torch

        f = _check_features("Context.adam_step_features", features, features.device)
        for t in (exp_avg, exp_avg_sq, grad_features):
            _check_features("Context.adam_step_features", t, f.device, f.shape[1])
        s = _torch_stream_arg(torch.cuda.current_stream(f.device) if stream is None else stream)
        self._ck(lib.gsb_adam_step_features(self.h, f.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(), grad_features.data_ptr(),
                                            f.shape[1], float(lr), C.byref(cfg), s))

    def render_into(self, u: Uniforms, out_ptr: int, fmt=FORMAT_RGBA32F, rows=None, stream=None, sync=True):
        """Render into DEVICE memory at out_ptr (e.g. tensor.data_ptr())."""
        rb, re, _ = self.band_rows(u, rows)
        self.frames += 1
        self._frame_hw = (u.height, u.width, self.frames)
        if sync:
            self._ck(lib.gsb_render(self.h, C.byref(u), rb, re, out_ptr, 0, MEM_DEVICE, fmt, stream_ptr(stream)))
        else:
            self._ck(lib.gsb_render_async(self.h, C.byref(u), rb, re, out_ptr, 0, fmt, stream_ptr(stream)))

    def stats(self) -> Stats:
        s = Stats()
        self._ck(lib.gsb_get_stats(self.h, C.byref(s)))
        return s

    def set_backward(self, on=True):
        """gsb_set_backward: the next frames keep what gsb_render_backward needs (tile-cull level 2 falls back to 1)."""
        self._ck(lib.gsb_set_backward(self.h, int(on)))

    def set_backward_deterministic(self, on=True):
        """gsb_set_backward_deterministic: the next backward calls reduce without floating-point atomics, so their outputs
        are bit-identical from call to call (and at tile-cull levels 0 and 1)."""
        self._ck(lib.gsb_set_backward_deterministic(self.h, int(on)))

    def render_backward(self, vertices_ptr, grad_image_ptr, grad_vertices_ptr, stream=None, row_pitch_bytes=0,
                        grad_uniforms_ptr=None, density_ptr=None):
        """gsb_render_backward on device pointers: dL/d(image) (H x W float4) -> dL/d(vertices) (n x 60, overwritten).
        With grad_uniforms_ptr (160 B of device memory), gsb_render_backward_camera: also dL/d(the frame's gsb_uniforms),
        overwritten; grad_vertices_ptr may then be None (a frozen scene).
        With density_ptr (n x 4 floats of device memory), gsb_render_backward_density: also accumulates the frame's
        density-control statistics into it; either gradient output may then be None, but not both."""
        self._backward(vertices_ptr, grad_image_ptr, grad_vertices_ptr, stream_ptr(stream), row_pitch_bytes,
                       grad_uniforms_ptr, density_ptr)

    def _backward(self, vertices_ptr, grad_image_ptr, grad_vertices_ptr, stream, row_pitch_bytes=0, grad_uniforms_ptr=None,
                  density_ptr=None, grad_depth_alpha_ptr=None, features=None, grad_feature_map=None, grad_features_ptr=None):
        """render_backward with `stream` already the C ABI's cudaStream_t argument.  With grad_depth_alpha_ptr (H x W float2
        of device memory, dL/d(D, A) of a render_depth frame), gsb_render_backward_depth; grad_image_ptr may then be None.
        With features ((n, C) tensor) and grad_feature_map ((H, W, C) tensor, dense pixels), gsb_render_backward_features."""
        if features is not None:
            self._ck(lib.gsb_render_backward_features(self.h, vertices_ptr, grad_image_ptr, row_pitch_bytes, grad_depth_alpha_ptr, 0,
                                                      features.data_ptr(), features.shape[1], grad_feature_map.data_ptr(),
                                                      grad_feature_map.stride()[0] * 4, grad_vertices_ptr, grad_uniforms_ptr,
                                                      grad_features_ptr, density_ptr, stream))
        elif grad_depth_alpha_ptr is not None:
            self._ck(lib.gsb_render_backward_depth(self.h, vertices_ptr, grad_image_ptr, row_pitch_bytes, grad_depth_alpha_ptr, 0,
                                                   grad_vertices_ptr, grad_uniforms_ptr, density_ptr, stream))
        elif density_ptr is not None:
            self._ck(lib.gsb_render_backward_density(self.h, vertices_ptr, grad_image_ptr, row_pitch_bytes, grad_vertices_ptr,
                                                     grad_uniforms_ptr, density_ptr, stream))
        elif grad_uniforms_ptr is None:
            self._ck(lib.gsb_render_backward(self.h, vertices_ptr, grad_image_ptr, row_pitch_bytes, grad_vertices_ptr, stream))
        else:
            self._ck(lib.gsb_render_backward_camera(self.h, vertices_ptr, grad_image_ptr, row_pitch_bytes, grad_vertices_ptr,
                                                    grad_uniforms_ptr, stream))

    def _backward_fisheye(self, vertices_ptr, grad_image_ptr, grad_vertices_ptr, stream, grad_uniforms_ptr=None, grad_lens_ptr=None,
                          density_ptr=None, grad_depth_alpha_ptr=None, features=None, grad_feature_map=None, grad_features_ptr=None,
                          row_pitch_bytes=0):
        """gsb_render_backward_fisheye on device pointers, `stream` the C ABI's cudaStream_t: _backward's arguments plus the
        camera gradient of the last (fisheye, OpenCV or orthographic) frame, grad_uniforms_ptr (160 B, dL/d gsb_uniforms, pose words only) and
        grad_lens_ptr (40 B, a gsb_camera_model of dL/d(fx, fy, cx, cy, k)), each overwritten and each may be None."""
        fptr, fch, gfm, fpitch = (None, 0, None, 0) if features is None else (
            features.data_ptr(), features.shape[1], grad_feature_map.data_ptr(), grad_feature_map.stride()[0] * 4)
        self._ck(lib.gsb_render_backward_fisheye(self.h, vertices_ptr, grad_image_ptr, row_pitch_bytes, grad_depth_alpha_ptr, 0, fptr,
                                                 fch, gfm, fpitch, grad_vertices_ptr, grad_uniforms_ptr, grad_lens_ptr,
                                                 grad_features_ptr, density_ptr, stream))

    def _render_whole_frame(self, u: Uniforms, device, depth=False):
        """The whole frame of u, recorded while gsb_set_backward is on, as a new tensor on torch's current stream; with
        depth, (image, depth_alpha) from gsb_render_depth, depth_alpha an (H, W, 2) tensor."""
        import torch

        img = torch.empty((u.height, u.width, 4), dtype=torch.float32, device=device)
        self.frames += 1
        self._frame_hw = (u.height, u.width, self.frames)
        stream = _torch_stream_arg(torch.cuda.current_stream(device))
        if not depth:
            self._ck(lib.gsb_render(self.h, C.byref(u), 0, ALL_ROWS, img.data_ptr(), 0, MEM_DEVICE, FORMAT_RGBA32F, stream))
            return img
        da = torch.empty((u.height, u.width, 2), dtype=torch.float32, device=device)
        self._ck(lib.gsb_render_depth(self.h, C.byref(u), 0, ALL_ROWS, img.data_ptr(), 0, MEM_DEVICE, FORMAT_RGBA32F,
                                      da.data_ptr(), 0, stream))
        self._depth_frame_id = self.frames
        return img, da

    def image_loss(self, image, target, lambda_dssim=0.2, grad_image=None, stream=None):
        """gsb_image_loss on torch tensors: the photometric loss (1 - lambda) L1 + lambda (1 - SSIM) of `image` against
        `target`, and, when grad_image is given, d loss / d image written into it (A = 0).  Returns the (4,) float64 device
        tensor (loss, L1, SSIM, MSE) without waiting for it.

        image and grad_image are (H, W, 4) float32 and target (H, W, 4) float32 or uint8 (read as v / 255), all CUDA tensors
        on the context's device; pixels are dense, rows may be padded (a view of wider rows).  Runs on `stream` (a torch
        stream), by default torch's current stream.  Bad shapes, dtypes or devices raise ValueError."""
        import torch

        image_pitch = self._frame_pitch("image", image, (torch.float32,), image.shape[:2] if image.dim() == 3 else None)
        H, W = image.shape[0], image.shape[1]
        target_pitch = self._frame_pitch("target", target, (torch.float32, torch.uint8), (H, W))
        grad_pitch = 0 if grad_image is None else self._frame_pitch("grad_image", grad_image, (torch.float32,), (H, W))
        result = torch.empty(4, dtype=torch.float64, device=image.device)
        s = _torch_stream_arg(torch.cuda.current_stream(image.device) if stream is None else stream)
        self._ck(lib.gsb_image_loss(self.h, W, H, image.data_ptr(), image_pitch, target.data_ptr(), target_pitch,
                                    FORMAT_RGBA8 if target.dtype == torch.uint8 else FORMAT_RGBA32F, float(lambda_dssim),
                                    None if grad_image is None else grad_image.data_ptr(), grad_pitch, result.data_ptr(), s))
        return result

    def adam_step(self, params, exp_avg, exp_avg_sq, grad_vertices, vertices, cfg: AdamConfig, stream=None, variance=None):
        """gsb_adam_step on torch tensors: one Adam step of the raw parameters `params` from grad_vertices (dL/d(activated
        record)), updating params, exp_avg and exp_avg_sq in place and writing the activated records into `vertices` and the
        context's scene (no upload needed).  All five are contiguous (n, 60) float32 CUDA tensors on the context's device,
        n the scene's size; cfg is an adam_config(...).  Runs on `stream` (a torch stream), by default torch's current
        stream, and does not wait for it.  Bad shapes, dtypes, devices or layouts raise ValueError.

        variance: an (n,) float32 CUDA tensor of Mip-Splatting's 3D filter (filter3d_variance; finite and >= 0, not checked
        here): the step is gsb_adam_step_filter3d, whose records carry the filtered scale and opacity (apply_filter_3d)."""
        import torch

        self._check_rows("adam_step", {"params": params, "exp_avg": exp_avg, "exp_avg_sq": exp_avg_sq,
                                       "grad_vertices": grad_vertices, "vertices": vertices})
        s = _torch_stream_arg(torch.cuda.current_stream(params.device) if stream is None else stream)
        if variance is None:
            self._ck(lib.gsb_adam_step(self.h, params.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                                       grad_vertices.data_ptr(), vertices.data_ptr(), C.byref(cfg), s))
        else:
            self._check_variance("adam_step", variance, params.shape[0])
            self._ck(lib.gsb_adam_step_filter3d(self.h, params.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                                                grad_vertices.data_ptr(), vertices.data_ptr(), variance.data_ptr(),
                                                C.byref(cfg), s))
        self.frames += 1  # the scene changed: the last frame can no longer be differentiated

    def _check_variance(self, caller, variance, n):
        """variance is a contiguous (n,) float32 CUDA tensor on the context's device; ValueError otherwise."""
        import torch

        if not isinstance(variance, torch.Tensor) or not variance.is_cuda or variance.device.index != self.device:
            raise ValueError(f"{caller}: variance must be a CUDA tensor on device {self.device}")
        if variance.dtype != torch.float32 or tuple(variance.shape) != (n,) or not variance.is_contiguous():
            raise ValueError(f"{caller}: variance must be a contiguous ({n},) float32 tensor, got {tuple(variance.shape)} "
                             f"{variance.dtype}")

    def filter3d_variance(self, vertices, cameras, lenses=None):
        """gsb_filter3d_variance on torch tensors: the (n,) float32 variance of Mip-Splatting's 3D smoothing filter of the
        Gaussians at the positions (columns 0-2) of `vertices`, a contiguous (n, 60) float32 CUDA tensor on the context's
        device (any n: no scene is needed), from `cameras`, a non-empty list of Uniforms (the training views): with d the
        least view depth over the cameras that see a Gaussian (the largest such d for one no camera sees) and f the largest
        focal length in pixels, variance = 0.2 (d / f)^2.  Runs on torch's current stream and returns when the variances are
        written; leaves the context's scene and last frame alone.  Bad arguments raise ValueError or GsbError.

        lenses: the cameras' lens models (gsb_filter3d_variance_lens), one CameraModel for every camera or a list of one per
        camera (a CameraModel of kind CAMERA_PINHOLE, e.g. CameraModel(), is that camera's UBO pinhole).  Each camera then
        sees a Gaussian as a frame through its lens does, and d / f becomes the least over those cameras of the footprint
        scale 1 / sigma_min(d uv / d t), the world size of one pixel at the camera's finest image axis.  None: the pinhole
        filter above."""
        import torch

        if not isinstance(vertices, torch.Tensor) or not vertices.is_cuda or vertices.device.index != self.device:
            raise ValueError(f"filter3d_variance: vertices must be a CUDA tensor on device {self.device}")
        if vertices.dtype != torch.float32 or vertices.dim() != 2 or vertices.shape[1] != 60 or not vertices.is_contiguous():
            raise ValueError(f"filter3d_variance: vertices must be a contiguous (n, 60) float32 tensor, got "
                             f"{tuple(vertices.shape)} {vertices.dtype}")
        cams = list(cameras)
        if not cams:
            raise ValueError("filter3d_variance: needs at least one camera")
        arr = (Uniforms * len(cams))(*cams)
        n = vertices.shape[0]
        out = torch.empty(n, dtype=torch.float32, device=vertices.device)
        s = _torch_stream_arg(torch.cuda.current_stream(vertices.device))
        if lenses is None:
            self._ck(lib.gsb_filter3d_variance(self.h, vertices.data_ptr(), n, arr, len(cams), out.data_ptr(), s))
            return out
        models = [lenses] * len(cams) if isinstance(lenses, CameraModel) else list(lenses)
        if len(models) != len(cams) or not all(isinstance(m, CameraModel) for m in models):
            raise ValueError(f"filter3d_variance: lenses must be one CameraModel or a list of {len(cams)}")
        marr = (CameraModel * len(models))(*models)
        self._ck(lib.gsb_filter3d_variance_lens(self.h, vertices.data_ptr(), n, arr, marr, len(cams), out.data_ptr(), s))
        return out

    def _check_rows(self, caller, arrays):
        """Every tensor of `arrays` (name -> tensor) is a contiguous (n, 60) float32 CUDA tensor on the context's device,
        n the scene's size; ValueError otherwise."""
        import torch

        n = self.num_gaussians
        for name, t in arrays.items():
            if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != self.device:
                raise ValueError(f"{caller}: {name} must be a CUDA tensor on device {self.device}")
            if t.dtype != torch.float32 or tuple(t.shape) != (n, 60) or not t.is_contiguous():
                raise ValueError(f"{caller}: {name} must be a contiguous ({n}, 60) float32 tensor, got {tuple(t.shape)} "
                                 f"{t.dtype}{'' if t.is_contiguous() else ' (not contiguous)'}")

    def mcmc_noise(self, params, vertices, scale, seed, step, stream=None):
        """gsb_mcmc_noise on torch tensors: adds 3DGS-MCMC's position noise Sigma (eps * gate(o) * scale) to every row of
        params, vertices and the resident scene, eps standard normals drawn by Philox4x32-10 from (seed, step, row), so the
        same arguments give the same words anywhere.  params and vertices are contiguous (n, 60) float32 CUDA tensors on the
        context's device; scale is the position learning rate times noise_lr.  Runs on `stream` (a torch stream), by default
        torch's current stream, and does not wait for it.  Bad shapes, dtypes, devices or layouts raise ValueError."""
        import torch

        self._check_rows("mcmc_noise", {"params": params, "vertices": vertices})
        s = _torch_stream_arg(torch.cuda.current_stream(params.device) if stream is None else stream)
        self._ck(lib.gsb_mcmc_noise(self.h, params.data_ptr(), vertices.data_ptr(), float(scale), int(seed) & (2**64 - 1),
                                    int(step) & (2**64 - 1), s))
        self.frames += 1  # the scene changed: the last frame can no longer be differentiated

    def mcmc_relocate(self, params, exp_avg, exp_avg_sq, vertices, dst, src, min_opacity=0.005, stream=None):
        """gsb_mcmc_relocate on torch tensors: row dst[j] becomes a copy of row src[j], after each source's opacity and scale
        are corrected for its r = 1 + (times it appears in src) copies; the moments of source and destination rows become
        zero.  The four arrays are as for adam_step; dst and src are 1-D int32 (or uint32) CUDA tensors of one length k on
        the context's device.  Runs on `stream` (a torch stream), by default torch's current stream, and returns once the
        rows are written.  An index >= n, a repeated destination or a destination that is also a source raise GsbError
        (ERR_INVALID) with nothing written; bad shapes, dtypes, devices or layouts raise ValueError."""
        import torch

        self._check_rows("mcmc_relocate", {"params": params, "exp_avg": exp_avg, "exp_avg_sq": exp_avg_sq,
                                           "vertices": vertices})
        for name, t in (("dst", dst), ("src", src)):
            if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != self.device:
                raise ValueError(f"mcmc_relocate: {name} must be a CUDA tensor on device {self.device}")
            if t.dtype not in (torch.int32, torch.uint32) or t.dim() != 1 or t.shape != dst.shape:
                raise ValueError(f"mcmc_relocate: {name} must be a 1-D int32 tensor of dst's length, got {tuple(t.shape)} {t.dtype}")
        k = dst.shape[0]
        dst, src = dst.contiguous(), src.contiguous()
        s = _torch_stream_arg(torch.cuda.current_stream(params.device) if stream is None else stream)
        self._ck(lib.gsb_mcmc_relocate(self.h, params.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                                       vertices.data_ptr(), dst.data_ptr(), src.data_ptr(), k, float(min_opacity), s))
        if k:
            self.frames += 1

    def init_from_points(self, xyz, rgb, opacity=0.1):
        """gsb_init_from_points on torch tensors: the (n, 60) float32 activated records of a point cloud, one isotropic
        Gaussian per point (Kerbl et al. 2023): scale sqrt of the mean squared distance to its three nearest neighbours
        (floored at 1e-7), `opacity`, identity rotation, SH DC (rgb - 0.5) / C0 and zero higher bands.  xyz is (n, 3)
        float32, rgb (n, 3) float32 in [0, 1] or uint8 (read as v / 255), both CUDA tensors on the context's device.  Runs
        on torch's current stream and returns when the records are written; needs no scene and leaves the context's scene
        and last frame alone.  Bad shapes, dtypes or devices raise ValueError."""
        import torch

        for name, t, dtypes in (("xyz", xyz, (torch.float32,)), ("rgb", rgb, (torch.float32, torch.uint8))):
            if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != self.device:
                raise ValueError(f"init_from_points: {name} must be a CUDA tensor on device {self.device}")
            if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] != xyz.shape[0]:
                raise ValueError(f"init_from_points: {name} must be (n, 3) with xyz's n, got {tuple(t.shape)}")
            if t.dtype not in dtypes:
                raise ValueError(f"init_from_points: {name} must be {' or '.join(str(d) for d in dtypes)}, got {t.dtype}")
        n = xyz.shape[0]
        out = torch.empty((n, 60), dtype=torch.float32, device=xyz.device)
        xyz = xyz.contiguous()
        rgb = (rgb.to(torch.float32) / 255 if rgb.dtype == torch.uint8 else rgb).contiguous()
        s = _torch_stream_arg(torch.cuda.current_stream(xyz.device))
        self._ck(lib.gsb_init_from_points(self.h, xyz.data_ptr(), rgb.data_ptr(), n, float(opacity), out.data_ptr(), s))
        return out

    def _frame_pitch(self, name, t, dtypes, hw, caller="image_loss"):
        """Row pitch in bytes of an (H, W, 4) CUDA tensor with dense pixels on this context's device; ValueError otherwise."""
        import torch

        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != self.device:
            raise ValueError(f"{caller}: {name} must be a CUDA tensor on device {self.device}")
        if t.dim() != 3 or t.shape[2] != 4 or hw is None or tuple(t.shape[:2]) != tuple(hw) or t.numel() == 0:
            raise ValueError(f"{caller}: {name} must be (H, W, 4) with the image's H and W >= 1, got {tuple(t.shape)}")
        if t.dtype not in dtypes:
            raise ValueError(f"{caller}: {name} must be {' or '.join(str(d) for d in dtypes)}, got {t.dtype}")
        if t.stride(2) != 1 or t.stride(1) != 4 or t.stride(0) < 4 * t.shape[1]:
            raise ValueError(f"{caller}: {name} must have dense pixels and rows in order, got strides {t.stride()}")
        return t.stride(0) * t.element_size()

    def _bilagrid_args(self, caller, image, grid):
        """(H, W, image pitch, (X, Y, L)) of a bilateral-grid call's image and (12, L, Y, X) grid; ValueError otherwise."""
        import torch

        pitch = self._frame_pitch("image", image, (torch.float32,), image.shape[:2] if image.dim() == 3 else None, caller)
        if not isinstance(grid, torch.Tensor) or not grid.is_cuda or grid.device.index != self.device:
            raise ValueError(f"{caller}: grid must be a CUDA tensor on device {self.device}")
        if grid.dim() != 4 or grid.shape[0] != 12 or grid.dtype != torch.float32 or not grid.is_contiguous():
            raise ValueError(f"{caller}: grid must be a contiguous (12, L, Y, X) float32 tensor, got {tuple(grid.shape)} "
                             f"{grid.dtype}{'' if grid.is_contiguous() else ' (not contiguous)'}")
        if not all(2 <= d <= 64 for d in grid.shape[1:]):
            raise ValueError(f"{caller}: grid dimensions must lie in [2, 64], got {tuple(grid.shape)}")
        return image.shape[0], image.shape[1], pitch, (grid.shape[3], grid.shape[2], grid.shape[1])

    def bilagrid_apply(self, image, grid, out=None, stream=None):
        """gsb_bilagrid_apply on torch tensors: the frame colour-corrected by the bilateral grid, out = A(p) (r, g, b, 1) with A
        sliced at the pixel's position and luma (DESIGN.md section 17), A copied.  image and out are (H, W, 4) float32 CUDA
        tensors on the context's device with dense pixels (rows may be padded); grid is a contiguous (12, L, Y, X) float32
        tensor, each dimension in [2, 64].  Returns out (a new tensor when None).  Runs on `stream` (a torch stream), by
        default torch's current stream, without waiting.  Bad shapes, dtypes or devices raise ValueError."""
        import torch

        H, W, pitch, (X, Y, L) = self._bilagrid_args("bilagrid_apply", image, grid)
        if out is None:
            out = torch.empty((H, W, 4), dtype=torch.float32, device=image.device)
        out_pitch = self._frame_pitch("out", out, (torch.float32,), (H, W), "bilagrid_apply")
        s = _torch_stream_arg(torch.cuda.current_stream(image.device) if stream is None else stream)
        self._ck(lib.gsb_bilagrid_apply(self.h, W, H, image.data_ptr(), pitch, grid.data_ptr(), X, Y, L, out.data_ptr(),
                                        out_pitch, s))
        return out

    def bilagrid_backward(self, image, grid, grad_out, grad_image=None, grad_grid=None, stream=None):
        """gsb_bilagrid_backward on torch tensors: d loss / d image (A = 0) into grad_image and d loss / d grid into grad_grid
        from grad_out = d loss / d out, both overwritten; either may be None, not both.  grad_out and grad_image are (H, W, 4)
        float32 and grad_grid a contiguous float32 tensor of the grid's shape, all on the context's device.  Bitwise
        reproducible.  Runs on `stream` (a torch stream), by default torch's current stream, without waiting.  Bad
        shapes, dtypes or devices raise ValueError."""
        import torch

        H, W, pitch, (X, Y, L) = self._bilagrid_args("bilagrid_backward", image, grid)
        go_pitch = self._frame_pitch("grad_out", grad_out, (torch.float32,), (H, W), "bilagrid_backward")
        gi_pitch = 0 if grad_image is None else self._frame_pitch("grad_image", grad_image, (torch.float32,), (H, W),
                                                                  "bilagrid_backward")
        if grad_image is None and grad_grid is None:
            raise ValueError("bilagrid_backward: grad_image and grad_grid are both None")
        if grad_grid is not None and (not isinstance(grad_grid, torch.Tensor) or grad_grid.device != grid.device
                                      or grad_grid.dtype != torch.float32 or grad_grid.shape != grid.shape
                                      or not grad_grid.is_contiguous()):
            raise ValueError(f"bilagrid_backward: grad_grid must be a contiguous float32 tensor of shape {tuple(grid.shape)} "
                             "on the grid's device")
        s = _torch_stream_arg(torch.cuda.current_stream(image.device) if stream is None else stream)
        self._ck(lib.gsb_bilagrid_backward(self.h, W, H, image.data_ptr(), pitch, grid.data_ptr(), X, Y, L,
                                           grad_out.data_ptr(), go_pitch, None if grad_image is None else grad_image.data_ptr(),
                                           gi_pitch, None if grad_grid is None else grad_grid.data_ptr(), s))

    def download(self, which) -> np.ndarray:
        nbytes = lib.gsb_debug_size(self.h, which)
        dt = {BUF_COV3D: np.float32, BUF_ATTR: ATTR_DTYPE, BUF_TILES_OVERLAP: np.uint32, BUF_PREFIX_SUM: np.uint32,
              BUF_KEYS_UNSORTED: np.uint64, BUF_VALS_UNSORTED: np.uint32, BUF_KEYS_SORTED: np.uint64,
              BUF_VALS_SORTED: np.uint32, BUF_TILE_BOUNDARY: np.uint32, BUF_DEPTH_ORDER: np.uint32,
              BUF_EMIT_OFFSETS: np.uint64}[which]
        out = np.empty(nbytes // np.dtype(dt).itemsize, dt)
        if nbytes or which == BUF_COV3D:
            self._ck(lib.gsb_debug_download(self.h, which, out.ctypes.data, nbytes))
        if which == BUF_COV3D:
            out = out.reshape(-1, 6)
        if which == BUF_TILE_BOUNDARY:
            out = out.reshape(-1, 2)
        return out

    def sort_pairs(self, keys_ptr, vals_ptr, keys_tmp_ptr, vals_tmp_ptr, m, key_bits=64, stream=None):
        self._ck(lib.gsb_sort_pairs(self.h, keys_ptr, vals_ptr, keys_tmp_ptr, vals_tmp_ptr, m, key_bits,
                                    stream_ptr(stream)))

    def sort_pairs32(self, keys_ptr, vals_ptr, keys_tmp_ptr, vals_tmp_ptr, m, key_bits=32, stream=None):
        self._ck(lib.gsb_sort_pairs32(self.h, keys_ptr, vals_ptr, keys_tmp_ptr, vals_tmp_ptr, m, key_bits,
                                      stream_ptr(stream)))


# ---------------------------------------------------------------- differentiable rendering (torch imported lazily)
_RenderFn = None
MAX_FEATURE_CHANNELS = 128  # GSB_MAX_FEATURE_CHANNELS
CUDA_STREAM_LEGACY = 1  # cudaStreamLegacy: the C ABI reads a NULL stream as "the context's own stream"


def _torch_stream_arg(torch_stream):
    """cudaStream_t for the C ABI that IS the given torch stream.  torch's default stream is the legacy NULL stream, which
    stream_ptr() would hand over as NULL -- the context's own stream, unordered with torch's work."""
    return C.c_void_p(torch_stream.cuda_stream or CUDA_STREAM_LEGACY)


def _check_density(caller, density, vertices):
    """ValueError unless density is None or the contiguous (n, 4) float32 table of the (n, 60) vertices, on their device."""
    import torch

    n = vertices.shape[0]
    if density is not None and (density.dtype != torch.float32 or tuple(density.shape) != (n, 4)
                                or density.device != vertices.device or not density.is_contiguous()):
        raise ValueError(f"{caller}: density must be a contiguous ({n}, 4) float32 tensor on the vertices' device")


def _check_features(caller, features, device, channels=None):
    """features as an (n, C) contiguous float32 tensor on `device`, 1 <= C <= 128 (C == channels when given); else ValueError."""
    import torch

    if (not isinstance(features, torch.Tensor) or features.dtype != torch.float32 or features.dim() != 2 or features.device != device
            or not features.is_contiguous() or not 1 <= features.shape[1] <= MAX_FEATURE_CHANNELS
            or (channels is not None and features.shape[1] != channels)):
        raise ValueError(f"{caller}: features must be a contiguous (n, C) float32 tensor on {device}, 1 <= C <= {MAX_FEATURE_CHANNELS}")
    return features


def _check_feature_map(caller, fmap, hw, features):
    """ValueError unless fmap is an (H, W, C) float32 tensor on the features' device with dense pixels, C = features' width."""
    import torch

    shape = (hw[0], hw[1], features.shape[1])
    if (not isinstance(fmap, torch.Tensor) or fmap.dtype != torch.float32 or tuple(fmap.shape) != shape
            or fmap.device != features.device or fmap.stride()[1:] != (features.shape[1], 1)):
        raise ValueError(f"{caller}: the feature map must be a {shape} float32 tensor on {features.device} with dense pixels")


def _render_fn():
    global _RenderFn
    if _RenderFn is None:
        import torch

        class RenderFn(torch.autograd.Function):
            @staticmethod
            def forward(fctx, ctx, vertices, u, ubo, density, background, depth, features, lens, sh_degree):
                v = vertices.detach().contiguous()
                fctx.depth = bool(depth)
                fctx.features = None
                if features is not None:
                    if features.shape[0] != v.shape[0]:
                        raise ValueError("render_torch: features must have one row per vertex")
                    fctx.features = _check_features("render_torch", features.detach().contiguous(), v.device)
                _check_density("render_torch", density, v)
                fctx.density = density
                fctx.lens_like = None
                cam = None
                if lens is not None:  # this frame through the tensor's lens, of the context's kind and max_theta, or the
                    w = lens.detach().to("cpu", torch.float32).reshape(-1)  # fisheye's default on a pinhole context
                    if ctx.camera is not None:
                        cam = lens_camera(w, ctx.camera.max_theta, ctx.camera.kind)
                    else:
                        cam = lens_camera(w, fisheye_camera(*w[:4].tolist(), w[4:].tolist()).max_theta)
                    fctx.lens_like = (lens.dtype, lens.device)
                if ubo is not None:  # the camera's float fields come from the tensor, the frame size from u
                    if ctx.camera is not None and cam is None:
                        raise ValueError("render_torch: ubo= on a lens camera model needs lens= (its camera gradient is "
                                         "gsb_render_backward_fisheye's)")
                    u = unpack_uniforms(ubo.detach().to("cpu", torch.float32).numpy(), u.width, u.height)
                    fctx.ubo_like = (ubo.dtype, ubo.device)
                ctx.set_backward(True)
                torch.cuda.current_stream(v.device).synchronize()  # the upload runs on the context's stream: v must be complete
                ctx.upload(v)

                def frame_bg():
                    if background is None:
                        return ctx._render_whole_frame(u, v.device, fctx.depth)
                    # this frame over the tensor's colour; the context's own setting is restored after it
                    fctx.bg_like = (background.dtype, background.device)
                    previous = ctx._background
                    ctx.set_background(background.detach().to("cpu", torch.float32).reshape(3).tolist())
                    try:
                        return ctx._render_whole_frame(u, v.device, fctx.depth)
                    finally:
                        ctx.set_background(previous)

                def frame():
                    if sh_degree is None:
                        return frame_bg()
                    # this frame at the given degree; the context's own setting is restored after it
                    previous = ctx.sh_degree
                    ctx.set_sh_degree(sh_degree)
                    try:
                        return frame_bg()
                    finally:
                        ctx.set_sh_degree(previous)

                if cam is None:
                    out = frame()
                else:  # the context's own model is restored after the frame (a lens it refuses raises and changes nothing)
                    previous_cam = ctx.camera
                    ctx.set_camera_model(cam)
                    try:
                        out = frame()
                    finally:
                        ctx.set_camera_model(previous_cam)
                fctx.gs_ctx, fctx.frame, fctx.vertices = ctx, ctx.frames, v
                if fctx.features is None:
                    return out
                fmap = ctx.render_features(fctx.features)
                return (*out, fmap) if fctx.depth else (out, fmap)

            @staticmethod
            def backward(fctx, grad_img, *grads):
                grad_da = grads[0] if fctx.depth else None
                grad_fm = grads[-1] if fctx.features is not None else None
                ctx = fctx.gs_ctx
                if ctx.frames != fctx.frame:
                    raise RuntimeError("render_torch: another frame was rendered on this context between forward and backward")
                v = fctx.vertices
                g = grad_img.detach().to(torch.float32).contiguous()
                gda = None  # depth frames: dL/d(D, A), zeros where torch gave none
                if fctx.depth:
                    gda = (torch.zeros(tuple(g.shape[:2]) + (2,), dtype=torch.float32, device=v.device) if grad_da is None
                           else grad_da.detach().to(torch.float32).contiguous())
                need_v, need_ubo, need_bg = fctx.needs_input_grad[1], fctx.needs_input_grad[3], fctx.needs_input_grad[5]
                need_f = fctx.features is not None and fctx.needs_input_grad[7]
                need_lens = fctx.lens_like is not None and fctx.needs_input_grad[8]
                grad_v = torch.empty_like(v) if need_v else None
                grad_ubo = grad_bg = grad_f = grad_lens = None
                # enqueued on torch's current stream (the engine runs backward on the forward's stream), so the gradients
                # are complete for whatever torch enqueues after them
                stream = _torch_stream_arg(torch.cuda.current_stream(v.device))
                gu = torch.empty(40, dtype=torch.float32, device=v.device) if need_ubo else None  # a whole gsb_uniforms
                ctx.set_backward_deterministic(torch.are_deterministic_algorithms_enabled())
                if fctx.lens_like is not None:  # a frame through lens=: every output in one gsb_render_backward_fisheye pass
                    f = fctx.features if fctx.features is not None and (need_f or grad_fm is not None) else None
                    gfm = None
                    if f is not None:
                        gfm = (torch.zeros((g.shape[0], g.shape[1], f.shape[1]), dtype=torch.float32, device=v.device)
                               if grad_fm is None else grad_fm.detach().to(torch.float32).contiguous())
                    grad_f = torch.empty_like(f) if need_f else None
                    gl = torch.empty(10, dtype=torch.float32, device=v.device) if need_lens else None  # a gsb_camera_model
                    if need_v or need_ubo or need_lens or need_f:
                        geometry = need_v or need_ubo or need_lens
                        ctx._backward_fisheye(v.data_ptr(), g.data_ptr(), grad_v.data_ptr() if need_v else None, stream,
                                              grad_uniforms_ptr=gu.data_ptr() if need_ubo else None,
                                              grad_lens_ptr=gl.data_ptr() if need_lens else None,
                                              density_ptr=None if fctx.density is None or not geometry else fctx.density.data_ptr(),
                                              grad_depth_alpha_ptr=None if gda is None else gda.data_ptr(), features=f,
                                              grad_feature_map=gfm, grad_features_ptr=grad_f.data_ptr() if need_f else None)
                    if need_lens:
                        dtype, device = fctx.lens_like
                        grad_lens = gl[1:1 + LENS_WORDS].to(device=device, dtype=dtype)
                elif fctx.features is not None and (need_f or (grad_fm is not None and (need_v or need_ubo))):  # one pass for all
                    f = fctx.features
                    gfm = (torch.zeros((g.shape[0], g.shape[1], f.shape[1]), dtype=torch.float32, device=v.device) if grad_fm is None
                           else grad_fm.detach().to(torch.float32).contiguous())
                    grad_f = torch.empty_like(f) if need_f else None
                    ctx._backward(v.data_ptr(), g.data_ptr(), grad_v.data_ptr() if need_v else None, stream,
                                  grad_uniforms_ptr=gu.data_ptr() if need_ubo else None,
                                  density_ptr=None if fctx.density is None or not (need_v or need_ubo) else fctx.density.data_ptr(),
                                  grad_depth_alpha_ptr=None if gda is None else gda.data_ptr(), features=f, grad_feature_map=gfm,
                                  grad_features_ptr=grad_f.data_ptr() if need_f else None)
                elif need_v or need_ubo:
                    ctx._backward(v.data_ptr(), g.data_ptr(), grad_v.data_ptr() if need_v else None, stream,
                                  grad_uniforms_ptr=gu.data_ptr() if need_ubo else None,
                                  density_ptr=None if fctx.density is None else fctx.density.data_ptr(),
                                  grad_depth_alpha_ptr=None if gda is None else gda.data_ptr())
                if need_ubo:
                    dtype, device = fctx.ubo_like
                    grad_ubo = gu[UBO_FLOAT_WORDS].to(device=device, dtype=dtype)
                if need_bg:  # sum_p T_final g, on the same stream
                    dtype, device = fctx.bg_like
                    grad_bg = ctx.background_gradient(g, torch.cuda.current_stream(v.device)).to(device=device, dtype=dtype)
                return None, grad_v, None, grad_ubo, None, grad_bg, None, grad_f, grad_lens, None

        _RenderFn = RenderFn
    return _RenderFn


def render_torch(ctx: "Context", vertices, u: Uniforms, ubo=None, density=None, background=None, depth=False, features=None,
                 lens=None, sh_degree=None):
    """Differentiable frame: vertices is a CUDA float32 tensor (n, 60) of GSScene::Vertex records (activated parameters, as
    gsb_scene_upload takes them).  Uploads it from device memory, renders the whole frame as an (H, W, 4) RGBA32F tensor and,
    on backward, returns dL/dvertices through gsb_render_backward.  Turns gsb_set_backward on for `ctx`.  The frame on the
    context must still be this one when backward runs.

    ubo (optional): a (UBO_FLOATS,) tensor of the camera's float fields in ABI order (uniforms_torch makes one from a pose);
    its values replace u's, u still gives the frame size, and backward also returns dL/dubo (gsb_render_backward_camera).
    Only the inputs that require grad are differentiated: frozen vertices cost no n x 60 gradient.

    density (optional): a contiguous (n, 4) float32 tensor on the vertices' device that backward accumulates this frame's
    density-control statistics into (gsb_render_backward_density, on torch's stream): screen-space gradient norm and absolute
    gradient norm in NDC units, the view count and the max pixel radius; see densify_and_prune.  Backward runs only when
    vertices, ubo or background requires grad.

    background (optional): a (3,) tensor; the frame is rendered over its colour (gsb_set_background) and the context's own
    setting is restored after the forward.  If it requires grad, backward also returns dL/dbackground = sum_p T_final(p)
    dL/dimage(p) (gsb_background_gradient, on torch's stream) -- also for frozen vertices, a learned background alone.

    Under torch.use_deterministic_algorithms(True), backward turns gsb_set_backward_deterministic on for `ctx` (otherwise
    off): every gradient and density statistic is then bit-identical for the same inputs, at some cost in time.  With
    torch's default settings backward takes the atomic path, whose results may differ in the last bit from run to run.

    The frame is projected through the context's camera model (Context.set_camera_model); ubo= on a fisheye, OpenCV or
    orthographic context raises ValueError unless lens= is given.

    lens (optional): an (8,) tensor (fx, fy, cx, cy, k[0..3]) (lens_tensor makes one).  The frame is rendered through
    lens_camera(lens, max_theta, kind), kind and max_theta those of the context's lens model if one is set (k1, k2, p1, p2
    for an OpenCV model), else a fisheye at fisheye_camera's default max_theta for these k, and the context's own model is
    restored after the forward (a lens gsb_set_camera_model refuses raises
    GsbError and changes nothing).  Backward runs gsb_render_backward_fisheye: dL/dlens when lens requires grad, dL/dubo
    (camera_position and view rows 0-2 only; the rest is 0) when ubo requires grad, and the other inputs' gradients as
    without lens=.  It composes with depth=, features=, density=, background= and the deterministic mode.

    depth=True renders with gsb_render_depth and returns (img, depth_alpha), depth_alpha an (H, W, 2) tensor of (D, A):
    D = sum f alpha T, f the view-space z (the distance from the camera for a fisheye model, z for OpenCV and orthographic), and A = 1 - T_final, the
    accumulated opacity.  Backward then takes dL/dimg and dL/d(depth_alpha), either of them unused (zero), through
    gsb_render_backward_depth; it composes with ubo=, density=, background= and the deterministic mode.  Expected depth is
    D / A.clamp_min(1e-10), inverse depth its reciprocal, and a mask loss reads A directly.

    features (optional): an (n, C) float32 CUDA tensor of per-Gaussian features, C <= 128.  The frame then also returns its
    (H, W, C) feature map F_c = sum f_ic alpha_i T_i over 0 (gsb_render_features): (img, fmap), or (img, depth_alpha, fmap)
    with depth=True.  Backward differentiates the image, depth / alpha and map in one gsb_render_backward_features pass, into
    vertices, ubo, density and -- when it requires grad -- features.

    sh_degree (optional): 0..3; the frame's colour sums the SH bands <= sh_degree only (gsb_set_sh_degree) and the context's
    own setting is restored after the forward; None uses the context's setting.  Backward follows the frame's degree: the
    coefficients of higher bands get a gradient of exactly 0.  It composes with ubo=, lens=, depth=, features=, density=,
    background= and the deterministic mode."""
    return _render_fn().apply(ctx, vertices, u, ubo, density, background, depth, features, lens, sh_degree)


_LossFn = None


def _loss_fn():
    global _LossFn
    if _LossFn is None:
        import torch

        class LossFn(torch.autograd.Function):
            @staticmethod
            def forward(fctx, ctx, image, target, lambda_dssim):
                img = image.detach()
                # the loss and its gradient in one call; only the loss when the image needs no gradient
                grad = torch.empty(img.shape, dtype=torch.float32, device=img.device) if fctx.needs_input_grad[1] else None
                result = ctx.image_loss(img, target.detach(), lambda_dssim, grad)  # on torch's current stream
                fctx.grad = grad
                return result[0].to(torch.float32)

            @staticmethod
            def backward(fctx, grad_loss):
                return None, fctx.grad * grad_loss, None, None

        _LossFn = LossFn
    return _LossFn


def image_loss_torch(ctx: "Context", image, target, lambda_dssim=0.2):
    """Differentiable photometric loss of 3DGS training (Kerbl et al. 2023) through gsb_image_loss, as a float32 scalar tensor:
    (1 - lambda_dssim) L1 + lambda_dssim (1 - SSIM), means over the RGB values, SSIM with an 11 x 11 Gaussian window
    (sigma 1.5) and zero padding.  image is the (H, W, 4) float32 CUDA tensor render_torch returns, target an (H, W, 4) float32
    or uint8 (read as v / 255) tensor on the same device; A is ignored.  Runs on torch's current stream and never waits on the
    host; backward returns the gradient the forward computed, scaled by the upstream gradient.  The result and the gradient
    are bitwise reproducible for the same inputs.  Bad shapes, dtypes or devices raise ValueError."""
    return _loss_fn().apply(ctx, image, target, float(lambda_dssim))


_BilagridFn = None


def _bilagrid_fn():
    global _BilagridFn
    if _BilagridFn is None:
        import torch

        class BilagridFn(torch.autograd.Function):
            @staticmethod
            def forward(fctx, ctx, image, grid):
                img, grd = image.detach(), grid.detach().contiguous()
                fctx.ctx = ctx
                fctx.save_for_backward(img, grd)
                return ctx.bilagrid_apply(img, grd)  # on torch's current stream

            @staticmethod
            def backward(fctx, grad_out):
                img, grd = fctx.saved_tensors
                want_image, want_grid = fctx.needs_input_grad[1], fctx.needs_input_grad[2]
                if not (want_image or want_grid):
                    return None, None, None
                gi = torch.empty(img.shape, dtype=torch.float32, device=img.device) if want_image else None
                gg = torch.empty_like(grd) if want_grid else None
                go = grad_out.to(torch.float32)
                if go.stride(2) != 1 or go.stride(1) != 4:
                    go = go.contiguous()
                fctx.ctx.bilagrid_backward(img, grd, go, gi, gg)
                if gi is not None:
                    gi[..., 3] = go[..., 3]  # A is copied
                return None, gi, gg

        _BilagridFn = BilagridFn
    return _BilagridFn


def bilateral_grid_torch(ctx: "Context", image, grid):
    """Differentiable bilateral-grid colour correction (Wang et al. 2024; gsplat's BilateralGrid) through gsb_bilagrid_apply:
    the (H, W, 4) float32 frame (render_torch's or SceneAdam.render's) with each pixel's RGB mapped by the 3 x 4 affine
    matrix sliced from `grid` at its position and luma, A copied (DESIGN.md section 17).  grid is a (12, L, Y, X) float32
    tensor, typically grids[i] of an identity_bilateral_grids(n) parameter, so autograd's indexing backward scatters into it.
    The backward (gsb_bilagrid_backward) returns d/d image and d/d grid for whichever require grad, bitwise reproducibly.
    Runs on torch's current stream and never waits on the host."""
    return _bilagrid_fn().apply(ctx, image, grid)


def identity_bilateral_grids(n, shape=(16, 16, 8), device=None):
    """n identity bilateral grids, A = [I | 0] at every node, as an (n, 12, L, Y, X) float32 tensor; shape is (X, Y, L)."""
    import torch

    X, Y, L = shape
    g = torch.zeros((n, 12, L, Y, X), dtype=torch.float32, device=device)
    for c in range(3):
        g[:, 4 * c + c] = 1.0
    return g


def bilateral_grid_tv(grids):
    """Total-variation regulariser of bilateral grids (n, 12, L, Y, X) (or one (12, L, Y, X) grid): over the three grid axes,
    the sum of the mean squared difference of neighbouring nodes, the mean taken over coefficients and node pairs and then
    over the n grids.  Plain torch: the grids are small."""
    g = grids if grids.dim() == 5 else grids.unsqueeze(0)
    return sum(g.diff(dim=d).square().mean() for d in (2, 3, 4))


def composite_target(target, background):
    """An (H, W, 4) RGBA target (float32, or uint8 read as v / 255) composited over `background` (3 values or a (3,) tensor):
    rgb a + bg (1 - a) as an (H, W, 4) float32 tensor with A = 1 -- what a frame rendered over that background (gsb_set_background)
    is compared against.  Runs on the target's device."""
    import torch

    t = target.to(torch.float32) / 255.0 if target.dtype == torch.uint8 else target.to(torch.float32)
    if t.dim() != 3 or t.shape[2] != 4:
        raise ValueError("composite_target: target must be (H, W, 4)")
    bg = torch.as_tensor(background, dtype=torch.float32).to(t.device).reshape(3)
    a = t[..., 3:4]
    out = torch.empty_like(t)
    out[..., :3] = t[..., :3] * a + bg * (1.0 - a)
    out[..., 3] = 1.0
    return out


def image_metrics(ctx: "Context", image, target):
    """Evaluation metrics of an (H, W, 4) float32 CUDA frame against a float32 or uint8 target through gsb_image_loss, on the
    host: {"l1", "ssim", "mse", "psnr"} with PSNR = -10 log10(MSE) for values in [0, 1] (inf for identical RGB)."""
    import math

    _, l1, ssim, mse = (float(v) for v in ctx.image_loss(image, target).cpu())
    return {"l1": l1, "ssim": ssim, "mse": mse, "psnr": -10.0 * math.log10(mse) if mse > 0 else math.inf}


def densify_and_prune(vertices, density, *, grad_threshold, scene_extent, percent_dense=0.01, min_opacity=0.005,
                      max_screen_size=None, use_absgrad=False, generator=None):
    """Adaptive density control (Kerbl et al. 2023, section 5) on activated (n, 60) GSScene::Vertex records, in torch on any
    device.  density is the (n, 4) table render_torch(..., density=) accumulates; resetting it is the caller's job.

    avg = density[:, 1 if use_absgrad else 0] / max(density[:, 2], 1), s_max = the largest of the row's three scales:
      clone  avg >= grad_threshold and s_max <= percent_dense * scene_extent: the row is kept and appended again as it is;
      split  avg >= grad_threshold and s_max >  percent_dense * scene_extent: the row is replaced by two children at
             p + R(q) (s * eps) with scale s / 1.6, the rest of the row copied (R(q) from the quaternion as stored, eps ~ N(0, I)
             drawn as one torch.randn((2 k, 3)) from `generator` for the k split rows, rows 0..k-1 for the first children);
      prune  then, on the result, every row whose opacity < min_opacity and, when max_screen_size is given, every row whose
             source's density[:, 3] (max pixel radius) > max_screen_size or whose own s_max > 0.1 * scene_extent.
    Output order: the kept rows in their order, the clones, the first children, the second children, pruned rows removed.
    Returns (new_vertices, source): source (int64, on vertices' device) is the old row each new row comes from, so the
    caller can gather its optimizer state (and other per-row tensors) with it."""
    import torch

    v = vertices.detach()
    n = v.shape[0]
    if density.shape != (n, 4):
        raise ValueError(f"densify_and_prune: density must be ({n}, 4), got {tuple(density.shape)}")
    d = density.detach().to(device=v.device, dtype=torch.float32)
    avg = d[:, 1 if use_absgrad else 0] / d[:, 2].clamp(min=1.0)
    s_max = v[:, 4:7].max(1).values
    hot = avg >= grad_threshold
    small = s_max <= percent_dense * scene_extent
    clone, split = hot & small, hot & ~small
    rows = torch.arange(n, device=v.device)
    split_rows = rows[split]
    k = split_rows.numel()
    eps = torch.randn((2 * k, 3), generator=generator, dtype=v.dtype, device=v.device)
    parent = v[split_rows].repeat(2, 1)
    q = parent[:, 8:12]
    qw, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([  # the rotation whose columns are the Gaussian's axes: Sigma = R diag(s^2) R^T
        torch.stack([1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy)], -1),
        torch.stack([2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx)], -1),
        torch.stack([2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * (qx * qx + qy * qy)], -1),
    ], -2)
    children = parent.clone()
    children[:, 0:3] = parent[:, 0:3] + (R @ (parent[:, 4:7] * eps)[:, :, None])[:, :, 0]
    children[:, 4:7] = parent[:, 4:7] / 1.6
    source = torch.cat([rows[~split], rows[clone], split_rows, split_rows])
    out = torch.cat([v[~split], v[clone], children])
    prune = out[:, 7] < min_opacity
    if max_screen_size is not None:
        prune |= (d[source, 3] > max_screen_size) | (out[:, 4:7].max(1).values > 0.1 * scene_extent)
    keep = ~prune
    return out[keep].contiguous(), source[keep]


def apply_filter_3d(vertices, variance):
    """Mip-Splatting's 3D smoothing filter (get_scaling_with_3D_filter, get_opacity_with_3D_filter) applied to activated
    (n, 60) records as differentiable torch ops, the variance (n,) held constant: with s the scales and o the opacity,
    q = s s, d = q + v, e = sqrt(d), r = q / d, c = sqrt((r0 r1) r2); the result's scales are e and its opacity o c, every
    other column as given.  In float32 on CUDA each op is the one gsb_adam_step_filter3d does, in its order.  For training
    through render_torch: render_torch(ctx, apply_filter_3d(vertices, variance), u)."""
    import torch

    v = variance.detach().to(device=vertices.device, dtype=vertices.dtype).reshape(-1, 1)
    q = vertices[:, 4:7] * vertices[:, 4:7]
    d = q + v
    r = q / d
    c = ((r[:, 0] * r[:, 1]) * r[:, 2]).sqrt()
    return torch.cat([vertices[:, 0:4], d.sqrt(), (vertices[:, 7] * c)[:, None], vertices[:, 8:60]], 1)


def activate_parameters(params):
    """The activated (n, 60) records of raw parameters, as gsb_adam_step writes them, in torch: (p, 1), exp(log s),
    sigmoid(logit), q / |q|, SH."""
    import torch

    p = params.detach()
    q = p[:, 8:12]
    return torch.cat([p[:, 0:3], torch.ones_like(p[:, 3:4]), p[:, 4:7].exp(), torch.sigmoid(p[:, 7:8]),
                      q / q.norm(dim=1, keepdim=True), p[:, 12:60]], 1).contiguous()


def raw_parameters(vertices):
    """The raw parameters gsb_adam_step optimises, of activated (n, 60) records: position, column 3 as given, log(scale),
    logit(opacity) (opacity clamped to [1e-6, 1 - 1e-6]), the quaternion and SH as given."""
    import torch

    p = vertices.detach().clone()
    p[:, 4:7] = p[:, 4:7].log()
    p[:, 7] = torch.logit(p[:, 7], eps=1e-6)
    return p


def adam_state_after_densify(params, exp_avg, exp_avg_sq, vertices, new_vertices, source):
    """The raw parameters and Adam moments of densify_and_prune's output (new_vertices, source) of `vertices`: every row's
    are gathered from its source row; a split child -- recognised by scale columns that differ from its source's (s / 1.6 !=
    s for every finite s > 0) -- takes its raw position and log scale from new_vertices and starts with zero moments
    (gsplat's convention).  Returns (params, exp_avg, exp_avg_sq)."""
    import torch

    p, m, v = params[source], exp_avg[source], exp_avg_sq[source]
    child = (new_vertices[:, 4:7] != vertices[source, 4:7]).any(1)
    p[child, 0:3] = new_vertices[child, 0:3]
    p[child, 4:7] = new_vertices[child, 4:7].log()
    m[child] = 0.0
    v[child] = 0.0
    return p.contiguous(), m.contiguous(), v.contiguous()


def mcmc_sample(weights, k, generator=None):
    """k row indices drawn with replacement in proportion to `weights` (n non-negative finite values, positive sum), by
    inverse-CDF sampling: the float64 cumulative sum, torch.rand(k, dtype=float64, generator=generator) times the total, and
    searchsorted(right=True), clamped to the last row of positive weight.  Zero-weight rows are never chosen, any n works
    (torch.multinomial stops at 2^24 categories), and the work is done on the CPU, so a seeded CPU generator gives the same
    rows whatever device the weights are on.  Returns an int64 tensor on the weights' device."""
    import torch

    w = weights.detach().to("cpu", torch.float64).reshape(-1)
    n = w.shape[0]
    if k < 0 or n == 0:
        raise ValueError(f"mcmc_sample: needs k >= 0 and at least one weight, got k = {k}, n = {n}")
    cdf = torch.cumsum(w, 0)
    total = float(cdf[-1])
    if not (total > 0.0 and total < float("inf")) or bool((w < 0).any()):
        raise ValueError("mcmc_sample: weights must be non-negative and finite with a positive sum")
    u = torch.rand(int(k), dtype=torch.float64, generator=generator) * total
    idx = torch.searchsorted(cdf, u, right=True)
    last = int(torch.searchsorted(cdf, cdf[-1:], right=False))  # u * total may round up to the total itself
    return idx.clamp_(max=min(n - 1, last)).to(weights.device)


class SceneAdam:
    """Trains the scene resident on `ctx` with gsb_adam_step: the fused chain rule through the activations, Adam and the
    scene update in one kernel, so a step needs no upload and waits on nothing.  A training step reads

        img = opt.render(u); ctx.image_loss(img, target, 0.2, grad_image=g); opt.step(g)

    with one host wait per step, inside gsb_render's arena check.  Owns, as (n, 60) float32 tensors on ctx's device:
    `params` (raw_parameters(vertices)), `exp_avg`, `exp_avg_sq`, `vertices` (the activated records the frames and the
    backward pass read; at first the given ones) and `grad` (the last step's dL/d vertices).

    lr: six learning rates in ADAM_GROUPS order (position, scale, opacity, rotation, SH DC, SH rest), read at every step,
    so the caller may change them (a schedule).  selective=True updates only the rows of the Gaussians that survived the
    frame's culls (the "selective Adam" of Mallick et al. 2024); False is torch.optim.Adam's dense update of every row.
    Turns gsb_set_backward on for ctx and uploads `vertices` once; under torch.use_deterministic_algorithms(True) the
    backward pass runs deterministically, as in render_torch.

    background: the colour render() composites over (gsb_set_background; None = the context's own setting).
    random_background=True: every render() draws a fresh uniform [0, 1)^3 colour from a torch.Generator seeded with `seed`
    (Inria's --random_background: the empty space must stay transparent to match every colour), to be compared against
    composite_target(rgba_target, opt.background).  `background` holds the colour of the last render() as 3 floats.

    sh_degree: the spherical-harmonics degree render() draws at (gsb_set_sh_degree, 0..3), read at every render() like lr,
    so the caller may raise it on a schedule -- Inria's oneupSHdegree every 1000 steps, gsplat's sh_degree_interval:

        opt.sh_degree = min(it // 1000, 3)
        img = opt.render(u); ctx.image_loss(img, target, 0.2, grad_image=g); opt.step(g)

    The backward pass gives the coefficients of the bands above the frame's degree a gradient of exactly 0, and Adam leaves
    a row with zero gradient and zero moments bit-identical, so those bands stay as they are until their degree arrives.  A
    scene from init_from_points has zero higher bands: they start from zero when their degree arrives.

    3D Gaussian Splatting as Markov Chain Monte Carlo (Kheradmand et al. 2024, gsplat's MCMCStrategy) instead of
    densify(): the opacity and scale regularisers in step(), position noise after every step (inject_noise, seeded by
    `seed` and the step count) and a periodic relocate() that moves dead Gaussians onto live ones and grows the scene up to
    a budget of cap_max Gaussians:

        img = opt.render(u)
        ctx.image_loss(img, target, 0.2, grad_image=g)
        opt.step(g, opacity_reg=0.01, scale_reg=0.01)
        opt.inject_noise()
        if 500 < it < 25000 and it % 100 == 0:
            opt.relocate(cap_max)

    Per-image appearance (exposure, white balance, vignetting) with bilateral grids (Wang et al. 2024, gsplat's
    BilateralGrid) needs no change here: the frame is corrected by bilateral_grid_torch before the loss, and the image
    gradient it returns is what step() takes; the grids are an ordinary torch parameter with their own optimizer:

        grids = torch.nn.Parameter(identity_bilateral_grids(n_images, device="cuda"))
        grid_opt = torch.optim.Adam([grids], lr=2e-3, eps=1e-15)
        img = opt.render(u).requires_grad_()
        out = bilateral_grid_torch(ctx, img, grids[i])
        loss = image_loss_torch(ctx, out, target) + 10.0 * bilateral_grid_tv(grids)
        loss.backward(); opt.step(img.grad); grid_opt.step(); grid_opt.zero_grad()

    Mip-Splatting's 3D smoothing filter (Yu et al. 2024), which keeps a scene free of needles and erosion holes when it is
    rendered closer or larger than its training views: filter_cameras, the list of training Uniforms, turns it on.  Then
    `params` stay the unfiltered raw parameters, `variance` holds each Gaussian's filter (Context.filter3d_variance) and
    `vertices` the filtered records (apply_filter_3d of the activated params), which frames render and step() trains
    through gsb_adam_step_filter3d.  filter_lenses gives the training views' lens models (Context.filter3d_variance's
    `lenses`: one CameraModel for all views or a list of one per view), so that fisheye and OpenCV views, mixed lenses
    included, see each Gaussian and resolve it as their frames do; without it the filter reads each view's UBO pinhole
    (tan_fov and ndc2Pix), whatever the context's camera model.
    Mip-Splatting recomputes the filter every 100 steps once densification has ended:

        if it >= densify_until and it % 100 == 0:
            opt.update_filter_3d()

    densify() decides on the unfiltered records and recomputes the filter for the new scene; inject_noise() and relocate()
    (3DGS-MCMC) raise ValueError with a filter.  The filtered records are an ordinary scene: a plain viewer renders the
    trained scene, filter included, from write_ply(path, ply_records(raw_parameters(opt.vertices))).

    Feature fields (Gaussian Grouping, LangSplat, Feature 3DGS): features, an (n, C) float32 tensor (C <= 128), makes the
    optimizer own `features` (a copy), its moments `feature_exp_avg` / `feature_exp_avg_sq` and `grad_features`, trained with
    Adam at feature_lr (identity activation; `selective` applies).  render(u, features=True) also returns the feature map
    (gsb_render_features), and step(..., grad_feature_map=) runs one gsb_render_backward_features pass, then the feature step
    (gsb_adam_step_features), then the scene step.  densify() gathers the feature rows by `source` (split children copy their
    parent's row and start with zero moments, as adam_state_after_densify does for the scene), and relocate() copies the
    source rows onto the relocated ones with zero moments and appends features[src] when it grows."""

    def __init__(self, ctx: "Context", vertices, lr, betas=(0.9, 0.999), eps=1e-15, selective=True, background=None,
                 random_background=False, seed=0, filter_cameras=None, features=None, feature_lr=0.0, filter_lenses=None,
                 sh_degree=3):
        import torch

        if not isinstance(vertices, torch.Tensor) or not vertices.is_cuda or vertices.dim() != 2 or vertices.shape[1] != 60:
            raise ValueError("SceneAdam: vertices must be an (n, 60) CUDA tensor")
        self.ctx, self.lr, self.betas, self.eps, self.selective = ctx, list(lr), tuple(betas), float(eps), bool(selective)
        self.steps = 0
        self.seed = int(seed)
        self.background = None if background is None else [float(x) for x in background]
        self.sh_degree = sh_degree
        self._generator = torch.Generator().manual_seed(int(seed)) if random_background else None
        self.filter_cameras = None if filter_cameras is None else list(filter_cameras)
        self.filter_lenses = filter_lenses
        self.variance = None
        self._adopt(vertices.detach().to(torch.float32).contiguous().clone(), None)
        self.features = self.feature_lr = None
        if features is not None:
            f = features.detach().to(torch.float32).contiguous().clone()
            _check_features("SceneAdam", f, vertices.device)
            if f.shape[0] != vertices.shape[0]:
                raise ValueError("SceneAdam: features must have one row per vertex")
            self.feature_lr = float(feature_lr)
            self._adopt_features(f, torch.zeros_like(f), torch.zeros_like(f))
        if self.filter_cameras is not None:
            self._set_filter(self._filter_variance(), self.vertices)
        ctx.set_backward(True)
        self._upload()

    def _adopt(self, vertices, state):
        import torch

        self.vertices = vertices
        if state is None:
            state = (raw_parameters(vertices), torch.zeros_like(vertices), torch.zeros_like(vertices))
        self.params, self.exp_avg, self.exp_avg_sq = state
        self.grad = torch.empty_like(vertices)

    def _adopt_features(self, features, exp_avg, exp_avg_sq):
        import torch

        self.features, self.feature_exp_avg, self.feature_exp_avg_sq = features, exp_avg, exp_avg_sq
        self.grad_features = torch.empty_like(features)

    def _set_filter(self, variance, unfiltered):
        """Adopts a filter: `variance` (checked finite and >= 0 here, once) and vertices = the filtered `unfiltered`."""
        import torch

        if not bool(torch.isfinite(variance).all()) or bool((variance < 0).any()):
            raise ValueError("SceneAdam: the filter variance must be finite and >= 0")
        self.variance = variance
        self.vertices = apply_filter_3d(unfiltered, variance).contiguous()

    def _filter_variance(self):
        return self.ctx.filter3d_variance(self.params, self.filter_cameras, self.filter_lenses)

    def update_filter_3d(self, cameras=None, lenses=None):
        """Recomputes the 3D filter from the current positions and the training cameras (`cameras`, which then replace
        filter_cameras; None: filter_cameras) through their lenses (`lenses`, which then replace filter_lenses; None:
        filter_lenses), re-activates every row through it and uploads the scene."""
        if cameras is not None:
            self.filter_cameras = list(cameras)
        if lenses is not None:
            self.filter_lenses = lenses
        if self.filter_cameras is None:
            raise ValueError("SceneAdam.update_filter_3d: no training cameras (filter_cameras)")
        self._set_filter(self._filter_variance(), activate_parameters(self.params))
        self._upload()

    def _upload(self):
        import torch

        torch.cuda.current_stream(self.vertices.device).synchronize()  # the upload runs on the context's own stream
        self.ctx.upload(self.vertices)

    def render(self, u: Uniforms, depth=False, features=False):
        """The resident scene's frame of u as an (H, W, 4) float32 tensor, rendered on torch's current stream with the
        backward state recorded, over the optimizer's background (fixed or a fresh random colour).  No upload.  depth=True:
        (image, depth_alpha) from gsb_render_depth (see render_torch), for step(..., grad_depth_alpha=).  features=True (an
        optimizer with features): the (H, W, C) feature map is appended to what is returned, for step(..., grad_feature_map=)."""
        import torch

        if features and self.features is None:
            raise ValueError("SceneAdam.render: features=True needs an optimizer made with features=")
        if self._generator is not None:
            self.background = torch.rand(3, generator=self._generator).tolist()
        if self.background is not None:
            self.ctx.set_background(self.background)
        self.ctx.set_sh_degree(self.sh_degree)
        out = self.ctx._render_whole_frame(u, self.vertices.device, depth)
        if not features:
            return out
        fmap = self.ctx.render_features(self.features)
        return (*out, fmap) if depth else (out, fmap)

    def step(self, grad_image, density=None, opacity_reg=0.0, scale_reg=0.0, grad_depth_alpha=None, grad_feature_map=None,
             grad_uniforms=None, grad_lens=None):
        """One training step from dL/d(the last render()'s image), an (H, W, 4) float32 tensor: gsb_render_backward into
        `grad` (gsb_render_backward_density, accumulating into `density`, an (n, 4) float32 tensor, when given), then
        gsb_adam_step.  Everything runs on torch's current stream; nothing waits on the host.

        opacity_reg, scale_reg: 3DGS-MCMC's regularisers opacity_reg * mean(opacity) + scale_reg * mean(scale) (the mean
        over the n opacities and the 3 n scales), whose gradient opacity_reg / n and scale_reg / (3 n) is added to `grad`'s
        columns 7 and 4-6 before the Adam step (gsplat uses 0.01 for both).  At 0, nothing is added.

        grad_depth_alpha: dL/d(depth_alpha) of the last render(u, depth=True), an (H, W, 2) float32 tensor, trained through
        gsb_render_backward_depth; grad_image may then be None (no colour loss).  ValueError if the last render had no depth.

        grad_feature_map: dL/d(the last render's feature map), an (H, W, C) float32 tensor (an optimizer with features): the
        backward is then gsb_render_backward_features, and `features` take their Adam step before the scene does.

        grad_uniforms, grad_lens: optional (40,) and (8,) float32 CUDA tensors, overwritten by the same backward pass with
        dL/d(the frame's gsb_uniforms, all 40 words) and dL/d(fx, fy, cx, cy, k[0..3]) of the frame's lens (k1..k4 for a
        fisheye, k1, k2, p1, p2 for OpenCV).  A pinhole frame fills grad_uniforms through gsb_render_backward_camera's words
        (grad_lens: ValueError); a fisheye, OpenCV or orthographic frame fills both through gsb_render_backward_fisheye (pose words only).  `grad`, the features and the step are the same as without them.
        Joint pose refinement, with per-view poses (and a lens tensor) in a torch optimizer:

            gu = torch.empty(40, device="cuda")
            ubo = uniforms_torch(pos[i], rot[i], fov, near, far, W, H)  # pos[i], rot[i] require grad
            img = opt.render(unpack_uniforms(ubo.detach().cpu().numpy(), W, H))
            ctx.image_loss(img, target[i], 0.2, grad_image=g)
            opt.step(g, grad_uniforms=gu)
            ubo.backward(gu[UBO_FLOAT_WORDS]); pose_opt.step(); pose_opt.zero_grad()

        For a lens, render through ctx.set_camera_model(lens_camera(lens, max_theta, kind)) and add lens.grad += the grad_lens."""
        import torch

        ctx, v = self.ctx, self.vertices
        if grad_depth_alpha is not None and not ctx._depth_frame:
            raise ValueError("SceneAdam.step: grad_depth_alpha needs a frame of render(u, depth=True)")
        if grad_feature_map is not None and self.features is None:
            raise ValueError("SceneAdam.step: grad_feature_map needs an optimizer made with features=")
        if grad_image is None and grad_depth_alpha is None and grad_feature_map is None:
            raise ValueError("SceneAdam.step: no gradient (grad_image, grad_depth_alpha and grad_feature_map are all None)")
        gfm = None
        if grad_feature_map is not None:
            gfm = grad_feature_map.detach().to(torch.float32).contiguous()
            _check_feature_map("SceneAdam.step", gfm, ctx._frame_size("SceneAdam.step"), self.features)
        g = None if grad_image is None else grad_image.detach().to(torch.float32).contiguous()
        gda = None if grad_depth_alpha is None else grad_depth_alpha.detach().to(torch.float32).contiguous()
        stream = _torch_stream_arg(torch.cuda.current_stream(v.device))
        ctx.set_backward_deterministic(torch.are_deterministic_algorithms_enabled())
        _check_density("SceneAdam.step", density, v)
        for name, t, size in (("grad_uniforms", grad_uniforms, 40), ("grad_lens", grad_lens, LENS_WORDS)):
            if t is not None and (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != (size,)
                                  or t.device != v.device or not t.is_contiguous()):
                raise ValueError(f"SceneAdam.step: {name} must be a contiguous ({size},) float32 tensor on {v.device}")
        common = dict(density_ptr=None if density is None else density.data_ptr(),
                      grad_depth_alpha_ptr=None if gda is None else gda.data_ptr(),
                      features=None if gfm is None else self.features, grad_feature_map=gfm,
                      grad_features_ptr=None if gfm is None else self.grad_features.data_ptr())
        gu = None if grad_uniforms is None else grad_uniforms.data_ptr()
        if ctx.camera is None:
            if grad_lens is not None:
                raise ValueError("SceneAdam.step: grad_lens needs a fisheye, OpenCV or orthographic frame (Context.set_camera_model)")
            ctx._backward(v.data_ptr(), None if g is None else g.data_ptr(), self.grad.data_ptr(), stream, grad_uniforms_ptr=gu,
                          **common)
        elif grad_uniforms is None and grad_lens is None:
            ctx._backward(v.data_ptr(), None if g is None else g.data_ptr(), self.grad.data_ptr(), stream, **common)
        else:
            gl = None if grad_lens is None else torch.empty(10, dtype=torch.float32, device=v.device)  # a gsb_camera_model
            ctx._backward_fisheye(v.data_ptr(), None if g is None else g.data_ptr(), self.grad.data_ptr(), stream,
                                  grad_uniforms_ptr=gu, grad_lens_ptr=None if gl is None else gl.data_ptr(), **common)
            if gl is not None:
                grad_lens.copy_(gl[1:1 + LENS_WORDS])
        n = v.shape[0]
        if opacity_reg:
            self.grad[:, 7] += opacity_reg / n
        if scale_reg:
            self.grad[:, 4:7] += scale_reg / (3 * n)
        self.steps += 1
        cfg = adam_config(self.lr, self.betas, self.eps, self.steps, self.selective)
        if gfm is not None:  # before the scene step, while the frame (its survivors, for selective) is still valid
            ctx.adam_step_features(self.features, self.feature_exp_avg, self.feature_exp_avg_sq, self.grad_features,
                                   self.feature_lr, cfg)
        ctx.adam_step(self.params, self.exp_avg, self.exp_avg_sq, self.grad, v,
                      adam_config(self.lr, self.betas, self.eps, self.steps, self.selective), variance=self.variance)

    def densify(self, density, **kwargs):
        """densify_and_prune(vertices, density, **kwargs) of the resident scene: `vertices` becomes its output, params and
        the moments follow through adam_state_after_densify, and the new scene is uploaded.  Returns `source`.  With the 3D
        filter the decisions are made on the unfiltered records (activate_parameters(params), as Mip-Splatting's
        get_scaling and get_opacity), and the filter is recomputed for the new scene before the upload."""
        unfiltered = self.vertices if self.variance is None else activate_parameters(self.params)
        new, source = densify_and_prune(unfiltered, density, **kwargs)
        if self.features is not None:  # split children (scale changed, as adam_state_after_densify finds them): zero moments
            child = (new[:, 4:7] != unfiltered[source, 4:7]).any(1)
            m, s = self.feature_exp_avg[source], self.feature_exp_avg_sq[source]
            m[child] = 0.0
            s[child] = 0.0
            self._adopt_features(self.features[source].contiguous(), m.contiguous(), s.contiguous())
        self._adopt(new, adam_state_after_densify(self.params, self.exp_avg, self.exp_avg_sq, unfiltered, new, source))
        if self.variance is not None:
            self._set_filter(self._filter_variance(), new)
        self._upload()
        return source

    def inject_noise(self, noise_lr=5e5):
        """3DGS-MCMC's position noise on the resident scene (gsb_mcmc_noise) with scale lr[0] * noise_lr, the optimizer's
        seed and its step count: every row moves by Sigma eps, gated to zero as its opacity approaches 1.  Runs on torch's
        current stream without a host wait.  Not defined with the 3D filter: ValueError."""
        self._no_filter("inject_noise")
        self.ctx.mcmc_noise(self.params, self.vertices, float(self.lr[0]) * float(noise_lr), self.seed, self.steps)

    def _no_filter(self, caller):
        if self.variance is not None:
            raise ValueError(f"SceneAdam.{caller}: 3DGS-MCMC is not defined with the 3D filter (filter_cameras)")

    def relocate(self, cap_max, min_opacity=0.005, growth=0.05, generator=None):
        """3DGS-MCMC's relocation and growth (gsplat's MCMCStrategy), in two phases; returns (n_relocated, n_added).
          relocate  the dead rows, vertices[:, 7] <= min_opacity, each become a copy of a live row drawn with mcmc_sample in
                    proportion to opacity (gsb_mcmc_relocate corrects the sources' opacity and scale for their copies); n
                    is unchanged and nothing is uploaded.  Skipped when no row is alive.
          add       k = max(0, min(cap_max, floor((1 + growth) n)) - n) sources drawn over all rows in proportion to
                    opacity are appended (params and vertices copied, moments zero), the scene is uploaded once, and
                    gsb_mcmc_relocate makes rows n .. n + k - 1 their copies.
        generator: a CPU torch.Generator for the draws (None: torch's default).  Not defined with the 3D filter: ValueError."""
        import math

        import torch

        self._no_filter("relocate")
        v = self.vertices
        dev = v.device
        n = v.shape[0]
        op = v[:, 7]
        dead = op <= min_opacity
        n_dead = int(dead.sum())
        n_relocated = 0
        if 0 < n_dead < n:
            src = mcmc_sample(torch.where(dead, torch.zeros_like(op), op), n_dead, generator)
            dst = torch.nonzero(dead)[:, 0]
            self.ctx.mcmc_relocate(self.params, self.exp_avg, self.exp_avg_sq, v, dst.to(torch.int32), src.to(torch.int32),
                                   min_opacity)
            if self.features is not None:
                self.features[dst] = self.features[src]
                self.feature_exp_avg[dst] = 0.0
                self.feature_exp_avg_sq[dst] = 0.0
            n_relocated = n_dead
        k = max(0, min(int(cap_max), int(math.floor((1.0 + growth) * n))) - n)
        if k > 0:
            src = mcmc_sample(self.vertices[:, 7], k, generator)
            zeros = torch.zeros((k, 60), dtype=torch.float32, device=dev)
            self._adopt(torch.cat([self.vertices, self.vertices[src]]).contiguous(),
                        (torch.cat([self.params, self.params[src]]).contiguous(),
                         torch.cat([self.exp_avg, zeros]).contiguous(), torch.cat([self.exp_avg_sq, zeros]).contiguous()))
            if self.features is not None:
                fz = torch.zeros((k, self.features.shape[1]), dtype=torch.float32, device=dev)
                self._adopt_features(torch.cat([self.features, self.features[src]]).contiguous(),
                                     torch.cat([self.feature_exp_avg, fz]).contiguous(), torch.cat([self.feature_exp_avg_sq, fz]).contiguous())
            self._upload()
            dst = torch.arange(n, n + k, dtype=torch.int32, device=dev)
            self.ctx.mcmc_relocate(self.params, self.exp_avg, self.exp_avg_sq, self.vertices, dst, src.to(torch.int32),
                                   min_opacity)
        return n_relocated, k


def _uniforms_restated(position, rotation_wxyz, fov_deg, near, far, width, height):
    """Renderer::makeUniforms and host/gsmath.h restated in float64 torch ops (differentiable in position, rotation and fov):
    view = inverse(translate(position) mat4_cast(q)) with q as given (not normalised), tan_fovx = tan(radians(fov) / 2),
    tan_fovy = tan_fovx H / W, proj = perspective(2 atan(tan_fovy), W / H, near, far) view, then rows y, z of view and row y
    of proj negated.  Returns the UBO_FLOATS float fields in ABI order."""
    import torch

    p, q, fov = position, rotation_wxyz, fov_deg
    w, x, y, z = q[0], q[1], q[2], q[3]
    one, zero = torch.ones_like(w), torch.zeros_like(w)
    R = torch.stack([  # mat4_cast: rows of the rotation
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)]),
        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)]),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]),
    ])
    M = torch.cat([torch.cat([R, p[:, None]], 1), torch.stack([zero, zero, zero, one])[None, :]], 0)  # translate * rotation
    view = torch.linalg.inv(M)
    tan_fovx = torch.tan(torch.deg2rad(fov) / 2)
    tan_fovy = tan_fovx * float(height) / float(width)
    aspect = float(width) / float(height)
    persp = torch.stack([
        torch.stack([1 / (aspect * tan_fovy), zero, zero, zero]),
        torch.stack([zero, 1 / tan_fovy, zero, zero]),
        torch.stack([zero, zero, -(far + near) / (far - near) * one, -(2 * far * near) / (far - near) * one]),
        torch.stack([zero, zero, -one, zero]),
    ])
    proj = persp @ view
    flip = torch.tensor([1.0, -1.0, -1.0, 1.0], dtype=view.dtype)[:, None]
    view = view * flip
    proj = proj * torch.tensor([1.0, -1.0, 1.0, 1.0], dtype=proj.dtype)[:, None]
    return torch.cat([p, one[None], proj.T.reshape(16), view.T.reshape(16), tan_fovx[None], tan_fovy[None]])


def uniforms_torch(position, rotation_wxyz, fov_deg, near, far, width, height):
    """Differentiable gsb_uniforms of a camera pose, for render_torch(..., ubo=): a (UBO_FLOATS,) float32 tensor of the float
    fields in ABI order (camera_position[4], proj_mat[16], view_mat[16], tan_fovx, tan_fovy) on position's device.

    Its value is exactly what gsh_uniforms_from_camera (Renderer::makeUniforms) produces for the float32 inputs, bit for bit,
    so a pose renders the viewer's image of that pose.  Its gradient is that of the float64 restatement of makeUniforms
    (position (3,), rotation_wxyz (4,) used as given -- normalise it in torch if it is a free parameter -- and fov_deg may
    each be a tensor that requires grad; near, far, width and height are constants)."""
    import torch

    position, rotation_wxyz, fov_deg = (torch.as_tensor(t) for t in (position, rotation_wxyz, fov_deg))
    device = position.device
    host = uniforms_from_camera(position.detach().to("cpu", torch.float32).numpy(),
                                rotation_wxyz.detach().to("cpu", torch.float32).numpy(),
                                float(fov_deg.detach().to(torch.float32)), near, far, width, height)
    value = torch.from_numpy(pack_uniforms(host)).to(torch.float64)
    r = _uniforms_restated(*(t.to("cpu", torch.float64) for t in (position, rotation_wxyz, fov_deg)),
                           float(near), float(far), width, height)
    # straight-through: the host's value with the restatement's gradient.  Written as value - (r' - r) rather than
    # value + (r - r'): r' - r is +0, and x - (+0) keeps x's sign even when x is -0 (the flipped rows hold -0 entries).
    return (value - (r.detach() - r)).to(torch.float32).to(device)


# ---------------------------------------------------------------- one frame over several GPUs
def shard_slice(n_total: int, rank: int, world: int):
    """(first, count) of the Gaussians rank `rank` holds (gsb_shard_slice)."""
    first, count = C.c_uint64(), C.c_uint64()
    assert lib.gsb_shard_slice(n_total, rank, world, C.byref(first), C.byref(count)) == OK
    return first.value, count.value


def _frame_shape(u: Uniforms, fmt):
    return (u.height, u.width, 4), (np.float32 if fmt == FORMAT_RGBA32F else np.uint8)


class Group:
    """gsb_group: one process drives `devices` (ids may repeat: several ranks on one GPU)."""

    def __init__(self, devices):
        devices = list(devices)
        arr = (C.c_int * len(devices))(*devices)
        h = _vp()
        rc = lib.gsb_group_create(len(devices), arr, C.byref(h))
        if rc != OK:
            raise GsbError(rc, lib.gsb_shard_last_error().decode())
        self.h = h
        self.size = len(devices)

    def close(self):
        if self.h:
            lib.gsb_group_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != OK:
            raise GsbError(rc, lib.gsb_group_last_error(self.h).decode())

    def context(self, rank) -> "Context":
        return Context(handle=_vp(lib.gsb_group_context(self.h, rank)))

    def upload(self, vertices: np.ndarray):
        v = _f32(vertices).reshape(-1, 60)
        self._ck(lib.gsb_group_scene_upload(self.h, v.ctypes.data, v.shape[0], MEM_HOST))

    def render(self, u: Uniforms, fmt=FORMAT_RGBA32F) -> np.ndarray:
        shape, dt = _frame_shape(u, fmt)
        out = np.empty(shape, dt)
        self._ck(lib.gsb_group_render(self.h, C.byref(u), out.ctypes.data, 0, MEM_HOST, fmt))
        return out

    def render_async(self, u: Uniforms, fmt=FORMAT_BGRA8):
        self._ck(lib.gsb_group_render_async(self.h, C.byref(u), fmt))


def shard_unique_id() -> bytes:
    buf = (C.c_ubyte * 128)()
    rc = lib.gsb_shard_unique_id(buf)
    if rc != OK:
        raise GsbError(rc, lib.gsb_shard_last_error().decode())
    return bytes(buf)


class ShardedContext(Context):
    """gsb_create_sharded: this process is rank `rank` of `world` (one process per GPU)."""

    def __init__(self, device, rank, world, unique_id: bytes):
        h = _vp()
        idbuf = (C.c_ubyte * 128).from_buffer_copy(unique_id)
        rc = lib.gsb_create_sharded(device, rank, world, idbuf, C.byref(h))
        if rc != OK:
            raise GsbError(rc, lib.gsb_shard_last_error().decode() or lib.gsb_last_error(None).decode())
        super().__init__(device, handle=h)
        self._own = True
        self.rank, self.world = rank, world

    def upload_slice(self, slice_vertices: np.ndarray, n_total: int):
        v = _f32(slice_vertices).reshape(-1, 60)
        self._ck(lib.gsb_scene_upload_sharded(self.h, v.ctypes.data, n_total, MEM_HOST))

    def render_sharded(self, u: Uniforms, fmt=FORMAT_RGBA32F, stream=None) -> np.ndarray:
        shape, dt = _frame_shape(u, fmt)
        out = np.empty(shape, dt)
        self._ck(lib.gsb_render_sharded(self.h, C.byref(u), out.ctypes.data, 0, MEM_HOST, fmt, stream_ptr(stream)))
        return out

    def render_sharded_into(self, u: Uniforms, out_ptr, fmt, mem=MEM_DEVICE, stream=None):
        self._ck(lib.gsb_render_sharded(self.h, C.byref(u), out_ptr, 0, mem, fmt, stream_ptr(stream)))

    def render_sharded_async(self, u: Uniforms, fmt, stream=None):
        self._ck(lib.gsb_render_sharded_async(self.h, C.byref(u), fmt, stream_ptr(stream)))

    def frame_ptr(self) -> int:
        return lib.gsb_shard_frame(self.h)


# ---------------------------------------------------------------- the C++ host Renderer (vkgs_* style bridge)
class HostRenderer:
    """C++ `Renderer` (3dgs.cpp_b200/host/Renderer.h) driven through the gsh_* C bridge."""

    def __init__(self, scene_path, device=0, width=1280, height=720, fmt=FORMAT_BGRA8, mode=MODE_EXACT):
        self.h = host.gsh_initialize(str(scene_path).encode(), device, width, height, fmt, mode)
        if not self.h:
            raise RuntimeError(host.gsh_last_error().decode())
        self.width, self.height, self.fmt = width, height, fmt

    def _ck(self, rc):
        if rc != 0:
            raise RuntimeError(host.gsh_last_error().decode())

    def close(self):
        if self.h:
            host.gsh_cleanup(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_camera(self, pos, quat_wxyz, fov=45.0, near=0.1, far=1000.0):
        p, q = _f32(pos, 3), _f32(quat_wxyz, 4)
        self._ck(host.gsh_set_camera(self.h, p.ctypes.data, q.ctypes.data, fov, near, far))

    def get_camera(self):
        p, q, f = np.zeros(3, np.float32), np.zeros(4, np.float32), C.c_float()
        self._ck(host.gsh_get_camera(self.h, p.ctypes.data, q.ctypes.data, C.byref(f)))
        return p, q, f.value

    def movement(self, x, y, z):
        self._ck(host.gsh_movement(self.h, x, y, z))

    def pan(self, dx, dy):
        self._ck(host.gsh_pan_translation(self.h, dx, dy))

    def keys(self, keys):
        arr = (C.c_int * 6)(*[int(k) for k in keys])
        self._ck(host.gsh_key_input(self.h, arr))

    def draw(self) -> np.ndarray:
        self._ck(host.gsh_draw(self.h))
        return self._frame(self.width, self.height, self.fmt)

    def render(self, width, height, fmt=FORMAT_RGBA32F) -> np.ndarray:
        self._ck(host.gsh_render(self.h, width, height, fmt, None, 0))
        return self._frame(width, height, fmt)

    def _frame(self, w, h, fmt):
        n = C.c_size_t()
        p = host.gsh_frame(self.h, C.byref(n))
        dt = np.float32 if fmt == FORMAT_RGBA32F else np.uint8
        buf = (C.c_char * n.value).from_address(p)
        return np.frombuffer(buf, dtype=dt).reshape(h, w, 4).copy()

    def stats(self) -> Stats:
        s = Stats()
        self._ck(host.gsh_stats(self.h, C.byref(s)))
        return s

    @property
    def num_vertices(self):
        return host.gsh_num_vertices(self.h)
