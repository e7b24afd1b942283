"""ctypes wrapper over oracle/liboracle.so (gs_oracle.c).

TEST INFRASTRUCTURE ONLY: may be imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs -- never by the product (3dgs.cpp_b200/).
Parity: the shader stages are pinned to the reference's own shaders run on the CPU (ref_shaders.py,
tests/test_ref_shaders.py); the host camera math and PLY load are not (see gs_oracle.h).
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB_PATH = HERE / "liboracle.so"


def build(force=False):
    if force or not LIB_PATH.exists() or LIB_PATH.stat().st_mtime < (HERE / "gs_oracle.c").stat().st_mtime:
        subprocess.run(["make", "-C", str(HERE), "-B" if force else "-s"], check=True, capture_output=True)
    return LIB_PATH


build()
lib = C.CDLL(str(LIB_PATH))


class Uniforms(C.Structure):
    _fields_ = [("camera_position", C.c_float * 4), ("proj_mat", C.c_float * 16), ("view_mat", C.c_float * 16),
                ("width", C.c_uint32), ("height", C.c_uint32), ("tan_fovx", C.c_float), ("tan_fovy", C.c_float)]


ATTR_DTYPE = np.dtype([("conic_opacity", "<f4", 4), ("color_radii", "<f4", 4), ("aabb", "<u4", 4),
                       ("uv", "<f4", 2), ("depth", "<f4"), ("magic", "<u4")])


class Frame(C.Structure):
    _fields_ = [("n", C.c_uint64), ("m", C.c_uint64), ("width", C.c_uint32), ("height", C.c_uint32),
                ("tiles_x", C.c_uint32), ("tiles_y", C.c_uint32), ("attr", C.c_void_p), ("tiles", C.c_void_p),
                ("scan", C.c_void_p), ("keys", C.c_void_p), ("vals", C.c_void_p), ("keys_unsorted", C.c_void_p),
                ("vals_unsorted", C.c_void_p), ("ranges", C.c_void_p), ("consumed", C.c_void_p),
                ("rgba", C.c_void_p), ("t_stage", C.c_double * 6)]


_vp = C.c_void_p
lib.gso_set_exp_mode.argtypes = [C.c_int]
lib.gso_set_exp_mode.restype = None
lib.gso_get_exp_mode.restype = C.c_int
lib.gso_exp_shared.argtypes = [C.c_float]
lib.gso_exp_shared.restype = C.c_float
lib.gso_load_records.argtypes = [_vp, C.c_uint64, _vp]
lib.gso_load_records.restype = None
lib.gso_load_ply.argtypes = [C.c_char_p, C.POINTER(C.c_uint64)]
lib.gso_load_ply.restype = C.POINTER(C.c_float)
lib.gso_free.argtypes = [_vp]
lib.gso_free.restype = None
lib.gso_cov3d.argtypes = [_vp, C.c_uint64, C.c_float, _vp]
lib.gso_cov3d.restype = None
lib.gso_uniforms_from_camera.argtypes = [_vp, _vp, C.c_float, C.c_float, C.c_float, C.c_uint32, C.c_uint32,
                                         C.POINTER(Uniforms)]
lib.gso_uniforms_from_camera.restype = None
lib.gso_camera_translate.argtypes = [_vp, _vp, _vp]
lib.gso_camera_translate.restype = None
lib.gso_pack_unorm8.argtypes = [_vp, C.c_uint64, C.c_int, _vp]
lib.gso_pack_unorm8.restype = None
lib.gso_sort.argtypes = [_vp, _vp, C.c_uint64]
lib.gso_sort.restype = None
lib.gso_render_frame.argtypes = [_vp, _vp, C.c_uint64, C.POINTER(Uniforms), C.c_uint32, C.c_uint32, C.POINTER(Frame)]
lib.gso_render_frame.restype = C.c_int
lib.gso_frame_free.argtypes = [C.POINTER(Frame)]
lib.gso_frame_free.restype = None
lib.gso_num_threads.restype = C.c_int
lib.gso_preprocess.argtypes = [_vp, _vp, C.c_uint64, C.POINTER(Uniforms), C.c_uint32, C.c_uint32, _vp, _vp]
lib.gso_preprocess.restype = None

lib.gso_set_num_threads.argtypes = [C.c_int]
lib.gso_set_num_threads.restype = None


class SynthParams(C.Structure):
    _fields_ = [("center", C.c_float * 3), ("half_extent", C.c_float * 3), ("log_scale_min", C.c_float),
                ("log_scale_max", C.c_float), ("opacity_min", C.c_float), ("opacity_max", C.c_float),
                ("sh_dc_range", C.c_float), ("sh_rest_sigma", C.c_float)]


lib.gso_synth_records.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(SynthParams), _vp]
lib.gso_synth_records.restype = None

STAGES = ["preprocess", "prefix_sum", "preprocess_sort", "sort", "tile_boundary", "render"]
ALL_ROWS = 0xFFFFFFFF


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def set_exp_mode(mode: int):
    lib.gso_set_exp_mode(mode)


def exp_shared(x: float) -> float:
    return lib.gso_exp_shared(x)


def num_threads() -> int:
    return lib.gso_num_threads()


def set_num_threads(n: int):
    lib.gso_set_num_threads(int(n))


def synth_params(center=(0, 0, 0), half_extent=(3, 3, 3), log_scale_min=None, log_scale_max=None, opacity_min=-2.0,
                 opacity_max=4.0, sh_dc_range=1.0, sh_rest_sigma=0.1) -> SynthParams:
    """Defaults = BASELINE config 1 (the product's gsh_synth_default_params)."""
    p = SynthParams()
    p.center[:] = list(center)
    p.half_extent[:] = list(half_extent)
    p.log_scale_min = np.float32(np.log(np.float32(0.01))) if log_scale_min is None else log_scale_min
    p.log_scale_max = np.float32(np.log(np.float32(0.15))) if log_scale_max is None else log_scale_max
    p.opacity_min, p.opacity_max, p.sh_dc_range, p.sh_rest_sigma = opacity_min, opacity_max, sh_dc_range, sh_rest_sigma
    return p


def synth_records(seed: int, n: int, params: SynthParams | None = None, first: int = 0) -> np.ndarray:
    params = params or synth_params()
    out = np.empty((n, 62), np.float32)
    lib.gso_synth_records(seed, first, n, C.byref(params), out.ctypes.data)
    return out


def load_records(records) -> np.ndarray:
    rec = _f32(records).reshape(-1, 62)
    out = np.empty((rec.shape[0], 60), np.float32)
    lib.gso_load_records(rec.ctypes.data, rec.shape[0], out.ctypes.data)
    return out


def load_ply(path) -> np.ndarray:
    n = C.c_uint64(0)
    p = lib.gso_load_ply(str(path).encode(), C.byref(n))
    if not p:
        raise RuntimeError(f"oracle could not load {path}")
    try:
        return np.ctypeslib.as_array(p, shape=(n.value, 60)).copy() if n.value else np.empty((0, 60), np.float32)
    finally:
        lib.gso_free(p)


def cov3d(vertices, scale_factor=1.0) -> np.ndarray:
    v = _f32(vertices).reshape(-1, 60)
    out = np.empty((v.shape[0], 6), np.float32)
    lib.gso_cov3d(v.ctypes.data, v.shape[0], scale_factor, out.ctypes.data)
    return out


def uniforms_from_camera(pos, quat_wxyz, fov_deg, near, far, width, height) -> Uniforms:
    u = Uniforms()
    p, q = _f32(pos), _f32(quat_wxyz)
    lib.gso_uniforms_from_camera(p.ctypes.data, q.ctypes.data, fov_deg, near, far, width, height, C.byref(u))
    return u


def camera_translate(pos, quat_wxyz, t) -> np.ndarray:
    p, q, tt = _f32(pos).copy(), _f32(quat_wxyz), _f32(t)
    lib.gso_camera_translate(p.ctypes.data, q.ctypes.data, tt.ctypes.data)
    return p


def pack_unorm8(rgba, bgra=False) -> np.ndarray:
    a = _f32(rgba)
    out = np.empty(a.shape, np.uint8)
    lib.gso_pack_unorm8(a.ctypes.data, a.size // 4, int(bgra), out.ctypes.data)
    return out


def sort_pairs(keys, vals):
    k = np.ascontiguousarray(keys, np.uint64).copy()
    v = np.ascontiguousarray(vals, np.uint32).copy()
    lib.gso_sort(k.ctypes.data, v.ctypes.data, k.size)
    return k, v


def preprocess(vertices, cov, u, rows=None):
    """A3 only (preprocess.comp): returns (attr, tiles_overlap)."""
    v = _f32(vertices).reshape(-1, 60)
    cv = _f32(cov).reshape(-1, 6)
    ou = Uniforms.from_buffer_copy(bytes(u))
    rb, re = (0, ALL_ROWS) if rows is None else rows
    attr = np.zeros(v.shape[0], ATTR_DTYPE)
    tiles = np.zeros(v.shape[0], np.uint32)
    lib.gso_preprocess(v.ctypes.data, cv.ctypes.data, v.shape[0], C.byref(ou), rb, re, attr.ctypes.data, tiles.ctypes.data)
    return attr, tiles


def uniforms_bytes(u) -> bytes:
    return bytes(memoryview(u))[:160] if not isinstance(u, Uniforms) else bytes(u)


lib.gso_set_step_probe.argtypes = [_vp, C.c_float]
lib.gso_set_step_probe.restype = None


def render_frame_probed(vertices, cov, u, rows=None, rel_delta=2e-3):
    """render_frame + the step-function probe: returns (frame, mask) where mask[y, x] is True for pixels that evaluate
    `alpha < 1/255` or `test_T < 1e-4` within rel_delta of the threshold (the only places where two exp flavours may
    legitimately disagree by more than rounding noise)."""
    ou = Uniforms.from_buffer_copy(bytes(u))
    mask = np.zeros((ou.height, ou.width), np.uint8)
    lib.gso_set_step_probe(mask.ctypes.data, rel_delta)
    try:
        f = render_frame(vertices, cov, u, rows)
    finally:
        lib.gso_set_step_probe(None, 0.0)
    return f, mask.astype(bool)


def render_frame(vertices, cov, u, rows=None, light=False) -> dict:
    """Runs the whole oracle frame; returns every intermediate as numpy arrays (light=True: counts and stage times only,
    for timing)."""
    v = _f32(vertices).reshape(-1, 60)
    cv = _f32(cov).reshape(-1, 6)
    ou = Uniforms.from_buffer_copy(bytes(u))  # accept the product's ctypes struct too (same 160-B layout)
    rb, re = (0, ALL_ROWS) if rows is None else rows
    f = Frame()
    rc = lib.gso_render_frame(v.ctypes.data, cv.ctypes.data, v.shape[0], C.byref(ou), rb, re, C.byref(f))
    if rc != 0:
        lib.gso_frame_free(C.byref(f))
        raise MemoryError("oracle frame allocation failed")
    try:
        n, m, T = f.n, f.m, f.tiles_x * f.tiles_y
        if light:
            return {"n": n, "m": m, "tiles_x": f.tiles_x, "tiles_y": f.tiles_y, "t_stage": dict(zip(STAGES, list(f.t_stage)))}

        def arr(ptr, dtype, count):
            if count == 0:
                return np.empty(0, dtype)
            nbytes = np.dtype(dtype).itemsize * count
            return np.frombuffer((C.c_char * nbytes).from_address(ptr), dtype=dtype, count=count).copy()

        out = {
            "n": n, "m": m, "tiles_x": f.tiles_x, "tiles_y": f.tiles_y,
            "attr": arr(f.attr, ATTR_DTYPE, n), "tiles": arr(f.tiles, np.uint32, n), "scan": arr(f.scan, np.uint32, n),
            "keys": arr(f.keys, np.uint64, m), "vals": arr(f.vals, np.uint32, m),
            "keys_unsorted": arr(f.keys_unsorted, np.uint64, m), "vals_unsorted": arr(f.vals_unsorted, np.uint32, m),
            "ranges": arr(f.ranges, np.uint32, 2 * T).reshape(-1, 2), "consumed": arr(f.consumed, np.uint32, T),
            "rgba": arr(f.rgba, np.float32, f.width * f.height * 4).reshape(f.height, f.width, 4),
            "t_stage": dict(zip(STAGES, list(f.t_stage))),
        }
        return out
    finally:
        lib.gso_frame_free(C.byref(f))
