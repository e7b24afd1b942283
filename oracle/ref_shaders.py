"""ctypes wrapper over oracle/_ref/libgsref.so: the reference renderer's compute shaders, translated to C++ and run on
the CPU stage by stage (ref_driver.cpp).  TEST INFRASTRUCTURE ONLY.  Built by `make -C oracle ref` (and so by
__graft_entry__.build()) when the reference tree is present; without it, load() raises with instructions."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

import oracle as o

HERE = Path(__file__).resolve().parent
LIB_PATH = HERE / "_ref" / "libgsref.so"
_lib = None


def load():
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise RuntimeError(f"{LIB_PATH} is missing: `python __graft_entry__.py build` builds it when it finds the "
                               "reference source tree (shg8/3DGS.cpp; set GS_REFERENCE to its directory), or run "
                               "`make -C oracle ref REFERENCE=<dir>`")
        lib = C.CDLL(str(LIB_PATH))
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        sigs = {"gsr_set_exp_mode": ([C.c_int], None), "gsr_cov3d": ([vp, u64, C.c_float, vp], None),
                "gsr_preprocess": ([vp, vp, u64, C.POINTER(o.Uniforms), vp, vp], None),
                "gsr_scan": ([vp, u64, vp], u32), "gsr_emit_keys": ([vp, vp, u64, u32, u64, vp, vp], None),
                "gsr_sort": ([vp, vp, u64], None), "gsr_tile_ranges": ([vp, u64, u32, vp], None),
                "gsr_blend": ([vp, u64, vp, u64, vp, u32, u32, vp], None),
                "gsr_render_frame": ([vp, u64, C.POINTER(o.Uniforms), C.POINTER(o.Frame)], C.c_int),
                "gsr_frame_free": ([C.POINTER(o.Frame)], None)}
        for name, (args, res) in sigs.items():
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = res
        _lib = lib
    return _lib


def _f32(a, cols):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def _u(u):
    return o.Uniforms.from_buffer_copy(bytes(u))


def set_exp_mode(mode: int):
    load().gsr_set_exp_mode(mode)


def cov3d(vertices, scale_factor=1.0):
    v = _f32(vertices, 60)
    out = np.empty((v.shape[0], 6), np.float32)
    load().gsr_cov3d(v.ctypes.data, v.shape[0], scale_factor, out.ctypes.data)
    return out


def preprocess(vertices, cov, u, attr=None, tiles=None):
    """preprocess.comp into `attr` / `tiles` (the caller's initial contents stay where the shader writes nothing)."""
    v, cv = _f32(vertices, 60), _f32(cov, 6)
    attr = np.zeros(v.shape[0], o.ATTR_DTYPE) if attr is None else np.ascontiguousarray(attr, o.ATTR_DTYPE).copy()
    tiles = np.zeros(v.shape[0], np.uint32) if tiles is None else np.ascontiguousarray(tiles, np.uint32).copy()
    ou = _u(u)
    load().gsr_preprocess(v.ctypes.data, cv.ctypes.data, v.shape[0], C.byref(ou), attr.ctypes.data, tiles.ctypes.data)
    return attr, tiles


def scan(tiles):
    t = np.ascontiguousarray(tiles, np.uint32)
    out = np.zeros(t.size, np.uint32)
    total = load().gsr_scan(t.ctypes.data, t.size, out.ctypes.data)
    return out, int(total)


def emit_keys(attr, scan_, tile_x, m):
    a = np.ascontiguousarray(attr, o.ATTR_DTYPE)
    s = np.ascontiguousarray(scan_, np.uint32)
    keys, vals = np.zeros(m, np.uint64), np.zeros(m, np.uint32)
    load().gsr_emit_keys(a.ctypes.data, s.ctypes.data, a.size, tile_x, m, keys.ctypes.data, vals.ctypes.data)
    return keys, vals


def sort_pairs(keys, vals):
    k = np.ascontiguousarray(keys, np.uint64).copy()
    v = np.ascontiguousarray(vals, np.uint32).copy()
    load().gsr_sort(k.ctypes.data, v.ctypes.data, k.size)
    return k, v


def tile_ranges(keys, num_tiles):
    k = np.ascontiguousarray(keys, np.uint64)
    out = np.empty(2 * num_tiles, np.uint32)
    load().gsr_tile_ranges(k.ctypes.data, k.size, num_tiles, out.ctypes.data)
    return out.reshape(-1, 2)


def blend(attr, vals, ranges, width, height):
    a = np.ascontiguousarray(attr, o.ATTR_DTYPE)
    v = np.ascontiguousarray(vals, np.uint32)
    r = np.ascontiguousarray(ranges, np.uint32)
    out = np.zeros((height, width, 4), np.float32)
    load().gsr_blend(a.ctypes.data, a.size, v.ctypes.data, v.size, r.ctypes.data, width, height, out.ctypes.data)
    return out


def render_frame(vertices, u) -> dict:
    """The whole frame from the vertices (precomp_cov3d included); the same keys as oracle.render_frame but `consumed`."""
    v = _f32(vertices, 60)
    ou = _u(u)
    f = o.Frame()
    lib = load()
    if lib.gsr_render_frame(v.ctypes.data, v.shape[0], C.byref(ou), C.byref(f)) != 0:
        lib.gsr_frame_free(C.byref(f))
        raise MemoryError("reference frame allocation failed")
    try:
        n, m, T = f.n, f.m, f.tiles_x * f.tiles_y

        def arr(ptr, dtype, count):
            if count == 0:
                return np.empty(0, dtype)
            nbytes = np.dtype(dtype).itemsize * count
            return np.frombuffer((C.c_char * nbytes).from_address(ptr), dtype=dtype, count=count).copy()

        return {"n": n, "m": m, "tiles_x": f.tiles_x, "tiles_y": f.tiles_y,
                "attr": arr(f.attr, o.ATTR_DTYPE, n), "tiles": arr(f.tiles, np.uint32, n), "scan": arr(f.scan, np.uint32, n),
                "keys": arr(f.keys, np.uint64, m), "vals": arr(f.vals, np.uint32, m),
                "keys_unsorted": arr(f.keys_unsorted, np.uint64, m), "vals_unsorted": arr(f.vals_unsorted, np.uint32, m),
                "ranges": arr(f.ranges, np.uint32, 2 * T).reshape(-1, 2),
                "rgba": arr(f.rgba, np.float32, f.width * f.height * 4).reshape(f.height, f.width, 4)}
    finally:
        lib.gsr_frame_free(C.byref(f))
