"""References of the anti-aliased mode (gsb_set_antialiased).  Test infrastructure only.

The mode keeps the dilated cov2d (preprocess.comp:63-65) for the conic, radius and tiles and scales each survivor's opacity
by comp = sqrt(max(0, det0 / det)), det0 = c00 c11 - c10 c01 over the undilated entries, det over the dilated ones, both in
the product order of preprocess.comp:138.  Both references here are layered on the existing ones, which stay as they are:

* `oracle_frame` runs the oracle stage by stage (gso_preprocess, then the scan, emission, sort, ranges and blend of
  gs_oracle.c) with the compensated opacity put into the attributes in between.  Only the opacity changes, so the survivor
  set, AABBs and keys are the plain frame's.  gso_preprocess does not return the undilated cov2d, so `cov2d_f32` restates
  that part of it in numpy fp32, op for op (numpy rounds each float32 operation once, like the oracle's -ffp-contract=off
  build).  Before using it, `oracle_frame` checks it against the oracle's own outputs on every survivor: the view depth
  and the three conic words bit for bit, which pin m01 and the dilated diagonal c + 0.3 exactly.  The low bits of c00 and
  c11 that the + 0.3 absorbs, and c10, enter only comp; those are pinned by tests/test_gpu_antialias.py, where the CUDA
  projection (csrc/gsb_geom.cuh, written separately) stores the same compensated opacity as this restatement, bit for bit,
  on every survivor of the c1, edge and scale scenes.
* `preprocess`, `reference` and `density_reference` are grad_ref's float64 functions with the opacity multiplied by comp.
  With K the dilated conic, det0 / det = det(I - 0.3 K) = (1 - 0.3 K00)(1 - 0.3 K11) - 0.09 K01^2, so comp is a
  differentiable function of grad_ref's conic; torch.where gives comp = 0 a zero gradient.
"""
from __future__ import annotations

import ctypes as C
from unittest import mock

import numpy as np
import torch

import grad_ref
import oracle as o

_f32 = np.float32
_vp = C.c_void_p
# A handle of our own on liboracle.so (the same loaded library, so set_exp_mode and the step probe apply), with the stages
# gs_oracle.h declares that oracle.py does not bind.
_lib = C.CDLL(str(o.LIB_PATH))
_lib.gso_scan_inclusive.argtypes = [_vp, C.c_uint64, _vp]
_lib.gso_scan_inclusive.restype = C.c_uint64
_lib.gso_emit_keys.argtypes = [_vp, _vp, C.c_uint64, C.c_uint32, _vp, _vp]
_lib.gso_emit_keys.restype = None
_lib.gso_sort.argtypes = [_vp, _vp, C.c_uint64]
_lib.gso_sort.restype = None
_lib.gso_tile_ranges.argtypes = [_vp, C.c_uint64, C.c_uint32, _vp]
_lib.gso_tile_ranges.restype = None
_lib.gso_set_step_probe.argtypes = [_vp, C.c_float]
_lib.gso_set_step_probe.restype = None
_lib.gso_blend.argtypes = [_vp, _vp, _vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _vp, _vp]
_lib.gso_blend.restype = None


# ---------------------------------------------------------------------------------------------------------------------
# fp32: the oracle with the compensation
# ---------------------------------------------------------------------------------------------------------------------
def cov2d_f32(vertices, cov, u):
    """gso_preprocess's (c00, c01, c10, c11) before the dilation and its view-space z, in fp32 with its rounding: J from
    get_projection_jacobian_approx, T = W J (mat3_mul), cov2d = T^T Sigma T as two mat3_mul calls."""
    v = np.asarray(vertices, _f32).reshape(-1, 60)
    cv = np.asarray(cov, _f32).reshape(-1, 6)
    vm = np.asarray(list(u.view_mat), _f32)
    px, py, pz = v[:, 0], v[:, 1], v[:, 2]
    with np.errstate(all="ignore"):
        def row(r):  # mat4_mul_vec4 of the view matrix and the vertex's position (x, y, z, w), row r
            s = vm[0 * 4 + r] * px
            s = s + vm[1 * 4 + r] * py
            s = s + vm[2 * 4 + r] * pz
            return s + vm[3 * 4 + r] * v[:, 3]

        t0, t1, t2 = row(0), row(1), row(2)
        limx, limy = _f32(1.3) * _f32(u.tan_fovx), _f32(1.3) * _f32(u.tan_fovy)
        tx = np.fmin(limx, np.fmax(-limx, t0 / t2)) * t2
        ty = np.fmin(limy, np.fmax(-limy, t1 / t2)) * t2
        fx = _f32(u.width) / (_f32(2.0) * _f32(u.tan_fovx))
        fy = _f32(u.height) / (_f32(2.0) * _f32(u.tan_fovy))
        zero = np.zeros_like(t2)
        J = [fx / t2, zero, -(fx * tx) / (t2 * t2), zero, fy / t2, -(fy * ty) / (t2 * t2), zero, zero, zero]
        view3 = [vm[c * 4 + r] for c in range(3) for r in range(3)]
        Wm = [view3[r * 3 + c] for c in range(3) for r in range(3)]  # mat3_transpose

        def mul(a, b):  # mat3_mul: o[c*3 + r] = ((a[0*3+r] b[c*3+0] + a[1*3+r] b[c*3+1]) + a[2*3+r] b[c*3+2])
            out = []
            for c in range(3):
                for r in range(3):
                    s = a[0 * 3 + r] * b[c * 3 + 0]
                    s = s + a[1 * 3 + r] * b[c * 3 + 1]
                    out.append(s + a[2 * 3 + r] * b[c * 3 + 2])
            return out

        Tm = mul(Wm, J)
        Tt = [Tm[r * 3 + c] for c in range(3) for r in range(3)]
        Sigma = [cv[:, 0], cv[:, 1], cv[:, 2], cv[:, 1], cv[:, 3], cv[:, 4], cv[:, 2], cv[:, 4], cv[:, 5]]
        c2 = mul(mul(Tt, Sigma), Tm)
    return c2[0], c2[1], c2[3], c2[4], t2


def compensation_f32(c00, c01, c10, c11):
    """(comp, det0, det) in fp32, the product's order: det = m00 m11 - m10 m01 with m = c + 0.3 I, det0 likewise."""
    with np.errstate(all="ignore"):
        m00, m11 = c00 + _f32(0.3), c11 + _f32(0.3)
        det = m00 * m11 - c10 * c01
        det0 = c00 * c11 - c10 * c01
        comp = np.sqrt(np.fmax(_f32(0.0), det0 / det))  # fmax(0, NaN) = 0
    return comp.astype(_f32), det0, det


def oracle_frame(vertices, cov, u, rows=None, probe_delta=None, antialiased=True) -> dict:
    """The oracle's frame of the anti-aliased mode: what oracle.render_frame returns (attr, tiles, scan, keys, vals,
    ranges, consumed, rgba, n, m, tiles_x, tiles_y) plus `comp` (n,) fp32 (0 for culled rows).  probe_delta: also return
    `steps`, the mask of oracle.render_frame_probed.  antialiased=False: the same stages without the compensation, which
    is oracle.render_frame's frame."""
    v = np.ascontiguousarray(vertices, _f32).reshape(-1, 60)
    cv = np.ascontiguousarray(cov, _f32).reshape(-1, 6)
    ou = o.Uniforms.from_buffer_copy(bytes(u))
    n, W, H = v.shape[0], int(ou.width), int(ou.height)
    tiles_x, tiles_y = (W + 15) // 16, (H + 15) // 16
    T = tiles_x * tiles_y
    rb, re = (0, o.ALL_ROWS) if rows is None else rows
    attr, tiles = o.preprocess(v, cv, ou, (rb, re))
    surv = attr["color_radii"][:, 3] != 0
    c00, c01, c10, c11, depth = cov2d_f32(v, cv, ou)
    comp_all, _, det = compensation_f32(c00, c01, c10, c11)
    with np.errstate(all="ignore"):  # the restatement is only used if it reproduces the oracle's outputs exactly
        ood = _f32(1.0) / det
        conic = np.stack([(c11 + _f32(0.3)) * ood, -c01 * ood, (c00 + _f32(0.3)) * ood], 1)
    assert np.array_equal(conic[surv].view(np.uint32), attr["conic_opacity"][surv, :3].view(np.uint32)) and \
        np.array_equal(depth[surv].view(np.uint32), attr["depth"][surv].view(np.uint32)), \
        "cov2d_f32 no longer restates gso_preprocess"
    comp = np.where(surv, comp_all, _f32(0.0)).astype(_f32)
    if antialiased:
        attr["conic_opacity"][:, 3] = np.where(surv, attr["conic_opacity"][:, 3] * comp, attr["conic_opacity"][:, 3])
    scan = np.zeros(n, np.uint32)
    m = int(_lib.gso_scan_inclusive(tiles.ctypes.data, n, scan.ctypes.data)) if n else 0
    keys = np.zeros(max(m, 1), np.uint64)
    vals = np.zeros(max(m, 1), np.uint32)
    _lib.gso_emit_keys(attr.ctypes.data, scan.ctypes.data, n, tiles_x, keys.ctypes.data, vals.ctypes.data)
    keys, vals = keys[:m].copy(), vals[:m].copy()
    _lib.gso_sort(keys.ctypes.data, vals.ctypes.data, m)
    ranges = np.zeros((T, 2), np.uint32)
    _lib.gso_tile_ranges(keys.ctypes.data, m, T, ranges.ctypes.data)
    rgba = np.zeros((H, W, 4), np.float32)
    consumed = np.zeros(T, np.uint32)
    mask = np.zeros((H, W), np.uint8)
    if probe_delta is not None:
        _lib.gso_set_step_probe(mask.ctypes.data, probe_delta)
    try:
        _lib.gso_blend(attr.ctypes.data, vals.ctypes.data, ranges.ctypes.data, W, H, rb, min(re, tiles_y),
                        rgba.ctypes.data, consumed.ctypes.data)
    finally:
        if probe_delta is not None:
            _lib.gso_set_step_probe(None, 0.0)
    out = {"n": n, "m": m, "tiles_x": tiles_x, "tiles_y": tiles_y, "attr": attr, "tiles": tiles, "scan": scan,
           "keys": keys, "vals": vals, "ranges": ranges, "consumed": consumed, "rgba": rgba, "comp": comp}
    if probe_delta is not None:
        out["steps"] = mask.astype(bool)
    return out


def oracle_frame_probed(vertices, cov, u, rows=None, rel_delta=2e-3):
    """oracle_frame with the step-function probe of oracle.render_frame_probed: (frame, mask)."""
    f = oracle_frame(vertices, cov, u, rows, probe_delta=rel_delta)
    return f, f.pop("steps")


# ---------------------------------------------------------------------------------------------------------------------
# float64: grad_ref with the compensation
# ---------------------------------------------------------------------------------------------------------------------
_plain_preprocess = grad_ref.preprocess


def compensation(conic: torch.Tensor) -> torch.Tensor:
    """sqrt(det0 / det) from the dilated conic (k, 3) = (K00, K01, K11): det(I - 0.3 K); 0 with a zero gradient where
    that is <= 0 (a flat Gaussian seen edge-on)."""
    r = (1 - 0.3 * conic[:, 0]) * (1 - 0.3 * conic[:, 2]) - 0.09 * conic[:, 1] * conic[:, 1]
    pos = r > 0
    return torch.where(pos, torch.sqrt(torch.where(pos, r, torch.ones_like(r))), torch.zeros_like(r))


def preprocess(v: torch.Tensor, u, cam=None):
    """grad_ref.preprocess with the opacity multiplied by compensation(conic)."""
    uv, conic, op, col, red = _plain_preprocess(v, u, cam)
    return uv, conic, op * compensation(conic), col, red


def _antialiased():
    """grad_ref's frame functions call its module-level preprocess: for the duration of one call, the compensated one."""
    return mock.patch.object(grad_ref, "preprocess", preprocess)


def reference(vertices, u, frame, grad_image=None, camera=False):
    """grad_ref.reference of the anti-aliased mode; `frame` is oracle_frame's (its lists are the plain frame's)."""
    with _antialiased():
        return grad_ref.reference(vertices, u, frame, grad_image, camera)


def density_reference(vertices, u, frame, grad_image):
    """grad_ref.density_reference of the anti-aliased mode."""
    with _antialiased():
        return grad_ref.density_reference(vertices, u, frame, grad_image)
