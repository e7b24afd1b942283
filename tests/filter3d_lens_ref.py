"""References of gsb_filter3d_variance_lens (DESIGN.md section 24), the 3D smoothing filter from cameras that each have their
own lens: the definition restated in float64 (numpy, with the lens maps of fisheye_ref and opencv_ref), and an fp32 numpy
model in the kernel's order of operations.  Test infrastructure only.

For Gaussian i and camera c (UBO u, lens model m; m None or of kind PINHOLE: the UBO's pinhole), with t = (x, y, z) the
view-space position: c sees i iff the frame's cull for the kind keeps i and its uv lies within the 15 % margins; the footprint
scale is s_ic = 1 / sigma_min(J), J = d uv / d t (vz / min(focal_x, focal_y) for a pinhole); s_i = min over the cameras that
see i, unseen rows take the largest seen s_i, and variance_i = 0.2 s_i^2.
"""
from __future__ import annotations

import math

import numpy as np

import fisheye_ref
import lens_ref
import opencv_ref

F = np.float32
PINHOLE, FISHEYE, OPENCV = 0, 1, 2


def kind(m):
    return PINHOLE if m is None else int(m.kind)


def _views(xyz, u, f):
    """clip_view (gsb_geom.cuh) in dtype f, op for op: (ndcx, ndcy, vx, vy, vz) of the points xyz (n, 3)."""
    p = np.ascontiguousarray(xyz, f).reshape(-1, 3)
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    pm, vm = np.array(u.proj_mat, F).astype(f), np.array(u.view_mat, F).astype(f)
    with np.errstate(all="ignore"):
        hx = ((pm[0] * px + pm[4] * py) + pm[8] * pz) + pm[12]
        hy = ((pm[1] * px + pm[5] * py) + pm[9] * pz) + pm[13]
        hw = ((pm[3] * px + pm[7] * py) + pm[11] * pz) + pm[15]
        p_w = f(1) / hw
        vx = ((vm[0] * px + vm[4] * py) + vm[8] * pz) + vm[12]
        vy = ((vm[1] * px + vm[5] * py) + vm[9] * pz) + vm[13]
        vz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14]
        return hx * p_w, hy * p_w, vx, vy, vz


def _in_box(uu, vv, u, f):
    W, H = f(u.width), f(u.height)
    return (uu >= f(-0.15) * W) & (uu <= f(1.15) * W) & (vv >= f(-0.15) * H) & (vv <= f(1.15) * H)


def pinhole_focal(u, f=F):
    """min(focal_x, focal_y) with jacobian()'s focal_x = (float)W / (2.0f tan_fovx), in dtype f."""
    return min(f(u.width) / (f(2) * f(u.tan_fovx)), f(u.height) / (f(2) * f(u.tan_fovy)))


def scale_from_gram(J, f):
    """1 / sigma_min of J (n, 2, 3) in dtype f in the kernel's order (lens_scale): lambda_min = det / lambda_max with
    det = |J0 x J1|^2."""
    J = np.asarray(J, f)
    j0, j1 = J[:, 0], J[:, 1]
    with np.errstate(all="ignore"):
        a = (j0[:, 0] * j0[:, 0] + j0[:, 1] * j0[:, 1]) + j0[:, 2] * j0[:, 2]
        c = (j1[:, 0] * j1[:, 0] + j1[:, 1] * j1[:, 1]) + j1[:, 2] * j1[:, 2]
        b = (j0[:, 0] * j1[:, 0] + j0[:, 1] * j1[:, 1]) + j0[:, 2] * j1[:, 2]
        x0 = j0[:, 1] * j1[:, 2] - j0[:, 2] * j1[:, 1]
        x1 = j0[:, 2] * j1[:, 0] - j0[:, 0] * j1[:, 2]
        x2 = j0[:, 0] * j1[:, 1] - j0[:, 1] * j1[:, 0]
        det = (x0 * x0 + x1 * x1) + x2 * x2
        dd = a - c
        lmax = ((a + c) + np.sqrt(dd * dd + (f(4) * b) * b)) * f(0.5)
        return f(1) / np.sqrt(det / lmax)


def lambda_min_textbook(J, f):
    """(a + c - sqrt((a - c)^2 + 4 b^2)) / 2 in dtype f: the form scale_from_gram avoids, for comparison."""
    J = np.asarray(J, f)
    j0, j1 = J[:, 0], J[:, 1]
    a = (j0[:, 0] * j0[:, 0] + j0[:, 1] * j0[:, 1]) + j0[:, 2] * j0[:, 2]
    c = (j1[:, 0] * j1[:, 0] + j1[:, 1] * j1[:, 1]) + j1[:, 2] * j1[:, 2]
    b = (j0[:, 0] * j1[:, 0] + j0[:, 1] * j1[:, 1]) + j0[:, 2] * j1[:, 2]
    dd = a - c
    return ((a + c) - np.sqrt(dd * dd + (f(4) * b) * b)) * f(0.5)


def camera_scale(xyz, u, m, f=F):
    """(s (n,), seen (n,)) of one camera in dtype f: float32 is the kernel's arithmetic op for op (but atan2, which neither
    numpy nor CUDA rounds correctly), float64 the definition.  Rows the camera does not see have s = inf."""
    ndcx, ndcy, vx, vy, vz = _views(xyz, u, f)
    t = np.stack([vx, vy, vz], 1)
    k = kind(m)
    with np.errstate(all="ignore"):
        if k == PINHOLE:
            uu = ((ndcx + f(1)) * f(u.width) - f(1)) * f(0.5)
            vv = ((ndcy + f(1)) * f(u.height) - f(1)) * f(0.5)
            ok = (vz > f(0.2)) & _in_box(uu, vv, u, f)
            s = vz / pinhole_focal(u, f)
        elif k == FISHEYE:
            cam = fisheye_ref.cam_tuple(m)
            lens = lens_ref.lens_values(m)
            x, y, z, r, d, theta, t2, b, scth, sg, c, e = lens_ref._geo(t, lens, f)
            ok = (d > f(0.2)) & (theta <= f(cam[5]))
            uu = f(cam[0]) * (sg * x) + f(cam[2])
            vv = f(cam[1]) * (sg * y) + f(cam[3])
            ok &= _in_box(uu, vv, u, f)
            s = scale_from_gram(fisheye_ref.jacobian(t, cam, f), f)
        else:
            cam = opencv_ref.cam_tuple(m)
            g = opencv_ref.geo(t, cam, f)
            bound = f(opencv_ref.tan2_bound(cam[5])) if f == F else math.tan(float(np.float32(cam[5]))) ** 2
            ok = (vz > f(0.2)) & (g["r2"] <= bound) & (g["det"] > f(0))
            uu = f(cam[0]) * g["xd"] + f(cam[2])
            vv = f(cam[1]) * g["yd"] + f(cam[3])
            ok &= _in_box(uu, vv, u, f)
            s = scale_from_gram(opencv_ref.jacobian(t, cam, f)[1], f)
        ok &= (s > 0) & np.isfinite(s)
    return np.where(ok, s, f(np.inf)).astype(f), ok


def _models(models, k):
    if models is None or not isinstance(models, (list, tuple)):
        return [models] * k
    assert len(models) == k
    return list(models)


def scales(xyz, cameras, models, f=F):
    """(s (n,), seen (n,)): the least scale over the cameras that see each row, in dtype f."""
    n = np.asarray(xyz).reshape(-1, 3).shape[0]
    s = np.full(n, np.inf, f)
    seen = np.zeros(n, bool)
    for u, m in zip(cameras, _models(models, len(cameras))):
        sc, ok = camera_scale(xyz, u, m, f)
        s = np.minimum(s, sc)
        seen |= ok
    return s, seen


def variance(xyz, cameras, models, f=F):
    """gsb_filter3d_variance_lens in dtype f: float32 is the kernel's words (bit for bit for pinhole and OpenCV cameras),
    float64 the definition."""
    s, seen = scales(xyz, cameras, models, f)
    if not seen.any():
        return np.zeros(s.shape[0], f)
    s = np.where(seen, s, s[seen].max())
    return (s * s) * f(0.2)


def borderline(xyz, cameras, models, px=0.05, rel=1e-4):
    """Rows within `px` pixels of a camera's 15 % margins or within `rel` (relative) of one of its culls, in float64: the rows
    where fp32 rounding (or atan2f) may flip "seen"."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    out = np.zeros(xyz.shape[0], bool)
    f = np.float64
    for u, m in zip(cameras, _models(models, len(cameras))):
        ndcx, ndcy, vx, vy, vz = _views(xyz, u, f)
        t = np.stack([vx, vy, vz], 1)
        k = kind(m)
        with np.errstate(all="ignore"):
            if k == PINHOLE:
                uu = ((ndcx + 1) * u.width - 1) * 0.5
                vv = ((ndcy + 1) * u.height - 1) * 0.5
                near = np.abs(vz - 0.2) < rel
            elif k == FISHEYE:
                cam = fisheye_ref.cam_tuple(m)
                x, y, z, r, d, theta, t2, b, scth, sg, c, e = lens_ref._geo(t, lens_ref.lens_values(m), f)
                uu, vv = cam[0] * (sg * x) + cam[2], cam[1] * (sg * y) + cam[3]
                near = (np.abs(d - 0.2) < rel) | (np.abs(theta - float(np.float32(cam[5]))) < rel)
            else:
                cam = opencv_ref.cam_tuple(m)
                g = opencv_ref.geo(t, cam, f)
                tan2 = opencv_ref.tan2_bound(cam[5])
                uu, vv = cam[0] * g["xd"] + cam[2], cam[1] * g["yd"] + cam[3]
                near = (np.abs(vz - 0.2) < rel) | (np.abs(g["r2"] - tan2) < rel * tan2) | (np.abs(g["det"]) < rel)
            for val, size in ((uu, u.width), (vv, u.height)):
                near |= (np.abs(val + 0.15 * size) < px) | (np.abs(val - 1.15 * size) < px)
        out |= near & np.isfinite(vz)
    return out


def ulps(a, b):
    """|a - b| in units in the last place of fp32, elementwise (a, b float32; -0 == +0)."""
    def ordered(v):
        i = np.asarray(v, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)

    return np.abs(ordered(a) - ordered(b))
