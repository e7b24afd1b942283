"""The scale scene of tests/test_gpu_backward_scale.py: the range of scales a trained scene spans -- huge Gaussians the camera
sits inside, sub-pixel ones at the 0.3 dilation floor, needles, far and near rows -- built as activated 60-float records
(tests/test_scale_coverage.py pins which regimes it reaches, and that every survivor is well-posed at fp32 resolution, so the
float64 reference is a fair judge of the backward pass on all of them).  Test infrastructure only; deterministic.

Groups (vertices() returns a mask per group, after a seeded permutation of the rows), at edge_scene's axis (1280 x 720) and
rotated_odd (333 x 217) cameras:
  backdrop  synthetic Gaussians in a 5 x 3 x 2 box at view depth 4-6, so that every tile has a list and the other groups
            sit in front of, among and behind ordinary rows.
  huge      HUGE_PER_CAMERA per camera, at view depth 0.3-3 in front of it, anisotropic (axis ratios 0.5-1) along that camera's
            axes, so b^2 << a c at it and the determinant of cov2d does not cancel; opacity 0.02-0.08, so the rows behind
            still receive gradient.  The camera lies inside the 1-sigma ellipsoid of every one.  det ~ sigma^4 is set per row:
            log-spaced for sigma = 1e4-1e6 px (det 1e16-1e24, either side of det^2's fp32 overflow at 1.84e19) and, for
            HUGE_SUBNORMAL of them, inside (9.2e18, 1.84e19), where 1 / det^2 is subnormal.
  tiny      scales 1e-7-1e-4 at view depth 4-6, random rotations: cov2d is the 0.3 I floor to within 1e-6 where all three
            scales are under ~3e-6 (38 at the axis camera, 131 at the farther and wider rotated_odd); opacity 0.3-0.9.
  needle    at the axis camera, whose view matrix has exact zeros, on the pixel row or column through the centre (v.y or v.x
            is exactly 0) with an identity rotation, so the off-diagonal of cov2d is exactly 0: needles along x, y and z and
            edge-on discs with axis ratios 1e2, 1e3 and 1e4, 3-40 px long (1 sigma).  rotated_odd sees them 4-5 x shorter and a few
            degrees off its pixel axes, where their determinant does not cancel either.  Also needles at +-45 degrees on the screen, 1-1.6
            px long (1 sigma), short enough that det's relative error stays under 1e-6.
  far       view depth 100-900 (there is no far cull; J is small there), 1-12 px.
  near      on the view axis of each camera at the view depths just above 0.2f (the near cull is v.z <= 0.2f), anisotropic
            along that camera's axes:
            the first N_NEAR steps of the 2^-21 grid above 0.2f at the axis camera (5 - z is exact there, as in
            edge_scene.near_depths), and at rotated_odd the first N_NEAR fp32 view depths above it whose rounding error is
            under 2e-7 relative.
Every row but the backdrop has red >= 0.15 and opacity <= 0.9.
"""
from __future__ import annotations

import functools

import numpy as np
import torch
from scipy.spatial.transform import Rotation

import edge_scene
import gs_b200 as g
import grad_ref

CAMERAS = edge_scene.BACKWARD_CAMERAS  # ("axis", "rotated_odd")
N_BACKDROP = 2000
HUGE_PER_CAMERA = 15
HUGE_SUBNORMAL = 4   # of HUGE_PER_CAMERA, with det inside the band where 1 / det^2 is subnormal
N_TINY = 300
NEEDLE_RATIOS = (1e2, 1e3, 1e4)
N_NEEDLE_AXIS = 36   # per ratio: axis-aligned needles and edge-on discs at the axis camera
N_NEEDLE_45 = 30
N_FAR = 200
N_NEAR = 10          # per camera
DET_CLIFF = float(np.sqrt(np.float64(np.finfo(np.float32).max)))     # 1.84e19: det * det overflows fp32 above it
DET_SUBNORMAL = float(1.0 / np.sqrt(np.float64(np.finfo(np.float32).tiny)))  # 9.2e18: 1 / det^2 is subnormal above it


def camera(name):
    return edge_scene.camera(name)


def focal(u):
    return float(u.width) / (2.0 * float(np.float32(u.tan_fovx)))


def _view(u):
    """The 4 x 4 view matrix of u in float64 (row-major M[r, c])."""
    return np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T


def _world(u, vx, vy, vz):
    """World points whose view-space coordinates at u are (vx, vy, vz) (float64)."""
    V = _view(u)
    v = np.stack([vx, vy, vz, np.ones_like(np.asarray(vz, np.float64))], -1)
    return (v @ np.linalg.inv(V).T)[..., :3]


def _camera_quat(u):
    """The stored quaternion (w, x, y, z) whose rotation rows (grad_ref's R, Sigma = R^T diag(s^2) R) are u's view axes."""
    Rv = _view(u)[:3, :3]
    x, y, z, w = Rotation.from_matrix(Rv.T).as_quat()  # grad_ref's R(q) is the transpose of the usual rotation matrix of q
    return np.array([w, x, y, z])


def _rows(n):
    v = np.zeros((n, 60), np.float32)
    v[:, 3] = 1.0
    v[:, 8] = 1.0
    return v


def _colour(rng, n):
    """DC coefficients for colours in [0.15, 0.95] (red well away from its clamp at 0) and small higher bands."""
    v = np.zeros((n, 48), np.float32)
    v[:, 0:3] = edge_scene._dc(rng.uniform(0.15, 0.95, (n, 3)))
    v[:, 3:48] = 0.01 * rng.standard_normal((n, 45))
    return v


def _backdrop():
    # per-axis log-scale U[ln 0.01, ln 0.03]: anisotropy under 3, so no determinant cancels beyond fp32's 1e-6
    p = g.synth_params(center=(0.0, 0.0, 0.0), half_extent=(2.5, 1.5, 1.0), log_scale_min=float(np.log(0.01)),
                       log_scale_max=float(np.log(0.03)))
    return g.activate_records(g.synth_records(77, N_BACKDROP, p))


def _snap_depth(u, p):
    """p (k, 3) float32 moved along its largest coordinate of the view axis to the fp32 neighbour (within 256 steps) where
    the fp32 view depth (clip_view's operation order) is nearest its float64 value.  Near a camera whose view depth is not
    an exact difference, v.z cancels, and its rounding error alone would move the conic by more than 1e-6."""
    V = _view(u)
    k = int(np.argmax(np.abs(V[2, :3])))
    out = np.array(p, np.float32)
    steps = np.arange(-256, 257)
    for r in range(out.shape[0]):
        cand = np.repeat(out[r:r + 1], steps.size, 0)
        cand[:, k] = (np.int64(out[r, k].view(np.int32)) + steps).astype(np.int32).view(np.float32)
        d32 = np.array([edge_scene._vz(u, c) for c in cand], np.float64)
        d64 = cand.astype(np.float64) @ V[2, :3] + V[2, 3]
        out[r] = cand[np.argmin(np.abs(d32 - d64) + 1e-12 * np.abs(steps))]
    return out


def _cov2d_det(vtx, u):
    """float64 det of cov2d (with the 0.3 dilation) at u, as grad_ref.preprocess: det = 1 / (A C - B^2) of its conic."""
    with torch.no_grad():
        conic = grad_ref.preprocess(torch.from_numpy(np.asarray(vtx, np.float64)), u)[1].numpy()
    return 1.0 / (conic[:, 0] * conic[:, 2] - conic[:, 1] ** 2)


def _huge(rng, cam):
    n = HUGE_PER_CAMERA
    u = camera(cam)
    f = focal(u)
    vz = np.exp(rng.uniform(np.log(0.3), np.log(3.0), n))
    cx, cy = rng.uniform(-0.3, 0.3, n) * float(u.width), rng.uniform(-0.3, 0.3, n) * float(u.height)  # px from the centre
    v = _rows(n)
    v[:, 0:3] = _snap_depth(u, _world(u, cx * vz / f, -cy * vz / f, vz))
    v[:, 8:12] = _camera_quat(u)
    ratio = rng.uniform(0.5, 1.0, (n, 3))
    ratio[:, 0] = 1.0
    target = np.exp(np.linspace(np.log(1e16), np.log(1e24), n - HUGE_SUBNORMAL))
    target = np.concatenate([target, np.exp(np.linspace(np.log(DET_SUBNORMAL * 1.1), np.log(DET_CLIFF * 0.9), HUGE_SUBNORMAL))])
    s = 1e4 * vz / f  # sigma 1e4 px, then scaled to the target det (det ~ s^4 once the dilation is negligible)
    v[:, 4:7] = s[:, None] * ratio
    for _ in range(3):
        det = _cov2d_det(v, u)
        v[:, 4:7] *= ((target / det) ** 0.25)[:, None].astype(np.float32)
    v[:, 7] = rng.uniform(0.02, 0.08, n)
    v[:, 12:60] = _colour(rng, n)
    return v


def _tiny(rng):
    n = N_TINY
    u = camera("axis")
    f = focal(u)
    vz = rng.uniform(4.0, 6.0, n)
    cx, cy = rng.uniform(-600, 600, n), rng.uniform(-330, 330, n)
    v = _rows(n)
    v[:, 0:3] = _world(u, cx * vz / f, -cy * vz / f, vz)
    v[:, 4:7] = np.exp(rng.uniform(np.log(1e-7), np.log(1e-4), (n, 3)))
    q = rng.standard_normal((n, 4))
    v[:, 8:12] = q / np.linalg.norm(q, axis=1, keepdims=True)
    v[:, 7] = rng.uniform(0.3, 0.9, n)
    v[:, 12:60] = _colour(rng, n)
    return v


def _needles(rng):
    """Axis-aligned needles and edge-on discs on the centre row / column of the axis camera, and short 45-degree needles.
    Returns (rows, ratio per row, kind per row: 0 axis-aligned, 1 at 45 degrees)."""
    u = camera("axis")
    f = focal(u)
    parts, ratios, kinds = [], [], []
    for ratio in NEEDLE_RATIOS:
        n = N_NEEDLE_AXIS
        v = _rows(n)
        vz = rng.uniform(2.0, 4.0, n)
        sigma = np.exp(rng.uniform(np.log(3.0), np.log(40.0), n))  # px of the long axis
        long_ = sigma * vz / f
        short = long_ / ratio
        kind = np.arange(n) % 4  # long along x, along y, along z, edge-on disc (in the x-z plane)
        on_row = kind != 1       # on the centre row (v.y = 0) unless the needle runs along y
        c = np.where(on_row, rng.uniform(-600, 600, n), rng.uniform(-330, 330, n))
        vx = np.where(on_row, c * vz / f, 0.0)
        vy = np.where(on_row, 0.0, -c * vz / f)
        v[:, 0:3] = _world(u, vx, vy, vz)
        v[:, 4:7] = short[:, None]
        v[kind == 0, 4] = long_[kind == 0]
        v[kind == 1, 5] = long_[kind == 1]
        v[kind == 2, 6] = long_[kind == 2]
        disc = kind == 3
        v[disc, 4], v[disc, 6] = long_[disc], long_[disc]
        v[:, 7] = rng.uniform(0.2, 0.9, n)
        v[:, 12:60] = _colour(rng, n)
        parts.append(v)
        ratios.append(np.full(n, ratio))
        kinds.append(np.zeros(n, np.int64))
    n = N_NEEDLE_45
    v = _rows(n)
    vz = rng.uniform(2.0, 4.0, n)
    cx, cy = rng.uniform(-600, 600, n), rng.uniform(-330, 330, n)
    v[:, 0:3] = _world(u, cx * vz / f, -cy * vz / f, vz)
    long_ = rng.uniform(1.0, 1.6, n) * vz / f
    ratio = np.array(NEEDLE_RATIOS)[np.arange(n) % 3]
    v[:, 4], v[:, 5], v[:, 6] = long_, long_ / ratio, long_ / ratio
    v[:, 8:12] = edge_scene._qz(np.where(np.arange(n) % 2 == 0, np.pi / 4, -np.pi / 4))
    v[:, 7] = rng.uniform(0.2, 0.9, n)
    v[:, 12:60] = _colour(rng, n)
    parts.append(v)
    ratios.append(ratio)
    kinds.append(np.ones(n, np.int64))
    return np.concatenate(parts), np.concatenate(ratios), np.concatenate(kinds)


def _far(rng):
    n = N_FAR
    u = camera("axis")
    f = focal(u)
    vz = np.exp(rng.uniform(np.log(100.0), np.log(900.0), n))
    cx, cy = rng.uniform(-600, 600, n), rng.uniform(-330, 330, n)
    v = _rows(n)
    v[:, 0:3] = _world(u, cx * vz / f, -cy * vz / f, vz)
    sigma = rng.uniform(1.0, 12.0, (n, 1)) * rng.uniform(0.5, 1.0, (n, 3))
    v[:, 4:7] = sigma * (vz / f)[:, None]
    q = rng.standard_normal((n, 4))
    v[:, 8:12] = q / np.linalg.norm(q, axis=1, keepdims=True)
    v[:, 7] = rng.uniform(0.3, 0.9, n)
    v[:, 12:60] = _colour(rng, n)
    return v


def near_depths():
    """(camera, x, y, z, view depth) of the near rows: on each camera's view axis at the fp32 view depths just above 0.2f
    (at the axis camera 5 - z is exact, so the first N_NEAR steps of its 2^-21 grid above 0.2f; at rotated_odd the first
    N_NEAR distinct ones found by stepping the point's largest coordinate along the axis)."""
    t = np.float32(0.2)
    out = []
    ua = camera("axis")
    step = np.float32(2.0 ** -21)
    lo = np.float32(np.floor(np.float64(t) / 2.0 ** -21) * 2.0 ** -21)
    for k in range(1, N_NEAR + 1):
        d = np.float32(lo + np.float32(k) * step)
        z = np.float32(5.0 - np.float64(d))
        assert edge_scene._vz(ua, (0.0, 0.0, z)) == d
        out.append(("axis", 0.0, 0.0, z, d))
    u = camera("rotated_odd")
    V = _view(u)
    p0 = _world(u, 0.0, 0.0, 0.2).astype(np.float32)
    # walk the point along the view axis in fp32 steps of its largest coordinate's component, keeping the first N_NEAR view
    # depths above 0.2f whose fp32 value is within 2e-7 relative of their float64 value (v.z cancels here, see _snap_depth)
    axis = _world(u, 0.0, 0.0, 1.0) - _world(u, 0.0, 0.0, 0.0)
    k = int(np.argmax(np.abs(axis)))
    found = {}
    p = p0.copy()
    for _ in range(1 << 16):
        d = edge_scene._vz(u, p)
        d64 = float(p.astype(np.float64) @ V[2, :3] + V[2, 3])
        if d > t and d not in found and abs(d - d64) <= 2e-7 * d64:
            found[d] = p.copy()
            if len(found) == N_NEAR:
                break
        p[k] = np.nextafter(p[k], np.float32(np.sign(axis[k]) * np.inf))
    assert len(found) == N_NEAR
    for d in sorted(found):
        x, y, z = found[d]
        out.append(("rotated_odd", x, y, z, d))
    return out


def _near(rng):
    rows = near_depths()
    v = _rows(len(rows))
    for k, (cam, x, y, z, _) in enumerate(rows):
        v[k, 0:3] = (x, y, z)
        # anisotropic along the camera's axes: the cancelling v.x, v.y enter cov2d at second order only
        v[k, 4:7] = 0.01 * rng.uniform(0.6, 1.0, 3)
        v[k, 8:12] = _camera_quat(camera(cam))
    v[:, 7] = rng.uniform(0.1, 0.3, len(rows))  # N_NEAR of them overlap on each camera's axis
    v[:, 12:60] = _colour(rng, len(rows))
    return v


def vertices():
    """(vertices (n, 60) float32, masks: group -> bool (n,), needle_ratio (n,): the axis ratio of each needle row, 0
    elsewhere, needle45 (n,) bool: the 45-degree needles)."""
    rng = np.random.default_rng(31)
    needles, ratio, kind = _needles(rng)
    parts = {"backdrop": _backdrop(), "huge": np.concatenate([_huge(rng, c) for c in CAMERAS]), "tiny": _tiny(rng),
             "needle": needles, "far": _far(rng), "near": _near(rng)}
    names = list(parts)
    group = np.concatenate([np.full(len(parts[k]), i) for i, k in enumerate(names)])
    vtx = np.concatenate([parts[k] for k in names])
    nr = np.zeros(vtx.shape[0])
    n45 = np.zeros(vtx.shape[0], bool)
    sel = group == names.index("needle")
    nr[sel], n45[sel] = ratio, kind == 1
    perm = rng.permutation(vtx.shape[0])
    vtx, group, nr, n45 = vtx[perm], group[perm], nr[perm], n45[perm]
    masks = {k: group == i for i, k in enumerate(names)}
    return np.ascontiguousarray(vtx, np.float32), masks, nr, n45


def red(vtx, u):
    """Unclamped red after SH (float64), per Gaussian."""
    with torch.no_grad():
        return grad_ref.preprocess(torch.from_numpy(np.asarray(vtx, np.float64)), u)[4].numpy()


def camera_vertices(huge_at=None):
    """vertices() for the camera gradient, a sum over every Gaussian that therefore needs none whose gradient is ill-posed
    (as stress_scene.camera_vertices): opacity capped at 0.95 (the 0.99 alpha clamp never binds) and the red DC coefficient
    moved for any Gaussian whose unclamped red lies within 1e-3 of 0 at one of CAMERAS.
    huge_at (a camera name): only the huge rows whose float64 det at that camera exceeds DET_SUBNORMAL.  A Gaussian much
    larger than the frame moves the image by ~1 / sigma^2, so in the whole scene the share of the rows past the cliff is
    far below the camera check's 1e-3; here it is most of the sum."""
    vtx, masks, _, _ = vertices()
    if huge_at is not None:
        vtx = vtx[masks["huge"] & (_cov2d_det(vtx, camera(huge_at)) > DET_SUBNORMAL)]
    vtx[:, 7] = np.minimum(vtx[:, 7], np.float32(0.95))
    for _ in range(20):
        moved = False
        for cam in CAMERAS:
            near = np.abs(red(vtx, camera(cam))) < 1e-3
            if near.any():
                vtx[near, 12] += np.float32(0.01 / grad_ref.SH_C0)
                moved = True
        if not moved:
            return vtx
    raise AssertionError("camera_vertices did not settle")


# the huge rows' sets of the backward check, by det (the oracle's fp32 conic's 1 / (A C - B^2)) at the camera: below the
# band where 1 / det^2 is subnormal, in it, and past det^2's overflow one decade at a time.  Their gradients fall as
# ~1 / sigma^2 - 1 / sigma^3 (sigma ~ det^(1/4)), so each decade gets its own absolute tolerance.
HUGE_BANDS = {"huge_below": (0.0, DET_SUBNORMAL), "huge_subnormal": (DET_SUBNORMAL, DET_CLIFF), "huge_past_1e20": (DET_CLIFF, 1e20),
              **{f"huge_past_1e{e + 1}": (10.0 ** e, 10.0 ** (e + 1)) for e in range(20, 26)}, "huge_past_inf": (1e26, np.inf)}


def frame_det(frame):
    co = frame["attr"]["conic_opacity"].astype(np.float64)
    with np.errstate(divide="ignore"):
        return 1.0 / (co[:, 0] * co[:, 2] - co[:, 1] ** 2)


def groups_at(masks, frame):
    """The row sets of the backward check in the oracle's `frame`: each group's survivors (radius non-zero), with the huge
    group split into the HUGE_BANDS it reaches."""
    survivor = frame["attr"]["color_radii"][:, 3] != 0
    sets = {k: m & survivor for k, m in masks.items() if k != "huge"}
    det = frame_det(frame)
    for name, (lo, hi) in HUGE_BANDS.items():
        rows = masks["huge"] & survivor & (det > lo) & (det <= hi)
        if rows.any():
            sets[name] = rows
    return sets


@functools.lru_cache(maxsize=None)
def backward_case(cam, camera_grad=None):
    """The scene at camera `cam` (camera_grad "all": camera_vertices(), "huge": camera_vertices(huge_at=cam)): its oracle
    frame (libm exp), a seeded upstream gradient that is zero on the step-probed pixels, grad_ref's float64 reference (with
    grad_ubo for the camera variants), the rows it keeps and, for vertices(), the sets of groups_at over them."""
    import oracle
    from backward_util import grad_image

    vtx, masks, _, _ = vertices()
    if camera_grad is not None:
        vtx = camera_vertices(huge_at=cam if camera_grad == "huge" else None)
    u = camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g_img = grad_image(u, steps)
    ref = grad_ref.reference(vtx, u, frame, g_img, camera=camera_grad is not None)
    keep = ~ref["exclude"]
    sets = {} if camera_grad is not None else {k: keep & m for k, m in groups_at(masks, frame).items()}
    return {"vtx": vtx, "u": u, "frame": frame, "g": g_img, "ref": ref, "keep": keep, "sets": sets}
