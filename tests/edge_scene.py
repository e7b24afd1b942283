"""The edge scene of tests/test_gpu_edge_parity.py: the inputs a trained or training scene contains and that
gs_b200.synth_records never produces, built as activated 60-float records (tests/test_edge_coverage.py pins which regimes it
reaches).  Test infrastructure only; deterministic.

Groups (vertices() returns a mask per group, after a seeded permutation of the rows):
  plane    a jittered 48 x 32 grid of flat discs at one fp32 z = 0, 4-10 deep per pixel at the axis camera, in six saturated
           DC colours (no two grid neighbours alike), opacity 0.3-0.9.  The axis camera's view matrix has exact zeros in
           its third row, so every plane row gets the same view depth: exact depth-key ties whose order decides the image.
  needle   300 Gaussians with scale ratios 1e2, 1e3 and 1e4 whose long axis projects to 20-600 px: at +-45 degrees to the
           pixel grid, at random orientations, and edge-on discs; opacity 0.01-0.05 (the cut ellipse lies far inside the
           AABB) or 0.5-1.6.  A fifth sit past the frame's edges, so their clipped AABBs are small enough for the level 1 cull.
  big      40 Gaussians of pixel radius 450-700 at 1280 x 720, the nearest of the scene but for the near group (so all of
           them fall into k_emit_coarse's first 1024-survivor chunk), opacity 0.02-0.035.
  near     at the near_plane camera: view depth on the float below 0.2f, on 0.2f and on the float above (found by scanning
           fp32 neighbours of z), and needles at view depth 0.2-0.3 far off axis whose projected centre lies beyond 2^31
           pixels while their footprint still covers the frame.  For these k_project's mid * mid overflows, so the pixel
           radius is +inf and the tile-AABB conversion saturates on +-inf (a finite argument >= 2^31 with a footprint that
           still reaches the frame would need a radius past fp32's range).  At the axis camera,
           the two view depths of its 2^-21 grid (5 - z is exact there) that bracket 0.2f.
  opacity  opacity 0, the float below 1/255, 1/255, the float above, densify_and_prune's min_opacity 0.005, and 0.99 with
           both neighbours, each centred exactly on a pixel of the axis camera (found by scanning fp32 neighbours of x and
           y), where alpha equals min(0.99, opacity): the alpha < 1/255 test and the clamp are met at equality.
  ident    40 identical rows.
  dup      200 verbatim copies of plane, needle and big rows (DUP_SOURCES); `pairs` lists (original, copy) row indices.
The permutation scatters originals and copies over the index range, so many pairs straddle the shard_slice boundaries.
"""
from __future__ import annotations

import functools

import numpy as np

import gs_b200 as g
import grad_ref
import scenes

# name -> (pos, quat, fov, W, H).  axis: c1's pose at 1280 x 720.  rotated_odd: a rotated pose at 333 x 217, where depth ties
# come only from duplicates.  near_plane: a camera 0.25 in front of the plane, where view depth is 0.25 - z rounded once, so
# every float near 0.2f is reachable (at the axis camera 5 - z is exact, a multiple of 2^-21).
CAMERA_POSES = {"axis": ([0, 0, 5], [1, 0, 0, 0], 45.0, 1280, 720),
                "rotated_odd": ([0.7, -0.5, 5.6], scenes.quat_axis_angle([0.8, 0.5, 0.3], 11), 50.0, 333, 217),
                "near_plane": ([0, 0, 0.25], [1, 0, 0, 0], 45.0, 160, 120)}
CAMERAS = tuple(CAMERA_POSES)
BACKWARD_CAMERAS = ("axis", "rotated_odd")
GRID = (48, 32)
N_NEEDLE = 300
N_BIG = 40
N_IDENT = 40
DUP_SOURCES = {"plane": 150, "needle": 40, "big": 10}
OPACITY_EDGES = [0.0, float(np.nextafter(np.float32(1 / 255), np.float32(0))), float(np.float32(1 / 255)),
                 float(np.nextafter(np.float32(1 / 255), np.float32(1))), 0.005,
                 float(np.nextafter(np.float32(0.99), np.float32(0))), float(np.float32(0.99)),
                 float(np.nextafter(np.float32(0.99), np.float32(1)))]
AXIS_FOCAL = 1280 / (2 * np.tan(np.radians(22.5)))  # pixels per unit at view depth 1, axis camera
COLOURS = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 1]], np.float64)


def camera(name):
    pos, q, fov, w, h = CAMERA_POSES[name]
    return g.uniforms_from_camera(pos, q, fov, 0.1, 1000.0, w, h)


def _rows(n):
    v = np.zeros((n, 60), np.float32)
    v[:, 3] = 1.0
    v[:, 8] = 1.0  # identity rotation
    return v


def _dc(rgb):
    """SH DC coefficients whose colour (DC * C0 + 0.5) is rgb."""
    return (np.asarray(rgb, np.float64) - 0.5) / grad_ref.SH_C0


def _qz(theta):
    return np.stack([np.cos(theta / 2), 0 * theta, 0 * theta, np.sin(theta / 2)], -1)


def _plane(rng):
    nx, ny = GRID
    gx, gy = np.meshgrid(np.linspace(-2.0, 2.0, nx), np.linspace(-1.15, 1.15, ny))
    i, j = np.meshgrid(np.arange(nx), np.arange(ny))
    v = _rows(nx * ny)
    v[:, 0] = gx.ravel() + rng.uniform(-0.02, 0.02, nx * ny)
    v[:, 1] = gy.ravel() + rng.uniform(-0.02, 0.02, nx * ny)
    v[:, 2] = 0.0
    v[:, 4] = rng.uniform(0.04, 0.06, nx * ny)
    v[:, 5] = rng.uniform(0.04, 0.06, nx * ny)
    v[:, 6] = 0.004
    v[:, 7] = rng.uniform(0.3, 0.9, nx * ny)
    v[:, 8:12] = _qz(rng.uniform(0, np.pi, nx * ny))
    v[:, 12:15] = _dc(COLOURS[((i + 2 * j) % 6).ravel()])
    v[:, 15:60] = 0.03 * rng.standard_normal((nx * ny, 45))
    return v


def _needles(rng):
    n = N_NEEDLE
    v = _rows(n)
    vz = rng.uniform(1.5, 4.5, n)
    ratio = np.array([1e2, 1e3, 1e4])[np.arange(n) % 3]
    sigma_px = np.exp(rng.uniform(np.log(20 / 3), np.log(600 / 3), n))  # 3 sigma of the long axis: 20-600 px
    kind = (np.arange(n) // 3) % 6  # 0, 1: +45 degrees, 2, 3: -45 degrees, 4: random orientation, 5: edge-on disc
    theta = np.where(kind < 2, np.pi / 4, -np.pi / 4)
    # centre in pixels from the frame centre.  Two fifths lie outside a corner of the frame and point into it along the
    # diagonal: their AABB, clipped to the frame, is at most ~11 x 11 tiles, so k_emit's level 1 row spans (not the
    # whole-block expansion of AABBs over EMIT_BIG tiles) handle these A C / det ~ 1e4 conics.
    cx, cy = rng.uniform(-640, 640, n), rng.uniform(-360, 360, n)
    corner = np.arange(n) % 5 >= 3
    sigma_px = np.where(corner, rng.uniform(110, 135, n), sigma_px)
    ratio = np.where(corner & (ratio < 1e3), 1e4, ratio)
    kind = np.where(corner, kind % 4, kind)
    # the corner (sx 640, sy 360): the long axis, +45 degrees in the world = (1, -1) on the screen (y down), must point from
    # the centre to the frame, and the centre sits d px past the corner on both axes, d a little under the needle's reach
    sx = rng.choice([-1.0, 1.0], n)
    sy = np.where(kind < 2, -sx, sx)
    d = 0.7 * 3 * sigma_px - rng.uniform(20, 80, n)
    cx = np.where(corner, sx * (640 + d), cx)
    cy = np.where(corner, sy * (360 + d), cy)
    v[:, 0], v[:, 1], v[:, 2] = cx * vz / AXIS_FOCAL, -cy * vz / AXIS_FOCAL, 5.0 - vz
    long_ = sigma_px * vz / AXIS_FOCAL
    q = _qz(theta)
    rq = rng.standard_normal((n, 4))
    q = np.where((kind == 4)[:, None], rq / np.linalg.norm(rq, axis=1, keepdims=True), q)
    # edge-on disc: scales (L, L, L / ratio) turned 90 degrees about the in-plane axis (cos phi, sin phi, 0), phi = +-45
    phi = np.where(np.arange(n) % 2 == 0, np.pi / 4, -np.pi / 4)
    disc_q = np.stack([np.full(n, np.cos(np.pi / 4)), np.cos(phi) * np.sin(np.pi / 4), np.sin(phi) * np.sin(np.pi / 4),
                       np.zeros(n)], -1)
    disc = kind == 5
    q = np.where(disc[:, None], disc_q, q)
    v[:, 8:12] = q
    v[:, 4] = long_
    v[:, 5] = np.where(disc, long_, long_ / ratio)
    v[:, 6] = long_ / ratio
    faint = np.arange(n) % 2 == 0
    v[:, 7] = np.where(faint, rng.uniform(0.01, 0.05, n), rng.uniform(0.5, 1.6, n))
    v[:, 12:15] = rng.uniform(-1.5, 1.5, (n, 3))
    v[:, 15:60] = 0.05 * rng.standard_normal((n, 45))
    return v


def _big(rng):
    n = N_BIG
    v = _rows(n)
    vz = rng.uniform(0.6, 1.0, n)
    cx, cy = rng.uniform(-150, 150, n), rng.uniform(-80, 80, n)
    v[:, 0], v[:, 1], v[:, 2] = cx * vz / AXIS_FOCAL, -cy * vz / AXIS_FOCAL, 5.0 - vz
    sigma_px = rng.uniform(450, 700, n) / 3
    s = sigma_px * vz / AXIS_FOCAL
    v[:, 4], v[:, 5], v[:, 6] = s, s * rng.uniform(0.8, 1.0, n), s * rng.uniform(0.8, 1.0, n)
    v[:, 7] = rng.uniform(0.02, 0.035, n)
    v[:, 8:12] = _qz(rng.uniform(0, np.pi, n))
    v[:, 12:15] = rng.uniform(-1.0, 1.0, (n, 3))
    v[:, 15:60] = 0.05 * rng.standard_normal((n, 45))
    return v


def _vz(u, p):
    """The view depth of clip_view / the oracle, in their fp32 operation order."""
    vm = np.asarray(list(u.view_mat), np.float32)
    p = np.asarray(p, np.float32)
    return ((vm[2] * p[0] + vm[6] * p[1]) + vm[10] * p[2]) + vm[14]


def _z_for_depth(u, x, y, target):
    """The fp32 z nearest the camera-side whose view depth at u is exactly `target` (scanning fp32 neighbours), or None."""
    z = np.float32(u.camera_position[2] - target)
    for _ in range(64):
        d = _vz(u, (x, y, z))
        if d == target:
            return z
        z = np.nextafter(z, np.float32(np.inf) if d > target else np.float32(-np.inf))
    return None


def near_depths():
    """(name, x, y, z, view depth) of the near rows on the view axis: the float below 0.2f, 0.2f and the float above at the
    near_plane camera, and the two grid neighbours of 0.2f at the axis camera."""
    out = []
    u = camera("near_plane")
    t = np.float32(0.2)
    for name, d in (("below", np.nextafter(t, np.float32(0))), ("at", t), ("above", np.nextafter(t, np.float32(1)))):
        z = _z_for_depth(u, 0.0, 0.0, d)
        assert z is not None, name
        out.append(("near_plane/" + name, 0.0, 0.0, z, d))
    ua = camera("axis")
    step = np.float32(2.0 ** -21)
    lo = np.float32(np.floor(np.float64(t) / 2.0 ** -21) * 2.0 ** -21)
    for name, d in (("axis/below", lo), ("axis/above", np.float32(lo + step))):
        z = np.float32(5.0 - np.float64(d))
        assert _vz(ua, (0.0, 0.0, z)) == d
        out.append((name, 0.0, 0.0, z, d))
    return out


def _near(rng):
    rows = near_depths()
    v = _rows(len(rows) + 6)
    for k, (_, x, y, z, _) in enumerate(rows):
        v[k, 0:3] = (x, y, z)
        v[k, 4:7] = 0.01
        v[k, 7] = 0.6
        v[k, 12:15] = _dc([0.2, 0.9, 0.4])
    # far off axis at the near_plane camera (view depth 0.2-0.3): needles along x (or y) from a centre tens of billions of
    # pixels away, long enough that the footprint covers the frame.  mid * mid overflows in k_project: the radius is +inf and
    # the float -> int conversion of the tile AABB saturates on +-inf
    k0 = len(rows)
    vz = np.float32(0.25) - np.float32([0.03, 0.0, -0.04, 0.02, -0.02, 0.01])
    dist = np.array([5e7, -6e7, 8e7, 5e7, -7e7, 6e7])
    along_y = np.array([False, False, False, True, True, True])
    for k in range(6):
        r = k0 + k
        z = np.float32(0.25) - vz[k]
        v[r, 0:3] = (0.0, dist[k], z) if along_y[k] else (dist[k], 0.0, z)
        v[r, 4:7] = (0.5 * abs(dist[k]), 50.0, 50.0)
        if along_y[k]:
            v[r, 8:12] = _qz(np.array(np.pi / 2))
        v[r, 7] = rng.uniform(0.3, 0.7)
        v[r, 12:15] = rng.uniform(-1.0, 1.0, 3)
    return v


def _scan_to_pixel_centre(u, row, axis, span=4096):
    """row with its coordinate `axis` (0: x, 1: y) moved to the fp32 neighbour nearest the given value at which the oracle's
    projected centre uv[axis] at u is an integer, i.e. exactly on a pixel (power is 0 there, so alpha = min(0.99, opacity))."""
    import oracle

    x0 = np.float32(row[axis])
    steps = np.arange(-span, span + 1)
    cand = (np.int64(x0.view(np.int32)) + steps).astype(np.int32).view(np.float32)
    rows = np.repeat(row[None, :], cand.size, 0)
    rows[:, axis] = cand
    uv = oracle.preprocess(rows, oracle.cov3d(rows), u)[0]["uv"][:, axis]
    hit = np.nonzero(uv == np.round(uv))[0]
    assert hit.size, "no fp32 neighbour puts the centre on a pixel"
    out = row.copy()
    out[axis] = cand[hit[np.argmin(np.abs(steps[hit]))]]
    return out


def _opacity_edges():
    """The opacity-edge rows at view depth 3 of the axis camera, 70 px apart, each centred exactly on a pixel: their alpha
    there is min(0.99, opacity) itself, so the blend's alpha < 1/255 test and the 0.99 clamp are met at equality."""
    n = len(OPACITY_EDGES)
    v = _rows(n)
    vz = 3.0
    # pixel (x, y) = (700 + 70 k, 520) is (x - 639.5, y - 359.5) px from the axis: start there, then scan.  (Right of and
    # below the centre, ndc + 1 lies in [1, 2), where its grid is fine enough to put uv on an integer.)
    px = 700.0 + 70.0 * np.arange(n)
    v[:, 0], v[:, 1], v[:, 2] = (px - 639.5) * vz / AXIS_FOCAL, -(520.0 - 359.5) * vz / AXIS_FOCAL, 5.0 - vz
    v[:, 4:7] = 12.0 * vz / AXIS_FOCAL
    v[:, 7] = OPACITY_EDGES
    v[:, 12:15] = _dc([0.9, 0.9, 0.1])
    u = camera("axis")
    for k in range(n):
        v[k] = _scan_to_pixel_centre(u, _scan_to_pixel_centre(u, v[k], 0), 1)
    return v


def _ident():
    v = _rows(N_IDENT)
    v[:, 0:3] = (0.35, -0.2, 2.5)
    v[:, 4:7] = (0.08, 0.05, 0.03)
    v[:, 7] = 0.15
    v[:, 8:12] = _qz(np.array(0.4))
    v[:, 12:15] = _dc([0.1, 0.3, 0.95])
    return v


def vertices(variant="full"):
    """(vertices (n, 60) float32, masks: group -> bool (n,), pairs: (k, 2) int64 of (original, copy) row indices).
    variant "backward": the scene without the needle and near groups (and their copies), whose gradients are ill-posed at
    fp32 resolution; "no_needles": without the needle group (and its copies)."""
    rng = np.random.default_rng(2024)
    parts = {"plane": _plane(rng), "needle": _needles(rng), "big": _big(rng), "near": _near(rng),
             "opacity": _opacity_edges(), "ident": _ident()}
    names = list(parts)
    group = np.concatenate([np.full(len(parts[k]), i) for i, k in enumerate(names)])
    base = np.concatenate([parts[k] for k in names])
    src = np.concatenate([rng.choice(np.nonzero(group == names.index(k))[0], c, replace=False)
                          for k, c in DUP_SOURCES.items()])
    vtx = np.concatenate([base, base[src]])
    group = np.concatenate([group, group[src]])
    is_dup = np.zeros(vtx.shape[0], bool)
    is_dup[base.shape[0]:] = True
    pairs = np.stack([src, base.shape[0] + np.arange(src.size)], 1)
    if variant == "backward":
        keep = (group != names.index("needle")) & (group != names.index("near"))
    elif variant == "no_needles":
        keep = group != names.index("needle")
    else:
        assert variant == "full", variant
        keep = np.ones(vtx.shape[0], bool)
    # drop the rows that are not kept, then permute: new index of old row r is inv[r]
    old = np.nonzero(keep)[0]
    perm = rng.permutation(old.size)  # new row k is old row old[perm[k]]
    new_of_old = np.full(vtx.shape[0], -1)
    new_of_old[old[perm]] = np.arange(old.size)
    vtx, group, is_dup = vtx[old[perm]], group[old[perm]], is_dup[old[perm]]
    pairs = new_of_old[pairs]
    pairs = pairs[(pairs >= 0).all(1)]
    masks = {k: (group == i) & ~is_dup for i, k in enumerate(names)}
    masks["dup"] = is_dup
    return np.ascontiguousarray(vtx, np.float32), masks, pairs


@functools.lru_cache(maxsize=None)
def backward_case(cam):
    """The backward variant at camera `cam`: its oracle frame (libm exp), a seeded upstream gradient that is zero on the
    step-probed pixels, and grad_ref's float64 reference.  `pairs`: the duplicate pairs of plane rows (opacity 0.3-0.9) whose
    rows both have a gradient norm of at least a tenth of the 99th percentile; `sets`: the row subsets the per-Gaussian
    check looks at separately.  Of the other pairs, the two copies' gradients differ by about the front copy's alpha (0.02 -
    0.035 for the big group) or lie under the absolute tolerance, so a swapped order is not visible there at all."""
    import oracle
    from backward_util import grad_image

    vtx, masks, pairs = vertices("backward")
    u = camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g_img = grad_image(u, steps)
    ref = grad_ref.reference(vtx, u, frame, g_img)
    keep = ~ref["exclude"]
    norm = np.linalg.norm(ref["grad"], axis=1)
    strong = keep & (norm >= 0.1 * np.percentile(norm[keep & (norm > 0)], 99))
    live = strong[pairs[:, 0]] & strong[pairs[:, 1]] & masks["plane"][pairs[:, 0]]
    in_pair = np.zeros(vtx.shape[0], bool)
    in_pair[pairs[live].ravel()] = True
    sets = {"dup_pairs": in_pair, "plane": keep & masks["plane"], "big": keep & masks["big"]}
    return {"vtx": vtx, "u": u, "frame": frame, "g": g_img, "ref": ref, "keep": keep, "sets": sets, "pairs": pairs[live]}
