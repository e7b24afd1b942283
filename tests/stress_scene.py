"""The stress scene of the backward tests (tests/test_gpu_backward_regimes.py) and the float64 measure of which regimes of
the reverse walk it reaches (tests/test_stress_coverage.py pins them).  Test infrastructure only.

scenes.c1() keeps every per-tile list under 256 entries and every opacity under sigmoid(4) = 0.982, so a reference
comparison on it never walks past the first batch of k_blend_backward nor meets the 0.99 alpha clamp.  This scene is 40 k
synthetic Gaussians packed into a 3 x 3 x 3 box: lists of ~1 000 entries per tile at c1's camera, and deterministic edits
that add
  - a faint region (x > 0.5, a quarter of the opacity), whose pixels walk past list position 512 and break deep in it;
  - opaque Gaussians (opacity 1 and 1.6; raw vertices allow > 1), whose centres hit the clamp alpha = min(0.99, raw);
  - Gaussians with a negative red DC coefficient, whose red is clamped at 0 after SH;
  - large Gaussians just outside 1.3 tan_fov at moderate depth, whose footprint still reaches the image: the clamp of
    t.x / t.z and t.y / t.z in the projection Jacobian binds for them.
"""
from __future__ import annotations

import numpy as np
import torch

import gs_b200 as g
import grad_ref
import scenes

# name -> (pos, quat, fov, W, H) as scenes.CAMERAS: c1's camera, and a 333 x 217 frame (not a multiple of the 16 x 16 tile)
# close enough to the box that its partial right and bottom tiles hold lists as long as the others
CAMERA_POSES = {"c1": scenes.CAMERAS["c1"],
                "odd_size_near": ([0.4, 0.2, 3.4], scenes.quat_axis_angle([1, 0, 0], -8), 45.0, 333, 217)}
CAMERAS = tuple(CAMERA_POSES)
N = 40_000
OPAQUE_EVERY = 20    # of the Gaussians with z > 0.5: every 20th gets opacity 1.0, every 20th (offset 10) opacity 1.6
FAINT_X = 0.5        # the others with x > 0.5 get a quarter of their opacity: pixels there walk far down their lists
NEG_RED_EVERY = 50   # every 50th Gaussian: red DC -3, red < 0 at every camera
N_EDGE = 48          # the fov-clamped Gaussians, appended after the N synthetic ones


def _edge_gaussians():
    """N_EDGE large Gaussians at view depth 2.5-4 of c1's camera (which looks down -z from (0, 0, 5)), their centres 1.35-1.7
    x the half field of view off axis -- past the 1.3 tan_fov clamp -- on all four sides, with scales of 0.35-0.55 so
    their 3-sigma footprint reaches back into the image."""
    rng = np.random.default_rng(5)
    u = scenes.camera("c1")
    v = np.zeros((N_EDGE, 60), np.float32)
    depth = rng.uniform(2.5, 4.0, N_EDGE)
    off = rng.uniform(1.35, 1.7, N_EDGE)
    side = np.arange(N_EDGE) % 4
    across = rng.uniform(-0.6, 0.6, N_EDGE)
    tx, ty = float(u.tan_fovx), float(u.tan_fovy)
    x = np.where(side < 2, np.where(side == 0, 1, -1) * off * tx, across * tx) * depth
    y = np.where(side >= 2, np.where(side == 2, 1, -1) * off * ty, across * ty) * depth
    v[:, 0], v[:, 1], v[:, 2], v[:, 3] = x, y, 5.0 - depth, 1.0
    v[:, 4:7] = rng.uniform(0.35, 0.55, (N_EDGE, 3))
    v[:, 7] = rng.uniform(0.3, 0.8, N_EDGE)
    q = rng.standard_normal((N_EDGE, 4))
    v[:, 8:12] = q / np.linalg.norm(q, axis=1, keepdims=True)
    v[:, 12:15] = rng.uniform(-0.5, 1.5, (N_EDGE, 3))
    v[:, 15:60] = 0.05 * rng.standard_normal((N_EDGE, 45))
    return v


def edits(vtx):
    """Masks of the synthetic rows the edits of vertices() select: opaque (opacity 1.0 or 1.6, scale halved), faint (opacity
    x 0.25) and neg_red (red DC -3)."""
    i = np.arange(vtx.shape[0])
    front = vtx[:, 2] > 0.5  # the third of the box nearest c1's camera
    opaque = front & (i % OPAQUE_EVERY == 0)
    opaque_above_one = front & (i % OPAQUE_EVERY == OPAQUE_EVERY // 2)
    faint = (vtx[:, 0] > FAINT_X) & ~opaque & ~opaque_above_one
    return {"opaque": opaque, "opaque_above_one": opaque_above_one, "faint": faint, "neg_red": i % NEG_RED_EVERY == 7}


def vertices():
    """The stress scene: (N + N_EDGE) x 60 activated records."""
    rec = g.synth_records(42, N, g.synth_params(half_extent=(1.5, 1.5, 1.5)))
    vtx = g.activate_records(rec)
    m = edits(vtx)
    vtx[m["opaque"], 7] = 1.0
    vtx[m["opaque_above_one"], 7] = 1.6
    vtx[m["opaque"] | m["opaque_above_one"], 4:7] *= np.float32(0.5)
    vtx[m["faint"], 7] *= np.float32(0.25)
    vtx[m["neg_red"], 12] = -3.0
    return np.ascontiguousarray(np.concatenate([vtx, _edge_gaussians()]), np.float32)


def camera_vertices():
    """vertices() for the camera gradient, a sum over every Gaussian that therefore needs none whose gradient is ill-posed
    (as test_gpu_backward_camera.camera_scene does for c1): opacity capped at 0.95 (the 0.99 alpha clamp never binds) and the
    red DC coefficient moved for any Gaussian whose unclamped red lies within 1e-3 of 0 at one of CAMERAS."""
    vtx = vertices()
    vtx[:, 7] = np.minimum(vtx[:, 7], np.float32(0.95))
    for _ in range(20):
        moved = False
        for cam in CAMERAS:
            near = np.abs(red(vtx, camera(cam))) < 1e-3
            if near.any():
                vtx[near, 12] += np.float32(0.01 / grad_ref.SH_C0)  # red + 0.01 at every camera
                moved = True
        if not moved:
            return vtx
    raise AssertionError("camera_vertices did not settle")


def camera(name):
    pos, q, fov, w, h = CAMERA_POSES[name]
    return g.uniforms_from_camera(pos, q, fov, 0.1, 1000.0, w, h)


def red(vtx, u):
    """Unclamped red after SH (float64), per Gaussian."""
    with torch.no_grad():
        return grad_ref.preprocess(torch.from_numpy(np.asarray(vtx, np.float64)), u)[4].numpy()


def fov_clamped(vtx, u):
    """Gaussians whose view-space t.x / t.z or t.y / t.z lies outside +-1.3 tan_fov (the Jacobian's clamp binds)."""
    v = np.asarray(vtx, np.float64)
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    pv = np.concatenate([v[:, 0:3], np.ones((v.shape[0], 1))], 1) @ V.T
    limx, limy = 1.3 * float(np.float32(u.tan_fovx)), 1.3 * float(np.float32(u.tan_fovy))
    return (np.abs(pv[:, 0] / pv[:, 2]) > limx) | (np.abs(pv[:, 1] / pv[:, 2]) > limy)


def walk_coverage(vtx, u, frame, grad_image):
    """What the reverse walk meets on the oracle's lists `frame`, decided in float64 like grad_ref:
      max_last (tiles,)     the largest last-contributor list position + 1 over the tile's pixels: where the walk starts
      break_pos (H, W)      list position + 1 of the entry at which the pixel breaks (T' < 1e-4), 0 if it never does
      clamped (n,)          bool: contributor to some pixel with a non-zero upstream gradient at raw alpha > 0.99"""
    v_all, used, local = grad_ref.survivors(vtx, frame)
    with torch.no_grad():
        uv, conic, op, col, _ = grad_ref.preprocess(torch.tensor(v_all[used].astype(np.float64)), u)
    gimg = np.asarray(grad_image)[..., :3]
    max_last = np.zeros(frame["ranges"].shape[0], np.int64)
    break_pos = np.zeros((int(u.height), int(u.width)), np.int64)
    clamped = np.zeros(v_all.shape[0], bool)
    for tl in grad_ref.tiles(u, frame, local):
        with torch.no_grad():
            _, contrib, raw, valid = grad_ref.blend_tile(uv[tl.idx], conic[tl.idx], op[tl.idx], col[tl.idx], tl.fx, tl.fy)
        contrib, valid, raw = contrib.numpy(), valid.numpy(), raw.numpy()
        L = contrib.shape[1]
        pos1 = np.arange(1, L + 1)
        last = np.where(contrib, pos1[None, :], 0).max(1)
        max_last[tl.t] = last.max()
        broken = valid & ~contrib  # the break entry and the valid entries behind it
        first_broken = np.where(broken, pos1[None, :], L + 1).min(1)
        break_pos[tl.py, tl.px] = np.where(first_broken <= L, first_broken, 0)
        live = (gimg[tl.py, tl.px] != 0).any(1)
        hit = (contrib & (raw > 0.99) & live[:, None]).any(0)
        clamped[tl.ids[hit]] = True
    return {"max_last": max_last, "break_pos": break_pos, "clamped": clamped}
