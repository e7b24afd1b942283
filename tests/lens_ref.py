"""Float64 reference of the fisheye camera gradient (gsb_render_backward_fisheye): the closed-form lens derivatives the kernel
uses (fisheye_lens_grad), evaluated in numpy, and a float64 torch frame whose view matrix, camera position and lens
(fx, fy, cx, cy, k1..k4) are leaves.  The blend and its depth / alpha and feature columns are depth_ref's and features_ref's,
the projection fisheye_ref's.  Test infrastructure only.
"""
from __future__ import annotations

import numpy as np
import torch

import depth_ref
import features_ref
import fisheye_ref
import grad_ref

# gsb_uniforms word offsets (ABI order, 40 words with width and height at 36, 37)
U_CAMPOS, U_PROJ, U_VIEW, U_TANX, U_TANY = 0, 4, 20, 38, 39
# the words of a fisheye frame's camera gradient that can be non-zero: camera_position.xyz and view_mat rows 0-2
LIVE_UBO = np.array([j < 3 or (U_VIEW <= j < U_VIEW + 16 and (j & 3) != 3) for j in range(40)])


def lens_values(cam):
    """(fx, fy, cx, cy, k1..k4) of a CameraModel (or fisheye_ref.cam_tuple) as a float64 array."""
    fx, fy, cx, cy, k, _ = fisheye_ref.cam_tuple(cam)
    return np.array([fx, fy, cx, cy, *k], np.float64)


def _geo(t, lens, f):
    """fisheye_geo of the kernel in dtype f, op for op: (x, y, z, r, d, theta, t2, b, scth, s, c, e)."""
    t = np.asarray(t, f)
    x, y, z = t[:, 0], t[:, 1], t[:, 2]
    L = [f(v) for v in lens]
    k = L[4:]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.sqrt(x * x + y * y)
        d = np.sqrt((x * x + y * y) + z * z)
        theta = np.arctan2(r, z).astype(f)
        t2 = theta * theta
        b = np.where(r > 0, theta / r, f(1) / d)
        P1 = k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3]))
        Q1 = f(3) * k[0] + t2 * (f(5) * k[1] + t2 * (f(7) * k[2] + t2 * (f(9) * k[3])))
        terms = fisheye_ref.KERNEL_TERMS if f == np.float32 else len(fisheye_ref.S_COEF)
        S_ser = fisheye_ref._series_S(t2.astype(f), terms).astype(f)
        scth_dir = ((r * z) / (d * d)) / theta
        S = np.where(theta < fisheye_ref.SERIES_THETA, S_ser, (scth_dir - f(1)) / t2)
        scth = np.where(theta < fisheye_ref.SERIES_THETA, f(1) + t2 * S_ser, scth_dir)
        c = ((S + Q1 * scth) - P1) * ((b * b) * b)
        s = (f(1) + t2 * P1) * b
        e = (f(1) + t2 * Q1) / (d * d)
    return x, y, z, r, d, theta, t2, b, scth, s, c, e


def closed_form(t, cam, dtype=np.float64):
    """The kernel's closed-form lens derivatives at the view-space positions t (k, 3), in `dtype` op for op:
    duv (k, 2, 8) = d uv / d(fx, fy, cx, cy, k1..k4) and dJ (k, 2, 3, 8) = d J / d(the same) (zero for cx, cy)."""
    f = dtype
    lens = lens_values(cam)
    fx, fy = f(lens[0]), f(lens[1])
    x, y, z, r, d, theta, t2, b, scth, s, c, e = _geo(t, lens, f)
    n = x.shape[0]
    duv = np.zeros((n, 2, 8), f)
    dJ = np.zeros((n, 2, 3, 8), f)
    xyc = (x * y) * c
    duv[:, 0, 0], duv[:, 1, 1] = s * x, s * y
    duv[:, 0, 2], duv[:, 1, 3] = 1, 1
    dJ[:, 0, 0, 0], dJ[:, 0, 1, 0], dJ[:, 0, 2, 0] = s + (x * x) * c, xyc, -(x * e)
    dJ[:, 1, 0, 1], dJ[:, 1, 1, 1], dJ[:, 1, 2, 1] = xyc, s + (y * y) * c, -(y * e)
    b3 = (b * b) * b
    pw = np.ones_like(t2)  # t2^(j-1)
    for j in range(1, 5):
        ds = b * (pw * t2)
        dc = pw * ((f(2 * j + 1) * scth - f(1)) * b3)
        de = f(2 * j + 1) * (pw * t2) / (d * d)
        col = 3 + j
        duv[:, 0, col], duv[:, 1, col] = fx * (x * ds), fy * (y * ds)
        dJ[:, 0, 0, col], dJ[:, 0, 1, col], dJ[:, 0, 2, col] = fx * (ds + (x * x) * dc), fx * ((x * y) * dc), -fx * (x * de)
        dJ[:, 1, 0, col], dJ[:, 1, 1, col], dJ[:, 1, 2, col] = fy * ((x * y) * dc), fy * (ds + (y * y) * dc), -fy * (y * de)
        pw = pw * t2
    return duv, dJ


def _cam_of(L, max_theta=0.0):
    return (L[0], L[1], L[2], L[3], L[4:8], max_theta)


def autograd(t, cam):
    """(duv, dJ) of closed_form by autograd of fisheye_ref.project with the lens as a float64 leaf (float64)."""
    L0 = torch.tensor(lens_values(cam))
    duv, dJ = [], []
    for p in torch.tensor(np.asarray(t, np.float64)):
        duv.append(torch.func.jacrev(lambda L: fisheye_ref.project(p[None], _cam_of(L))[0])(L0))
        dJ.append(torch.func.jacrev(lambda L: torch.func.jacrev(lambda q: fisheye_ref.project(q[None], _cam_of(L))[0])(p))(L0))
    return torch.stack(duv).numpy(), torch.stack(dJ).numpy()


# ---------------------------------------------------------------------------------------------------------------------
# the float64 frame with camera and lens leaves
# ---------------------------------------------------------------------------------------------------------------------
def leaves(u, cam):
    """The float64 leaves of a fisheye frame's camera: grad_ref.camera_leaves(u) (view_mat and camera_position are read)
    and the lens (8,)."""
    cl = grad_ref.camera_leaves(u)
    cl["lens"] = torch.tensor(lens_values(cam)).requires_grad_()
    return cl


def pre(cl, max_theta, antialiased=False):
    """A depth_ref-style preprocess (v, u, _) -> (uv, conic, op, colour, red, f = |t|) through the leaves cl (leaves())."""
    def fn(v, u, _cam=None):
        _, _, op, col, red = grad_ref.preprocess(v, u, cl)  # opacity and colour; the view direction reads camera_position
        s, q = v[:, 4:7], v[:, 8:12]
        qw, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        R = torch.stack([
            torch.stack([1 - 2 * qy * qy - 2 * qz * qz, 2 * qx * qy + 2 * qz * qw, 2 * qx * qz - 2 * qy * qw], -1),
            torch.stack([2 * qx * qy - 2 * qz * qw, 1 - 2 * qx * qx - 2 * qz * qz, 2 * qy * qz + 2 * qx * qw], -1),
            torch.stack([2 * qx * qz + 2 * qy * qw, 2 * qy * qz - 2 * qx * qw, 1 - 2 * qx * qx - 2 * qy * qy], -1),
        ], -2)
        M = s[:, :, None] * R
        Sigma = M.transpose(1, 2) @ M
        V = cl["view_mat"].reshape(4, 4).T
        ph = torch.cat([v[:, 0:3], torch.ones_like(v[:, :1])], 1)
        t = (ph @ V.T)[:, :3]
        lens = _cam_of(cl["lens"], max_theta)
        with torch.enable_grad():
            tg = t if t.requires_grad else t.detach().requires_grad_()
            uv = fisheye_ref.project(tg, lens)
            # J = d uv / d t, differentiable in t and the lens (each uv row depends on its own t row only)
            J = torch.stack([torch.autograd.grad(uv[:, a].sum(), tg, create_graph=True)[0] for a in range(2)], 1)
        T = J @ V[:3, :3]
        cov = T @ Sigma @ T.transpose(1, 2)
        a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
        det = a * c - b * b
        conic = torch.stack([c / det, -b / det, a / det], -1)
        if antialiased:
            import aa_ref

            op = op * aa_ref.compensation(conic)
        return uv, conic, op, col, red, torch.linalg.norm(tg, dim=1)

    return fn


def reference(vertices, u, cam, frame, grad_image=None, grad_da=None, features=None, grad_fm=None, antialiased=False):
    """The float64 frame of `frame`'s lists ({"vals", "ranges"}) through the lens cam and, with an upstream gradient --
    grad_image (H, W, >= 3), grad_da (H, W, 2) or, with features (n, C), grad_fm (H, W, C) -- dL/dvertices (n, 60),
    grad_ubo (40,) in gsb_uniforms' word layout (zero outside LIVE_UBO), grad_lens (8,), `exclude` (n,) as in depth_ref and,
    with features, grad_features (n, C)."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    max_theta = fisheye_ref.cam_tuple(cam)[5]
    cl = leaves(u, cam)
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=True)
    fn = pre(cl, max_theta, antialiased)
    info = {}
    if features is None:
        vals = depth_ref.frame_values(leaf, u, frame, local, pre=fn, info=info)
        g = np.zeros((H, W, 5))
        if grad_image is not None:
            g[..., :3] = np.asarray(grad_image, np.float64)[..., :3]
        if grad_da is not None:
            g[..., 3:] = np.asarray(grad_da, np.float64)[..., :2]
    else:
        F = np.asarray(features, np.float64)
        feat = torch.tensor(F[used], requires_grad=True)
        vals = features_ref.frame_values(leaf, feat, u, frame, local, pre=fn, info=info)
        g = np.zeros((H, W, 3 + F.shape[1]))
        if grad_image is not None:
            g[..., :3] = np.asarray(grad_image, np.float64)[..., :3]
        if grad_fm is not None:
            g[..., 3:] = np.asarray(grad_fm, np.float64)
    (vals * torch.tensor(g)).sum().backward()
    near_clamp = np.zeros(used.size, bool)
    for tl, contrib, raw in info["tiles"]:
        live = torch.tensor((g[tl.py, tl.px] != 0).any(1))[:, None]
        hit = (contrib & live & ((raw - 0.99).abs() < 1e-4)).any(0).numpy()
        near_clamp[local[tl.ids][hit]] = True
    grad = np.zeros((n, 60))
    grad[used] = leaf.grad.numpy()
    grad[:, 3] = 0.0
    exclude = np.zeros(n, bool)
    exclude[used] = near_clamp | (info["red"].abs().numpy() < 1e-4)
    gu = np.zeros(40)
    gu[U_CAMPOS:U_CAMPOS + 4] = cl["camera_position"].grad.numpy()
    gu[U_VIEW:U_VIEW + 16] = cl["view_mat"].grad.numpy()
    gu[~LIVE_UBO] = 0.0
    out = {"values": vals.detach().numpy(), "grad": grad, "grad_ubo": gu, "grad_lens": cl["lens"].grad.numpy(), "exclude": exclude}
    if features is not None:
        gf = np.zeros((n, F.shape[1]))
        gf[used] = feat.grad.numpy()
        out["grad_features"] = gf
    return out


def cpu_frame(vertices, u, cam):
    """Per-tile lists ({"vals", "ranges"}) of the float64 restatement, without a GPU: each Gaussian k_project keeps enters
    every tile of its AABB (fisheye_ref.aabb), each list in the order of the depth key d, then the index."""
    v = np.asarray(vertices, np.float64).reshape(-1, 60)
    box = fisheye_ref.aabb(v, u, cam)
    with torch.no_grad():
        d = torch.linalg.norm(fisheye_ref.view_positions(torch.tensor(v), u), dim=1).numpy()
    tx, ty = (u.width + 15) // 16, (u.height + 15) // 16
    vals, ranges = [], np.zeros((tx * ty, 2), np.uint32)
    for t in range(tx * ty):
        x, y = t % tx, t // tx
        ids = np.nonzero((box[:, 0] <= x) & (x < box[:, 2]) & (box[:, 1] <= y) & (y < box[:, 3]))[0]
        ids = ids[np.lexsort((ids, d[ids]))]
        ranges[t] = (len(vals), len(vals) + ids.size)
        vals.extend(ids.tolist())
    return {"vals": np.asarray(vals, np.uint32), "ranges": ranges}


def translation_residual(grad, g_ubo, u):
    """Moving every Gaussian by delta equals t_view += V3 delta and camera_position -= delta:
    sum_i dL/dp_i = V3^T g(view translation) - g(camera_position).  Returns (residual (3,), scale)."""
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    lhs = grad[:, 0:3].sum(0)
    rhs = V[:3, :3].T @ g_ubo[U_VIEW + 12:U_VIEW + 15] - g_ubo[U_CAMPOS:U_CAMPOS + 3]
    scale = np.abs(grad[:, 0:3]).sum(0).max() + np.abs(rhs).max()
    return lhs - rhs, scale


def step_pixels(vertices, u, cam, frame, antialiased=False, rel=1e-3):
    """(H, W) bool: the pixels where the float64 restatement lies within `rel` (relative) of one of the blend's step
    functions for some entry of its list -- alpha = 1/255, the 0.99 clamp, T = 1e-4 for the break -- so that the fp32 frame
    may take the other side.  A summed camera gradient cannot leave out a row, so such pixels get no upstream gradient."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    W, H = int(u.width), int(u.height)
    leaf = torch.tensor(v_all[used].astype(np.float64))
    uv, conic, op, _, _, _ = pre(leaves(u, cam), fisheye_ref.cam_tuple(cam)[5], antialiased)(leaf, u)
    uv, conic, op = uv.detach(), conic.detach(), op.detach()
    mask = np.zeros((H, W), bool)
    for tl in grad_ref.tiles(u, frame, local):
        i = tl.idx
        dx, dy = uv[i, 0][None, :] - tl.fx[:, None], uv[i, 1][None, :] - tl.fy[:, None]
        A, B, C = conic[i][None, :, 0], conic[i][None, :, 1], conic[i][None, :, 2]
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        raw = op[i][None, :] * torch.exp(torch.clamp(power, max=0.0))
        alpha = torch.clamp(raw, max=0.99)
        valid = (power <= 0) & (alpha >= 1.0 / 255.0)
        t_after = torch.cumprod(1 - torch.where(valid, alpha, torch.zeros_like(alpha)), 1)
        near = (((raw * 255.0 - 1.0).abs() < rel) | ((raw / 0.99 - 1.0).abs() < rel)
                | (valid & ((t_after * 1e4 - 1.0).abs() < rel)))
        mask[tl.py, tl.px] = near.any(1).numpy()
    return mask
