"""Float64 torch restatement of the forward (SURVEY Appendix A3 preprocess.comp + A8 render.comp), the reference the GPU
backward (gsb_render_backward, _camera and _density) is compared against.  Test infrastructure only.

List membership is the oracle's fp32 decision: every tile blends over the oracle's own sorted list (render_frame's `vals`
and `ranges`), while uv, conic, opacity, colour, alpha and T are differentiable float64.  The per-pixel tests of render.comp
(power > 0, alpha < 1/255, the T' < 1e-4 break) are evaluated in float64 on those lists; the pixels where fp32 and float64
may decide them differently are the ones oracle.render_frame_probed flags.

The camera gradient takes the UBO's float fields -- camera_position, proj_mat, view_mat, tan_fovx, tan_fovy -- as float64
leaf tensors (camera_leaves), each an independent input as in the ABI.  The density statistics take the offsets
(dx, dy) = uv - pixel of every (pixel, entry) pair as leaves, so that each pixel's own dL_p/duv is available before the sum
over pixels.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def _mat(m16):
    """Column-major float[16] (std140 mat4) -> 4 x 4 float64 tensor M with M[r, c]."""
    return torch.tensor(np.asarray(list(m16), np.float64).reshape(4, 4).T.copy())


def camera_leaves(u):
    """The float fields of u as float64 leaf tensors that require grad, in ABI order: camera_position (4,), proj_mat and
    view_mat (16,) column-major, tan_fovx and tan_fovy (scalars)."""
    def leaf(x):
        return torch.tensor(np.asarray(x, np.float64)).requires_grad_()

    return {"camera_position": leaf(list(u.camera_position)), "proj_mat": leaf(list(u.proj_mat)),
            "view_mat": leaf(list(u.view_mat)), "tan_fovx": leaf(u.tan_fovx), "tan_fovy": leaf(u.tan_fovy)}


def preprocess(v: torch.Tensor, u, cam=None):
    """preprocess.comp for the rows of v (k x 60, float64): uv (k, 2), conic (k, 3) = (A, B, C) of
    power = -A/2 dx^2 - C/2 dy^2 - B dx dy, opacity (k,), colour (k, 3) and the unclamped red (k,).  The camera comes from
    cam (camera_leaves(u)) when given, from the UBO u otherwise; u always gives width and height."""
    W, H = float(u.width), float(u.height)
    p, s, op, q = v[:, 0:3], v[:, 4:7], v[:, 7], v[:, 8:12]
    sh = v[:, 12:60].reshape(-1, 16, 3)
    # precomp_cov3d.comp: Sigma = M^T M, M = diag(s) R, R from the quaternion as stored (w, x, y, z)
    qw, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    # R[:, r, c] = common.glsl's R[c][r]
    R = torch.stack([
        torch.stack([1 - 2 * qy * qy - 2 * qz * qz, 2 * qx * qy + 2 * qz * qw, 2 * qx * qz - 2 * qy * qw], -1),
        torch.stack([2 * qx * qy - 2 * qz * qw, 1 - 2 * qx * qx - 2 * qz * qz, 2 * qy * qz + 2 * qx * qw], -1),
        torch.stack([2 * qx * qz + 2 * qy * qw, 2 * qy * qz - 2 * qx * qw, 1 - 2 * qx * qx - 2 * qy * qy], -1),
    ], -2)
    M = s[:, :, None] * R
    Sigma = M.transpose(1, 2) @ M
    if cam is None:
        P, V = _mat(u.proj_mat), _mat(u.view_mat)
        tan_fovx, tan_fovy = float(u.tan_fovx), float(u.tan_fovy)
        cam_pos = torch.tensor(np.asarray(list(u.camera_position)[:3], np.float64))
    else:
        P, V = cam["proj_mat"].reshape(4, 4).T, cam["view_mat"].reshape(4, 4).T  # M[r, c] from column-major
        tan_fovx, tan_fovy = cam["tan_fovx"], cam["tan_fovy"]
        cam_pos = cam["camera_position"][:3]
    ph = torch.cat([p, torch.ones_like(p[:, :1])], 1)
    hc = ph @ P.T
    pv = ph @ V.T
    vx, vy, vz = pv[:, 0], pv[:, 1], pv[:, 2]
    limx, limy = (torch.as_tensor(1.3 * t, dtype=torch.float64) for t in (tan_fovx, tan_fovy))
    tx = torch.minimum(torch.maximum(vx / vz, -limx), limx) * vz
    ty = torch.minimum(torch.maximum(vy / vz, -limy), limy) * vz
    fx, fy = W / (2.0 * tan_fovx), H / (2.0 * tan_fovy)
    z = torch.zeros_like(vz)
    J = torch.stack([torch.stack([fx / vz, z, -(fx * tx) / (vz * vz)], -1),
                     torch.stack([z, fy / vz, -(fy * ty) / (vz * vz)], -1)], -2)
    T = J @ V[:3, :3]
    cov = T @ Sigma @ T.transpose(1, 2)
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a * c - b * b
    conic = torch.stack([c / det, -b / det, a / det], -1)
    ndc = hc[:, :2] / hc[:, 3:4]
    uv = torch.stack([((ndc[:, 0] + 1) * W - 1) * 0.5, ((ndc[:, 1] + 1) * H - 1) * 0.5], -1)
    # compute_sh (preprocess.comp:73-108)
    d = p - cam_pos
    d = d / torch.sqrt((d * d).sum(1, keepdim=True))
    x, y, zz = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, z2 = x * x, y * y, zz * zz
    basis = torch.stack([
        torch.full_like(x, SH_C0), -SH_C1 * y, SH_C1 * zz, -SH_C1 * x,
        SH_C2[0] * x * y, SH_C2[1] * y * zz, SH_C2[2] * (2 * z2 - xx - yy), SH_C2[3] * zz * x, SH_C2[4] * (xx - yy),
        SH_C3[0] * (3 * xx - yy) * y, SH_C3[1] * x * y * zz, SH_C3[2] * (4 * z2 - xx - yy) * y,
        SH_C3[3] * zz * (2 * z2 - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * z2 - xx - yy), SH_C3[5] * (xx - yy) * zz,
        SH_C3[6] * x * (xx - 3 * yy)], -1)
    col = (basis[:, :, None] * sh).sum(1) + 0.5
    red = col[:, 0]
    col = torch.stack([torch.where(red < 0, torch.zeros_like(red), red), col[:, 1], col[:, 2]], -1)
    return uv, conic, op, col, red


def blend_offsets(dx, dy, conic, op, col):
    """render.comp:61-98 over one tile's list (the rows of conic ... in list order) for the offsets (dx, dy) = uv - pixel
    (P, L).  Returns rgb (P, 3), the contributor mask (P, L), raw alpha (P, L) and the mask of the entries that pass
    render.comp's power and alpha tests (P, L), contributors and the entries from the break on."""
    A, B, C = conic[None, :, 0], conic[None, :, 1], conic[None, :, 2]
    power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
    raw = op[None, :] * torch.exp(torch.clamp(power, max=0.0))
    alpha = torch.clamp(raw, max=0.99)
    with torch.no_grad():
        valid = (power <= 0) & (alpha >= 1.0 / 255.0)
        a0 = torch.where(valid, alpha, torch.zeros_like(alpha))
        t_after = torch.cumprod(1 - a0, 1)
        after_break = torch.cumsum((valid & (t_after < 1e-4)).to(torch.int32), 1) > 0  # the break and everything after it
        contrib = valid & ~after_break
    a = torch.where(contrib, alpha, torch.zeros_like(alpha))
    t_before = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), 1 - a[:, :-1]], 1), 1)
    rgb = ((a * t_before)[:, :, None] * col[None, :, :]).sum(1)
    return rgb, contrib, raw.detach(), valid


def blend_tile(uv, conic, op, col, fx, fy):
    """blend_offsets for the pixels (fx, fy) (P,) and the list's uv (L, 2)."""
    return blend_offsets(uv[None, :, 0] - fx[:, None], uv[None, :, 1] - fy[:, None], conic, op, col)


class Tile(NamedTuple):
    t: int               # tile index
    py: np.ndarray       # the tile's pixels inside the frame, row-major: rows (P,) and columns (P,)
    px: np.ndarray
    fx: torch.Tensor     # their coordinates as float64 (P,)
    fy: torch.Tensor
    ids: np.ndarray      # the tile's list: Gaussian indices in list order (L,)
    idx: torch.Tensor    # the same as rows of the survivors' tensors (survivors(...)'s local numbering)


def survivors(vertices, frame):
    """The Gaussians in some list of `frame`: (all vertices as float32 (n, 60), their sorted indices `used`, local (n,) =
    the row of each in used, -1 for the others)."""
    v_all = np.asarray(vertices, np.float32).reshape(-1, 60)
    used = np.unique(frame["vals"].astype(np.int64))
    local = np.full(v_all.shape[0], -1, np.int64)
    local[used] = np.arange(used.size)
    return v_all, used, local


def tiles(u, frame, local):
    """The non-empty tiles of the oracle's lists `frame` (oracle.render_frame), in tile order."""
    W, H = int(u.width), int(u.height)
    tiles_x = (W + 15) // 16
    ranges = frame["ranges"]
    vals = frame["vals"].astype(np.int64)
    for t in range(ranges.shape[0]):
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        if e <= s:
            continue
        tx, ty = t % tiles_x, t // tiles_x
        xs = np.arange(tx * 16, min(W, tx * 16 + 16))
        ys = np.arange(ty * 16, min(H, ty * 16 + 16))
        gy, gx = np.meshgrid(ys, xs, indexing="ij")
        py, px = gy.ravel(), gx.ravel()
        ids = vals[s:e]
        yield Tile(t, py, px, torch.tensor(px, dtype=torch.float64), torch.tensor(py, dtype=torch.float64), ids,
                   torch.tensor(local[ids]))


def reference(vertices, u, frame, grad_image=None, camera=False, cut_conic=None):
    """Float64 image (H, W, 3) of the frame whose oracle lists are `frame` (oracle.render_frame of the same vertices / u) and,
    if grad_image (H, W, >= 3) is given, dL/dvertices (n, 60) for L = sum(grad_image[..., :3] * image) plus `exclude` (n,):
    Gaussians whose gradient is ill-posed at float64 / fp32 resolution (unclamped red within 1e-4 of 0, or raw alpha within
    1e-4 of the 0.99 clamp on a pixel with a non-zero upstream gradient).  camera=True also returns grad_ubo: dL/d(the 38
    float fields of u in ABI order: camera_position[4], proj_mat[16], view_mat[16], tan_fovx, tan_fovy).  cut_conic (n,)
    bool: the conics of these Gaussians are detached, so no gradient flows through them (what a backward pass that drops
    the conic path of those rows would compute)."""
    v_all, used, local = survivors(vertices, frame)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=grad_image is not None)
    cam = camera_leaves(u) if camera else None
    with torch.set_grad_enabled(grad_image is not None):
        uv, conic, op, col, red = preprocess(leaf, u, cam)
        if cut_conic is not None:
            cut = torch.from_numpy(np.asarray(cut_conic, bool)[used])[:, None]
            conic = torch.where(cut, conic.detach(), conic)
    # per-tile blends against detached copies; their gradients are chained through preprocess once at the end
    parts = [t.detach().clone().requires_grad_(grad_image is not None) for t in (uv, conic, op, col)]
    image = np.zeros((H, W, 3), np.float64)
    near_clamp = np.zeros(used.size, bool)
    gimg = None if grad_image is None else torch.tensor(np.asarray(grad_image, np.float64)[..., :3])
    for tl in tiles(u, frame, local):
        with torch.set_grad_enabled(gimg is not None):
            rgb, contrib, raw, _ = blend_tile(*(p[tl.idx] for p in parts), tl.fx, tl.fy)
        image[tl.py, tl.px] = rgb.detach().numpy()
        if gimg is not None:
            g = gimg[tl.py, tl.px]
            (rgb * g).sum().backward()
            live = (g != 0).any(1)[:, None]
            hit = (contrib & live & ((raw - 0.99).abs() < 1e-4)).any(0).numpy()
            near_clamp[local[tl.ids][hit]] = True
    if gimg is None:
        return {"image": image}
    torch.autograd.backward([uv, conic, op, col], [p.grad if p.grad is not None else torch.zeros_like(p) for p in parts])
    grad = np.zeros((n, 60), np.float64)
    grad[used] = leaf.grad.numpy()
    grad[:, 3] = 0.0
    exclude = np.zeros(n, bool)
    exclude[used] = near_clamp | (red.detach().abs().numpy() < 1e-4)
    out = {"image": image, "grad": grad, "exclude": exclude}
    if camera:
        out["grad_ubo"] = np.concatenate([np.zeros(t.numel()) if t.grad is None else np.atleast_1d(t.grad.numpy())
                                          for t in cam.values()])
    return out


def density_reference(vertices, u, frame, grad_image):
    """gsb_render_backward_density's statistics for L = sum(grad_image[..., :3] * image) over the oracle's lists `frame`:
      duv (n, 2)      dL/d uv summed over pixels (pixel units)
      abs_duv (n, 2)  sum over pixels of |dL_p/d uv|, per component
      density (n, 4)  what one gsb_render_backward_density call adds to a zeroed buffer: the two norms in NDC units
                      (d u / d ndc.x = W / 2), 1 per survivor, the radius
      survivor (n,)   bool, radii (n,) float32: the oracle's GSB_BUF_ATTR color_radii[3], non-zero exactly for the Gaussians
                      that survived the culls"""
    v_all, used, local = survivors(vertices, frame)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    with torch.no_grad():
        uv, conic, op, col, _ = preprocess(torch.tensor(v_all[used].astype(np.float64)), u)
    gimg = torch.tensor(np.asarray(grad_image, np.float64)[..., :3])
    duv = torch.zeros((used.size, 2), dtype=torch.float64)
    abs_duv = torch.zeros((used.size, 2), dtype=torch.float64)
    for tl in tiles(u, frame, local):
        dx = (uv[tl.idx, 0][None, :] - tl.fx[:, None]).requires_grad_()
        dy = (uv[tl.idx, 1][None, :] - tl.fy[:, None]).requires_grad_()
        with torch.enable_grad():
            rgb = blend_offsets(dx, dy, conic[tl.idx], op[tl.idx], col[tl.idx])[0]
            (rgb * gimg[tl.py, tl.px]).sum().backward()
        # d dx / d u = 1: dx.grad[p, l] is pixel p's own dL_p/du of entry l
        pix = torch.stack([dx.grad, dy.grad], -1)  # (P, L, 2)
        duv.index_add_(0, tl.idx, pix.sum(0))
        abs_duv.index_add_(0, tl.idx, pix.abs().sum(0))
    radii = frame["attr"]["color_radii"][:, 3].copy()
    survivor = radii != 0
    full_duv, full_abs = np.zeros((n, 2)), np.zeros((n, 2))
    full_duv[used], full_abs[used] = duv.numpy(), abs_duv.numpy()
    half = np.array([0.5 * W, 0.5 * H])
    density = np.zeros((n, 4))
    density[:, 0] = np.linalg.norm(full_duv * half, axis=1)
    density[:, 1] = np.linalg.norm(full_abs * half, axis=1)
    density[:, 2] = survivor
    density[:, 3] = radii
    return {"duv": full_duv, "abs_duv": full_abs, "density": density, "survivor": survivor, "radii": radii}
