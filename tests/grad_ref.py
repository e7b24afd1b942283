"""Float64 torch restatement of the forward (SURVEY Appendix A3 preprocess.comp + A8 render.comp), the reference the GPU
backward (gsb_render_backward) is compared against.  Test infrastructure only.

List membership is the oracle's fp32 decision: every tile blends over the oracle's own sorted list (render_frame's `vals`
and `ranges`), while uv, conic, opacity, colour, alpha and T are differentiable float64.  The per-pixel tests of render.comp
(power > 0, alpha < 1/255, the T' < 1e-4 break) are evaluated in float64 on those lists; the pixels where fp32 and float64
may decide them differently are the ones oracle.render_frame_probed flags.
"""
from __future__ import annotations

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


def preprocess(v: torch.Tensor, u):
    """preprocess.comp for the rows of v (k x 60, float64): uv (k, 2), conic (k, 3) = (A, B, C) of
    power = -A/2 dx^2 - C/2 dy^2 - B dx dy, opacity (k,), colour (k, 3) and the unclamped red (k,)."""
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
    P, V = _mat(u.proj_mat), _mat(u.view_mat)
    ph = torch.cat([p, torch.ones_like(p[:, :1])], 1)
    hc = ph @ P.T
    pv = ph @ V.T
    vx, vy, vz = pv[:, 0], pv[:, 1], pv[:, 2]
    limx, limy = 1.3 * float(np.float32(u.tan_fovx)), 1.3 * float(np.float32(u.tan_fovy))
    tx = torch.clamp(vx / vz, -limx, limx) * vz
    ty = torch.clamp(vy / vz, -limy, limy) * vz
    fx, fy = W / (2.0 * u.tan_fovx), H / (2.0 * u.tan_fovy)
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
    d = p - torch.tensor(np.asarray(list(u.camera_position)[:3], np.float64))
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


def _blend_tile(uv, conic, op, col, fx, fy):
    """render.comp:61-98 for the pixels (fx, fy) (P,) over one tile's list (the rows of uv ... in list order).
    Returns rgb (P, 3), contributor mask (P, L) and raw alpha (P, L)."""
    dx = uv[None, :, 0] - fx[:, None]
    dy = uv[None, :, 1] - fy[:, None]
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
    return rgb, contrib, raw.detach()


def reference(vertices, u, frame, grad_image=None):
    """Float64 image (H, W, 3) of the frame whose oracle lists are `frame` (oracle.render_frame of the same vertices / u) and,
    if grad_image (H, W, >= 3) is given, dL/dvertices (n, 60) for L = sum(grad_image[..., :3] * image) plus `exclude` (n,):
    Gaussians whose gradient is ill-posed at float64 / fp32 resolution (unclamped red within 1e-4 of 0, or raw alpha within
    1e-4 of the 0.99 clamp on a pixel with a non-zero upstream gradient)."""
    v_all = np.asarray(vertices, np.float32).reshape(-1, 60)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    tiles_x = (W + 15) // 16
    ranges = frame["ranges"]
    vals = frame["vals"].astype(np.int64)
    used = np.unique(vals)
    local = np.full(n, -1, np.int64)
    local[used] = np.arange(used.size)
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=grad_image is not None)
    with torch.set_grad_enabled(grad_image is not None):
        uv, conic, op, col, red = preprocess(leaf, u)
    # per-tile blends against detached copies; their gradients are chained through preprocess once at the end
    parts = [t.detach().clone().requires_grad_(grad_image is not None) for t in (uv, conic, op, col)]
    image = np.zeros((H, W, 3), np.float64)
    near_clamp = np.zeros(used.size, bool)
    gimg = None if grad_image is None else torch.tensor(np.asarray(grad_image, np.float64)[..., :3])
    for t in range(ranges.shape[0]):
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        if e <= s:
            continue
        tx, ty = t % tiles_x, t // tiles_x
        xs = np.arange(tx * 16, min(W, tx * 16 + 16))
        ys = np.arange(ty * 16, min(H, ty * 16 + 16))
        gy, gx = np.meshgrid(ys, xs, indexing="ij")
        fx, fy = torch.tensor(gx.ravel(), dtype=torch.float64), torch.tensor(gy.ravel(), dtype=torch.float64)
        idx = torch.tensor(local[vals[s:e]])
        with torch.set_grad_enabled(gimg is not None):
            rgb, contrib, raw = _blend_tile(parts[0][idx], parts[1][idx], parts[2][idx], parts[3][idx], fx, fy)
        image[gy.ravel(), gx.ravel()] = rgb.detach().numpy()
        if gimg is not None:
            g = gimg[gy.ravel(), gx.ravel()]
            (rgb * g).sum().backward()
            live = (g != 0).any(1)[:, None]
            hit = (contrib & live & ((raw - 0.99).abs() < 1e-4)).any(0).numpy()
            near_clamp[local[vals[s:e]][hit]] = True
    if gimg is None:
        return {"image": image}
    torch.autograd.backward([uv, conic, op, col], [p.grad if p.grad is not None else torch.zeros_like(p) for p in parts])
    grad = np.zeros((n, 60), np.float64)
    grad[used] = leaf.grad.numpy()
    grad[:, 3] = 0.0
    exclude = np.zeros(n, bool)
    exclude[used] = near_clamp | (red.detach().abs().numpy() < 1e-4)
    return {"image": image, "grad": grad, "exclude": exclude}
