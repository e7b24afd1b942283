"""The camera gradient of the float64 reference (tests/grad_ref.py), which gsb_render_backward_camera is compared against.
Test infrastructure only.

grad_ref.preprocess takes the camera from the UBO as constants; `preprocess` below is the same restatement of
preprocess.comp with the camera's float fields -- camera_position, proj_mat, view_mat, tan_fovx, tan_fovy -- as float64
tensors, so that autograd also returns their gradient.  Each field is an independent input, as in the ABI.  The blend is
grad_ref's own (_blend_tile over the oracle's lists); test_camera_grad.py pins `preprocess` and the vertex gradient of
`reference` to grad_ref's.
"""
from __future__ import annotations

import numpy as np
import torch

from grad_ref import SH_C0, SH_C1, SH_C2, SH_C3, _blend_tile


def camera_leaves(u):
    """The float fields of u as float64 leaf tensors that require grad, in ABI order: camera_position (4,), proj_mat and
    view_mat (16,) column-major, tan_fovx and tan_fovy (scalars)."""
    def leaf(x):
        return torch.tensor(np.asarray(x, np.float64)).requires_grad_()

    return {"camera_position": leaf(list(u.camera_position)), "proj_mat": leaf(list(u.proj_mat)),
            "view_mat": leaf(list(u.view_mat)), "tan_fovx": leaf(u.tan_fovx), "tan_fovy": leaf(u.tan_fovy)}


def preprocess(v: torch.Tensor, u, cam):
    """grad_ref.preprocess with the camera taken from cam (camera_leaves(u)); u gives width and height only."""
    W, H = float(u.width), float(u.height)
    p, s, op, q = v[:, 0:3], v[:, 4:7], v[:, 7], v[:, 8:12]
    sh = v[:, 12:60].reshape(-1, 16, 3)
    qw, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([
        torch.stack([1 - 2 * qy * qy - 2 * qz * qz, 2 * qx * qy + 2 * qz * qw, 2 * qx * qz - 2 * qy * qw], -1),
        torch.stack([2 * qx * qy - 2 * qz * qw, 1 - 2 * qx * qx - 2 * qz * qz, 2 * qy * qz + 2 * qx * qw], -1),
        torch.stack([2 * qx * qz + 2 * qy * qw, 2 * qy * qz - 2 * qx * qw, 1 - 2 * qx * qx - 2 * qy * qy], -1),
    ], -2)
    M = s[:, :, None] * R
    Sigma = M.transpose(1, 2) @ M
    P, V = cam["proj_mat"].reshape(4, 4).T, cam["view_mat"].reshape(4, 4).T  # M[r, c] from column-major
    tan_fovx, tan_fovy = cam["tan_fovx"], cam["tan_fovy"]
    ph = torch.cat([p, torch.ones_like(p[:, :1])], 1)
    hc = ph @ P.T
    pv = ph @ V.T
    vx, vy, vz = pv[:, 0], pv[:, 1], pv[:, 2]
    limx, limy = 1.3 * tan_fovx, 1.3 * tan_fovy
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
    d = p - cam["camera_position"][:3]
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


def reference(vertices, u, frame, grad_image):
    """grad_ref.reference's gradient of L = sum(grad_image[..., :3] * image) over the oracle lists `frame`, with the camera
    differentiable too: {"grad": dL/dvertices (n, 60), "exclude": as grad_ref's, "grad_ubo": dL/d(the 38 float fields of u
    in ABI order: camera_position[4], proj_mat[16], view_mat[16], tan_fovx, tan_fovy)}."""
    v_all = np.asarray(vertices, np.float32).reshape(-1, 60)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    tiles_x = (W + 15) // 16
    ranges = frame["ranges"]
    vals = frame["vals"].astype(np.int64)
    used = np.unique(vals)
    local = np.full(n, -1, np.int64)
    local[used] = np.arange(used.size)
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=True)
    cam = camera_leaves(u)
    uv, conic, op, col, red = preprocess(leaf, u, cam)
    # per-tile blends against detached copies; their gradients are chained through preprocess once at the end
    parts = [t.detach().clone().requires_grad_() for t in (uv, conic, op, col)]
    near_clamp = np.zeros(used.size, bool)
    gimg = torch.tensor(np.asarray(grad_image, np.float64)[..., :3])
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
        rgb, contrib, raw = _blend_tile(parts[0][idx], parts[1][idx], parts[2][idx], parts[3][idx], fx, fy)
        g = gimg[gy.ravel(), gx.ravel()]
        (rgb * g).sum().backward()
        live = (g != 0).any(1)[:, None]
        hit = (contrib & live & ((raw - 0.99).abs() < 1e-4)).any(0).numpy()
        near_clamp[local[vals[s:e]][hit]] = True
    torch.autograd.backward([uv, conic, op, col], [p.grad if p.grad is not None else torch.zeros_like(p) for p in parts])
    grad = np.zeros((n, 60), np.float64)
    grad[used] = leaf.grad.numpy()
    grad[:, 3] = 0.0
    exclude = np.zeros(n, bool)
    exclude[used] = near_clamp | (red.detach().abs().numpy() < 1e-4)
    grad_ubo = np.concatenate([np.zeros(t.numel()) if t.grad is None else np.atleast_1d(t.grad.numpy()) for t in cam.values()])
    return {"grad": grad, "exclude": exclude, "grad_ubo": grad_ubo}
