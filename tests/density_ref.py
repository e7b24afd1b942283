"""Float64 reference of gsb_render_backward_density's statistics.  Test infrastructure only.

It reuses grad_ref.preprocess and restates grad_ref's tile blend with the offsets (dx, dy) = uv - pixel as float64 leaves of
shape (pixels, entries), so each pixel's own dL_p/du and dL_p/dv of every entry is available before the sum over pixels:
dL/du = sum_p dL_p/du gives column 0, sum_p |dL_p/du| column 1.  The survivor set and the radii come from the oracle's
GSB_BUF_ATTR layout (color_radii[3], non-zero exactly for the Gaussians that survived the culls).
"""
from __future__ import annotations

import numpy as np
import torch

import grad_ref


def blend_tile_offsets(dx, dy, conic, op, col):
    """grad_ref._blend_tile with (dx, dy) (P, L) given instead of uv and the pixel coordinates.  Returns rgb (P, 3)."""
    A, B, C = conic[None, :, 0], conic[None, :, 1], conic[None, :, 2]
    power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
    raw = op[None, :] * torch.exp(torch.clamp(power, max=0.0))
    alpha = torch.clamp(raw, max=0.99)
    with torch.no_grad():
        valid = (power <= 0) & (alpha >= 1.0 / 255.0)
        a0 = torch.where(valid, alpha, torch.zeros_like(alpha))
        t_after = torch.cumprod(1 - a0, 1)
        after_break = torch.cumsum((valid & (t_after < 1e-4)).to(torch.int32), 1) > 0
        contrib = valid & ~after_break
    a = torch.where(contrib, alpha, torch.zeros_like(alpha))
    t_before = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), 1 - a[:, :-1]], 1), 1)
    return ((a * t_before)[:, :, None] * col[None, :, :]).sum(1)


def reference(vertices, u, frame, grad_image):
    """For L = sum(grad_image[..., :3] * image) over the oracle's lists `frame` (oracle.render_frame of the same vertices / u):
      duv (n, 2)      dL/d uv summed over pixels (pixel units)
      abs_duv (n, 2)  sum over pixels of |dL_p/d uv|, per component
      density (n, 4)  what one gsb_render_backward_density call adds to a zeroed buffer: the two norms in NDC units
                      (d u / d ndc.x = W / 2), 1 per survivor, the radius
      survivor (n,)   bool, radii (n,) float32: the oracle's color_radii[3]"""
    v_all = np.asarray(vertices, np.float32).reshape(-1, 60)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    tiles_x = (W + 15) // 16
    ranges = frame["ranges"]
    vals = frame["vals"].astype(np.int64)
    used = np.unique(vals)
    local = np.full(n, -1, np.int64)
    local[used] = np.arange(used.size)
    with torch.no_grad():
        uv, conic, op, col, _ = grad_ref.preprocess(torch.tensor(v_all[used].astype(np.float64)), u)
    gimg = torch.tensor(np.asarray(grad_image, np.float64)[..., :3])
    duv = torch.zeros((used.size, 2), dtype=torch.float64)
    abs_duv = torch.zeros((used.size, 2), dtype=torch.float64)
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
        dx = (uv[idx, 0][None, :] - fx[:, None]).requires_grad_()
        dy = (uv[idx, 1][None, :] - fy[:, None]).requires_grad_()
        with torch.enable_grad():
            rgb = blend_tile_offsets(dx, dy, conic[idx], op[idx], col[idx])
            (rgb * gimg[gy.ravel(), gx.ravel()]).sum().backward()
        # d dx / d u = 1: dx.grad[p, l] is pixel p's own dL_p/du of entry l
        pix = torch.stack([dx.grad, dy.grad], -1)  # (P, L, 2)
        duv.index_add_(0, idx, pix.sum(0))
        abs_duv.index_add_(0, idx, pix.abs().sum(0))
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
