"""References of the rendered feature maps (gsb_render_features, gsb_render_backward_features).  Test infrastructure only.

For a pixel whose contributors are i = 1..k in list order, F_c = sum f_ic alpha_i T_i over 0, f an (n, C) table of
per-Gaussian features in the scene's row order.  Both references extend depth_ref's to C columns:

* `blend32` restates gso_blend in numpy fp32 over a frame's own lists (depth_ref.blend32's walk, exp mode 1), with the C
  feature columns accumulated like colour channels: (f * alpha) * T, one rounding per op, from +0.
* `reference` is grad_ref's float64 blend with the colour columns extended by the C features over 0; it is differentiable in
  the vertices, the camera leaves (grad_ref.camera_leaves) and the features.
"""
from __future__ import annotations

import numpy as np
import torch

import bg_ref
import depth_ref
import grad_ref

_f32 = np.float32


def blend32(frame, width, height, features):
    """(H, W, C) fp32 feature map of the oracle frame `frame` (exp mode 1) for features (n, C) indexed like the vertices.
    Pixels of empty tiles and pixels without contributors: 0."""
    W, H = int(width), int(height)
    feats = np.asarray(features, np.float32)
    C = feats.shape[1]
    tiles_x = (W + 15) // 16
    attr, vals, ranges = frame["attr"], frame["vals"].astype(np.int64), frame["ranges"]
    out = np.zeros((H, W, C), np.float32)
    one, cut_a, cut_t = _f32(1.0), _f32(1.0 / 255.0), _f32(0.0001)
    for t in range(ranges.shape[0]):
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        if e <= s:
            continue
        tx, ty = t % tiles_x, t // tiles_x
        ys, xs = np.arange(ty * 16, min(H, ty * 16 + 16)), np.arange(tx * 16, min(W, tx * 16 + 16))
        gy, gx = np.meshgrid(ys, xs, indexing="ij")
        py, px = gy.ravel(), gx.ravel()
        a = attr[vals[s:e]]
        f = feats[vals[s:e]]
        co, uv = a["conic_opacity"], a["uv"]
        with np.errstate(all="ignore"):
            dx = uv[None, :, 0] - px.astype(np.float32)[:, None]
            dy = uv[None, :, 1] - py.astype(np.float32)[:, None]
            power = _f32(-0.5) * ((co[None, :, 0] * dx) * dx + (co[None, :, 2] * dy) * dy) - (co[None, :, 1] * dx) * dy
            live = ~(power > 0)
            ex = bg_ref.exp_shared(np.where(live, power, _f32(0.0)))
            alpha = np.fmin(_f32(0.99), co[None, :, 3] * ex)
            valid = live & ~(alpha < cut_a)
            factor = np.where(valid, one - alpha, one).astype(np.float32)
            t_after = np.multiply.accumulate(factor, axis=1, dtype=np.float32)
            brk = valid & (t_after < cut_t)
            first = np.where(brk.any(1), brk.argmax(1), brk.shape[1])
            contrib = valid & (np.arange(brk.shape[1])[None, :] < first[:, None])
            t_before = np.concatenate([np.ones((t_after.shape[0], 1), np.float32), t_after[:, :-1]], 1)
            for c in range(C):
                terms = np.where(contrib, (f[None, :, c] * alpha) * t_before, _f32(0.0)).astype(np.float32)
                terms = np.concatenate([np.zeros((terms.shape[0], 1), np.float32), terms], 1)
                out[py, px, c] = np.add.accumulate(terms, axis=1, dtype=np.float32)[:, -1]
    return out


def colours(frame, n):
    """(n, 3) fp32: each Gaussian's colour as the frame's records hold it (0 for Gaussians in no list)."""
    f = np.zeros((n, 3), np.float32)
    used = np.unique(frame["vals"].astype(np.int64))
    f[used] = frame["attr"]["color_radii"][used, :3]
    return f


def depth_keys(frame, n):
    """(n, 1) fp32: each Gaussian's depth key as the frame's records hold it (0 for Gaussians in no list)."""
    f = np.zeros((n, 1), np.float32)
    used = np.unique(frame["vals"].astype(np.int64))
    f[used, 0] = frame["attr"]["depth"][used]
    return f


def frame_values(leaf, feat, u, frame, local, cam=None, pre=None, info=None):
    """(H, W, 3 + C) float64: the image over black and the feature map of the frame whose lists are `frame`, for the survivor
    rows `leaf` and their features `feat` (L, C) (grad_ref.survivors' numbering `local`)."""
    pre = pre or depth_ref.pinhole()
    W, H = int(u.width), int(u.height)
    uv, conic, op, col, red, _ = pre(leaf, u, cam)
    cols = torch.cat([col, feat], 1)
    flat = torch.zeros((H * W, cols.shape[1]), dtype=torch.float64)
    idx, vals = [], []
    for tl in grad_ref.tiles(u, frame, local):
        i = tl.idx
        dx, dy = uv[i, 0][None, :] - tl.fx[:, None], uv[i, 1][None, :] - tl.fy[:, None]
        out, contrib, raw, _ = grad_ref.blend_offsets(dx, dy, conic[i], op[i], cols[i])
        idx.append(torch.tensor(tl.py * W + tl.px))
        vals.append(out)
        if info is not None:
            info.setdefault("tiles", []).append((tl, contrib, raw))
    if info is not None:
        info["red"] = red.detach()
    if idx:
        flat = flat.index_put((torch.cat(idx),), torch.cat(vals))
    return flat.reshape(H, W, cols.shape[1])


def reference(vertices, u, frame, features, grad_image=None, grad_fm=None, camera=False, pre=None):
    """The float64 (H, W, 3 + C) frame of `frame`'s lists and, with an upstream gradient -- grad_image (H, W, >= 3) and grad_fm
    (H, W, C), either may be None (zero) -- dL/dvertices (n, 60), dL/dfeatures (n, C), `exclude` (n,) as in depth_ref, and
    with camera=True grad_ubo (the 38 float fields)."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    n = v_all.shape[0]
    F = np.asarray(features, np.float64)
    C = F.shape[1]
    W, H = int(u.width), int(u.height)
    want = grad_image is not None or grad_fm is not None
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=want)
    feat = torch.tensor(F[used], requires_grad=want)
    cam = grad_ref.camera_leaves(u) if camera else None
    info = {}
    with torch.set_grad_enabled(want):
        vals = frame_values(leaf, feat, u, frame, local, cam, pre, info)
    out = {"values": vals.detach().numpy()}
    if not want:
        return out
    g = np.zeros((H, W, 3 + C))
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
    gf = np.zeros((n, C))
    gf[used] = feat.grad.numpy()
    exclude = np.zeros(n, bool)
    exclude[used] = near_clamp | (info["red"].abs().numpy() < 1e-4)
    out.update(grad=grad, grad_features=gf, exclude=exclude)
    if camera:
        out["grad_ubo"] = np.concatenate([np.zeros(t.numel()) if t.grad is None else np.atleast_1d(t.grad.numpy())
                                          for t in cam.values()])
    return out
