"""References of the rendered depth and alpha (gsb_render_depth, gsb_render_backward_depth).  Test infrastructure only.

For a pixel whose contributors are i = 1..k in list order, D = sum f_i alpha_i T_i (f the record's depth: view-space z, or the
distance |t| for a fisheye frame) and A = 1 - T_final.  Both references are layered on grad_ref / bg_ref / fisheye_ref, as
bg_ref and aa_ref are:

* `blend32` restates gso_blend in numpy fp32 over a frame's own lists and attributes (bg_ref.transmittance's restatement,
  with the exp of oracle exp mode 1), extended by D: (f * alpha) * T added like a colour channel.  Its colour is checked
  against the oracle's image bit for bit before D and A = 1 - T are used.
* `frame_values` is grad_ref's float64 blend with the colour columns extended by (f, 1): channels 3 and 4 are D and A.
  Channels 0-2 are the image over the background bg (T_final * bg added, bg on the pixels of empty tiles), where D = A = 0.
  It is differentiable in the vertices, the camera leaves (grad_ref.camera_leaves) and bg.
"""
from __future__ import annotations

import numpy as np
import torch

import bg_ref
import grad_ref

_f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# fp32: the oracle's blend, restated for D and T_final
# ---------------------------------------------------------------------------------------------------------------------
def blend32(frame, width, height):
    """(T, rgb, D) over the frame's lists (exp mode 1): each pixel's final transmittance (H, W), gso_blend's colour (H, W, 3)
    and D (H, W), all fp32 with one rounding per op.  Pixels of empty tiles: T = 1, colour 0, D = 0."""
    W, H = int(width), int(height)
    tiles_x = (W + 15) // 16
    attr, vals, ranges = frame["attr"], frame["vals"].astype(np.int64), frame["ranges"]
    T = np.ones((H, W), np.float32)
    rgb = np.zeros((H, W, 3), np.float32)
    D = np.zeros((H, W), np.float32)
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
        co, uv = a["conic_opacity"], a["uv"]
        chans = [a["color_radii"][:, c] for c in range(3)] + [a["depth"].astype(np.float32)]
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
            T_fin = np.where(first > 0, t_before[np.arange(t_after.shape[0]), np.minimum(first, brk.shape[1] - 1)], one)
            T_fin = np.where(first == brk.shape[1], t_after[:, -1], T_fin).astype(np.float32)
            sums = []
            for c in chans:
                terms = np.where(contrib, (c[None, :] * alpha) * t_before, _f32(0.0)).astype(np.float32)
                terms = np.concatenate([np.zeros((terms.shape[0], 1), np.float32), terms], 1)
                sums.append(np.add.accumulate(terms, axis=1, dtype=np.float32)[:, -1])
        for c in range(3):
            rgb[py, px, c] = sums[c]
        D[py, px] = sums[3]
        T[py, px] = T_fin
    return T, rgb, D


def depth_alpha32(frame, u, rows=None):
    """(rows, W, 2) fp32 (D, 1 - T_final) of the oracle frame `frame` (oracle.render_frame or aa_ref.oracle_frame at exp mode
    1; rows: its band of tile rows, None for the whole frame; its image is whole-frame either way), after checking that
    blend32 reproduces the band's image bit for bit."""
    T, rgb, D = blend32(frame, u.width, u.height)
    band = slice(0, int(u.height)) if rows is None else slice(rows[0] * 16, min(int(u.height), rows[1] * 16))
    assert np.array_equal(rgb[band].view(np.uint32), np.ascontiguousarray(frame["rgba"][band, :, :3]).view(np.uint32)), \
        "blend32 no longer restates gso_blend"
    return np.stack([D[band], _f32(1.0) - T[band]], -1).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# float64: grad_ref's blend with the (f, 1) columns
# ---------------------------------------------------------------------------------------------------------------------
def pinhole(antialiased=False):
    """The preprocess of a pinhole frame: grad_ref's (aa_ref's when antialiased) plus f = view row 2 . (p, 1)."""
    def pre(v, u, cam):
        if antialiased:
            import aa_ref

            uv, conic, op, col, red = aa_ref.preprocess(v, u, cam)
        else:
            uv, conic, op, col, red = grad_ref.preprocess(v, u, cam)
        V = grad_ref._mat(u.view_mat) if cam is None else cam["view_mat"].reshape(4, 4).T
        ph = torch.cat([v[:, 0:3], torch.ones_like(v[:, :1])], 1)
        return uv, conic, op, col, red, ph @ V[2]

    return pre


def fisheye(cam_model):
    """The preprocess of a fisheye frame (fisheye_ref) plus f = |t|, the distance from the camera."""
    import fisheye_ref

    def pre(v, u, cam):
        assert cam is None, "no camera gradient through the fisheye lens"
        uv, conic, op, col, red, _ = fisheye_ref.preprocess(v, u, cam_model)
        return uv, conic, op, col, red, torch.linalg.norm(fisheye_ref.view_positions(v, u), dim=1)

    return pre


def frame_values(leaf, u, frame, local, bg=None, cam=None, pre=None, info=None):
    """(H, W, 5) float64: the image over bg (3), D and A of the frame whose lists are `frame`, for the survivor rows `leaf`
    (grad_ref.survivors' numbering `local`).  Differentiable in leaf, cam (camera_leaves) and bg (a (3,) tensor, or values,
    or None for black).  info (a dict): receives per tile (tile, contrib, raw alpha) for the exclusion of ill-posed rows."""
    pre = pre or pinhole()
    W, H = int(u.width), int(u.height)
    uv, conic, op, col, red, f = pre(leaf, u, cam)
    col5 = torch.cat([col, f[:, None], torch.ones_like(f)[:, None]], 1)
    if bg is None:
        bgt = torch.zeros(3, dtype=torch.float64)
    else:
        bgt = bg if isinstance(bg, torch.Tensor) else torch.tensor(np.asarray(bg, np.float64).reshape(3))
    bg5 = torch.cat([bgt, torch.zeros(2, dtype=torch.float64)])
    flat = bg5[None, :].expand(H * W, 5)
    idx, vals = [], []
    for tl in grad_ref.tiles(u, frame, local):
        i = tl.idx
        dx, dy = uv[i, 0][None, :] - tl.fx[:, None], uv[i, 1][None, :] - tl.fy[:, None]
        out, contrib, raw, _ = grad_ref.blend_offsets(dx, dy, conic[i], op[i], col5[i])
        A_, B_, C_ = conic[i][None, :, 0], conic[i][None, :, 1], conic[i][None, :, 2]
        power = -0.5 * (A_ * dx * dx + C_ * dy * dy) - B_ * dx * dy
        alpha = torch.clamp(op[i][None, :] * torch.exp(torch.clamp(power, max=0.0)), max=0.99)
        t_final = torch.prod(1 - torch.where(contrib, alpha, torch.zeros_like(alpha)), 1)
        out = out + t_final[:, None] * bg5[None, :]
        idx.append(torch.tensor(tl.py * W + tl.px))
        vals.append(out)
        if info is not None:
            info.setdefault("tiles", []).append((tl, contrib, raw))
    if info is not None:
        info["red"] = red.detach()
    if idx:
        flat = flat.index_put((torch.cat(idx),), torch.cat(vals))
    return flat.reshape(H, W, 5)


def reference(vertices, u, frame, grad_image=None, grad_da=None, bg=None, camera=False, pre=None):
    """The float64 frame (H, W, 5) of `frame`'s lists and, when an upstream gradient is given -- grad_image (H, W, >= 3), grad_da
    (H, W, 2), either may be None (zero) -- dL/dvertices (n, 60) for L = sum g . (image, D, A), `exclude` (n,) as in grad_ref
    (unclamped red within 1e-4 of 0, raw alpha within 1e-4 of the 0.99 clamp on a pixel with an upstream gradient), and
    with camera=True grad_ubo (the 38 float fields), with a tensor bg its gradient in bg.grad."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    want = grad_image is not None or grad_da is not None
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=want)
    cam = grad_ref.camera_leaves(u) if camera else None
    info = {}
    with torch.set_grad_enabled(want):
        vals = frame_values(leaf, u, frame, local, bg, cam, pre, info)
    out = {"values": vals.detach().numpy()}
    if not want:
        return out
    g = np.zeros((H, W, 5))
    if grad_image is not None:
        g[..., :3] = np.asarray(grad_image, np.float64)[..., :3]
    if grad_da is not None:
        g[..., 3:] = np.asarray(grad_da, np.float64)[..., :2]
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
    out.update(grad=grad, exclude=exclude)
    if camera:
        out["grad_ubo"] = np.concatenate([np.zeros(t.numel()) if t.grad is None else np.atleast_1d(t.grad.numpy())
                                          for t in cam.values()])
    return out
