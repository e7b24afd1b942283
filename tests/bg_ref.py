"""References of the background colour (gsb_set_background).  Test infrastructure only.

With a background bg every colour channel of every pixel is c + T_final * bg (fp32 multiply, then add), T_final being the
transmittance after the pixel's last contributor (at the T' < 1e-4 break, the T before the breaking entry; 1 for a pixel
no entry reaches).  The oracle and grad_ref stay as they are; both references here are layered on them (the pattern of
aa_ref.py):

* `transmittance` restates gs_oracle.c's gso_blend in numpy fp32 over a frame's own lists and attributes (oracle.render_frame's
  or aa_ref.oracle_frame's), with the oracle's shared-definition exp (exp mode 1) restated op for op.  numpy rounds every
  float32 operation once, like the oracle's -ffp-contract=off build; fmaf is formed in float64 and rounded once to float32
  through round-to-odd, which is exact.  The transmittance never leaves gso_blend, so before it is used the restatement's
  own colour is checked against the oracle's image bit for bit on every pixel: both come from the same alphas, contributor
  sets and T chain.  `oracle_frame` adds T * bg to the oracle's image in numpy fp32.
* `reference` and `density_reference` are grad_ref's float64 functions with `blend_offsets` patched to add T_final * bg,
  T_final being the product of (1 - alpha) over the contributors; the pixels of empty tiles get bg.  bg may be a float64
  leaf tensor, and `grad_background` is the float64 sum of T * g over all pixels.
"""
from __future__ import annotations

from unittest import mock

import numpy as np
import torch

import grad_ref
import oracle as o

_f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# fp32: the oracle's blend, restated for its final transmittance
# ---------------------------------------------------------------------------------------------------------------------
def fmaf(a, b, c):
    """C's fmaf on float32 arrays: a * b + c rounded once.  a * b is exact in float64; the float64 sum is made exact by
    TwoSum and rounded to odd, from which the rounding to float32 (24 bits, 53 >= 2 * 24 + 2) is the correctly rounded one."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    inexact = e != 0
    away = inexact & ((e > 0) != (s > 0))  # |s| > |s + e|: truncation is one ulp toward zero
    s = np.where(away, np.nextafter(s, 0.0), s)
    bits = s.view(np.int64) | inexact.astype(np.int64)
    return bits.view(np.float64).astype(np.float32)


def exp_shared(x):
    """gso_exp_shared (oracle exp mode 1) on a float32 array, op for op."""
    x = np.asarray(x, np.float32)
    with np.errstate(all="ignore"):
        x = np.where(x < _f32(-87.0), _f32(-87.0), x).astype(np.float32)
        t = x * _f32(1.44269504088896341)
        magic = _f32(12582912.0)
        tm = (t + magic).astype(np.float32)
        n = tm - magic
        r = fmaf(n, _f32(-0.693359375), x)
        r = fmaf(n, _f32(2.12194440e-4), r)
        p = fmaf(_f32(8.290082216262817e-3), r, _f32(4.1899293661117554e-2))
        p = fmaf(p, r, _f32(1.6667647659778595e-1))
        p = fmaf(p, r, _f32(4.9999138712882996e-1))
        p = fmaf(p, r, _f32(9.999997019767761e-1))
        p = fmaf(p, r, _f32(1.0))
    y = p.view(np.uint32) + (tm.view(np.uint32) << np.uint32(23))
    return y.view(np.float32)


def transmittance(frame, width, height):
    """(T, rgb): each pixel's final transmittance (H, W) fp32 and the colour gso_blend computes (H, W, 3) fp32 over the
    frame's lists (exp mode 1).  Pixels of empty tiles: T = 1, colour 0."""
    W, H = int(width), int(height)
    tiles_x = (W + 15) // 16
    attr, vals, ranges = frame["attr"], frame["vals"].astype(np.int64), frame["ranges"]
    T = np.ones((H, W), np.float32)
    rgb = np.zeros((H, W, 3), np.float32)
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
        co, uv, col = a["conic_opacity"], a["uv"], a["color_radii"][:, :3]
        with np.errstate(all="ignore"):
            dx = uv[None, :, 0] - px.astype(np.float32)[:, None]
            dy = uv[None, :, 1] - py.astype(np.float32)[:, None]
            power = _f32(-0.5) * ((co[None, :, 0] * dx) * dx + (co[None, :, 2] * dy) * dy) - (co[None, :, 1] * dx) * dy
            live = ~(power > 0)
            ex = exp_shared(np.where(live, power, _f32(0.0)))
            alpha = np.fmin(_f32(0.99), co[None, :, 3] * ex)
            valid = live & ~(alpha < cut_a)
            factor = np.where(valid, one - alpha, one).astype(np.float32)
            t_after = np.multiply.accumulate(factor, axis=1, dtype=np.float32)  # sequential, one rounding per step
            brk = valid & (t_after < cut_t)
            first = np.where(brk.any(1), brk.argmax(1), brk.shape[1])
            idx = np.arange(brk.shape[1])[None, :]
            contrib = valid & (idx < first[:, None])
            t_before = np.concatenate([np.ones((t_after.shape[0], 1), np.float32), t_after[:, :-1]], 1)
            T_fin = np.where(first > 0, t_before[np.arange(t_after.shape[0]), np.minimum(first, brk.shape[1] - 1)], one)
            T_fin = np.where(first == brk.shape[1], t_after[:, -1], T_fin).astype(np.float32)
            for c in range(3):
                terms = np.where(contrib, (col[None, :, c] * alpha) * t_before, _f32(0.0)).astype(np.float32)
                terms = np.concatenate([np.zeros((terms.shape[0], 1), np.float32), terms], 1)
                rgb[py, px, c] = np.add.accumulate(terms, axis=1, dtype=np.float32)[:, -1]
        T[py, px] = T_fin
    return T, rgb


def composite(rgba, T, bg):
    """rgba[..., :3] + T * bg in fp32 (multiply, then add), A = 1: what gsb_set_background frames store."""
    out = np.array(rgba, np.float32, copy=True)
    bgv = np.asarray(bg, np.float32).reshape(3)
    for c in range(3):
        out[..., c] = out[..., c] + T * bgv[c]
    out[..., 3] = _f32(1.0)
    return out


def with_transmittance(frame, u):
    """frame plus `T`: the restated transmittance, after checking that the restatement reproduces frame['rgba'] bit for
    bit (the frame must come from exp mode 1)."""
    T, rgb = transmittance(frame, u.width, u.height)
    assert np.array_equal(rgb.view(np.uint32), np.ascontiguousarray(frame["rgba"][..., :3]).view(np.uint32)), \
        "transmittance() no longer restates gso_blend"
    out = dict(frame)
    out["T"] = T
    return out


def oracle_frame(vertices, cov, u, bg, antialiased=False, rows=None):
    """The oracle's frame over bg (oracle exp mode 1 must be set): oracle.render_frame's (or, antialiased, aa_ref.oracle_frame's)
    dict plus `T` (H, W) and `rgba` composited over bg.  `rgba_black` keeps the oracle's own image."""
    if antialiased:
        import aa_ref

        f = aa_ref.oracle_frame(vertices, cov, u, rows)
    else:
        f = o.render_frame(vertices, cov, u, rows)
    f = with_transmittance(f, u)
    f["rgba_black"] = f["rgba"]
    f["rgba"] = composite(f["rgba"], f["T"], bg)
    return f


# ---------------------------------------------------------------------------------------------------------------------
# float64: grad_ref with the background term
# ---------------------------------------------------------------------------------------------------------------------
_plain_blend_offsets = grad_ref.blend_offsets


def _background(bg):
    """grad_ref's frame functions call its module-level blend_offsets: for one call, the one that adds T_final * bg."""
    bgt = bg if isinstance(bg, torch.Tensor) else torch.tensor(np.asarray(bg, np.float64).reshape(3))

    def blend_offsets(dx, dy, conic, op, col):
        rgb, contrib, raw, valid = _plain_blend_offsets(dx, dy, conic, op, col)
        A, B, C = conic[None, :, 0], conic[None, :, 1], conic[None, :, 2]
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        alpha = torch.clamp(op[None, :] * torch.exp(torch.clamp(power, max=0.0)), max=0.99)
        a = torch.where(contrib, alpha, torch.zeros_like(alpha))
        t_final = torch.prod(1 - a, 1)
        return rgb + t_final[:, None] * bgt[None, :], contrib, raw, valid

    return mock.patch.object(grad_ref, "blend_offsets", blend_offsets), bgt


def _empty_tile_pixels(u, frame):
    """(H, W) bool: the pixels of the tiles whose list is empty."""
    W, H = int(u.width), int(u.height)
    tiles_x = (W + 15) // 16
    r = frame["ranges"]
    empty_tile = (r[:, 1] <= r[:, 0]).reshape(-1, tiles_x)
    return np.repeat(np.repeat(empty_tile, 16, 0), 16, 1)[:H, :W]


def transmittance64(vertices, u, frame):
    """Float64 T_final (H, W) over the frame's lists: grad_ref's blend with a unit background and black colours."""
    with torch.no_grad():
        uv, conic, op, col, _ = grad_ref.preprocess(torch.tensor(np.asarray(vertices, np.float32)[np.unique(frame["vals"].astype(np.int64))]
                                                                 .astype(np.float64)), u)
    _, used, local = grad_ref.survivors(vertices, frame)
    T = np.ones((int(u.height), int(u.width)))
    for tl in grad_ref.tiles(u, frame, local):
        _, contrib, _, _ = grad_ref.blend_tile(uv[tl.idx], conic[tl.idx], op[tl.idx], col[tl.idx], tl.fx, tl.fy)
        A, B, C = conic[tl.idx][None, :, 0], conic[tl.idx][None, :, 1], conic[tl.idx][None, :, 2]
        dx, dy = uv[tl.idx][None, :, 0] - tl.fx[:, None], uv[tl.idx][None, :, 1] - tl.fy[:, None]
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        alpha = torch.clamp(op[tl.idx][None, :] * torch.exp(torch.clamp(power, max=0.0)), max=0.99)
        T[tl.py, tl.px] = torch.prod(1 - torch.where(contrib, alpha, torch.zeros_like(alpha)), 1).numpy()
    return T


def grad_background(T, grad_image):
    """float64 sum over all pixels of T * g (3,)."""
    g = np.asarray(grad_image, np.float64)[..., :3]
    return (np.asarray(T, np.float64)[..., None] * g).sum((0, 1))


def reference(vertices, u, frame, bg, grad_image=None, camera=False):
    """grad_ref.reference of a frame over bg: the image gets T_final * bg (bg on the pixels of empty tiles), the gradients
    the background's share of the chain rule.  bg: 3 values or a float64 (3,) tensor (a leaf: its .grad then holds the tiles'
    share of dL/dbg; `grad_background` below is the whole of it)."""
    patch, bgt = _background(bg)
    with patch:
        out = grad_ref.reference(vertices, u, frame, grad_image, camera)
    empty = _empty_tile_pixels(u, frame)
    out["image"][empty] += bgt.detach().numpy()[None, :]
    return out


def density_reference(vertices, u, frame, bg, grad_image):
    """grad_ref.density_reference of a frame over bg."""
    patch, _ = _background(bg)
    with patch:
        return grad_ref.density_reference(vertices, u, frame, grad_image)
