"""Float64 restatement of the orthographic camera of gsb_set_camera_model (DESIGN.md section 26), layered on grad_ref,
sh_degree_ref and aa_ref as those are on each other, and a numpy fp32 restatement of k_project's record words in the kernel's
operation order.  The blend and its depth / alpha and feature columns are depth_ref's and features_ref's.  Test
infrastructure only.

The camera, for the view-space position t = (x, y, z) of clip_view's view rows: uv = (fx x + cx, fy y + cy), kept when
z > 0.2, J = [fx, 0, 0; 0, fy, 0], cov2d = J W Sigma W^T J^T + 0.3 I, depth key z, and the SH colour seen along the camera's
forward axis: the direction normalize(view row 2), the same for every Gaussian.
"""
from __future__ import annotations

import numpy as np
import torch

import depth_ref
import features_ref
import grad_ref
import sh_degree_ref

U_CAMPOS, U_VIEW = 0, 20
# the words of an orthographic frame's camera gradient that can be non-zero: view rows 0-2 (camera_position is not read)
LIVE_UBO = np.array([U_VIEW <= j < U_VIEW + 16 and (j & 3) != 3 for j in range(40)])
_f32 = np.float32


def cam_tuple(cam):
    """(fx, fy, cx, cy) of a gs_b200.CameraModel or of such a tuple."""
    if isinstance(cam, tuple):
        return cam[:4]
    return (float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy))


def lens_values(cam):
    """(fx, fy, cx, cy, 0, 0, 0, 0) as a float64 array: lens_tensor's layout."""
    return np.array([*cam_tuple(cam), 0.0, 0.0, 0.0, 0.0], np.float64)


def project(t, cam):
    """uv (k, 2) of the view-space positions t (k, 3), differentiable in t and in tensor lens values."""
    fx, fy, cx, cy = cam_tuple(cam)
    return torch.stack([fx * t[:, 0] + cx, fy * t[:, 1] + cy], -1)


def jacobian(cam):
    """J = d uv / d t (2, 3), float64."""
    fx, fy, _, _ = (float(x) for x in cam_tuple(cam))
    return np.array([[fx, 0.0, 0.0], [0.0, fy, 0.0]])


def grad_t(cam, duv, df=None):
    """The closed form of ortho_grad: dL/dt (k, 3) = J^T duv, plus df (k,) on z for the depth key f = z."""
    fx, fy, _, _ = (float(x) for x in cam_tuple(cam))
    duv = np.asarray(duv, np.float64)
    out = np.stack([fx * duv[:, 0], fy * duv[:, 1], np.zeros(len(duv))], 1)
    if df is not None:
        out[:, 2] += df
    return out


def lens_grad(t, dJ, duv):
    """The closed form of ortho_lens_grad: dL/d(fx, fy, cx, cy) (k, 4) of Phi = sum dJ * J + duv . uv."""
    t, dJ, duv = (np.asarray(a, np.float64) for a in (t, dJ, duv))
    return np.stack([duv[:, 0] * t[:, 0] + dJ[:, 0, 0], duv[:, 1] * t[:, 1] + dJ[:, 1, 1], duv[:, 0], duv[:, 1]], 1)


def view_positions(v, V):
    ph = torch.cat([v[:, 0:3], torch.ones_like(v[:, :1])], 1)
    return (ph @ V.T)[:, :3]


def forward_dir(view_mat):
    """view row 2 ([2], [6], [10] of the column-major view matrix), the SH direction before normalisation."""
    return view_mat[2::4][:3] if isinstance(view_mat, torch.Tensor) else np.asarray(list(view_mat), np.float64)[[2, 6, 10]]


def colour(v, view_mat, sh_degree=3):
    """The SH colour (k, 3) (red clamped at 0) and the unclamped red (k,) of the rows of v, seen along normalize(view row 2):
    sh_degree_ref.sh_colour of the point view row 2 from the origin, which leaves p out."""
    e = forward_dir(view_mat)
    e = e if isinstance(e, torch.Tensor) else torch.tensor(e)
    w = torch.cat([e.expand(v.shape[0], 3), v[:, 3:]], 1)
    return sh_degree_ref.sh_colour(w, torch.zeros(3, dtype=torch.float64), sh_degree)


# ---------------------------------------------------------------------------------------------------------------------
# the float64 frame with camera and lens leaves
# ---------------------------------------------------------------------------------------------------------------------
def leaves(u, cam):
    """The float64 leaves of an orthographic frame's camera: grad_ref.camera_leaves(u) and the lens (8,)."""
    cl = grad_ref.camera_leaves(u)
    cl["lens"] = torch.tensor(lens_values(cam)).requires_grad_()
    return cl


def pre(cl, antialiased=False, sh_degree=3):
    """A depth_ref-style preprocess (v, u, _) -> (uv, conic, op, colour, red, f = z) through the leaves cl (leaves())."""
    def fn(v, u, _cam=None):
        s, op, q = v[:, 4:7], v[:, 7], v[:, 8:12]
        qw, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        R = torch.stack([
            torch.stack([1 - 2 * qy * qy - 2 * qz * qz, 2 * qx * qy + 2 * qz * qw, 2 * qx * qz - 2 * qy * qw], -1),
            torch.stack([2 * qx * qy - 2 * qz * qw, 1 - 2 * qx * qx - 2 * qz * qz, 2 * qy * qz + 2 * qx * qw], -1),
            torch.stack([2 * qx * qz + 2 * qy * qw, 2 * qy * qz - 2 * qx * qw, 1 - 2 * qx * qx - 2 * qy * qy], -1),
        ], -2)
        M = s[:, :, None] * R
        Sigma = M.transpose(1, 2) @ M
        V = cl["view_mat"].reshape(4, 4).T
        t = view_positions(v, V)
        L = cl["lens"]
        uv = project(t, (L[0], L[1], L[2], L[3]))
        zero = torch.zeros((), dtype=torch.float64)
        J = torch.stack([torch.stack([L[0], zero, zero]), torch.stack([zero, L[1], zero])])
        T = J[None] @ V[:3, :3]
        cov = T @ Sigma @ T.transpose(1, 2)
        a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
        det = a * c - b * b
        conic = torch.stack([c / det, -b / det, a / det], -1)
        if antialiased:
            import aa_ref

            op = op * aa_ref.compensation(conic)
        col, red = colour(v, cl["view_mat"], sh_degree)
        return uv, conic, op, col, red, t[:, 2]

    return fn


def reference(vertices, u, cam, frame, grad_image=None, grad_da=None, features=None, grad_fm=None, antialiased=False,
              sh_degree=3):
    """The float64 frame of `frame`'s lists ({"vals", "ranges"}) through the orthographic camera cam: "image" (H, W, 3),
    "depth_alpha" (H, W, 2) (D with f = z, and A) and, with an upstream gradient -- grad_image (H, W, >= 3), grad_da (H, W, 2)
    or, with features (n, C), grad_fm (H, W, C) -- dL/dvertices "grad" (n, 60), "grad_ubo" (40,) (zero outside LIVE_UBO),
    "grad_lens" (8,) (k words 0), "exclude" (n,) as in depth_ref and, with features, "grad_features" (n, C)."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    cl = leaves(u, cam)
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=True)
    fn = pre(cl, antialiased, sh_degree)
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
    out = {"image": vals[..., :3].detach().numpy(), "depth_alpha": vals[..., 3:5].detach().numpy()}
    if not g.any():
        return out
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
    gu[U_VIEW:U_VIEW + 16] = cl["view_mat"].grad.numpy()
    gu[~LIVE_UBO] = 0.0
    assert cl["camera_position"].grad is None or not cl["camera_position"].grad.any()
    gl = cl["lens"].grad.numpy().copy()
    gl[4:] = 0.0  # k is 0 by definition: not a parameter of the camera
    out.update(grad=grad, grad_ubo=gu, grad_lens=gl, exclude=exclude)
    if features is not None:
        gf = np.zeros((n, F.shape[1]))
        gf[used] = feat.grad.numpy()
        out["grad_features"] = gf
    return out


def step_pixels(vertices, u, cam, frame, antialiased=False, rel=1e-3):
    """(H, W) bool: the pixels where the float64 restatement lies within `rel` of one of the blend's step functions, which
    get no upstream gradient in the camera comparisons (as opencv_ref.step_pixels)."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    W, H = int(u.width), int(u.height)
    leaf = torch.tensor(v_all[used].astype(np.float64))
    uv, conic, op, _, _, _ = pre(leaves(u, cam), antialiased)(leaf, u)
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


# ---------------------------------------------------------------------------------------------------------------------
# fp32: k_project's record words, op for op
# ---------------------------------------------------------------------------------------------------------------------
_SH_C = (0.28209479177387814, 0.4886025119029199, 1.0925484305920792, -1.0925484305920792, 0.31539156525252005,
         -1.0925484305920792, 0.5462742152960396, -0.5900435899266435, 2.890611442640554, -0.4570457994644658,
         0.3731763325901154, -0.4570457994644658, 1.445305721320277, -0.5900435899266435)


def colour32(sh, view_mat, sh_degree=3):
    """compute_sh / compute_sh_degree of the kernel in fp32 for the SH rows sh (k, 48) seen along view row 2: (k, 3)."""
    C = [_f32(c) for c in _SH_C]
    C0, C1, C20, C21, C22, C23, C24, C30, C31, C32, C33, C34, C35, C36 = C
    vm = np.asarray(list(view_mat), np.float32)
    dx, dy, dz = vm[2] - _f32(0), vm[6] - _f32(0), vm[10] - _f32(0)
    ln = np.sqrt(_f32(dx * dx + dy * dy) + dz * dz, dtype=np.float32)
    x, y, z = _f32(dx / ln), _f32(dy / ln), _f32(dz / ln)
    xx, yy = _f32(x * x), _f32(y * y)
    two, three, four = _f32(2), _f32(3), _f32(4)
    w6 = _f32(_f32(_f32(two * z) * z - xx) - yy)
    w8 = _f32(xx - yy)
    w9 = _f32(_f32(three * x) * x - yy)
    w11 = _f32(_f32(_f32(four * z) * z - xx) - yy)
    w12 = _f32(_f32(_f32(two * z) * z - _f32(three * x) * x) - _f32(three * y) * y)
    w15 = _f32(xx - _f32(three * y) * y)
    terms = [lambda a, s: C0 * s, lambda a, s: a - (C1 * s) * y, lambda a, s: a + (C1 * s) * z, lambda a, s: a - (C1 * s) * x,
             lambda a, s: a + ((C20 * s) * x) * y, lambda a, s: a + ((C21 * s) * y) * z, lambda a, s: a + (C22 * s) * w6,
             lambda a, s: a + ((C23 * s) * z) * x, lambda a, s: a + (C24 * s) * w8, lambda a, s: a + ((C30 * s) * w9) * y,
             lambda a, s: a + (((C31 * s) * x) * y) * z, lambda a, s: a + ((C32 * s) * w11) * y,
             lambda a, s: a + ((C33 * s) * z) * w12, lambda a, s: a + ((C34 * s) * x) * w11,
             lambda a, s: a + ((C35 * s) * w8) * z, lambda a, s: a + ((C36 * s) * x) * w15]
    sh = np.asarray(sh, np.float32).reshape(-1, 16, 3)
    nk = (sh_degree + 1) ** 2
    out = np.zeros((sh.shape[0], 3), np.float32)
    with np.errstate(all="ignore"):
        for ch in range(3):
            c = np.zeros(sh.shape[0], np.float32)
            for k in range(nk):
                c = terms[k](c, sh[:, k, ch]).astype(np.float32)
            out[:, ch] = c + _f32(0.5)
    out[:, 0] = np.where(out[:, 0] < 0, _f32(0), out[:, 0])
    return out


def record32(vertices, cov3d, u, cam):
    """k_project's words per Gaussian, in fp32 op for op: a dict of kept (n,), uv (n, 2), conic (n, 3), radii (n,),
    aabb (n, 4) (x0, y0, x1, y1; zeros where culled), depth (n,).  cov3d (n, 6) are the frame's own Sigma words
    (GSB_BUF_COV3D)."""
    v = np.asarray(vertices, np.float32).reshape(-1, 60)
    S = np.asarray(cov3d, np.float32).reshape(-1, 6)
    vm = np.asarray(list(u.view_mat), np.float32)
    fx, fy, cx, cy = (_f32(x) for x in cam_tuple(cam))
    px, py, pz = v[:, 0], v[:, 1], v[:, 2]
    with np.errstate(all="ignore"):
        vx = ((vm[0] * px + vm[4] * py) + vm[8] * pz) + vm[12]
        vy = ((vm[1] * px + vm[5] * py) + vm[9] * pz) + vm[13]
        vz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14]
        T0 = [fx * vm[r * 4 + 0] for r in range(3)]
        T1 = [fy * vm[r * 4 + 1] for r in range(3)]
        Sg = [[S[:, 0], S[:, 1], S[:, 2]], [S[:, 1], S[:, 3], S[:, 4]], [S[:, 2], S[:, 4], S[:, 5]]]
        tm0 = [(T0[0] * Sg[k][0] + T0[1] * Sg[k][1]) + T0[2] * Sg[k][2] for k in range(3)]
        tm1 = [(T1[0] * Sg[k][0] + T1[1] * Sg[k][1]) + T1[2] * Sg[k][2] for k in range(3)]
        m00 = ((tm0[0] * T0[0] + tm0[1] * T0[1]) + tm0[2] * T0[2]) + _f32(0.3)
        m01 = (tm1[0] * T0[0] + tm1[1] * T0[1]) + tm1[2] * T0[2]
        m10 = (tm0[0] * T1[0] + tm0[1] * T1[1]) + tm0[2] * T1[2]
        m11 = ((tm1[0] * T1[0] + tm1[1] * T1[1]) + tm1[2] * T1[2]) + _f32(0.3)
        det = m00 * m11 - m10 * m01
        ood = _f32(1) / det
        conic = np.stack([m11 * ood, -m01 * ood, m00 * ood], 1)
        mid = _f32(0.5) * (m00 + m11)
        sq = np.sqrt(np.fmax(_f32(0.1), mid * mid - det))
        lam = np.fmax(mid + sq, mid - sq)
        radii = np.ceil(_f32(3) * np.sqrt(lam))
        uvx, uvy = fx * vx + cx, fy * vy + cy
        tx, ty = (int(u.width) + 15) // 16, (int(u.height) + 15) // 16

        def tile(a, hi):
            a = np.where(np.isnan(a), 0, a)
            return np.clip(np.trunc(np.clip(a, -2.0 ** 31, 2.0 ** 31 - 1)), 0, hi).astype(np.int64)

        s16 = _f32(16)
        box = np.stack([tile((uvx - radii) / s16, tx), tile((uvy - radii) / s16, ty),
                        tile((((uvx + radii) + s16) - _f32(1)) / s16, tx), tile((((uvy + radii) + s16) - _f32(1)) / s16, ty)], 1)
    front = vz > _f32(0.2)
    ok = front & ~(det <= 0)
    nt = (box[:, 2] - box[:, 0]) * (box[:, 3] - box[:, 1])
    kept = ok & (nt != 0)
    box[~kept] = 0
    return {"kept": kept, "uv": np.stack([uvx, uvy], 1).astype(np.float32), "conic": conic.astype(np.float32),
            "radii": radii.astype(np.float32), "aabb": box, "depth": vz.astype(np.float32)}


def pinhole_pullback(t, focal, D):
    """The cross-check of the CPU tests: a float64 pinhole of focal f D whose camera sits D farther back along the view axis
    maps t = (x, y, z) to (f D x / (z + D), f D y / (z + D)) with J = f D / (z + D) [1, 0, -x / (z + D); 0, 1, -y / (z + D)],
    which tends to the orthographic (f x, f y) and [f, 0, 0; 0, f, 0] as D grows.  Returns (uv (k, 2), J (k, 2, 3))."""
    t = np.asarray(t, np.float64)
    x, y, z = t[:, 0], t[:, 1], t[:, 2] + D
    s = focal * D / z
    J = np.zeros((len(t), 2, 3))
    J[:, 0, 0], J[:, 0, 2] = s, -s * x / z
    J[:, 1, 1], J[:, 1, 2] = s, -s * y / z
    return np.stack([s * x, s * y], 1), J
