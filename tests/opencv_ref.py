"""Float64 restatement of the OpenCV (Brown-Conrady radial-tangential) lens of gsb_set_camera_model (DESIGN.md section 23), the
closed forms of the kernels (gsb_geom.cuh opencv_geo, opencv_jacobian, opencv_grad, opencv_lens_grad) evaluated in numpy op for
op, and a float64 torch frame whose view matrix, camera position and lens (fx, fy, cx, cy, k1, k2, p1, p2) are leaves.  The
blend and its depth / alpha and feature columns are depth_ref's and features_ref's.  Test infrastructure only.

The lens, for the view-space position t = (x, y, z): xn = x / z, yn = y / z, r2 = xn^2 + yn^2, R = 1 + k1 r2 + k2 r2^2,
xd = xn R + 2 p1 xn yn + p2 (r2 + 2 xn^2), yd = yn R + p1 (r2 + 2 yn^2) + 2 p2 xn yn, uv = (fx xd + cx, fy yd + cy).  A
Gaussian is kept when z > 0.2, r2 <= tan^2(max_theta) (rounded to fp32 once) and det d(xd, yd) / d(xn, yn) > 0.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import depth_ref
import features_ref
import grad_ref

# gsb_uniforms word offsets (ABI order) and the words of a lens frame's camera gradient that can be non-zero
U_CAMPOS, U_VIEW = 0, 20
LIVE_UBO = np.array([j < 3 or (U_VIEW <= j < U_VIEW + 16 and (j & 3) != 3) for j in range(40)])


def cam_tuple(cam):
    """(fx, fy, cx, cy, k (4,), max_theta) of a gs_b200.CameraModel or of such a tuple."""
    if isinstance(cam, tuple):
        return cam
    return (float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy), [float(x) for x in cam.k], float(cam.max_theta))


def lens_values(cam):
    """(fx, fy, cx, cy, k1, k2, p1, p2) as a float64 array."""
    fx, fy, cx, cy, k, _ = cam_tuple(cam)
    return np.array([fx, fy, cx, cy, *k], np.float64)


def tan2_bound(max_theta):
    """k_project's cull bound: tan^2 of the fp32 max_theta in double, rounded to fp32 once (as launch_project does)."""
    t = math.tan(float(np.float32(max_theta)))
    return float(np.float32(t * t))


def project(t, cam):
    """uv (k, 2) of the view-space positions t (k, 3), float64 torch, differentiable in t and in a tensor lens (the map
    itself: autograd of this is the reference D, J and lens derivatives)."""
    fx, fy, cx, cy, k, _ = cam_tuple(cam)
    k1, k2, p1, p2 = k
    x, y, z = t[:, 0], t[:, 1], t[:, 2]
    xn, yn = x / z, y / z
    r2 = xn * xn + yn * yn
    R = 1 + r2 * (k1 + r2 * k2)
    xd = xn * R + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * R + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    return torch.stack([fx * xd + cx, fy * yd + cy], -1)


def distort(n, cam):
    """(xd, yd) (k, 2) of the normalised points n (k, 2), float64 torch (project's inner map)."""
    t = torch.cat([n, torch.ones_like(n[:, :1])], 1)
    return project(t, (1.0, 1.0, 0.0, 0.0) + tuple(cam_tuple(cam)[4:]))


def geo(t, cam, f=np.float64):
    """opencv_geo of the kernel in dtype f, op for op: a dict of xn, yn, r2, R, Rp, xd, yd, D00, D01, D11, e0, e1, det."""
    t = np.asarray(t, f)
    x, y, z = t[:, 0], t[:, 1], t[:, 2]
    k1, k2, p1, p2 = (f(v) for v in cam_tuple(cam)[4])
    two, six = f(2), f(6)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        xn, yn = x / z, y / z
        xx, yy, xy = xn * xn, yn * yn, xn * yn
        r2 = xx + yy
        R = f(1) + r2 * (k1 + r2 * k2)
        Rp = k1 + (two * k2) * r2
        g = dict(xn=xn, yn=yn, r2=r2, R=R, Rp=Rp)
        g["xd"] = xn * R + ((two * p1) * xy + p2 * (r2 + two * xx))
        g["yd"] = yn * R + (p1 * (r2 + two * yy) + (two * p2) * xy)
        g["D00"] = ((R + (two * xx) * Rp) + (two * p1) * yn) + (six * p2) * xn
        g["D11"] = ((R + (two * yy) * Rp) + (six * p1) * yn) + (two * p2) * xn
        g["D01"] = ((two * xy) * Rp + (two * p1) * xn) + (two * p2) * yn
        g["e0"] = g["D00"] * xn + g["D01"] * yn
        g["e1"] = g["D01"] * xn + g["D11"] * yn
        g["det"] = g["D00"] * g["D11"] - g["D01"] * g["D01"]
    return g


def jacobian(t, cam, f=np.float64):
    """The kernel's closed-form (D (k, 2, 2), J (k, 2, 3)) (opencv_geo, opencv_jacobian) in dtype f, op for op."""
    fx, fy = f(cam_tuple(cam)[0]), f(cam_tuple(cam)[1])
    z = np.asarray(t, f)[:, 2]
    g = geo(t, cam, f)
    D = np.stack([np.stack([g["D00"], g["D01"]], -1), np.stack([g["D01"], g["D11"]], -1)], -2)
    J = np.empty((z.shape[0], 2, 3), f)
    J[:, 0, 0], J[:, 0, 1], J[:, 0, 2] = (fx * g["D00"]) / z, (fx * g["D01"]) / z, -(fx * g["e0"]) / z
    J[:, 1, 0], J[:, 1, 1], J[:, 1, 2] = (fy * g["D01"]) / z, (fy * g["D11"]) / z, -(fy * g["e1"]) / z
    return D, J


def _dj(cam, g, dJ, f):
    fx, fy = f(cam_tuple(cam)[0]), f(cam_tuple(cam)[1])
    A0, A1, A2 = fx * dJ[:, 0, 0], fx * dJ[:, 0, 1], fx * dJ[:, 0, 2]
    B0, B1, B2 = fy * dJ[:, 1, 0], fy * dJ[:, 1, 1], fy * dJ[:, 1, 2]
    return A2, B2, A0 - A2 * g["xn"], (A1 + B0) - (A2 * g["yn"] + B2 * g["xn"]), B1 - B2 * g["yn"]


def grad_t(t, cam, dJ, duv, f=np.float64):
    """opencv_grad in dtype f, op for op: dL/dt (k, 3) of Phi = sum dJ * J + duv . uv for upstream dJ (k, 2, 3), duv (k, 2)."""
    fx, fy, _, _, k, _ = cam_tuple(cam)
    fx, fy, k8, p1, p2 = f(fx), f(fy), f(8) * f(k[1]), f(k[2]), f(k[3])
    t = np.asarray(t, f)
    dJ, duv = np.asarray(dJ, f), np.asarray(duv, f)
    z = t[:, 2]
    g = geo(t, cam, f)
    xn, yn, Rp = g["xn"], g["yn"], g["Rp"]
    A2, B2, a, m, c = _dj(cam, g, dJ, f)
    psi = (a * g["D00"] + m * g["D01"]) + c * g["D11"]
    H000 = ((f(6) * xn) * Rp + ((k8 * xn) * xn) * xn) + f(6) * p2
    H001 = ((f(2) * yn) * Rp + ((k8 * xn) * xn) * yn) + f(2) * p1
    H011 = ((f(2) * xn) * Rp + ((k8 * yn) * yn) * xn) + f(2) * p2
    H111 = ((f(6) * yn) * Rp + ((k8 * yn) * yn) * yn) + f(6) * p1
    psx = ((a * H000 + m * H001) + c * H011) - (A2 * g["D00"] + B2 * g["D01"])
    psy = ((a * H001 + m * H011) + c * H111) - (A2 * g["D01"] + B2 * g["D11"])
    Lu, Lv = fx * duv[:, 0], fy * duv[:, 1]
    gx = psx / z + (Lu * g["D00"] + Lv * g["D01"])
    gy = psy / z + (Lu * g["D01"] + Lv * g["D11"])
    return np.stack([gx / z, gy / z, -((gx * xn + gy * yn) + psi / z) / z], 1)


def lens_grad(t, cam, dJ, duv, f=np.float64):
    """opencv_lens_grad in dtype f, op for op: dL/d(fx, fy, cx, cy, k1, k2, p1, p2) (k, 8) of the same Phi."""
    fx, fy = f(cam_tuple(cam)[0]), f(cam_tuple(cam)[1])
    t = np.asarray(t, f)
    dJ, duv = np.asarray(dJ, f), np.asarray(duv, f)
    z = t[:, 2]
    g = geo(t, cam, f)
    xn, yn, r2 = g["xn"], g["yn"], g["r2"]
    xx, yy, xy = xn * xn, yn * yn, xn * yn
    du, dv = duv[:, 0], duv[:, 1]
    out = np.zeros((t.shape[0], 8), f)
    out[:, 0] = du * g["xd"] + ((dJ[:, 0, 0] * g["D00"] + dJ[:, 0, 1] * g["D01"]) - dJ[:, 0, 2] * g["e0"]) / z
    out[:, 1] = dv * g["yd"] + ((dJ[:, 1, 0] * g["D01"] + dJ[:, 1, 1] * g["D11"]) - dJ[:, 1, 2] * g["e1"]) / z
    out[:, 2], out[:, 3] = du, dv
    _, _, a, m, c = _dj(cam, g, dJ, f)
    Lu, Lv = fx * du, fy * dv
    s, q, Ld = a + c, ((a * xx + m * xy) + c * yy), Lu * xn + Lv * yn
    two = f(2)
    out[:, 4] = (r2 * s + two * q) / z + r2 * Ld
    out[:, 5] = r2 * ((r2 * s + f(4) * q) / z + r2 * Ld)
    out[:, 6] = (((two * a) * yn + (two * m) * xn) + (f(6) * c) * yn) / z + (Lu * (two * xy) + Lv * (r2 + two * yy))
    out[:, 7] = (((f(6) * a) * xn + (two * m) * yn) + (two * c) * xn) / z + (Lu * (r2 + two * xx) + Lv * (two * xy))
    return out


def _cam_of(L, max_theta=0.0):
    return (L[0], L[1], L[2], L[3], [L[4], L[5], L[6], L[7]], max_theta)


def autograd(t, cam, dJ, duv):
    """By autograd of project (float64): D (k, 2, 2), J (k, 2, 3), dL/dt (k, 3) and dL/dlens (k, 8) of
    Phi = sum dJ * J + duv . uv, the lens a leaf."""
    L0 = torch.tensor(lens_values(cam))
    D, J, gt, gl = [], [], [], []
    for p, w, g in zip(torch.tensor(np.asarray(t, np.float64)), torch.tensor(np.asarray(dJ, np.float64)),
                       torch.tensor(np.asarray(duv, np.float64))):
        n = (p[:2] / p[2])[None]
        D.append(torch.func.jacrev(lambda q: distort(q[None], cam)[0])(n[0]))
        J.append(torch.func.jacrev(lambda q: project(q[None], cam)[0])(p))

        def phi(q, L):
            jac = torch.func.jacrev(lambda s: project(s[None], _cam_of(L))[0])(q)
            return (jac * w).sum() + (project(q[None], _cam_of(L))[0] * g).sum()

        a, b = torch.func.grad(phi, argnums=(0, 1))(p, L0)
        gt.append(a)
        gl.append(b)
    return tuple(torch.stack(x).numpy() for x in (D, J, gt, gl))


def kept(t, cam):
    """(k,) bool: k_project's cull of the view-space positions t (float64 for the fp32 kernel: callers allow for rows at a
    rounding boundary)."""
    t = np.asarray(t, np.float64)
    g = geo(t, cam)
    with np.errstate(invalid="ignore"):
        return (t[:, 2] > 0.2) & (g["r2"] <= tan2_bound(cam_tuple(cam)[5])) & (g["det"] > 0)


def radial_increasing(k1, k2, max_theta, samples=200001):
    """The setter's rule by a dense scan: d(r R(r^2)) / dr = 1 + 3 k1 u + 5 k2 u^2 > 0 at every sample u of [0, tan^2 max_theta]."""
    u = np.linspace(0.0, math.tan(max_theta) ** 2, samples)
    return bool(np.all(1.0 + u * (3.0 * k1 + u * (5.0 * k2)) > 0.0))


# ---------------------------------------------------------------------------------------------------------------------
# the float64 frame with camera and lens leaves
# ---------------------------------------------------------------------------------------------------------------------
def leaves(u, cam):
    """The float64 leaves of an OpenCV frame's camera: grad_ref.camera_leaves(u) and the lens (8,)."""
    cl = grad_ref.camera_leaves(u)
    cl["lens"] = torch.tensor(lens_values(cam)).requires_grad_()
    return cl


def view_positions(v, V):
    ph = torch.cat([v[:, 0:3], torch.ones_like(v[:, :1])], 1)
    return (ph @ V.T)[:, :3]


def pre(cl, antialiased=False):
    """A depth_ref-style preprocess (v, u, _) -> (uv, conic, op, colour, red, f = z) through the leaves cl (leaves())."""
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
        t = view_positions(v, V)
        lens = _cam_of(cl["lens"])
        with torch.enable_grad():
            tg = t if t.requires_grad else t.detach().requires_grad_()
            uv = project(tg, lens)
            J = torch.stack([torch.autograd.grad(uv[:, a].sum(), tg, create_graph=True)[0] for a in range(2)], 1)
        T = J @ V[:3, :3]
        cov = T @ Sigma @ T.transpose(1, 2)
        a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
        det = a * c - b * b
        conic = torch.stack([c / det, -b / det, a / det], -1)
        if antialiased:
            import aa_ref

            op = op * aa_ref.compensation(conic)
        return uv, conic, op, col, red, tg[:, 2]

    return fn


def reference(vertices, u, cam, frame, grad_image=None, grad_da=None, features=None, grad_fm=None, antialiased=False):
    """The float64 frame of `frame`'s lists ({"vals", "ranges"}) through the lens cam: "image" (H, W, 3), "depth_alpha"
    (H, W, 2) (D with f = z, and A) and, with an upstream
    gradient -- grad_image (H, W, >= 3), grad_da (H, W, 2) or, with features (n, C), grad_fm (H, W, C) -- dL/dvertices
    "grad" (n, 60), "grad_ubo" (40,) (zero outside LIVE_UBO), "grad_lens" (8,), "exclude" (n,) as in depth_ref and, with
    features, "grad_features" (n, C)."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    cl = leaves(u, cam)
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=True)
    fn = pre(cl, antialiased)
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
    gu[U_CAMPOS:U_CAMPOS + 4] = cl["camera_position"].grad.numpy()
    gu[U_VIEW:U_VIEW + 16] = cl["view_mat"].grad.numpy()
    gu[~LIVE_UBO] = 0.0
    out.update(grad=grad, grad_ubo=gu, grad_lens=cl["lens"].grad.numpy(), exclude=exclude)
    if features is not None:
        gf = np.zeros((n, F.shape[1]))
        gf[used] = feat.grad.numpy()
        out["grad_features"] = gf
    return out


def aabb(vertices, u, cam):
    """The tile AABB (x0, y0, x1, y1) (n, 4) of every Gaussian k_project keeps under the lens, zeros for culled ones, from the
    float64 conic and uv (preprocess.comp:146-164 with the lens's uv and cov2d).  A bound can differ from the fp32 kernel's
    at a rounding boundary, which callers allow for.  Kept rows with a non-finite radius or centre are -1."""
    v = torch.tensor(np.asarray(vertices, np.float64).reshape(-1, 60))
    cl = leaves(u, cam)
    with torch.no_grad():
        t = view_positions(v, cl["view_mat"].detach().reshape(4, 4).T)
        keep = kept(t.numpy(), cam)
    uv, conic, _, _, _, _ = pre(cl)(v, u)
    uv, conic = uv.detach(), conic.detach()
    A, B, C = conic[:, 0], conic[:, 1], conic[:, 2]
    det_c = A * C - B * B
    a, c = C / det_c, A / det_c
    det = a * c - (B / det_c) ** 2
    mid = 0.5 * (a + c)
    sq = torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    rad = torch.ceil(3 * torch.sqrt(torch.maximum(mid + sq, mid - sq)))
    tx, ty = (u.width + 15) // 16, (u.height + 15) // 16
    box = torch.stack([torch.clamp(torch.trunc((uv[:, 0] - rad) / 16), 0, tx), torch.clamp(torch.trunc((uv[:, 1] - rad) / 16), 0, ty),
                       torch.clamp(torch.trunc((uv[:, 0] + rad + 15) / 16), 0, tx), torch.clamp(torch.trunc((uv[:, 1] + rad + 15) / 16), 0, ty)], 1)
    finite = torch.isfinite(box).all(1).numpy()
    box = torch.where(torch.isfinite(box), box, torch.zeros_like(box)).numpy().astype(np.int64)
    box[~keep | ((box[:, 2] - box[:, 0]) * (box[:, 3] - box[:, 1]) == 0)] = 0
    box[keep & ~finite] = -1
    return box


def step_pixels(vertices, u, cam, frame, antialiased=False, rel=1e-3):
    """(H, W) bool: the pixels where the float64 restatement lies within `rel` of one of the blend's step functions (as
    lens_ref.step_pixels), which get no upstream gradient in the camera comparisons."""
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
