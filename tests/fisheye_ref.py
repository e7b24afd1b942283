"""Float64 restatement of the fisheye projection of gsb_set_camera_model (DESIGN.md section 19) and an fp32 numpy model of the
kernel's formulas.  The blend, the tiling and the SH colour are grad_ref's; only the projection is new here.  Test
infrastructure only.

The lens, for the view-space position t = (x, y, z): r = |(x, y)|, d = |t|, theta = atan2(r, z), rho = theta P(theta^2) with
P = 1 + k1 t2 + k2 t2^2 + k3 t2^3 + k4 t2^4, and uv = (fx (rho / r) x + cx, fy (rho / r) y + cy).  A Gaussian is kept when
d > 0.2 and theta <= max_theta.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import grad_ref

# the kernel's switch from S's Taylor series to its direct form (gsb_geom.cuh FISHEYE_SERIES_THETA)
SERIES_THETA = 1.0
# S(t2) = (sin(2 theta) / 2 - theta) / theta^3 = sum_n a_n t2^(n-1), a_n = (-1)^n 4^n / (2n + 1)!.  The kernel sums the first
# KERNEL_TERMS (truncation < 2e-10 relative at theta = 1, below fp32's resolution); the float64 restatement sums 14 (< 1e-30).
S_COEF = [(-1) ** n * 4.0 ** n / math.factorial(2 * n + 1) for n in range(1, 15)]
KERNEL_TERMS = 7


def cam_tuple(cam):
    """(fx, fy, cx, cy, k (4,), max_theta) of a gs_b200.CameraModel or of such a tuple."""
    if isinstance(cam, tuple):
        return cam
    return (float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy), [float(x) for x in cam.k], float(cam.max_theta))


def project(t, cam):
    """uv (k, 2) of the view-space positions t (k, 3), float64 torch, differentiable (the map itself, written with atan2 and
    the polynomial: autograd of this is the reference Jacobian).  r = 0 rows give (cx, cy) through s = 1 / d there."""
    fx, fy, cx, cy, k, _ = cam_tuple(cam)
    x, y, z = t[:, 0], t[:, 1], t[:, 2]
    r = torch.sqrt(x * x + y * y)
    d = torch.sqrt(x * x + y * y + z * z)
    theta = torch.atan2(r, z)
    t2 = theta * theta
    rho = theta * (1 + t2 * (k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3]))))
    s = torch.where(r > 0, rho / torch.where(r > 0, r, torch.ones_like(r)), 1.0 / d)
    return torch.stack([fx * s * x + cx, fy * s * y + cy], -1)


def _series_S(t2, terms):
    coef = [t2.dtype.type(a) for a in S_COEF[:terms]]
    acc = np.zeros_like(t2) + coef[-1]
    for a in coef[-2::-1]:
        acc = a + t2 * acc
    return acc


def jacobian(t, cam, dtype=np.float64, series=True):
    """The closed-form J = d uv / d t (k, 2, 3) of the kernel (gsb_geom.cuh fisheye_geo / fisheye_jacobian), evaluated in
    `dtype` op for op in numpy: float64 for the reference, float32 for the model of the kernel's arithmetic.  series=False
    evaluates c = (rho' cos sin - rho) / r^3 in its direct form for every theta (what the series replaces).  The series
    has the kernel's KERNEL_TERMS terms in float32 and 14 in float64."""
    fx, fy, cx, cy, k, _ = cam_tuple(cam)
    f = dtype
    t = np.asarray(t, f)
    x, y, z = t[:, 0], t[:, 1], t[:, 2]
    k = [f(v) for v in k]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.sqrt(x * x + y * y)
        d = np.sqrt((x * x + y * y) + z * z)
        theta = np.arctan2(r, z).astype(f)
        t2 = theta * theta
        b = np.where(r > 0, theta / r, f(1) / d)
        P1 = k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3]))
        Q1 = f(3) * k[0] + t2 * (f(5) * k[1] + t2 * (f(7) * k[2] + t2 * (f(9) * k[3])))
        if series:
            S_ser = _series_S(t2.astype(f), KERNEL_TERMS if f == np.float32 else len(S_COEF)).astype(f)
            scth_dir = ((r * z) / (d * d)) / theta
            S = np.where(theta < SERIES_THETA, S_ser, (scth_dir - f(1)) / t2)
            scth = np.where(theta < SERIES_THETA, f(1) + t2 * S_ser, scth_dir)
            c = ((S + Q1 * scth) - P1) * ((b * b) * b)
        else:  # c = (rho' cos(theta) sin(theta) - rho) / r^3, cos = z / d, sin = r / d
            rho = theta * (f(1) + t2 * P1)
            c = ((f(1) + t2 * Q1) * ((z / d) * (r / d)) - rho) / ((r * r) * r)
        s = (f(1) + t2 * P1) * b
        e = (f(1) + t2 * Q1) / (d * d)
    xyc = (x * y) * c
    J = np.empty((t.shape[0], 2, 3), f)
    J[:, 0, 0], J[:, 0, 1], J[:, 0, 2] = f(fx) * (s + (x * x) * c), f(fx) * xyc, -f(fx) * (x * e)
    J[:, 1, 0], J[:, 1, 1], J[:, 1, 2] = f(fy) * xyc, f(fy) * (s + (y * y) * c), -f(fy) * (y * e)
    return J


def jacobian_autograd(t, cam):
    """d uv / d t (k, 2, 3) by autograd of project (float64)."""
    tt = torch.tensor(np.asarray(t, np.float64))
    return torch.func.vmap(torch.func.jacrev(lambda p: project(p[None], cam)[0]))(tt).numpy()


def view_positions(v, u):
    """The view-space positions (k, 3) of the vertex rows v (k x 60 float64 torch) under the UBO u."""
    V = grad_ref._mat(u.view_mat)
    ph = torch.cat([v[:, 0:3], torch.ones_like(v[:, :1])], 1)
    return (ph @ V.T)[:, :3]


def preprocess(v, u, cam):
    """grad_ref.preprocess with the fisheye projection: uv (k, 2), conic (k, 3), opacity, colour, unclamped red, and the
    kept mask (k,) of the lens's cull (d > 0.2 and theta <= max_theta).  Sigma and the SH colour are grad_ref's."""
    _, _, _, _, _, max_theta = cam_tuple(cam)
    _, _, op, col, red = grad_ref.preprocess(v, u)  # opacity and colour do not depend on the projection
    s, q = v[:, 4:7], v[:, 8:12]
    qw, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([
        torch.stack([1 - 2 * qy * qy - 2 * qz * qz, 2 * qx * qy + 2 * qz * qw, 2 * qx * qz - 2 * qy * qw], -1),
        torch.stack([2 * qx * qy - 2 * qz * qw, 1 - 2 * qx * qx - 2 * qz * qz, 2 * qy * qz + 2 * qx * qw], -1),
        torch.stack([2 * qx * qz + 2 * qy * qw, 2 * qy * qz - 2 * qx * qw, 1 - 2 * qx * qx - 2 * qy * qy], -1),
    ], -2)
    M = s[:, :, None] * R
    Sigma = M.transpose(1, 2) @ M
    t = view_positions(v, u)
    uv = project(t, cam)
    # J = d uv / d t as a differentiable function of t (its own derivative is J's second derivatives)
    J = torch.func.vmap(torch.func.jacrev(lambda p: project(p[None], cam)[0]))(t)
    W = grad_ref._mat(u.view_mat)[:3, :3]
    T = J @ W
    cov = T @ Sigma @ T.transpose(1, 2)
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a * c - b * b
    conic = torch.stack([c / det, -b / det, a / det], -1)
    with torch.no_grad():
        d = torch.linalg.norm(t, dim=1)
        theta = torch.atan2(torch.linalg.norm(t[:, :2], dim=1), t[:, 2])
        kept = (d > 0.2) & (theta <= max_theta)
    return uv, conic, op, col, red, kept


def reference(vertices, u, cam, frame, grad_image=None):
    """grad_ref.reference for a fisheye frame: the float64 image (H, W, 3) blended with grad_ref's blend over the lists
    `frame` ({"vals", "ranges"}: the GPU frame's own level-0 lists) and, with grad_image, dL/dvertices (n, 60) and `exclude`
    (grad_ref's ill-posed rows)."""
    v_all, used, local = grad_ref.survivors(vertices, frame)
    n = v_all.shape[0]
    W, H = int(u.width), int(u.height)
    want = grad_image is not None
    leaf = torch.tensor(v_all[used].astype(np.float64), requires_grad=want)
    with torch.set_grad_enabled(want):
        uv, conic, op, col, red, _ = preprocess(leaf, u, cam)
    parts = [p.detach().clone().requires_grad_(want) for p in (uv, conic, op, col)]
    image = np.zeros((H, W, 3), np.float64)
    near_clamp = np.zeros(used.size, bool)
    gimg = None if grad_image is None else torch.tensor(np.asarray(grad_image, np.float64)[..., :3])
    for tl in grad_ref.tiles(u, frame, local):
        with torch.set_grad_enabled(want):
            rgb, contrib, raw, _ = grad_ref.blend_tile(*(p[tl.idx] for p in parts), tl.fx, tl.fy)
        image[tl.py, tl.px] = rgb.detach().numpy()
        if want:
            g = gimg[tl.py, tl.px]
            (rgb * g).sum().backward()
            live = (g != 0).any(1)[:, None]
            hit = (contrib & live & ((raw - 0.99).abs() < 1e-4)).any(0).numpy()
            near_clamp[local[tl.ids][hit]] = True
    if not want:
        return {"image": image}
    torch.autograd.backward([uv, conic, op, col], [p.grad if p.grad is not None else torch.zeros_like(p) for p in parts])
    grad = np.zeros((n, 60), np.float64)
    grad[used] = leaf.grad.numpy()
    grad[:, 3] = 0.0
    exclude = np.zeros(n, bool)
    exclude[used] = near_clamp | (red.detach().abs().numpy() < 1e-4)
    return {"image": image, "grad": grad, "exclude": exclude}


def aabb(vertices, u, cam):
    """The tile AABB (x0, y0, x1, y1) (n, 4) of every Gaussian k_project keeps under the lens, zeros for culled ones, from the
    float64 conic and uv (preprocess.comp:146-164 with the fisheye's uv and cov2d).  Float64 against the kernel's fp32: a
    bound can differ at a rounding boundary, which callers allow for.  Rows kept with a non-finite radius or centre are -1:
    there the kernel's saturating float-to-int conversions decide, which this does not restate."""
    v = torch.tensor(np.asarray(vertices, np.float64).reshape(-1, 60))
    with torch.no_grad():
        uv, conic, _, _, _, kept = preprocess(v, u, cam)
    A, B, C = conic[:, 0], conic[:, 1], conic[:, 2]
    det_c = A * C - B * B
    a, c = C / det_c, A / det_c  # cov2d diagonal
    det = a * c - (B / det_c) ** 2
    mid = 0.5 * (a + c)
    lam = torch.maximum(mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1)), mid - torch.sqrt(torch.clamp(mid * mid - det, min=0.1)))
    rad = torch.ceil(3 * torch.sqrt(lam))
    tx, ty = (u.width + 15) // 16, (u.height + 15) // 16
    box = torch.stack([torch.clamp(torch.trunc((uv[:, 0] - rad) / 16), 0, tx), torch.clamp(torch.trunc((uv[:, 1] - rad) / 16), 0, ty),
                       torch.clamp(torch.trunc((uv[:, 0] + rad + 15) / 16), 0, tx), torch.clamp(torch.trunc((uv[:, 1] + rad + 15) / 16), 0, ty)], 1)
    finite = torch.isfinite(box).all(1).numpy()
    box = torch.where(torch.isfinite(box), box, torch.zeros_like(box)).numpy().astype(np.int64)
    box[~kept.numpy() | ((box[:, 2] - box[:, 0]) * (box[:, 3] - box[:, 1]) == 0)] = 0  # k_project stores zeros for culled rows
    box[kept.numpy() & ~finite] = -1  # an infinite float64 radius or centre: the kernel's saturating conversions decide
    return box


def record32(vertices, cov, u, cam):
    """An fp32 numpy model of k_project's fisheye record: uv (n, 2) and conic (n, 3) from the fp32 cov3d words `cov`
    (oracle.cov3d) in the kernel's op order (clip_view's view position, fisheye_geo, fisheye_jacobian, cov2d, the conic)."""
    f = np.float32
    v = np.asarray(vertices, f).reshape(-1, 60)
    vm = np.asarray(list(u.view_mat), f)
    px, py, pz = v[:, 0], v[:, 1], v[:, 2]
    x = ((vm[0] * px + vm[4] * py) + vm[8] * pz) + vm[12]
    y = ((vm[1] * px + vm[5] * py) + vm[9] * pz) + vm[13]
    z = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14]
    fx, fy, cx, cy, k, _ = cam_tuple(cam)
    J = jacobian(np.stack([x, y, z], 1), cam, dtype=f)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.sqrt(x * x + y * y)
        d = np.sqrt((x * x + y * y) + z * z)
        theta = np.arctan2(r, z).astype(f)
        t2 = theta * theta
        b = np.where(r > 0, theta / r, f(1) / d)
        kk = [f(q) for q in k]
        s = (f(1) + t2 * (kk[0] + t2 * (kk[1] + t2 * (kk[2] + t2 * kk[3])))) * b
    uv = np.stack([f(fx) * (s * x) + f(cx), f(fy) * (s * y) + f(cy)], 1)
    T0 = np.stack([(vm[r * 4 + 0] * J[:, 0, 0] + vm[r * 4 + 1] * J[:, 0, 1]) + vm[r * 4 + 2] * J[:, 0, 2] for r in range(3)], 1)
    T1 = np.stack([(vm[r * 4 + 0] * J[:, 1, 0] + vm[r * 4 + 1] * J[:, 1, 1]) + vm[r * 4 + 2] * J[:, 1, 2] for r in range(3)], 1)
    c = np.asarray(cov, f).reshape(-1, 6)
    S = [[c[:, 0], c[:, 1], c[:, 2]], [c[:, 1], c[:, 3], c[:, 4]], [c[:, 2], c[:, 4], c[:, 5]]]
    tm0 = [(T0[:, 0] * S[q][0] + T0[:, 1] * S[q][1]) + T0[:, 2] * S[q][2] for q in range(3)]
    tm1 = [(T1[:, 0] * S[q][0] + T1[:, 1] * S[q][1]) + T1[:, 2] * S[q][2] for q in range(3)]
    m00 = ((tm0[0] * T0[:, 0] + tm0[1] * T0[:, 1]) + tm0[2] * T0[:, 2]) + f(0.3)
    m01 = (tm1[0] * T0[:, 0] + tm1[1] * T0[:, 1]) + tm1[2] * T0[:, 2]
    m10 = (tm0[0] * T1[:, 0] + tm0[1] * T1[:, 1]) + tm0[2] * T1[:, 2]
    m11 = ((tm1[0] * T1[:, 0] + tm1[1] * T1[:, 1]) + tm1[2] * T1[:, 2]) + f(0.3)
    ood = f(1) / (m00 * m11 - m10 * m01)
    conic = np.stack([m11 * ood, -m01 * ood, m00 * ood], 1)
    return uv.astype(np.float64), conic.astype(np.float64)
