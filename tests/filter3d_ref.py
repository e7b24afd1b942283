"""References of Mip-Splatting's 3D smoothing filter (DESIGN.md section 18): gsb_filter3d_variance restated op for op in
numpy fp32; Mip-Splatting's own compute_3D_filter restated in float64 from the camera poses; and the float64 filtered
activation, its chain rule and the filtered Adam step built on tests/adam_ref.py.  Test infrastructure only."""
import math

import numpy as np
import torch

import adam_ref

F = np.float32


def depth_f32(xyz, cameras):
    """(d, seen): the least view depth over the cameras that see each point and whether any does, in fp32 with the
    frame's arithmetic: clip_view (gsb_geom.cuh) and ndc2Pix, seen iff vz > 0.2f and u, v within [-0.15 W, 1.15 W]."""
    p = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    d = np.full(p.shape[0], np.inf, F)
    seen = np.zeros(p.shape[0], bool)
    with np.errstate(all="ignore"):
        for u in cameras:
            pm, vm = np.array(u.proj_mat, F), np.array(u.view_mat, F)
            hx = ((pm[0] * px + pm[4] * py) + pm[8] * pz) + pm[12]
            hy = ((pm[1] * px + pm[5] * py) + pm[9] * pz) + pm[13]
            hw = ((pm[3] * px + pm[7] * py) + pm[11] * pz) + pm[15]
            p_w = F(1) / hw
            ndcx, ndcy = hx * p_w, hy * p_w
            vz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14]
            W, H = F(u.width), F(u.height)
            x = ((ndcx + F(1)) * W - F(1)) * F(0.5)
            y = ((ndcy + F(1)) * H - F(1)) * F(0.5)
            ok = (vz > F(0.2)) & (x >= F(-0.15) * W) & (x <= F(1.15) * W) & (y >= F(-0.15) * H) & (y <= F(1.15) * H)
            d = np.where(ok, np.minimum(d, vz), d)
            seen |= ok
    return d, seen


def focal_f32(cameras):
    """The largest focal_x = (float)W / (2.0f tan_fovx) of the cameras, as jacobian() computes it."""
    return max(F(u.width) / (F(2) * F(u.tan_fovx)) for u in cameras)


def variance_f32(xyz, cameras):
    """gsb_filter3d_variance in numpy fp32: unseen rows take the largest seen d; t = d / f, (t t) 0.2f; all 0 if none seen."""
    d, seen = depth_f32(xyz, cameras)
    if not seen.any():
        return np.zeros(d.shape[0], F)
    d = np.where(seen, d, d[seen].max())
    t = d / focal_f32(cameras)
    return (t * t) * F(0.2)


def _rotation(q):
    """glm's mat4_cast of q = (w, x, y, z) as given: the camera's axes as columns, float64."""
    w, x, y, z = (float(c) for c in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _camera_points(xyz, pose):
    """(x, y, z, fx, fy, W, H) of the points in a pose (pos, quat wxyz, fov_deg, W, H): camera coordinates with z the view
    depth (this renderer's view_mat: rows y and z of the GL view negated), and the focal lengths in pixels."""
    pos, q, fov, W, H = pose
    c = (np.asarray(xyz, np.float64) - np.asarray(pos, np.float64)) @ _rotation(np.asarray(q, np.float32))
    tan_x = math.tan(math.radians(float(np.float32(fov))) / 2)
    tan_y = tan_x * H / W
    return c[:, 0], -c[:, 1], -c[:, 2], W / (2 * tan_x), H / (2 * tan_y), W, H


def variance_mip64(xyz, poses):
    """Mip-Splatting's compute_3D_filter in float64, from the poses: xyz_cam = R^T (p - T), seen iff z > 0.2 and the pixel
    x / z f_x + W / 2 (minus this renderer's half pixel) is within [-0.15 W, 1.15 W], likewise y; filter_3D = d / f sqrt(0.2),
    returned squared (the variance)."""
    n = np.asarray(xyz).shape[0]
    distance = np.full(n, np.inf)
    valid_points = np.zeros(n, bool)
    focal = 0.0
    with np.errstate(all="ignore"):
        for pose in poses:
            x, y, z, fx, fy, W, H = _camera_points(xyz, pose)
            u, v = x / z * fx + W / 2.0 - 0.5, y / z * fy + H / 2.0 - 0.5
            valid = (z > 0.2) & (u >= -0.15 * W) & (u <= W * 1.15) & (v >= -0.15 * H) & (v <= H * 1.15)
            distance[valid] = np.minimum(distance[valid], z[valid])
            valid_points |= valid
            focal = max(focal, fx)
    if not valid_points.any():
        return np.zeros(n)
    distance[~valid_points] = distance[valid_points].max()
    return (distance / focal * math.sqrt(0.2)) ** 2


def borderline(xyz, poses, px=1.0, dz=1e-4):
    """Points within `px` pixels of a camera's 15 % margins or within dz of vz = 0.2, where the half-pixel convention
    and fp32 rounding may flip "seen"."""
    out = np.zeros(np.asarray(xyz).shape[0], bool)
    with np.errstate(all="ignore"):
        for pose in poses:
            x, y, z, fx, fy, W, H = _camera_points(xyz, pose)
            u, v = x / z * fx + W / 2.0 - 0.5, y / z * fy + H / 2.0 - 0.5
            out |= np.abs(z - 0.2) < dz
            front = z > 0.2 - dz
            for val, size in ((u, W), (v, H)):
                out |= front & ((np.abs(val + 0.15 * size) < px) | (np.abs(val - 1.15 * size) < px))
    return out


# ---- the filtered activation and Adam step (float64) ----

def _f64(a):
    return torch.as_tensor(a).to(torch.float64)


def _filter_terms(params, variance):
    p, v = _f64(params), _f64(variance).reshape(-1, 1)
    s = p[:, 4:7].exp()
    q = s * s
    d = q + v
    e = d.sqrt()
    r = q / d
    c = ((r[:, 0] * r[:, 1]) * r[:, 2]).sqrt()
    o = torch.sigmoid(p[:, 7])
    return s, d, e, c, o, o * c, v


def activate(params, variance):
    """The filtered activated records: adam_ref.activate with scale e = sqrt(s^2 + v) and opacity o c."""
    out = adam_ref.activate(params)
    _, _, e, _, _, of, _ = _filter_terms(params, variance)
    out[:, 4:7] = e
    out[:, 7] = of
    return out


def chain(params, grad_vertices, variance):
    """dL/d(raw parameters) through the filtered activation, v held constant: d log s = (g s)(s / e) + (g_w o c)(v / d),
    d logit = ((g_w c) o)(1 - o); the other columns as adam_ref.chain."""
    g = _f64(grad_vertices)
    out = adam_ref.chain(params, g)
    s, d, e, c, o, of, v = _filter_terms(params, variance)
    out[:, 4:7] = (g[:, 4:7] * s) * (s / e) + (g[:, 7:8] * of[:, None]) * (v / d)
    out[:, 7] = ((g[:, 7] * c) * o) * (1 - o)
    return out


def step(params, exp_avg, exp_avg_sq, grad_vertices, cfg, variance, rows=None):
    """One gsb_adam_step_filter3d with gsb_adam_config `cfg`: (params, exp_avg, exp_avg_sq, vertices), float64."""
    P, M, V = adam_ref.adam_update(params, exp_avg, exp_avg_sq, chain(params, grad_vertices, variance), list(cfg.lr), cfg.beta1,
                                   cfg.beta2, cfg.eps, cfg.bias_correction1, cfg.bias_correction2_sqrt, rows)
    return P, M, V, activate(P, variance)


# ---- the footprint bound ----

def footprint_slack(conic, depth, d, f, u):
    """lambda_min of the undilated 2D covariance (the inverse of the fp32 conic (a, b, c) minus 0.3 I) minus the filter's
    bound 0.2 (min(f_x, f_y) d / (f vz))^2, and lambda_max for a tolerance, in float64.  conic: (m, 3), depth: vz (m,),
    d: each row's filter depth (m,), f: the filter's focal length, u: the camera."""
    a, b, c = (np.asarray(conic, np.float64)[:, k] for k in range(3))
    det = a * c - b * b
    m00, m01, m11 = c / det - 0.3, -b / det, a / det - 0.3
    mid = 0.5 * (m00 + m11)
    rad = np.sqrt(np.maximum(0.0, 0.25 * (m00 - m11) ** 2 + m01 * m01))
    fx = u.width / (2.0 * float(u.tan_fovx))
    fy = u.height / (2.0 * float(u.tan_fovy))
    bound = 0.2 * (min(fx, fy) * np.asarray(d, np.float64) / (float(f) * np.asarray(depth, np.float64))) ** 2
    return mid - rad - bound, mid + rad, bound
