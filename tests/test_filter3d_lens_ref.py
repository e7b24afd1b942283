"""tests/filter3d_lens_ref.py on the CPU: the float64 restatement of gsb_filter3d_variance_lens takes sigma_min from the lens
Jacobians that autograd gives, the stable lambda_min keeps its digits where the textbook form loses them, the fp32 model in
the kernel's order agrees with float64 within a stated ulp bound, and the filter combines cameras by an exact min: it does
not depend on their order, a union of camera sets is the min of their filters, and all-pinhole cameras of one focal give
gsb_filter3d_variance's words."""
import math

import numpy as np
import pytest
import torch

import filter3d_lens_ref as lr
import filter3d_ref as fr
import fisheye_ref
import opencv_ref
import scenes
from test_filter3d_ref import cloud, look_at_poses, uniforms

F = np.float32
PHONE = (-0.12, 0.03, 0.0008, -0.0006)  # a phone main camera calibrated as OPENCV
# The fp32 model against the float64 definition, on rows that avoid every margin and cull (filter3d_lens_ref.borderline):
# PINHOLE and OPENCV words differ only by fp32 rounding, FISHEYE ones also by numpy's atan2.  The largest part is the frame's
# own fp32 view-space position, which cancels for a Gaussian close to a camera far from the origin (25 ulp measured).
F32_ULPS = 32


def lens_for(gs, u, name):
    """A lens for the UBO u's frame: "phone" (OpenCV, fx != fy, off-centre principal point), "fish180" and "fish200" (an
    equidistant-like fisheye whose 90 or 100 deg rim touches the shorter frame edge, fx != fy, off-centre)."""
    fx = u.width / (2.0 * float(u.tan_fovx))
    cx, cy = u.width / 2.0 - 0.5, u.height / 2.0 - 0.5
    if name == "phone":
        return gs.opencv_camera(fx, fx * 1.02, cx + 3.25, cy - 2.5, PHONE)
    if name == "pinhole":
        return gs.CameraModel()
    rim = math.radians(90.0 if name == "fish180" else 100.0)
    f = min(u.width, u.height) / 2.0 / rim
    return gs.fisheye_camera(f, f * 0.98, cx + 1.5, cy - 0.75, (0.02, -0.004, 0.0, 0.0), rim)


def _views(gs, k, seed, names):
    cams = uniforms(gs, look_at_poses(k, seed=seed))
    return cams, [lens_for(gs, u, names[i % len(names)]) for i, u in enumerate(cams)]


def _sigma_autograd(t, J_fn):
    return np.array([np.linalg.svd(J_fn(p))[1][-1] for p in t])


def _opencv_J(cam):
    def J(p):
        tp = torch.tensor(p, dtype=torch.float64)
        return torch.func.jacrev(lambda q: opencv_ref.project(q[None], cam)[0])(tp).numpy()
    return J


def _fisheye_J(cam):
    return lambda p: fisheye_ref.jacobian_autograd(np.asarray(p)[None], cam)[0]


def _directions(theta, n=7):
    """Unit view-space rays at angle theta off the axis, at n azimuths."""
    phi = np.linspace(0.1, 2 * math.pi + 0.1, n, endpoint=False)
    return np.stack([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.full(n, np.cos(theta))], 1)


def test_sigma_min_matches_autograd_fisheye(gs):
    """On the axis, near max_theta and past 90 deg of a 200 deg lens: 1 / s = sigma_min of autograd's d uv / d t."""
    cam = fisheye_ref.cam_tuple(gs.fisheye_camera(400.0, 390.0, 320.0, 240.0, (0.02, -0.004, 0.001, -0.0002), math.radians(100)))
    rows = [_directions(1e-7) * 3.0, _directions(0.3) * 0.7, _directions(math.radians(60)) * 5.0,
            _directions(math.radians(95)) * 2.0, _directions(math.radians(99.9)) * 40.0]
    t = np.concatenate(rows)
    s = lr.scale_from_gram(fisheye_ref.jacobian(t, cam, np.float64), np.float64)
    want = _sigma_autograd(t, _fisheye_J(cam))
    err = np.abs(1.0 / s - want) / want
    assert float(err.max()) <= 1e-12, float(err.max())
    # the ray spans J's null space: sigma_min is the smaller image-plane rate
    J = fisheye_ref.jacobian(t, cam, np.float64)
    assert float(np.abs(np.einsum("nij,nj->ni", J, t)).max() / np.abs(J).max()) <= 1e-12


def test_sigma_min_matches_autograd_opencv(gs):
    """Random rays, the axis and rows beside a tangential fold (det D small and positive)."""
    cam = opencv_ref.cam_tuple(gs.opencv_camera(500.0, 520.0, 300.0, 200.0, (0.0, 0.0, 0.3, -0.25), math.radians(60)))
    rng = np.random.default_rng(0)
    t = np.concatenate([rng.uniform(-1, 1, (20, 3)) * [1.5, 1.5, 0] + [0, 0, 2.0], [[1e-9, -1e-9, 3.0], [0.0, 0.0, 1.0]]])
    # beside the fold: walk a ray outward until det D reaches 1e-3 of its value on the axis
    fold = []
    for phi in np.linspace(0.2, 6.2, 9):
        d = np.array([math.cos(phi), math.sin(phi)])
        lo, hi = 0.0, math.tan(math.radians(70))
        if opencv_ref.geo(np.array([[*(d * hi), 1.0]]), cam)["det"][0] > 1e-3:
            continue
        for _ in range(200):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if opencv_ref.geo(np.array([[*(d * mid), 1.0]]), cam)["det"][0] > 1e-3 else (lo, mid)
        fold.append([*(d * lo * 2.5), 2.5])
    assert len(fold) >= 3
    t = np.concatenate([t, fold])
    s = lr.scale_from_gram(opencv_ref.jacobian(t, cam, np.float64)[1], np.float64)
    want = _sigma_autograd(t, _opencv_J(cam))
    err = np.abs(1.0 / s - want) / want
    assert float(err.max()) <= 1e-12, float(err.max())
    J = opencv_ref.jacobian(t, cam, np.float64)[1]
    assert float(np.abs(np.einsum("nij,nj->ni", J, t)).max() / np.abs(J).max()) <= 1e-12


def test_stable_lambda_min_keeps_its_digits():
    """A compressed periphery: rows of very different length.  det / lambda_max stays within 8 ulps of the exact
    lambda_min of the fp32 J; (a + c - sqrt(...)) / 2 loses most of its digits."""
    J = np.array([[[3000.0, 0.5, -120.0], [0.25, 2.0, -0.75]]], F)
    exact = np.linalg.eigvalsh(J.astype(np.float64)[0] @ J.astype(np.float64)[0].T)[0]
    stable = lr.scale_from_gram(J, F)[0]
    s_exact = F(1.0 / math.sqrt(exact))
    err = int(lr.ulps(stable, s_exact))
    assert err <= 8, err
    textbook = lr.lambda_min_textbook(J, F)[0]
    rel = abs(float(textbook) - exact) / exact
    print(f"lambda_min {exact:.9g}: stable scale within {err} ulp, textbook relative error {rel:.2e}")
    assert rel > 1e-3


CASES = {  # name: (k, lens names cycled over the cameras)
    "pinhole": (7, ["pinhole"]),
    "phone": (7, ["phone"]),
    "fish180": (7, ["fish180"]),
    "fish200": (7, ["fish200"]),
    "mixed": (65, ["pinhole", "phone", "fish180", "fish200"]),
}


@pytest.mark.parametrize("name", list(CASES))
def test_fp32_model_agrees_with_float64(gs, name):
    k, names = CASES[name]
    cams, models = _views(gs, k, 11, names)
    xyz = cloud(6000, seed=k)
    xyz = xyz[~lr.borderline(xyz, cams, models)]
    _, seen = lr.scales(xyz, cams, models, np.float64)
    assert np.array_equal(seen, lr.scales(xyz, cams, models, F)[1])
    got = lr.variance(xyz, cams, models, F)
    want = lr.variance(xyz, cams, models, np.float64).astype(F)
    worst = int(lr.ulps(got, want).max())
    print(f"{name}: {xyz.shape[0]} rows, {int(seen.sum())} seen, fp32 model within {worst} ulp of float64")
    assert worst <= F32_ULPS
    assert seen.sum() > 200


def test_wide_lens_sees_behind_where_a_pinhole_cannot(gs):
    u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 60.0, 0.1, 1000.0, 640, 480)
    wide = lens_for(gs, u, "fish200")
    ndcx, ndcy, vx, vy, vz = lr._views(np.zeros((1, 3)), u, np.float64)
    # rows at 95 deg off the camera's axis, 3 units away
    t = _directions(math.radians(95), 16) * 3.0
    V = np.array(u.view_mat, np.float64).reshape(4, 4)  # column-major: V[c][r]
    R, tr = V[:3, :3], V[3, :3]
    xyz = (t - tr) @ np.linalg.inv(R)
    _, seen = lr.camera_scale(xyz, u, wide)
    assert seen.all()
    assert not lr.camera_scale(xyz, u, None)[1].any()


def test_order_invariance_and_union(gs):
    cams, models = _views(gs, 40, 5, ["pinhole", "phone", "fish180", "fish200"])
    xyz = cloud(5000, seed=5)
    v = lr.variance(xyz, cams, models)
    perm = np.random.default_rng(1).permutation(len(cams))
    assert np.array_equal(v.view(np.uint32), lr.variance(xyz, [cams[i] for i in perm], [models[i] for i in perm]).view(np.uint32))
    a, b = perm[:17], perm[17:]
    va, sa = lr.variance(xyz, [cams[i] for i in a], [models[i] for i in a]), lr.scales(xyz, [cams[i] for i in a], [models[i] for i in a])[1]
    vb, sb = lr.variance(xyz, [cams[i] for i in b], [models[i] for i in b]), lr.scales(xyz, [cams[i] for i in b], [models[i] for i in b])[1]
    both = sa & sb
    assert both.sum() > 100
    assert np.array_equal(v[both].view(np.uint32), np.minimum(va[both], vb[both]).view(np.uint32))


def common_focal_c1(gs):
    """c1's camera poses at one field of view and frame size (focal_x == focal_y == one value in fp32)."""
    return [gs.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 640, 480) for p, q, *_ in scenes.CAMERAS.values()]


def test_common_focal_pinholes_equal_the_pinhole_filter(gs):
    """min(vz / f) = fl(min vz / f): division by a positive constant is monotone under correct rounding."""
    cams = common_focal_c1(gs)
    assert len({lr.pinhole_focal(u) for u in cams}) == 1
    assert all(F(u.width) / (F(2) * F(u.tan_fovx)) == F(u.height) / (F(2) * F(u.tan_fovy)) for u in cams)
    _, vtx, _ = scenes.c1()
    for xyz in (vtx[:, 0:3], cloud(20_000, seed=2)):
        want = fr.variance_f32(xyz, cams)
        for models in (None, gs.CameraModel()):
            assert np.array_equal(lr.variance(xyz, cams, models).view(np.uint32), want.view(np.uint32))


def test_focals_that_differ_are_combined_per_camera(gs):
    """Mip-Splatting takes the least depth over all cameras and the largest focal over all cameras, separately; the lens
    filter takes the least depth / focal per camera.  With a near wide camera and a far long one they differ: the per-camera
    rule is never larger (f_max >= each f, d_min <= each d)."""
    near = gs.uniforms_from_camera([0, 0, 3], [1, 0, 0, 0], 90.0, 0.1, 1000.0, 640, 480)
    far = gs.uniforms_from_camera([0, 0, 12], [1, 0, 0, 0], 20.0, 0.1, 1000.0, 640, 480)
    xyz = cloud(3000, seed=4, half=0.5)
    old, new = fr.variance_f32(xyz, [near, far]), lr.variance(xyz, [near, far], None)
    _, seen = lr.scales(xyz, [near, far], None)
    assert seen.sum() > 1000
    assert bool((new[seen] >= old[seen]).all()) and bool((new[seen] > old[seen]).any())
