"""The OpenCV lens's closed forms (tests/opencv_ref.py, the kernels' formulas) against autograd of the float64 map, gradcheck of
the float64 frame, the translation identity, the fp32 model of the kernels' arithmetic, the setter's monotonicity rule and the
COLMAP constructors.  CPU only."""
import math

import numpy as np
import pytest
import torch

import opencv_ref
import scenes
from backward_util import translation_identity

LENSES = {  # (k1, k2, p1, p2)
    "k0": (0.0, 0.0, 0.0, 0.0),
    "barrel": (-0.28, 0.07, 0.0, 0.0),
    "pincushion": (0.12, 0.03, 0.0, 0.0),
    "tangential": (-0.1, 0.02, 0.004, -0.006),
}
# |p1|, |p2| large enough that det D reaches 0 inside max_theta: the cull's tangential fold
FOLD = (0.0, 0.0, 0.3, -0.25)


def _cam(k, fx=480.0, fy=510.0, cx=321.3, cy=238.7, max_theta=math.radians(50.0)):
    return (fx, fy, cx, cy, list(k), max_theta)


def _points(cam, n, seed, axis=False):
    """n view-space points with r <= tan(max_theta) at depths in [0.5, 6], and the on-axis point when `axis`."""
    rng = np.random.default_rng(seed)
    tmax = math.tan(cam[5])
    rr = tmax * np.sqrt(rng.uniform(0, 1, n))
    ang = rng.uniform(0, 2 * np.pi, n)
    z = rng.uniform(0.5, 6.0, n)
    t = np.stack([rr * np.cos(ang) * z, rr * np.sin(ang) * z, z], 1)
    if axis:
        t = np.concatenate([t, [[0.0, 0.0, 2.0]]])
    return t


def _upstream(n, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, 2, 3)), rng.standard_normal((n, 2))


def _check_closed_form(t, cam):
    dJ, duv = _upstream(t.shape[0], 5)
    D, J = opencv_ref.jacobian(t, cam)
    gt = opencv_ref.grad_t(t, cam, dJ, duv)
    gl = opencv_ref.lens_grad(t, cam, dJ, duv)
    aD, aJ, agt, agl = opencv_ref.autograd(t, cam, dJ, duv)
    for got, want, what in ((D, aD, "D"), (J, aJ, "J"), (gt, agt, "dL/dt"), (gl, agl, "dL/dlens")):
        err = np.abs(got - want).max() / max(1.0, np.abs(want).max())
        assert err <= 1e-12, (what, err)


@pytest.mark.parametrize("name", sorted(LENSES))
def test_closed_form_matches_autograd(name):
    cam = _cam(LENSES[name])
    _check_closed_form(_points(cam, 64, 1, axis=True), cam)


def test_closed_form_on_axis():
    cam = _cam(LENSES["tangential"])
    t = np.array([[0.0, 0.0, 0.3], [0.0, 0.0, 5.0], [1e-9, -1e-9, 1.0]])
    _check_closed_form(t, cam)
    D, _ = opencv_ref.jacobian(t[:1], cam)
    k1, k2, p1, p2 = LENSES["tangential"]
    assert np.allclose(D[0], [[1.0, 0.0], [0.0, 1.0]])  # D = I at the axis for any k: r2 = 0, xn = yn = 0


def test_closed_form_near_the_tangential_fold():
    cam = _cam(FOLD, max_theta=math.radians(60.0))
    t = _points(cam, 20000, 3)
    det = opencv_ref.geo(t, cam)["det"]
    assert (det < 0).any() and (det > 0).any()  # the fold lies inside the disc
    near = t[np.argsort(np.abs(det))[:32]]  # the points closest to det D = 0
    assert np.abs(opencv_ref.geo(near, cam)["det"]).max() < 0.01
    _check_closed_form(near, cam)
    assert not opencv_ref.kept(t, cam)[det <= 0].any()


def test_fp32_model_within_ulps():
    """The kernels' formulas in fp32 against the same formulas in float64: the Jacobian within 8 ulps of its largest entry,
    the uv within 4 ulps of the focal length (uv ~ f xd + c), the gradients within 64 ulps of their largest term."""
    for name, k in LENSES.items():
        cam = _cam(k)
        t = _points(cam, 2000, 11, axis=True)
        dJ, duv = _upstream(t.shape[0], 6)
        _, J64 = opencv_ref.jacobian(t, cam)
        _, J32 = opencv_ref.jacobian(t, cam, np.float32)
        scale = np.abs(J64).max((1, 2))
        assert (np.abs(J32 - J64).max((1, 2)) / (scale * 2.0 ** -23)).max() <= 8, name
        g64, g32 = opencv_ref.geo(t, cam), opencv_ref.geo(t, cam, np.float32)
        uv_err = np.abs(cam[0] * g32["xd"].astype(np.float64) - cam[0] * g64["xd"]).max()
        assert uv_err <= 4 * cam[0] * math.tan(cam[5]) * 2.0 ** -23 * 4, name
        for fn in (opencv_ref.grad_t, opencv_ref.lens_grad):
            a = fn(t, cam, dJ, duv)
            b = fn(t, cam, dJ.astype(np.float32), duv.astype(np.float32), np.float32).astype(np.float64)
            s = np.abs(a).max(1) + 1.0
            assert (np.abs(a - b).max(1) / (s * 2.0 ** -23)).max() <= 64, (name, fn.__name__)


def _small_frame():
    """A handful of Gaussians in front of the c1 camera, a 48 x 32 frame and its float64 restatement lists."""
    vtx = scenes.c1(n=24, seed=5)[1]
    u = scenes.camera("c1")
    u.width, u.height = 48, 32
    return vtx, u


def test_gradcheck_vertex_camera_and_lens_leaves():
    vtx, u = _small_frame()
    cam = _cam(LENSES["tangential"], fx=40.0, fy=42.0, cx=23.5, cy=15.5, max_theta=math.radians(60.0))
    cl = opencv_ref.leaves(u, cam)
    v = torch.tensor(vtx.astype(np.float64))
    with torch.no_grad():
        keep = opencv_ref.kept(opencv_ref.view_positions(v, cl["view_mat"].reshape(4, 4).T).numpy(), cam)
    v = v[torch.tensor(keep)][:6].clone().requires_grad_()
    assert v.shape[0] >= 3

    def out(vv, view, campos, lens):
        c = dict(cl, view_mat=view, camera_position=campos, lens=lens)
        uv, conic, op, col, _, f = opencv_ref.pre(c)(vv, u)
        return torch.cat([uv.reshape(-1), conic.reshape(-1), col.reshape(-1), f])

    args = (v, cl["view_mat"].detach().clone().requires_grad_(), cl["camera_position"].detach().clone().requires_grad_(),
            cl["lens"].detach().clone().requires_grad_())
    assert torch.autograd.gradcheck(out, args, eps=1e-6, atol=1e-5, rtol=1e-4)


def test_translation_identity():
    vtx, u = _small_frame()
    cam = _cam(LENSES["barrel"], fx=40.0, fy=42.0, cx=23.5, cy=15.5, max_theta=math.radians(60.0))
    v = np.asarray(vtx, np.float64)
    cl = opencv_ref.leaves(u, cam)
    with torch.no_grad():
        keep = opencv_ref.kept(opencv_ref.view_positions(torch.tensor(v), cl["view_mat"].reshape(4, 4).T).numpy(), cam)
    leaf = torch.tensor(v[keep], requires_grad=True)
    uv, conic, op, col, _, f = opencv_ref.pre(cl)(leaf, u)
    rng = np.random.default_rng(3)
    loss = sum((x * torch.tensor(rng.standard_normal(tuple(x.shape)))).sum() for x in (uv, conic, col, f))
    loss.backward()
    gu = np.zeros(40)
    gu[0:4] = cl["camera_position"].grad.numpy()
    gu[20:36] = cl["view_mat"].grad.numpy()
    grad = leaf.grad.numpy()
    res, scale = translation_identity(grad[:, 0:3].sum(0), np.abs(grad[:, 0:3]).sum(0), u, gu)
    assert (np.abs(res) <= 1e-9 * scale).all(), (res, scale)


@pytest.mark.parametrize("seed", range(4))
def test_setter_rule_against_a_dense_scan(gs, seed):
    """opencv_monotone_limit (the closed form the setter and opencv_camera's default use) against a dense scan of
    1 + 3 k1 u + 5 k2 u^2 > 0, on random coefficients around the edge of the rule."""
    rng = np.random.default_rng(seed)
    for _ in range(200):
        k1, k2 = rng.uniform(-1.5, 1.0), rng.uniform(-0.5, 1.0)
        u0 = gs.opencv_monotone_limit(k1, k2)
        for theta in (0.2, 0.7, 1.2, 1.5):
            inside = math.tan(theta) ** 2 < u0
            if abs(math.tan(theta) ** 2 - u0) > 1e-3 * max(1.0, u0):  # not at the boundary the scan resolves
                assert opencv_ref.radial_increasing(k1, k2, theta) == inside, (k1, k2, theta, u0)
        cam = gs.opencv_camera(500.0, 500.0, 0.0, 0.0, (k1, k2, 0.0, 0.0))
        assert 0.0 < cam.max_theta <= gs.OPENCV_MAX_THETA_CAP + 1e-7
        assert opencv_ref.radial_increasing(k1, k2, cam.max_theta)


def test_camera_from_colmap(gs):
    cases = {
        "SIMPLE_PINHOLE": ([500.0, 320.0, 240.0], (500.0, 500.0, 319.5, 239.5, (0.0, 0.0, 0.0, 0.0))),
        "PINHOLE": ([500.0, 510.0, 320.0, 241.0], (500.0, 510.0, 319.5, 240.5, (0.0, 0.0, 0.0, 0.0))),
        "SIMPLE_RADIAL": ([500.0, 320.0, 240.0, -0.125], (500.0, 500.0, 319.5, 239.5, (-0.125, 0.0, 0.0, 0.0))),
        "RADIAL": ([500.0, 320.0, 240.0, -0.25, 0.0625], (500.0, 500.0, 319.5, 239.5, (-0.25, 0.0625, 0.0, 0.0))),
        "OPENCV": ([500.0, 510.0, 320.0, 240.0, -0.25, 0.0625, 0.001, -0.002],
                   (500.0, 510.0, 319.5, 239.5, (-0.25, 0.0625, 0.001, -0.002))),
    }
    for model, (params, (fx, fy, cx, cy, k)) in cases.items():
        cam = gs.camera_from_colmap(model, params)
        assert cam.kind == gs.CAMERA_OPENCV, model
        assert (cam.fx, cam.fy, cam.cx, cam.cy) == (fx, fy, cx, cy), model
        assert np.array_equal(np.array(list(cam.k), np.float32), np.array(k, np.float32)), model
        assert opencv_ref.radial_increasing(k[0], k[1], cam.max_theta)
        want = gs.opencv_from_colmap(fx, fy, cx + 0.5, cy + 0.5, *k)
        assert bytes(cam) == bytes(want), model
    fish = gs.camera_from_colmap("OPENCV_FISHEYE", [300.0, 301.0, 320.0, 240.0, 0.01, 0.0, 0.0, 0.0])
    assert bytes(fish) == bytes(gs.fisheye_from_colmap(300.0, 301.0, 320.0, 240.0, 0.01, 0.0, 0.0, 0.0))
    assert gs.opencv_camera(1.0, 1.0, 0.0, 0.0).max_theta == np.float32(gs.OPENCV_MAX_THETA_CAP)
    for model in ("FULL_OPENCV", "THIN_PRISM_FISHEYE", "FOV", "RADIAL_FISHEYE", "SIMPLE_RADIAL_FISHEYE", "opencv"):
        with pytest.raises(ValueError):
            gs.camera_from_colmap(model, [1.0] * 12)
    with pytest.raises(ValueError):
        gs.camera_from_colmap("OPENCV", [500.0, 500.0, 320.0, 240.0])
    # lens_camera round trip with a kind
    t = gs.lens_tensor(gs.camera_from_colmap("OPENCV", cases["OPENCV"][0]))
    back = gs.lens_camera(t, 1.0, gs.CAMERA_OPENCV)
    assert back.kind == gs.CAMERA_OPENCV and np.array_equal(np.array(list(back.k), np.float32), t[4:].numpy())
    assert gs.lens_camera(t, 1.0).kind == gs.CAMERA_FISHEYE
    with pytest.raises(ValueError):
        gs.lens_camera(t, 1.0, gs.CAMERA_PINHOLE)
