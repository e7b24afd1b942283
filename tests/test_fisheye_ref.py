"""The fisheye restatement (tests/fisheye_ref.py) against autograd, mpmath and the pinhole oracle; the fp32 model of the
kernel's Jacobian near the axis; gs_b200's lens constructors.  CPU only."""
import math

import mpmath
import numpy as np
import pytest

import fisheye_ref

LENSES = {
    "equidistant": (400.0, 380.0, 319.5, 239.5, [0.0, 0.0, 0.0, 0.0], 3.0),
    "colmap_like": (300.0, 300.0, 320.0, 240.0, [0.03, -0.008, 0.0015, -0.0001], 1.7),
    "barrel": (250.0, 260.0, 300.0, 200.0, [-0.05, 0.004, -0.0002, 0.0], 1.9),
}
THETAS = [1e-8, 1e-6, 1e-4, 1e-3, 1e-2, 0.1, 0.5, 0.99, 1.0, 1.01, 1.5]


def _points(thetas, max_theta, seed=0):
    """View-space points at the angles thetas (<= max_theta) off the axis, random azimuth and distance."""
    rng = np.random.default_rng(seed)
    th = np.array([t for t in thetas if t <= max_theta] + [max_theta], np.float64)
    ph = rng.uniform(0, 2 * np.pi, th.size)
    d = rng.uniform(0.5, 20.0, th.size)
    return np.stack([d * np.sin(th) * np.cos(ph), d * np.sin(th) * np.sin(ph), d * np.cos(th)], 1), th


@pytest.mark.parametrize("lens", sorted(LENSES))
def test_closed_form_jacobian_matches_autograd(lens):
    cam = LENSES[lens]
    t, th = _points(THETAS, cam[5])
    want = fisheye_ref.jacobian_autograd(t, cam)
    got = fisheye_ref.jacobian(t, cam)
    scale = np.abs(want).max((1, 2), keepdims=True)
    assert (np.abs(got - want) <= 1e-12 * scale).all(), np.abs(got - want).max()
    # the direct form of c is the same function where it does not cancel
    far = th >= 0.5
    direct = fisheye_ref.jacobian(t[far], cam, series=False)
    assert (np.abs(direct - want[far]) <= 1e-12 * scale[far]).all()


def _mp_uv_jacobian(p, cam):
    fx, fy, cx, cy, k, _ = cam
    mpmath.mp.dps = 50
    x, y, z = (mpmath.mpf(float(v)) for v in p)

    def uv(x, y, z):
        r = mpmath.sqrt(x * x + y * y)
        th = mpmath.atan2(r, z)
        rho = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
        s = rho / r
        return [fx * s * x + cx, fy * s * y + cy]

    J = [[mpmath.diff(lambda *a: uv(*a)[i], (x, y, z), tuple(int(j == m) for m in range(3))) for j in range(3)]
         for i in range(2)]
    return np.array([float(v) for v in uv(x, y, z)]), np.array([[float(v) for v in row] for row in J])


@pytest.mark.parametrize("lens", ["colmap_like", "barrel"])
def test_restatement_against_mpmath(lens):
    import torch

    cam = LENSES[lens]
    t, _ = _points([1e-8, 1e-4, 1e-2, 0.3, 1.0, 1.4], cam[5], seed=1)
    uv = fisheye_ref.project(torch.tensor(t), cam).numpy()
    J = fisheye_ref.jacobian(t, cam)
    for i, p in enumerate(t):
        muv, mJ = _mp_uv_jacobian(p, cam)
        assert np.allclose(uv[i], muv, rtol=0, atol=1e-10 * np.abs(muv).max())
        assert (np.abs(J[i] - mJ) <= 1e-11 * np.abs(mJ).max()).all(), (i, J[i], mJ)


def test_fp32_jacobian_near_the_axis_is_within_a_few_ulps():
    """For theta <= 1e-3 the kernel's fp32 formulas give J within 8 ulps of its largest entry (each of J's entries is a
    handful of rounded ops on well-conditioned operands); the direct form of c loses its digits there."""
    cam = LENSES["colmap_like"]
    t, th = _points([1e-7, 1e-6, 1e-5, 1e-4, 3e-4, 1e-3], 1e-3, seed=2)
    t32 = t.astype(np.float32).astype(np.float64)  # the exact value at the fp32 inputs
    exact = fisheye_ref.jacobian(t32, cam)
    got = fisheye_ref.jacobian(t32, cam, dtype=np.float32).astype(np.float64)
    ulp = np.spacing(np.abs(exact).max((1, 2)).astype(np.float32)).astype(np.float64)[:, None, None]
    assert (np.abs(got - exact) <= 8 * ulp).all(), (np.abs(got - exact) / ulp).max()
    # c's own error, relative to c's exact value: the direct form is off by far more than an fp32 rounding
    x = t32[:, 0]
    with np.errstate(all="ignore"):
        direct = fisheye_ref.jacobian(t32, cam, dtype=np.float32, series=False).astype(np.float64)
    c_exact = exact[:, 0, 1] / (cam[0] * x * t32[:, 1])
    c_direct = direct[:, 0, 1] / (cam[0] * x * t32[:, 1])
    assert not (np.abs(c_direct - c_exact) <= 1e-3 * np.abs(c_exact)).all()


def test_on_axis_record_matches_the_pinhole_oracle(gs, oracle):
    """k = 0, fx = W / (2 tan_fovx), cx = (W - 1) / 2: for Gaussians with r / z <= 1e-4 the fisheye uv and cov2d differ
    from the pinhole's by O(theta^2) <= 1e-8 relative, less than an fp32 rounding; an fp32 model of k_project's fisheye
    record is within 2 ulps (uv) and 1e-5 relative (conic, through det's cancellation) of the oracle's."""
    W, H = 640, 480
    u = oracle.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, W, H)
    rng = np.random.default_rng(4)
    n = 500
    v = oracle.load_records(oracle.synth_records(3, n))
    z = rng.uniform(2.0, 8.0, n)
    ang = rng.uniform(0, 2 * np.pi, n)
    r = z * rng.uniform(0, 1e-4, n)
    v[:, 0], v[:, 1], v[:, 2] = r * np.cos(ang), r * np.sin(ang), 5.0 - z
    v[:, 4:7] = np.exp(rng.uniform(-4.5, -3.0, (n, 3)))
    attr, _ = oracle.preprocess(v, oracle.cov3d(v), u)
    cam = (W / (2 * u.tan_fovx), H / (2 * u.tan_fovy), (W - 1) / 2, (H - 1) / 2, [0.0] * 4, 3.0)
    uv32, conic32 = fisheye_ref.record32(v, oracle.cov3d(v), u, cam)
    live = attr["color_radii"][:, 3] > 0
    assert live.sum() > 0.9 * n
    ulp = np.spacing(np.abs(attr["uv"][live]).astype(np.float32)).astype(np.float64)
    assert (np.abs(uv32[live] - attr["uv"][live]) <= 2 * ulp).all()
    co = attr["conic_opacity"][live, :3].astype(np.float64)
    assert (np.abs(conic32[live] - co) <= 1e-5 * np.abs(co).max(1, keepdims=True)).all()


def test_fisheye_from_colmap_shifts_half_a_pixel(gs):
    c = gs.fisheye_from_colmap(500.0, 510.0, 640.0, 360.0, 0.1, -0.02, 0.003, -0.0004)
    assert c.kind == gs.CAMERA_FISHEYE
    assert (c.fx, c.fy, c.cx, c.cy) == (500.0, 510.0, 639.5, 359.5)
    assert np.allclose(list(c.k), [0.1, -0.02, 0.003, -0.0004], rtol=1e-6)


def test_default_max_theta(gs):
    assert math.isclose(gs.fisheye_camera(1, 1, 0, 0).max_theta, gs.FISHEYE_MAX_THETA_CAP, rel_tol=1e-3)
    # d theta_d / d theta = 1 - 1.5 t^2 reaches 0 at t = sqrt(2 / 3)
    m = gs.fisheye_camera(1, 1, 0, 0, k=(-0.5, 0, 0, 0)).max_theta
    assert math.sqrt(2 / 3) - 2e-4 <= m < math.sqrt(2 / 3)
    assert gs.fisheye_camera(1, 1, 0, 0, max_theta=0.7).max_theta == pytest.approx(0.7)
