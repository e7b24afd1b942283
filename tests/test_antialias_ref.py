"""The references of the anti-aliased mode (tests/aa_ref.py): the oracle's frame with the compensation and grad_ref's float64
function with it.  CPU only."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import aa_ref
import edge_scene
import grad_ref
import scale_scene
import scenes

EPS = float(np.finfo(np.float32).eps)


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside", "wide"])
def test_stagewise_oracle_without_compensation_is_render_frame(oracle, cam):
    """aa_ref.oracle_frame runs the oracle's own stages; with the compensation off it is oracle.render_frame bit for bit
    (attributes, lists, ranges, image), so the anti-aliased frame differs from the plain one only by its opacities."""
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    cov = oracle.cov3d(vtx)
    for mode in (0, 1):
        oracle.set_exp_mode(mode)
        try:
            ref = oracle.render_frame(vtx, cov, u)
            got = aa_ref.oracle_frame(vtx, cov, u, antialiased=False)
        finally:
            oracle.set_exp_mode(0)
        assert got["m"] == ref["m"] > 0
        for k in ("attr", "tiles", "scan", "keys", "vals", "ranges", "consumed", "rgba"):
            assert got[k].tobytes() == ref[k].tobytes(), (cam, mode, k)
    aa = aa_ref.oracle_frame(vtx, cov, u)
    assert aa["m"] == ref["m"] and aa["keys"].tobytes() == ref["keys"].tobytes()
    surv = ref["attr"]["color_radii"][:, 3] != 0
    op = ref["attr"]["conic_opacity"][:, 3]
    assert np.array_equal(aa["attr"]["conic_opacity"][:, 3], np.where(surv, op * aa["comp"], op))
    assert (aa["comp"][surv] < 1).any() and not np.array_equal(aa["rgba"], ref["rgba"])


def _scene_cases():
    rng = np.random.default_rng(5)
    _, vtx, _ = scenes.c1()
    for k in range(6):  # random orientations looking at the c1 cloud from 0.5 ... 12 away (the nearest from inside it)
        rot = Rotation.random(random_state=rng)
        x, y, z, w = rot.as_quat()
        pos = rot.apply([0.0, 0.0, float(rng.uniform(0.5, 12.0))])
        yield f"c1_random{k}", vtx, scenes.g.uniforms_from_camera(pos, [w, x, y, z], float(rng.uniform(30, 90)),
                                                                   0.1, 1000.0, 400, 300)
    ev = edge_scene.vertices()[0]
    for cam in edge_scene.CAMERAS:
        yield f"edge_{cam}", ev, edge_scene.camera(cam)
    sv = scale_scene.vertices()[0]
    for cam in scale_scene.CAMERAS:
        yield f"scale_{cam}", sv, scale_scene.camera(cam)


@pytest.mark.parametrize("case", list(range(6 + len(edge_scene.CAMERAS) + len(scale_scene.CAMERAS))))
def test_oracle_compensation_within_fp32_bounds(oracle, case):
    """The oracle's comp against sqrt(max(0, det0 / det)) in float64 of the same fp32 cov2d entries: |comp^2 - r| within
    the rounding of the two fp32 determinants, the division and the sqrt; comp <= 1 wherever c00, c11 >= 0 (then
    det >= det0 holds in fp32 too: rounding is monotone)."""
    name, vtx, u = list(_scene_cases())[case]
    cov = oracle.cov3d(vtx)
    frame = aa_ref.oracle_frame(vtx, cov, u)
    surv = frame["attr"]["color_radii"][:, 3] != 0
    assert surv.sum() > 10, name
    c00, c01, c10, c11, _ = (x[surv] for x in aa_ref.cov2d_f32(vtx, cov, u))
    comp = frame["comp"][surv].astype(np.float64)
    d00, d01, d10, d11 = (x.astype(np.float64) for x in (c00, c01, c10, c11))
    det0 = d00 * d11 - d10 * d01
    det = (d00 + np.float64(np.float32(0.3))) * (d11 + np.float64(np.float32(0.3))) - d10 * d01
    r = np.maximum(0.0, det0 / det)
    m00, m11 = d00 + 0.3, d11 + 0.3
    bound = 4 * EPS * ((np.abs(d00 * d11) + np.abs(d10 * d01)) / det
                       + r * ((np.abs(m00 * m11) + np.abs(d10 * d01)) / det + 2)) + 1e-30
    err = np.abs(comp * comp - r)
    assert (err <= bound).all(), (name, float((err / bound).max()))
    pos_diag = (c00 >= 0) & (c11 >= 0)
    assert (comp[pos_diag] <= 1).all(), name
    assert np.isfinite(comp).all()


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_aa_reference_image_matches_oracle(oracle, cam):
    """grad_ref with the compensation (aa_ref.reference) renders the anti-aliased oracle's image (libm exp) within 1e-4,
    away from the pixels whose step functions sit on their thresholds."""
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = aa_ref.oracle_frame_probed(vtx, oracle.cov3d(vtx), u)
    assert frame["m"] > 0 and steps.mean() < 0.05
    ref = aa_ref.reference(vtx, u, frame)["image"]
    err = np.abs(ref - frame["rgba"][..., :3].astype(np.float64)).max(-1)
    assert err[~steps].max() <= 1e-4, (cam, float(err[~steps].max()))
    plain = grad_ref.reference(vtx, u, frame)["image"]
    assert np.abs(plain - ref).max() > 1e-2  # the compensation is visible


def _gradcheck_rows():
    """Twelve c1 survivors well inside every branch: comp in (0.05, 0.95), red away from its clamp, t/t.z inside the clamp."""
    _, vtx, _ = scenes.c1()
    u = scenes.camera("c1")
    v = torch.from_numpy(vtx.astype(np.float64))
    with torch.no_grad():
        uv, conic, op, col, red = grad_ref.preprocess(v, u)
        comp = aa_ref.compensation(conic)
    ok = (comp > 0.05) & (comp < 0.95) & (red.abs() > 0.05) & (uv[:, 0] > 0) & (uv[:, 0] < 640) & (uv[:, 1] > 0) & (uv[:, 1] < 480)
    rows = torch.nonzero(ok).ravel()[:12]
    assert rows.numel() == 12
    return v[rows].clone(), u


def test_gradcheck_preprocess_vertices():
    v, u = _gradcheck_rows()
    leaf = v.clone().requires_grad_()

    def f(x):
        return aa_ref.preprocess(x, u)[2]  # the compensated opacity: every other output is grad_ref's, checked there

    assert torch.autograd.gradcheck(f, (leaf,), eps=1e-7, atol=1e-6, rtol=1e-5)


def test_gradcheck_preprocess_camera():
    v, u = _gradcheck_rows()
    cam = grad_ref.camera_leaves(u)
    names = list(cam)

    def f(*leaves):
        return aa_ref.preprocess(v, u, dict(zip(names, leaves)))[2]

    assert torch.autograd.gradcheck(f, tuple(cam.values()), eps=1e-7, atol=1e-6, rtol=1e-5)


def test_compensation_gradient_is_zero_where_comp_is_zero():
    conic = torch.tensor([[1 / 0.3, 0.0, 1.0], [4.0, 0.0, 1.0], [1.0, 0.2, 1.0]], dtype=torch.float64, requires_grad=True)
    comp = aa_ref.compensation(conic)
    comp.sum().backward()
    assert comp[0] == 0 and comp[1] == 0 and comp[2] > 0
    assert (conic.grad[:2] == 0).all() and torch.isfinite(conic.grad).all()


def test_isotropic_energy_is_preserved():
    """For an isotropic cov2d of sigma 0.05 ... 2 px: opacity comp sqrt(det(S + 0.3 I)) = opacity sqrt(det S), the
    integrated weight of the undilated Gaussian -- in fp32 (the product's op order) within a few ulp, and in float64."""
    sigma = np.geomspace(0.05, 2.0, 200)
    var = (sigma * sigma).astype(np.float32)
    zero = np.zeros_like(var)
    op = np.float32(0.8)
    comp, _, det = aa_ref.compensation_f32(var, zero, zero, var)
    lhs = np.float64(op) * comp.astype(np.float64) * np.sqrt(det.astype(np.float64))
    rhs = np.float64(op) * var.astype(np.float64)
    assert np.abs(lhs / rhs - 1).max() <= 8 * EPS
    v64 = sigma * sigma
    conic = torch.tensor(np.stack([1 / (v64 + 0.3), 0 * v64, 1 / (v64 + 0.3)], 1))
    c64 = aa_ref.compensation(conic).numpy()
    assert np.abs(c64 * (v64 + 0.3) / v64 - 1).max() <= 1e-12


def zoom_case(oracle, antialiased, n=200_000, W=640, H=480):
    """Many sub-pixel Gaussians (sigma about 0.2-0.7 px at W x H, a quarter of that at W/4 x H/4): (the W/4 x H/4 frame,
    the 4 x 4 box average of the W x H frame).  Low-res pixel X samples the full-res position 4X + 1.5, the centre of
    its box."""
    p = oracle.synth_params(half_extent=(2.0, 1.5, 1.0), log_scale_min=float(np.log(0.0015)),
                            log_scale_max=float(np.log(0.0045)), opacity_min=-3.0, opacity_max=1.0)
    vtx = oracle.load_records(oracle.synth_records(7, n, p))
    cov = oracle.cov3d(vtx)
    frames = []
    for w, h in ((W, H), (W // 4, H // 4)):
        u = oracle.uniforms_from_camera([0, 0, 6], [1, 0, 0, 0], 45.0, 0.1, 1000.0, w, h)
        frames.append(aa_ref.oracle_frame(vtx, cov, u, antialiased=antialiased)["rgba"][..., :3].astype(np.float64))
    box = frames[0].reshape(H // 4, 4, W // 4, 4, 3).mean((1, 3))
    return frames[1], box


def test_zoom_out_is_closer_to_the_box_average(oracle):
    """Rendered at a quarter of the resolution, a scene of sub-pixel Gaussians drawn without compensation gains weight
    (each splat grows to the 0.3 px^2 floor at full opacity); with it, the small frame stays near the box average of the
    large one.  The two mean L1 distances are recorded in DESIGN.md section 14."""
    oracle.set_exp_mode(0)
    d = {}
    for aa in (False, True):
        small, box = zoom_case(oracle, aa)
        d[aa] = float(np.abs(small - box).mean())
    print(f"zoom-out mean L1: plain {d[False]:.5f}, antialiased {d[True]:.5f}")
    assert d[True] < 0.5 * d[False], d
