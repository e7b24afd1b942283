"""The backward pass against the float64 references across the range of scales a trained scene spans (tests/scale_scene.py;
tests/test_scale_coverage.py pins which regimes it reaches and that the checks below would see a zero gradient on the
huge rows): Gaussians up to sigma = 1e6 px with the camera inside them, whose cov2d determinant is past the point where
det^2 overflows fp32, sub-pixel Gaussians at the 0.3 dilation floor, needles, and far and near rows.  Every group is
checked per Gaussian against a tolerance taken from its own rows."""
import numpy as np
import pytest

import scale_scene
from backward_util import CAMERA_GROUPS, DEAD, GROUPS, rel
from test_gpu_backward_regimes import PATHS, _backward, _check_density, _check_vertices

pytestmark = pytest.mark.gpu

# Measured on an H100 80GB HBM3 (400 W limit), both cameras, levels and paths: the largest per-Gaussian error / tolerance is
# 0.11 (the tiny rows' rotation), and the largest camera field-group error 2.1e-5.  With det^2 formed in fp32, the huge rows
# past 1.84e19 get zero scale and rotation gradients and the huge camera variant's view_3x3 group is off by 16-100 %.
CAMS = scale_scene.CAMERAS


@pytest.fixture(scope="module")
def case(oracle):
    """scale_scene.backward_case(cam) with the float64 density reference, once per camera."""
    import functools

    import grad_ref

    @functools.lru_cache(maxsize=None)
    def at(cam):
        b = dict(scale_scene.backward_case(cam))
        b["density"] = grad_ref.density_reference(b["vtx"], b["u"], b["frame"], b["g"])
        return b

    return at


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("cam", CAMS)
def test_backward_matches_reference(gs, case, cam, level, path):
    b = case(cam)
    gv, dens, _ = _backward(gs, b["vtx"], b["u"], b["g"], level=level, deterministic=PATHS[path], density=True)
    what = ("scale", cam, level, path)
    # the huge rows' bands of det hold 3-17 rows each
    _check_vertices(gv, b["ref"]["grad"], b["keep"], b["sets"], what, set_atol=True, min_rows=1)
    # the huge rows' scale and rotation gradients run through the reverse of the conic: non-zero wherever the reference is
    huge = np.any([rows for k, rows in b["sets"].items() if k.startswith("huge")], axis=0)
    ref = b["ref"]["grad"]
    for name in ("scale", "rotation"):
        cols = GROUPS[name]
        live = huge & (np.abs(ref[:, cols]).sum(1) > 0)
        assert live.sum() >= 20 and (gv[live][:, cols] != 0).any(1).all(), (what, name)
    _check_density(dens, b["density"], b["keep"], what)
    assert np.array_equal(dens[:, 2], b["density"]["survivor"].astype(np.float64)), what
    assert np.array_equal(dens[:, 3].astype(np.float32).view(np.uint32),
                          b["density"]["radii"].astype(np.float32).view(np.uint32)), what


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("variant", ["all", "huge"])
@pytest.mark.parametrize("cam", CAMS)
def test_camera_gradient_matches_reference(gs, oracle, cam, variant, level, path):
    """On the whole scene, and on its huge rows past det > 9.2e18 alone, where their conic path is most of the sum."""
    b = scale_scene.backward_case(cam, camera_grad=variant)
    assert not b["ref"]["exclude"].any()
    want = np.zeros(40)
    want[gs.UBO_FLOAT_WORDS] = b["ref"]["grad_ubo"]
    _, _, got = _backward(gs, b["vtx"], b["u"], b["g"], level=level, deterministic=PATHS[path], camera=True)
    got = got.astype(np.float64)
    assert np.isfinite(got).all()
    rels = {name: rel(got[idx], want[idx]) for name, idx in CAMERA_GROUPS.items()}
    print((cam, variant, level, path), "camera gradient relative error:", {k: f"{v:.3g}" for k, v in rels.items()})
    for name, r in rels.items():
        assert r <= 1e-3, (cam, variant, level, path, name, r)
    assert not got[DEAD].any()


@pytest.mark.parametrize("cam", CAMS)
def test_deterministic_levels_agree(gs, case, cam):
    """The deterministic path sums each Gaussian's per-instance terms in list order, and level 1 drops only instances that
    contribute nothing: its words equal level 0's."""
    b = case(cam)
    g0, d0, _ = _backward(gs, b["vtx"], b["u"], b["g"], level=0, deterministic=True, density=True)
    g1, d1, _ = _backward(gs, b["vtx"], b["u"], b["g"], level=1, deterministic=True, density=True)
    assert np.array_equal(g0.view(np.uint32), g1.view(np.uint32))
    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32))


@pytest.mark.parametrize("cam", CAMS)
def test_fast_mode_close_to_exact(gs, case, cam):
    b = case(cam)
    ge, de, _ = _backward(gs, b["vtx"], b["u"], b["g"], mode=0, density=True)
    gf, df, _ = _backward(gs, b["vtx"], b["u"], b["g"], mode=1, density=True)
    assert np.isfinite(gf).all() and np.isfinite(df).all()
    gf, ge, df, de = (a.astype(np.float64) for a in (gf, ge, df, de))
    for sname, rows in {"all": b["keep"], **b["sets"]}.items():
        for name, cols in GROUPS.items():
            if np.linalg.norm(ge[rows][:, cols]) > 0:
                err = rel(gf[rows][:, cols], ge[rows][:, cols])
                assert err <= 1e-3, (cam, sname, name, err)
    for c in (0, 1):
        assert rel(df[b["keep"], c], de[b["keep"], c]) <= 1e-3, (cam, c)


@pytest.mark.parametrize("cam", CAMS)
def test_frame_matches_oracle(gs, oracle, cam):
    """The scene's forward frame equals oracle mode 1 bit for bit at levels 0, 1 and 2: the backward tests above
    differentiate the frame the oracle's lists describe."""
    vtx = scale_scene.vertices()[0]
    u = scale_scene.camera(cam)
    oracle.set_exp_mode(1)
    try:
        ref = oracle.render_frame(vtx, oracle.cov3d(vtx), u)["rgba"]
    finally:
        oracle.set_exp_mode(0)
    ctx = gs.Context(0)
    try:
        ctx.upload(vtx)
        for level in (0, 1, 2):
            ctx.set_tile_cull(level)
            img = ctx.render(u, gs.FORMAT_RGBA32F)
            assert np.array_equal(img.view(np.uint32), ref.view(np.uint32)), (cam, level)
    finally:
        ctx.close()
