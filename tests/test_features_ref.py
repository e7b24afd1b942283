"""The references of the rendered feature maps (tests/features_ref.py) against the oracle, depth_ref and each other: no GPU."""
import numpy as np
import pytest

import depth_ref
import features_ref
import scenes


def _frame(oracle, vtx, u, mode):
    oracle.set_exp_mode(mode)
    try:
        return oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_colour_and_depth_features_restate_the_frame(oracle, cam):
    """With f the records' colours the fp32 walk gives the oracle's mode-1 image, with f their depth keys depth_ref's D,
    bit for bit."""
    vtx = scenes.c1()[1]
    u = scenes.camera(cam)
    frame, _ = _frame(oracle, vtx, u, 1)
    n = vtx.shape[0]
    rgb = features_ref.blend32(frame, u.width, u.height, features_ref.colours(frame, n))
    assert np.array_equal(rgb.view(np.uint32), np.ascontiguousarray(frame["rgba"][..., :3]).view(np.uint32))
    D = features_ref.blend32(frame, u.width, u.height, features_ref.depth_keys(frame, n))[..., 0]
    assert np.array_equal(D.view(np.uint32), depth_ref.depth_alpha32(frame, u)[..., 0].view(np.uint32))


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_fp32_restatement_is_close_to_float64(oracle, cam):
    """The fp32 map of random colour-like features is within 1e-5 of the float64 reference off the pixels where the frames'
    contributor sets differ (the oracle's step pixels)."""
    vtx = scenes.c1()[1]
    u = scenes.camera(cam)
    F = np.random.default_rng(3).uniform(0, 1, (vtx.shape[0], 5)).astype(np.float32)  # colour-like values
    frame32, steps = _frame(oracle, vtx, u, 1)
    frame64, _ = _frame(oracle, vtx, u, 0)
    f32 = features_ref.blend32(frame32, u.width, u.height, F)
    f64 = features_ref.reference(vtx, u, frame64, F)["values"][..., 3:]
    err = np.abs(f32 - f64)
    assert err[~steps].max() <= 1e-5, err[~steps].max()
    assert np.abs(f64).max() > 0.1


def test_float64_map_and_gradient_are_linear_in_the_features(oracle):
    """F(a f + b h) = a F(f) + b F(h); the feature gradient does not depend on f, and the colour columns do not depend on f."""
    vtx = scenes.c1()[1]
    u = scenes.camera("c1")
    frame, _ = _frame(oracle, vtx, u, 0)
    rng = np.random.default_rng(4)
    f, h = rng.normal(size=(vtx.shape[0], 3)), rng.normal(size=(vtx.shape[0], 3))
    F = lambda x: features_ref.reference(vtx, u, frame, x)["values"]  # noqa: E731
    mix = F(2.0 * f - 0.5 * h)
    assert np.abs(mix[..., 3:] - (2.0 * F(f)[..., 3:] - 0.5 * F(h)[..., 3:])).max() <= 1e-12
    assert np.array_equal(mix[..., :3], F(f)[..., :3])
    g = rng.normal(size=(u.height, u.width, 3))
    a = features_ref.reference(vtx, u, frame, f, grad_fm=g)["grad_features"]
    b = features_ref.reference(vtx, u, frame, h, grad_fm=g)["grad_features"]
    assert np.abs(a - b).max() <= 1e-12 and np.abs(a).max() > 0

