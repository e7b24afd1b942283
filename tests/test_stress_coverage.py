"""The stress scene of the backward tests (tests/stress_scene.py) reaches every regime of the reverse walk it is there for, so
that a later edit to the scene cannot quietly drop one: measured with the oracle's lists and the float64 reference only."""
import numpy as np
import pytest

import grad_ref
import stress_scene

# camera -> the least each count may be (about half of what the scene gives; the measured values are in the comments)
MIN_COUNTS = {
    # tiles whose walk starts past list position 512 (291), pixels that break past position 256 (71 679), non-excluded
    # Gaussians with a clamped-alpha contributor pair on a live pixel (332), red < 0 (300) and fov-clamped (53) survivors
    # with a gradient
    "c1": {"deep_tiles": 150, "deep_breaks": 35_000, "clamped": 150, "red_below_0": 150, "fov_clamped": 25},
    # (121, 29 540, 157, 167, 182), and partial tiles -- the frame is 333 x 217 -- whose walk starts past 256 (27 of 34)
    "odd_size_near": {"deep_tiles": 60, "deep_breaks": 15_000, "clamped": 80, "red_below_0": 85, "fov_clamped": 90,
                      "deep_partial_tiles": 15},
}


@pytest.mark.parametrize("cam", stress_scene.CAMERAS)
def test_stress_scene_reaches_every_regime(oracle, cam):
    vtx = stress_scene.vertices()
    u = stress_scene.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = np.random.default_rng(7).standard_normal((u.height, u.width, 4)).astype(np.float32)
    g[steps] = 0.0
    ref = grad_ref.reference(vtx, u, frame, g)
    cov = stress_scene.walk_coverage(vtx, u, frame, g)
    keep = ~ref["exclude"]
    has_grad = keep & (np.abs(ref["grad"]).sum(1) > 0)
    survivor = frame["attr"]["color_radii"][:, 3] != 0
    tiles_x, tiles_y = (u.width + 15) // 16, (u.height + 15) // 16
    tile = np.arange(tiles_x * tiles_y)
    partial = ((tile % tiles_x) * 16 + 16 > u.width) | ((tile // tiles_x) * 16 + 16 > u.height)
    counts = {
        "deep_tiles": int((cov["max_last"] > 512).sum()),  # >= 3 batches of 256 (atomic), >= 5 of 128 (deterministic)
        "deep_breaks": int((cov["break_pos"] > 256).sum()),
        "clamped": int((cov["clamped"] & keep).sum()),
        "red_below_0": int((has_grad & survivor & (stress_scene.red(vtx, u) < 0)).sum()),
        "fov_clamped": int((has_grad & survivor & stress_scene.fov_clamped(vtx, u)).sum()),
        "deep_partial_tiles": int((partial & (cov["max_last"] > 256)).sum()),
    }
    live = 1.0 - float(steps.mean())
    print(cam, counts, "live pixels", live)
    for name, least in MIN_COUNTS[cam].items():
        assert counts[name] >= least, (cam, name, counts[name], least)
    assert live >= 0.8, (cam, live)  # the step-probe mask leaves most pixels' gradient in the comparison
