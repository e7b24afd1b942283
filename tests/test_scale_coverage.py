"""The scale scene of the backward tests (tests/scale_scene.py) reaches every regime it is there for, every survivor is
well-posed at fp32 resolution, and the GPU checks would see a backward pass that loses the conic path of the huge rows:
measured with the oracle's fp32 frame and float64 arithmetic only."""
import numpy as np
import pytest
import torch

import grad_ref
import scale_scene
from backward_util import CAMERA_GROUPS, GROUPS, rel
from test_gpu_backward_regimes import RTOL, _atol

# the least each count may be: about half of what the scene gives (measured values in the comments).  det is the oracle's
# fp32 conic's 1 / (A C - B^2).
MIN_COUNTS = {
    # det > 2 x 1.84e19 (13), 9.2e18 < det < 1.84e19 (6), tiny rows whose cov2d is within 1e-6 of 0.3 I (38), axis-aligned
    # needles per ratio (36 each), 45-degree needles per ratio (10 each), view depth >= 100 (200), near rows (10)
    "axis": {"past_cliff": 7, "subnormal": 2, "tiny_floor": 19, "needle_1e+02": 18, "needle_1e+03": 18, "needle_1e+04": 18,
             "needle45_1e+02": 5, "needle45_1e+03": 5, "needle45_1e+04": 5, "far": 100, "near": 5},
    # (8, 5, 131, 36 x 3, 10 x 3, 180, 10)
    "rotated_odd": {"past_cliff": 4, "subnormal": 2, "tiny_floor": 65, "needle_1e+02": 18, "needle_1e+03": 18,
                    "needle_1e+04": 18, "needle45_1e+02": 5, "needle45_1e+03": 5, "needle45_1e+04": 5, "far": 90, "near": 5},
}


def _frame(cam):
    import oracle

    vtx, masks, ratio, n45 = scale_scene.vertices()
    u = scale_scene.camera(cam)
    attr, tiles = oracle.preprocess(vtx, oracle.cov3d(vtx), u)
    return vtx, masks, ratio, n45, u, attr, tiles > 0


def _conics(vtx, u):
    with torch.no_grad():
        return grad_ref.preprocess(torch.from_numpy(vtx.astype(np.float64)), u)[1].numpy()


def coverage(cam):
    vtx, masks, ratio, n45, u, attr, surv = _frame(cam)
    det = scale_scene.frame_det({"attr": attr})
    c = {"past_cliff": int((surv & (det > 2 * scale_scene.DET_CLIFF)).sum()),
         "subnormal": int((surv & (det > scale_scene.DET_SUBNORMAL) & (det < scale_scene.DET_CLIFF)).sum())}
    # cov2d = the inverse of the float64 conic: within 1e-6 of the 0.3 I dilation floor
    k = _conics(vtx, u)
    kd = k[:, 0] * k[:, 2] - k[:, 1] ** 2
    cov = np.stack([k[:, 2] / kd, -k[:, 1] / kd, k[:, 0] / kd], 1)
    floor = np.abs(cov - np.array([0.3, 0.0, 0.3])).max(1) < 1e-6
    c["tiny_floor"] = int((surv & masks["tiny"] & floor).sum())
    for r in scale_scene.NEEDLE_RATIOS:
        c[f"needle_{r:.0e}"] = int((surv & masks["needle"] & (ratio == r) & ~n45).sum())
        c[f"needle45_{r:.0e}"] = int((surv & masks["needle"] & (ratio == r) & n45).sum())
    depth = attr["depth"].astype(np.float64)
    c["far"] = int((surv & masks["far"] & (depth >= 100)).sum())
    c["near"] = int((surv & masks["near"] & (depth > 0.2) & (depth < 0.2 + 1e-5)).sum())
    return c


@pytest.mark.parametrize("cam", scale_scene.CAMERAS)
def test_scale_scene_reaches_every_regime(cam):
    counts = coverage(cam)
    print(cam, counts)
    for name, least in MIN_COUNTS[cam].items():
        assert counts[name] >= least, (cam, name, counts[name], least)


@pytest.mark.parametrize("cam", scale_scene.CAMERAS)
def test_every_survivor_is_well_posed(cam):
    """The oracle's fp32 conic of every survivor is within 1e-6 (relative, as a vector) of the float64 conic, so the float64
    reference judges the backward pass fairly on every row it keeps; and it excludes none."""
    vtx, masks, _, _, u, attr, surv = _frame(cam)
    k64 = _conics(vtx, u)
    k32 = attr["conic_opacity"][:, :3].astype(np.float64)
    err = np.linalg.norm(k32 - k64, axis=1) / np.linalg.norm(k64, axis=1)
    worst = {g: float(err[m & surv].max()) for g, m in masks.items() if (m & surv).any()}
    print(cam, "largest conic relative error per group:", {g: f"{v:.3g}" for g, v in worst.items()})
    assert (err[surv] <= 1e-6).all(), worst
    assert not scale_scene.backward_case(cam)["ref"]["exclude"].any()


@pytest.mark.parametrize("cam", scale_scene.CAMERAS)
def test_zero_conic_path_fails_the_vertex_check(cam):
    """For every huge row past det^2's overflow, the per-Gaussian tolerance of the scale and rotation groups (RTOL of its
    norm plus its det band's own absolute tolerance) lies below the norm of its reference gradient, by a factor of 1.5 at
    least: a backward pass that returns zeros there fails."""
    b = scale_scene.backward_case(cam)
    ref, det = b["ref"]["grad"], scale_scene.frame_det(b["frame"])
    past = 0
    for sname, rows in b["sets"].items():
        if not sname.startswith("huge_past"):
            continue
        assert (det[rows] > scale_scene.DET_CLIFF).all()
        past += int(rows.sum())
        for name in ("scale", "rotation"):
            cols = GROUPS[name]
            r = np.linalg.norm(ref[rows][:, cols], axis=1)
            margin = r / (RTOL * r + _atol(ref, rows, cols))
            print(cam, sname, name, "rows", int(rows.sum()), "smallest norm / tolerance", f"{margin.min():.3g}")
            assert (margin > 1.5).all(), (cam, sname, name, margin)
    assert past >= 6


@pytest.mark.parametrize("cam", scale_scene.CAMERAS)
def test_zero_conic_path_fails_the_camera_check(cam):
    """On the huge camera variant, dropping the conic path of the rows past det^2's overflow moves at least one field group
    of the camera gradient by ten times the 1e-3 the GPU check allows."""
    import gs_b200 as gs

    b = scale_scene.backward_case(cam, camera_grad="huge")
    past = (b["frame"]["attr"]["color_radii"][:, 3] != 0) & (scale_scene.frame_det(b["frame"]) > scale_scene.DET_CLIFF)
    assert past.sum() >= 4
    cut = grad_ref.reference(b["vtx"], b["u"], b["frame"], b["g"], camera=True, cut_conic=past)["grad_ubo"]
    want, got = np.zeros(40), np.zeros(40)
    want[gs.UBO_FLOAT_WORDS], got[gs.UBO_FLOAT_WORDS] = b["ref"]["grad_ubo"], cut
    rels = {name: rel(got[idx], want[idx]) for name, idx in CAMERA_GROUPS.items()}
    print(cam, "camera gradient without the conic path of", int(past.sum()), "rows:", {k: f"{v:.3g}" for k, v in rels.items()})
    assert max(rels.values()) > 1e-2
