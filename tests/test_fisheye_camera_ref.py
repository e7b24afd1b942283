"""The fisheye camera gradient's float64 reference (tests/lens_ref.py): the kernel's closed-form lens derivatives against
autograd of fisheye_ref.project, their fp32 model near the axis, gradcheck of the frame in the view matrix, camera position and
lens, the translation identity, and gs_b200's lens helpers.  CPU only."""
import math

import numpy as np
import pytest
import torch

import lens_ref
from test_fisheye_ref import LENSES, THETAS, _points

# both sides of FISHEYE_SERIES_THETA (1.0) and the axis down to 1e-8
LENS_THETAS = THETAS + [0.999999, 1.000001, 1.2, 1.69]


@pytest.mark.parametrize("lens", sorted(LENSES))
def test_closed_form_lens_derivatives_match_autograd(lens):
    cam = LENSES[lens]
    t, _ = _points(LENS_THETAS, cam[5], seed=1)
    want_uv, want_J = lens_ref.autograd(t, cam)
    got_uv, got_J = lens_ref.closed_form(t, cam)
    # per point and lens word, relative to the largest entry of that column over uv (J)
    s_uv = np.abs(want_uv).max(1, keepdims=True)
    s_J = np.abs(want_J).max((1, 2), keepdims=True)
    assert (np.abs(got_uv - want_uv) <= 1e-12 * np.maximum(s_uv, 1e-300)).all(), np.abs(got_uv - want_uv).max()
    assert (np.abs(got_J - want_J) <= 1e-12 * np.maximum(s_J, 1e-300)).all(), np.abs(got_J - want_J).max()


# the fp32 model of the same formulas: within FP32_ULPS ulps of each point's largest uv (J) derivative, from the axis to the
# lens's edge (about 5 ulps at most, just below FISHEYE_SERIES_THETA where the 7-term series meets its float64 sum)
FP32_ULPS = 8


@pytest.mark.parametrize("lens", sorted(LENSES))
def test_fp32_lens_derivatives_near_the_axis(lens):
    cam = LENSES[lens]
    t, _ = _points([1e-8, 1e-6, 1e-4, 1e-3, 1e-2, 0.1, 0.5, 0.9, 0.99, 1.2, 1.5], cam[5], seed=2)
    t = t.astype(np.float32).astype(np.float64)  # points fp32 can hold, so both models see the same input
    ref_uv, ref_J = lens_ref.closed_form(t, cam)
    got_uv, got_J = lens_ref.closed_form(t, cam, np.float32)
    assert np.isfinite(got_uv).all() and np.isfinite(got_J).all()
    ulp = np.finfo(np.float32).eps
    assert (np.abs(got_uv - ref_uv) <= FP32_ULPS * ulp * np.abs(ref_uv).max((1, 2), keepdims=True)).all()
    assert (np.abs(got_J - ref_J) <= FP32_ULPS * ulp * np.abs(ref_J).max((1, 2, 3), keepdims=True)).all()


def _small_scene(gs, n=24, seed=5):
    """n Gaussians in front of a 48 x 32 fisheye at 60-170 degrees of field, with a non-zero k."""
    rng = np.random.default_rng(seed)
    vtx = gs.activate_records(gs.synth_records(seed, n))
    th = rng.uniform(0.0, 1.3, n)
    ph = rng.uniform(0, 2 * np.pi, n)
    d = rng.uniform(1.5, 3.0, n)
    vtx[:, 0], vtx[:, 1], vtx[:, 2] = d * np.sin(th) * np.cos(ph), d * np.sin(th) * np.sin(ph), 5.0 - d * np.cos(th)
    vtx[:, 4:7] = np.exp(rng.uniform(-2.5, -1.5, (n, 3)))
    vtx[:, 7] = rng.uniform(0.3, 0.8, n)
    u = gs.uniforms_from_camera([0.05, -0.03, 5.0], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 48, 32)
    cam = gs.fisheye_camera(14.0, 14.5, 23.5, 15.5, (0.02, -0.004, 0.0005, 0.0), 1.5)
    return vtx.astype(np.float32), u, cam


@pytest.mark.parametrize("upstream", ["colour", "depth_alpha", "feature"])
@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
def test_reference_passes_gradcheck(gs, upstream, aa):
    vtx, u, cam = _small_scene(gs)
    frame = lens_ref.cpu_frame(vtx, u, cam)
    assert frame["vals"].size > 20
    rng = np.random.default_rng(3)
    H, W = int(u.height), int(u.width)
    feats = rng.standard_normal((vtx.shape[0], 3)) if upstream == "feature" else None
    g = rng.standard_normal((H, W, 3 if upstream != "depth_alpha" else 2))
    base = lens_ref.leaves(u, cam)
    max_theta = float(cam.max_theta)
    v_all, used, local = lens_ref.grad_ref.survivors(vtx, frame)
    leaf = torch.tensor(v_all[used].astype(np.float64))

    def loss(view, campos, lens):
        cl = {"camera_position": campos, "proj_mat": base["proj_mat"].detach(), "view_mat": view, "tan_fovx": base["tan_fovx"],
              "tan_fovy": base["tan_fovy"], "lens": lens}
        fn = lens_ref.pre(cl, max_theta, aa)
        if upstream == "feature":
            vals = lens_ref.features_ref.frame_values(leaf, torch.tensor(feats[used]), u, frame, local, pre=fn)[..., 3:]
        else:
            vals = lens_ref.depth_ref.frame_values(leaf, u, frame, local, pre=fn)
            vals = vals[..., :3] if upstream == "colour" else vals[..., 3:]
        return (vals * torch.tensor(g)).sum()

    args = tuple(base[k].detach().clone().requires_grad_() for k in ("view_mat", "camera_position", "lens"))
    assert torch.autograd.gradcheck(loss, args, eps=1e-7, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("upstream", ["colour", "depth_alpha"])
def test_translation_identity(gs, upstream):
    vtx, u, cam = _small_scene(gs, n=40, seed=9)
    frame = lens_ref.cpu_frame(vtx, u, cam)
    rng = np.random.default_rng(4)
    H, W = int(u.height), int(u.width)
    gi = rng.standard_normal((H, W, 4)) if upstream == "colour" else None
    gda = rng.standard_normal((H, W, 2)) if upstream == "depth_alpha" else None
    ref = lens_ref.reference(vtx, u, cam, frame, grad_image=gi, grad_da=gda)
    res, scale = lens_ref.translation_residual(ref["grad"], ref["grad_ubo"], u)
    assert np.abs(res).max() <= 1e-9 * scale, (res, scale)
    assert np.abs(ref["grad_lens"]).max() > 0 and not ref["grad_ubo"][~lens_ref.LIVE_UBO].any()


def test_lens_helpers_round_trip(gs):
    cams = [gs.fisheye_camera(412.3, 408.9, 319.5, 239.25, (0.031, -0.0079, 0.0013, -0.0001)),
            gs.fisheye_from_colmap(300.1, 299.7, 320.3, 240.9, -0.05, 0.004, -0.0002, 0.0),
            gs.fisheye_camera(1e-3, 7.5e5, -12.0, 1e4, (1e-30, 0.0, -0.0, 3.0e-7), math.pi / 2)]
    for cam in cams:
        t = gs.lens_tensor(cam)
        assert t.dtype == torch.float32 and tuple(t.shape) == (gs.LENS_WORDS,)
        back = gs.lens_camera(t, cam.max_theta)
        assert bytes(back) == bytes(cam)
        assert np.array_equal(gs.lens_tensor(back).numpy().view(np.uint32), t.numpy().view(np.uint32))
        assert np.array_equal(t.numpy(), np.array([cam.fx, cam.fy, cam.cx, cam.cy, *cam.k], np.float32))
    with pytest.raises(ValueError):
        gs.lens_camera(torch.zeros(7), 1.0)
