"""The references of the rendered depth and alpha (tests/depth_ref.py) against each other, the oracle and autograd: no GPU."""
import numpy as np
import pytest
import torch

import bg_ref
import depth_ref
import edge_scene
import grad_ref
import scenes
from backward_util import translation_identity


def _scene(name):
    if name == "edge":
        return edge_scene.vertices()[0], edge_scene.camera("axis")
    return scenes.c1()[1], scenes.camera(name)


def _frame(oracle, vtx, u, mode):
    oracle.set_exp_mode(mode)
    try:
        return oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside", "edge"])
def test_alpha_is_one_minus_the_product(oracle, cam):
    """The float64 A channel (colour 1 over 0) equals 1 - prod(1 - alpha) over the contributors, and D vanishes with A."""
    vtx, u = _scene(cam)
    frame, _ = _frame(oracle, vtx, u, 0)
    vals = depth_ref.reference(vtx, u, frame)["values"]
    T = bg_ref.transmittance64(vtx, u, frame)
    assert np.abs(vals[..., 4] - (1.0 - T)).max() <= 1e-12
    assert not vals[..., 3][vals[..., 4] == 0].any()


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_fp32_restatement_is_close_to_float64(oracle, cam):
    """The fp32 restatement reproduces the oracle's image bit for bit (depth_alpha32 checks it), and its D and A are within
    1e-4 relative of the float64 reference off the step pixels."""
    vtx, u = _scene(cam)
    frame32, steps = _frame(oracle, vtx, u, 1)
    da = depth_ref.depth_alpha32(frame32, u)
    frame64, _ = _frame(oracle, vtx, u, 0)
    ref = depth_ref.reference(vtx, u, frame64)["values"][..., 3:]
    err = np.abs(da - ref) / np.maximum(np.abs(ref), 1.0)
    assert err[~steps].max() <= 1e-4, err[~steps].max()
    assert da[..., 0].max() > 1.0 and (da[..., 1] > 0.5).mean() > 0.1


def test_fp32_restatement_on_the_edge_scene(oracle):
    vtx, u = _scene("edge")
    frame32, _ = _frame(oracle, vtx, u, 1)
    da = depth_ref.depth_alpha32(frame32, u)
    assert np.isfinite(da).all() and (da[..., 1] <= 1.0).all()


def _small_case():
    """A few Gaussians of c1 in a 40 x 24 frame: small enough for gradcheck."""
    vtx = scenes.c1()[1]
    u = scenes.camera("c1")
    rng = np.random.default_rng(5)
    sub = vtx[rng.choice(vtx.shape[0], 400, replace=False)].copy()
    import gs_b200 as gs

    small = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 40, 24)
    return sub, small


def test_gradcheck_vertices_camera_and_background(oracle):
    vtx, u = _small_case()
    frame, _ = _frame(oracle, vtx, u, 0)
    _, used, local = grad_ref.survivors(vtx, frame)
    assert used.size > 5
    base = torch.tensor(vtx[used].astype(np.float64))
    weights = torch.tensor(np.random.default_rng(2).standard_normal((u.height, u.width, 5)))

    def f_vertices(x):
        leaf = torch.cat([x, base[6:]])
        return (depth_ref.frame_values(leaf, u, frame, local, bg=(0.2, 0.4, 0.6)) * weights).sum()

    x0 = base[:6].clone().requires_grad_()
    assert torch.autograd.gradcheck(f_vertices, (x0,), eps=1e-7, atol=1e-5, rtol=1e-4)

    cam = grad_ref.camera_leaves(u)

    def f_camera(view_mat, camera_position):
        c = dict(cam)
        c["view_mat"], c["camera_position"] = view_mat, camera_position
        return (depth_ref.frame_values(base, u, frame, local, cam=c) * weights).sum()

    assert torch.autograd.gradcheck(f_camera, (cam["view_mat"], cam["camera_position"]), eps=1e-7, atol=1e-5, rtol=1e-4)

    def f_bg(bg):
        return (depth_ref.frame_values(base, u, frame, local, bg=bg) * weights).sum()

    assert torch.autograd.gradcheck(f_bg, (torch.tensor([0.2, 0.4, 0.6], dtype=torch.float64, requires_grad=True),))


def test_translation_identity_with_a_depth_only_gradient(oracle):
    """Moving every Gaussian by delta equals moving the camera by -delta (DESIGN.md section 10): with a depth-only upstream
    gradient the position gradients' sum equals the camera's side, view row 2 included."""
    vtx, u = _scene("c1")
    frame, steps = _frame(oracle, vtx, u, 0)
    gda = np.random.default_rng(4).standard_normal((u.height, u.width, 2))
    gda[..., 1] = 0.0
    gda[steps] = 0.0
    ref = depth_ref.reference(vtx, u, frame, None, gda, camera=True)
    g = ref["grad"][:, 0:3]
    res, scale = translation_identity(g.sum(0), np.abs(g).sum(0), u, ref["grad_ubo"])
    assert np.all(np.abs(res) <= 1e-9 * scale), (res, scale)
    assert np.abs(ref["grad_ubo"][20 + 14]) > 0  # view row 2's translation: the depth's own term
