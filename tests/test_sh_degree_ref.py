"""gsb_set_sh_degree's definition in the float64 reference (tests/sh_degree_ref.py): the frame and the gradient at
degree d are those of the scene with the bands above d zeroed, rendered at degree 3, except that the zeroed coefficients
get no gradient.  CPU only."""
import numpy as np
import pytest
import torch

import grad_ref
import scenes
import sh_degree_ref
from backward_util import grad_image


def zero_bands(vtx, d):
    """The scene with the SH coefficients of bands > d set to 0 (Z_d)."""
    z = np.array(vtx, np.float32, copy=True)
    z[:, 12 + 3 * (d + 1) ** 2:60] = 0.0
    return z


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
@pytest.mark.parametrize("d", [0, 1, 2])
def test_degree_d_is_degree_3_of_the_zeroed_scene(oracle, cam, d):
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    z = zero_bands(vtx, d)
    got = sh_degree_ref.reference(vtx, u, frame, g, camera=True, sh_degree=d)
    want = grad_ref.reference(z, u, frame, g, camera=True)
    assert np.abs(got["image"] - want["image"]).max() <= 1e-12
    live = 12 + 3 * (d + 1) ** 2
    scale = max(np.abs(want["grad"]).max(), 1.0)
    assert np.abs(got["grad"][:, :live] - want["grad"][:, :live]).max() <= 1e-12 * scale, (cam, d)
    assert not got["grad"][:, live:].any()
    assert np.abs(want["grad"][:, live:]).max() > 0  # the zeroed bands of Z_d do get a gradient at degree 3
    assert np.abs(got["grad_ubo"] - want["grad_ubo"]).max() <= 1e-12 * max(np.abs(want["grad_ubo"]).max(), 1.0)
    # at degree 3 the restated colour is grad_ref's
    full = sh_degree_ref.reference(vtx, u, frame, g, camera=True)
    plain = grad_ref.reference(vtx, u, frame, g, camera=True)
    assert np.abs(full["image"] - plain["image"]).max() <= 1e-12
    assert np.abs(full["grad"] - plain["grad"]).max() <= 1e-12 * max(np.abs(plain["grad"]).max(), 1.0)


@pytest.mark.parametrize("d", [0, 1, 2])
def test_gradcheck_of_vertex_and_camera_leaves(d):
    _, vtx, _ = scenes.c1()
    u = scenes.camera("c1")
    rows = torch.tensor(vtx[:200].astype(np.float64))
    with torch.no_grad():
        red = sh_degree_ref.preprocess(rows, u, sh_degree=d)[4]
        vz = grad_ref.preprocess(rows, u)[0]  # any finite survivor of the projection
    pick = torch.nonzero((red.abs() > 1e-2) & torch.isfinite(vz).all(1)).flatten()[:6]
    v = rows[pick].clone().requires_grad_()
    cam = grad_ref.camera_leaves(u)
    names = list(cam)

    def f(v, *leaves):
        out = sh_degree_ref.preprocess(v, u, dict(zip(names, leaves)), sh_degree=d)
        return tuple(t for t in out[:4])

    assert torch.autograd.gradcheck(f, (v, *(cam[k] for k in names)), eps=1e-6, atol=1e-5, rtol=1e-4)
