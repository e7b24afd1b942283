"""The camera side of reverse mode, on the CPU: gs_b200.uniforms_torch (the differentiable gsb_uniforms of a pose), the
UBO pack / unpack helpers, and the camera gradient of the float64 reference (tests/grad_ref.py) that the GPU's
gsb_render_backward_camera is compared against."""
import numpy as np
import pytest
import torch

import grad_ref
import scenes
from backward_util import translation_identity


def _random_poses(n=20, seed=11):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        pos = rng.uniform(-6.0, 6.0, 3).astype(np.float32)
        q = rng.standard_normal(4)
        q = (q / np.linalg.norm(q)).astype(np.float32)
        fov = np.float32(rng.uniform(20.0, 100.0))
        w, h = int(rng.integers(16, 2000)), int(rng.integers(16, 1200))
        yield pos, q, fov, w, h


def test_pack_unpack_round_trip(gs):
    u = scenes.camera("odd_size")
    f = gs.pack_uniforms(u)
    assert f.shape == (gs.UBO_FLOATS,) and f.dtype == np.float32
    back = gs.unpack_uniforms(f, u.width, u.height)
    assert bytes(back) == bytes(u)


def test_uniforms_torch_value_is_the_hosts_bit_for_bit(gs):
    for pos, q, fov, w, h in _random_poses():
        host = gs.pack_uniforms(gs.uniforms_from_camera(pos, q, fov, 0.1, 1000.0, w, h))
        got = gs.uniforms_torch(torch.from_numpy(pos), torch.from_numpy(q), float(fov), 0.1, 1000.0, w, h)
        assert got.dtype == torch.float32 and got.shape == (gs.UBO_FLOATS,)
        assert np.array_equal(got.numpy().view(np.uint32), host.view(np.uint32)), (pos, q, fov, w, h)
        # the float64 restatement whose gradient it carries computes the same function
        r = gs._uniforms_restated(*(torch.tensor(np.float64(x)) for x in (pos, q, fov)), 0.1, 1000.0, w, h).numpy()
        for sl in (slice(0, 4), slice(4, 20), slice(20, 36), slice(36, 38)):  # position, proj, view, tan_fov
            err = np.abs(r[sl] - host[sl]).max() / np.abs(host[sl]).max()
            assert err <= 1e-6, (sl, err, pos, q, fov, w, h)


def test_uniforms_restatement_gradcheck(gs):
    pos = torch.tensor([0.3, -1.2, 4.0], dtype=torch.float64, requires_grad=True)
    q = torch.tensor([0.9, 0.1, -0.3, 0.2], dtype=torch.float64, requires_grad=True)  # not normalised: used as given
    fov = torch.tensor(50.0, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda p, r, f: gs._uniforms_restated(p, r, f, 0.1, 1000.0, 640, 480), (pos, q, fov))


def test_uniforms_torch_carries_the_restatements_gradient(gs):
    pos = torch.tensor([0.3, -1.2, 4.0], requires_grad=True)
    q = torch.tensor([0.9, 0.1, -0.3, 0.2], requires_grad=True)
    fov = torch.tensor(50.0, requires_grad=True)
    # fp32-representable weights: the float32 output's upstream gradient is then the same as the restatement's
    w = torch.from_numpy(np.random.default_rng(2).standard_normal(gs.UBO_FLOATS).astype(np.float32)).double()
    (gs.uniforms_torch(pos, q, fov, 0.1, 1000.0, 640, 480).double() * w).sum().backward()
    p64, q64, f64 = (t.detach().double().requires_grad_() for t in (pos, q, fov))
    (gs._uniforms_restated(p64, q64, f64, 0.1, 1000.0, 640, 480) * w).sum().backward()
    for a, b in ((pos, p64), (q, q64), (fov, f64)):
        assert torch.allclose(a.grad.double(), b.grad, rtol=1e-6, atol=1e-9)


def test_reference_camera_gradient_obeys_the_translation_identity(oracle):
    _, vtx, u = scenes.c1()
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = np.random.default_rng(5).standard_normal((u.height, u.width, 4)).astype(np.float32)
    g[steps] = 0.0
    ref = grad_ref.reference(vtx, u, frame, g, camera=True)
    gu = ref["grad_ubo"]
    assert gu.shape == (38,) and np.abs(gu).max() > 0
    # the fields the forward does not read, or reads only through step functions, have no gradient
    assert gu[3] == 0 and not gu[4 + 2:20:4].any() and not gu[20 + 3:36:4].any()
    gp = ref["grad"][:, 0:3]
    res, scale = translation_identity(gp.sum(0), np.abs(gp).sum(0), u, gu)
    assert (np.abs(res) <= 1e-9 * scale).all(), (res, scale)
    # with the camera as leaves the reference differentiates the same function: same vertex gradient and exclusions
    plain = grad_ref.reference(vtx, u, frame, g)
    assert np.linalg.norm(plain["grad"] - ref["grad"]) <= 1e-12 * np.linalg.norm(plain["grad"])
    assert np.array_equal(plain["exclude"], ref["exclude"])


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_camera_restatement_is_grad_refs_preprocess(cam):
    """grad_ref.preprocess with the camera as tensors (camera_leaves) computes what it computes from the UBO."""
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    v = torch.from_numpy(vtx.astype(np.float64))
    with torch.no_grad():
        want = grad_ref.preprocess(v, u)
        got = grad_ref.preprocess(v, u, grad_ref.camera_leaves(u))
    for name, a, b in zip(("uv", "conic", "opacity", "colour", "red"), got, want):
        ok = torch.isfinite(b)
        assert torch.equal(ok, torch.isfinite(a)), name
        assert torch.allclose(a[ok], b[ok], rtol=1e-12, atol=1e-12), name
