"""gsb_render_backward_camera / render_torch(..., ubo=) / uniforms_torch: the gradient of a frame with respect to its camera
matches the float64 restatement of the forward (tests/grad_ref.py), obeys the translation identity at full
size, and refines a perturbed camera pose."""
import math

import numpy as np
import pytest

import grad_ref
import scenes
from backward_util import CAMERA_GROUPS, DEAD, expect, grad_image, rel, render, translation_identity

pytestmark = pytest.mark.gpu

ENTRY = "gsb_render_backward_camera"  # what its error messages start with
REF_CAMERAS = ("c1", "odd_size", "inside")
# pose refinement: Adam step sizes (position, quaternion) and step count
POSE_LR_POS, POSE_LR_ROT, POSE_STEPS = 2e-3, 5e-4, 100


def camera_scene():
    """scenes.c1() with no Gaussian whose gradient is ill-posed at the reference cameras, so the camera gradient -- a sum over
    every Gaussian -- can be compared whole: opacity capped at 0.95 (the 0.99 alpha clamp never binds) and the red DC
    coefficient moved for any Gaussian whose unclamped red lies within 1e-3 of 0 at one of REF_CAMERAS."""
    import torch

    _, vtx, _ = scenes.c1()
    vtx = vtx.copy()
    vtx[:, 7] = np.minimum(vtx[:, 7], np.float32(0.95))
    for _ in range(20):
        moved = False
        for cam in REF_CAMERAS:
            with torch.no_grad():
                red = grad_ref.preprocess(torch.from_numpy(vtx.astype(np.float64)), scenes.camera(cam))[4].numpy()
            near = np.abs(red) < 1e-3
            if near.any():
                vtx[near, 12] += np.float32(0.01 / grad_ref.SH_C0)  # red + 0.01 at every camera
                moved = True
        if not moved:
            return vtx
    raise AssertionError("camera_scene did not settle")


@pytest.fixture(scope="module")
def cam_vtx():
    return camera_scene()


@pytest.fixture
def bctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _camera_backward(ctx, vtx, g, with_vertices=True):
    """gsb_render_backward_camera of the context's last frame: (grad_vertices or None, the 40 words of dL/d(UBO)) in float64."""
    import torch

    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    gi = torch.from_numpy(g).cuda()
    gv = torch.full_like(v, float("nan")) if with_vertices else None
    gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda")
    ctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr() if with_vertices else None, grad_uniforms_ptr=gu.data_ptr())
    torch.cuda.synchronize()
    return (gv.cpu().numpy().astype(np.float64) if with_vertices else None), gu.cpu().numpy().astype(np.float64)


def _vertex_backward(ctx, vtx, g):
    import torch

    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    gi = torch.from_numpy(g).cuda()
    out = torch.full_like(v, float("nan"))
    ctx.render_backward(v.data_ptr(), gi.data_ptr(), out.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.float64)


def _words(gs, floats38):
    w = np.zeros(40)
    w[gs.UBO_FLOAT_WORDS] = floats38
    return w


@pytest.mark.parametrize("cam", REF_CAMERAS)
def test_camera_gradient_matches_float64_reference(gs, oracle, bctx, cam_vtx, cam):
    u = scenes.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(cam_vtx, oracle.cov3d(cam_vtx), u)
    g = grad_image(u, steps)
    ref = grad_ref.reference(cam_vtx, u, frame, g, camera=True)
    assert not ref["exclude"].any()
    want = _words(gs, ref["grad_ubo"])
    bctx.upload(cam_vtx)
    render(bctx, u)
    gv, got = _camera_backward(bctx, cam_vtx, g)
    assert np.isfinite(got).all() and np.isfinite(gv).all()
    for name, idx in CAMERA_GROUPS.items():
        r = rel(got[idx], want[idx])
        assert r <= 1e-3, (cam, name, r, got[idx], want[idx])
    assert not got[DEAD].any()  # camera_position.w, proj row 2, view row 3, width, height
    # the vertex gradient is gsb_render_backward's, and a frozen scene gives the same camera gradient
    assert rel(gv, _vertex_backward(bctx, cam_vtx, g)) <= 1e-6
    _, frozen = _camera_backward(bctx, cam_vtx, g, with_vertices=False)
    assert rel(frozen, got) <= 1e-6


def test_levels_agree(bctx, cam_vtx):
    u = scenes.camera("c1")
    g = grad_image(u, np.zeros((u.height, u.width), bool))
    bctx.upload(cam_vtx)
    got = []
    for level in (0, 1, 2):  # 2 falls back to 1 while recording
        render(bctx, u, level=level)
        got.append(_camera_backward(bctx, cam_vtx, g)[1])
    assert np.abs(got[0]).max() > 0
    assert rel(got[1], got[0]) <= 1e-6
    assert rel(got[2], got[0]) <= 1e-6


def test_fast_mode_close_to_exact(oracle, bctx, cam_vtx):
    u = scenes.camera("c1")
    oracle.set_exp_mode(0)
    _, steps = oracle.render_frame_probed(cam_vtx, oracle.cov3d(cam_vtx), u)
    g = grad_image(u, steps)
    bctx.upload(cam_vtx)
    render(bctx, u, mode=0)
    ge = _camera_backward(bctx, cam_vtx, g)[1]
    render(bctx, u, mode=1)
    gf = _camera_backward(bctx, cam_vtx, g)[1]
    assert rel(gf, ge) <= 1e-3


def test_nothing_visible_gives_zero(bctx):
    _, vtx, _ = scenes.c1()
    u = scenes.camera("away")
    bctx.upload(vtx)
    render(bctx, u)
    g = np.ones((u.height, u.width, 4), np.float32)
    gv, gu = _camera_backward(bctx, vtx, g)
    assert not gv.any() and not gu.any()
    assert not _camera_backward(bctx, vtx, g, with_vertices=False)[1].any()


def test_error_cases(gs, bctx):
    import torch

    _, vtx, u = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    gi = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    out = torch.empty_like(v)
    gu = torch.empty(40, dtype=torch.float32, device="cuda")

    def bw(c, vertices=True):
        return lambda: c.render_backward(v.data_ptr(), gi.data_ptr(), out.data_ptr() if vertices else None,
                                         grad_uniforms_ptr=gu.data_ptr())

    expect(gs, bctx, gs.ERR_NO_SCENE, bw(bctx), ENTRY)  # nothing uploaded
    bctx.upload(vtx)
    expect(gs, bctx, gs.ERR_NO_SCENE, bw(bctx), ENTRY)  # no frame yet
    bctx.set_backward(False)
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx, vertices=False), ENTRY)  # switch off
    bctx.set_backward(True)
    bctx.render(u, rows=(0, 2))
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx), ENTRY)  # a band
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID,  # a NULL grad_uniforms
           lambda: bctx._ck(gs.lib.gsb_render_backward_camera(bctx.h, v.data_ptr(), gi.data_ptr(), 0, out.data_ptr(), None, None)),
           ENTRY)
    bw(bctx)()  # the whole frame: fine
    bw(bctx, vertices=False)()
    bctx.upload(vtx)
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx), ENTRY)  # uploaded again after the frame
    # a pipelined frame that overflowed its arena (gsb_render_async never regrows; a fresh context holds N = 10 k instances)
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        fresh.set_backward(True)
        ui = scenes.camera("inside")
        dev = torch.empty((ui.height, ui.width, 4), dtype=torch.float32, device="cuda")
        fresh.render_into(ui, dev.data_ptr(), gs.FORMAT_RGBA32F, sync=False)
        torch.cuda.synchronize()
        expect(gs, fresh, gs.ERR_INVALID, bw(fresh), ENTRY)
        with pytest.raises(gs.GsbError):
            fresh.stats()  # reports (and clears) the overflow
    finally:
        fresh.close()
    # fp16 SH storage
    bctx.set_sh_storage(True)
    bctx.upload(vtx)
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx), ENTRY)
    # a sharded context (two ranks on one GPU)
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, bw(c0), ENTRY)
    finally:
        grp.close()


def test_translation_identity_at_full_size(gs):
    """Moving every Gaussian by delta is the same function as moving the camera by -delta: the sum of the position
    gradients over the 5.8 M Gaussians of bench.py's garden stand-in equals the camera-side terms."""
    import sys
    from pathlib import Path

    import torch

    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    u = bench.cameras(gs, wl)[0]
    ctx = gs.Context(0)
    try:
        ctx.set_tile_cull(1)
        ctx.set_backward(True)
        v = torch.from_numpy(bench.make_scene(gs, wl)).cuda()
        ctx.upload(v)
        ctx.render_into(u, torch.empty((u.height, u.width, 4), dtype=torch.float32, device="cuda").data_ptr())
        gi = torch.randn((u.height, u.width, 4), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
        gv = torch.empty_like(v)
        gu = torch.empty(40, dtype=torch.float32, device="cuda")
        ctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), grad_uniforms_ptr=gu.data_ptr())
        torch.cuda.synchronize()
        gp = gv[:, 0:3].double()
        psum, pabs = gp.sum(0).cpu().numpy(), gp.abs().sum(0).cpu().numpy()
        g38 = gu.cpu().numpy().astype(np.float64)[gs.UBO_FLOAT_WORDS]
    finally:
        ctx.close()
    res, scale = translation_identity(psum, pabs, u, g38)
    print("translation identity: residual", res, "scale", scale)
    assert np.abs(g38).max() > 0
    assert (np.abs(res) <= 1e-5 * scale).all(), (res, scale)


def test_render_torch_ubo_gradient_is_ordered_on_torchs_stream(gs, bctx, cam_vtx):
    import torch

    u = scenes.camera("c1")
    g = grad_image(u, np.zeros((u.height, u.width), bool))
    gt = torch.from_numpy(g).cuda()
    v = torch.from_numpy(cam_vtx).cuda().requires_grad_()
    ubo = torch.from_numpy(gs.pack_uniforms(u)).cuda().requires_grad_()
    img = gs.render_torch(bctx, v, u, ubo)
    (img * gt).sum().backward()
    got_v = v.grad.cpu().numpy().astype(np.float64)
    got_u = ubo.grad.cpu().numpy().astype(np.float64)
    want_v, want_u = _camera_backward(bctx, cam_vtx, g)  # the same frame, differentiated again and synchronised
    assert np.abs(want_u).max() > 0
    assert rel(got_u, want_u[gs.UBO_FLOAT_WORDS]) <= 1e-6
    assert rel(got_v, want_v) <= 1e-6
    # frozen vertices: no vertex gradient, the same camera gradient
    vf = torch.from_numpy(cam_vtx).cuda()
    ubo2 = torch.from_numpy(gs.pack_uniforms(u)).cuda().requires_grad_()
    img = gs.render_torch(bctx, vf, u, ubo2)
    (img * gt).sum().backward()
    assert vf.grad is None
    assert rel(ubo2.grad.cpu().numpy().astype(np.float64), want_u[gs.UBO_FLOAT_WORDS]) <= 1e-6
    # a ubo that needs no gradient renders its camera and differentiates the scene only
    u2 = scenes.camera("odd_size")
    v2 = torch.from_numpy(cam_vtx).cuda().requires_grad_()
    img = gs.render_torch(bctx, v2, u2, torch.from_numpy(gs.pack_uniforms(u2)))
    assert np.array_equal(img.detach().cpu().numpy(), bctx.render(u2))
    assert img.shape == (u2.height, u2.width, 4)


def _quat_angle_deg(a, b):
    d = abs(float(np.dot(a / np.linalg.norm(a), b / np.linalg.norm(b))))
    return math.degrees(2.0 * math.acos(min(1.0, d)))


def test_pose_refinement(gs, bctx):
    """Adam on (position, quaternion normalised in torch) through uniforms_torch + render_torch recovers a perturbed
    camera: both pose errors at least halve and the photometric loss falls below a quarter of its start."""
    import torch

    _, vtx, _ = scenes.c1()
    pos0, q0, fov, W, H = [0.0, 0.0, 5.0], [1.0, 0.0, 0.0, 0.0], 45.0, 640, 480
    u = gs.uniforms_from_camera(pos0, q0, fov, 0.1, 1000.0, W, H)
    v = torch.from_numpy(vtx).cuda()
    with torch.no_grad():
        target = gs.render_torch(bctx, v, u)[..., :3].clone()
    pos = torch.tensor([0.03, -0.02, 5.04], dtype=torch.float64, requires_grad=True)  # 5.4 cm off
    q = torch.tensor(scenes.quat_axis_angle([0.3, 1.0, 0.2], 1.0), dtype=torch.float64, requires_grad=True)  # 1 degree off
    opt = torch.optim.Adam([{"params": [pos], "lr": POSE_LR_POS}, {"params": [q], "lr": POSE_LR_ROT}])

    def errors():
        return (float(np.linalg.norm(pos.detach().numpy() - pos0)), _quat_angle_deg(q.detach().numpy(), np.array(q0)))

    e_pos0, e_rot0 = errors()
    losses = []
    for _ in range(POSE_STEPS):
        opt.zero_grad()
        ubo = gs.uniforms_torch(pos, q / q.norm(), fov, 0.1, 1000.0, W, H)
        img = gs.render_torch(bctx, v, u, ubo)
        loss = ((img[..., :3] - target) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    with torch.no_grad():
        ubo = gs.uniforms_torch(pos, q / q.norm(), fov, 0.1, 1000.0, W, H)
        final = float(((gs.render_torch(bctx, v, u, ubo)[..., :3] - target) ** 2).sum())
    e_pos, e_rot = errors()
    print(f"pose refinement: loss {losses[0]:.4g} -> {final:.4g}; translation error {100 * e_pos0:.2f} -> {100 * e_pos:.2f} cm; "
          f"rotation error {e_rot0:.3f} -> {e_rot:.3f} deg; losses every 10 steps {[round(x, 3) for x in losses[::10]]}")
    assert final < 0.25 * losses[0], (losses[0], final)
    assert e_pos <= 0.5 * e_pos0, (e_pos0, e_pos)
    assert e_rot <= 0.5 * e_rot0, (e_rot0, e_rot)
