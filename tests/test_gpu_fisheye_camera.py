"""gsb_render_backward_fisheye on the GPU: the camera and lens gradients of fisheye frames against the float64 reference
(tests/lens_ref.py) blended over the frame's own level-0 lists, its other outputs against the existing entries, determinism,
the error codes, the translation identity at full size, render_torch(lens=, ubo=), pose refinement and lens self-calibration
through the lens, and SceneAdam.step's camera outputs."""

import numpy as np
import pytest

import lens_ref
import scenes
from backward_util import expect, grad_image, rel, translation_identity
from test_gpu_backward_camera import POSE_LR_POS, POSE_LR_ROT, POSE_STEPS, _quat_angle_deg
from test_gpu_fisheye import _frame_lists, _grad_case, _lens

pytestmark = pytest.mark.gpu

ENTRY = "gsb_render_backward_fisheye"
# field groups of the fisheye camera gradient: gsb_uniforms words and lens words (fx, fy, cx, cy, k1..k4)
UBO_GROUPS = {"camera_position": [0, 1, 2], "view_3x3": [20 + c * 4 + r for c in range(3) for r in range(3)],
              "view_translation": [32, 33, 34]}
LENS_GROUPS = {"focal": [0, 1], "principal_point": [2, 3], "k": [4, 5, 6, 7]}
DEAD_UBO = np.nonzero(~lens_ref.LIVE_UBO)[0]


def _torch():
    import torch

    return torch


@pytest.fixture
def fctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _case(gs, name):
    """odd_size gets a non-zero k (test_gpu_fisheye's "odd_size" lens); inside is the 180-degree lens from inside the cloud."""
    return _grad_case(gs, name)


def _call(gs, ctx, v, gi=None, gda=None, feats=None, gfm=None, vertices=True, camera=True, lens=True, density=False,
          features_grad=False, stream=None):
    """One gsb_render_backward_fisheye call on torch tensors: (grad_vertices, grad_uniforms (40,), grad_lens (10,),
    grad_features, density) as float64 numpy arrays (None where not asked for)."""
    torch = _torch()
    gv = torch.full_like(v, float("nan")) if vertices else None
    gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda") if camera else None
    gl = torch.full((10,), float("nan"), dtype=torch.float32, device="cuda") if lens else None
    gf = torch.full_like(feats, float("nan")) if features_grad else None
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if density else None
    s = gs._torch_stream_arg(stream or torch.cuda.current_stream())
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    ctx._backward_fisheye(ptr(v), ptr(gi), ptr(gv), s, grad_uniforms_ptr=ptr(gu), grad_lens_ptr=ptr(gl), density_ptr=ptr(dens),
                          grad_depth_alpha_ptr=ptr(gda), features=feats, grad_feature_map=gfm, grad_features_ptr=ptr(gf))
    torch.cuda.synchronize()
    out = lambda t: None if t is None else t.cpu().numpy().astype(np.float64)  # noqa: E731
    return out(gv), out(gu), out(gl), out(gf), out(dens)


def _upstream(u, kind, steps, n, seed=7):
    """(grad_image (H, W, 4), grad_da (H, W, 2), features (n, 3), grad_fm (H, W, 3)) for one kind of upstream gradient, zero on
    the pixels `steps`; the unused ones are None."""
    rng = np.random.default_rng(seed)
    H, W = int(u.height), int(u.width)
    keep = ~steps[..., None]
    gi = gda = feats = gfm = None
    if kind == "colour":
        gi = (grad_image(u, seed=seed) * keep).astype(np.float32)
    elif kind in ("depth", "alpha"):
        gda = np.zeros((H, W, 2), np.float32)
        gda[..., 0 if kind == "depth" else 1] = rng.standard_normal((H, W)) * keep[..., 0]
    else:
        feats = rng.standard_normal((n, 3)).astype(np.float32)
        gfm = (rng.standard_normal((H, W, 3)) * keep).astype(np.float32)
    return gi, gda, feats, gfm


def _render(gs, ctx, u, depth, level=0):
    ctx.set_tile_cull(level)
    if depth:
        ctx.render_depth(u)
    else:
        ctx.render(u)


REF_RUNS = [("c1", "colour", False), ("c1", "colour", True), ("odd_size", "colour", False), ("odd_size", "colour", True),
            ("inside", "colour", False), ("inside", "colour", True), ("wide", "colour", False), ("wide", "colour", True),
            ("c1", "depth", False), ("c1", "alpha", True), ("c1", "feature", False),
            ("wide", "depth", True), ("wide", "alpha", False), ("odd_size", "feature", True)]


@pytest.mark.parametrize("name,kind,aa", REF_RUNS, ids=[f"{n}-{k}-{'aa' if a else 'plain'}" for n, k, a in REF_RUNS])
def test_camera_and_lens_gradients_match_float64_reference(gs, fctx, name, kind, aa):
    torch = _torch()
    vtx, u, cam = _case(gs, name)
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    fctx.set_antialiased(aa)
    fctx.set_backward(True)
    _, frame = _frame_lists(gs, fctx, u, vtx, cam)
    steps = lens_ref.step_pixels(vtx, u, cam, frame, aa)
    assert steps.mean() < 0.05
    gi, gda, feats, gfm = _upstream(u, kind, steps, vtx.shape[0])
    ref = lens_ref.reference(vtx, u, cam, frame, grad_image=gi, grad_da=gda, features=feats, grad_fm=gfm, antialiased=aa)
    v = torch.from_numpy(vtx).cuda()
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    for det in (False, True):
        fctx.set_backward_deterministic(det)
        _render(gs, fctx, u, gda is not None)
        _, gu, gl, _, _ = _call(gs, fctx, v, t(gi), t(gda), t(feats), t(gfm), vertices=False)
        for group, words in UBO_GROUPS.items():
            r = rel(gu[words], ref["grad_ubo"][words])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
        for group, words in LENS_GROUPS.items():
            r = rel(gl[1:9][words], ref["grad_lens"][words])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
        assert not gu[DEAD_UBO].any() and gl[0] == 0 and gl[9] == 0
    fctx.set_backward_deterministic(False)
    fctx.set_antialiased(False)


def test_other_outputs_equal_the_existing_entries(gs, fctx):
    torch = _torch()
    vtx, u, cam = _case(gs, "wide")
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    fctx.set_backward(True)
    v = torch.from_numpy(vtx).cuda()
    g = torch.from_numpy(grad_image(u)).cuda()
    rng = np.random.default_rng(2)
    gda = torch.from_numpy(rng.standard_normal((u.height, u.width, 2)).astype(np.float32)).cuda()
    feats = torch.from_numpy(rng.standard_normal((vtx.shape[0], 5)).astype(np.float32)).cuda()
    gfm = torch.from_numpy(rng.standard_normal((u.height, u.width, 5)).astype(np.float32)).cuda()
    for det in (True, False):
        fctx.set_backward_deterministic(det)
        fctx.render_depth(u)
        gv, gu, gl, gf, dens = _call(gs, fctx, v, g, gda, feats, gfm, density=True, features_grad=True)
        # the same frame through gsb_render_backward_features
        wv, wf = torch.empty_like(v), torch.empty_like(feats)
        wd = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
        fctx.render_backward_features(v.data_ptr(), feats, gfm, wv.data_ptr(), wf.data_ptr(), grad_image_ptr=g.data_ptr(),
                                      grad_depth_alpha_ptr=gda.data_ptr(), density_ptr=wd.data_ptr())
        torch.cuda.synchronize()
        want = [x.cpu().numpy().astype(np.float64) for x in (wv, wf, wd)]
        for got, w in zip((gv, gf, dens), want):
            if det:
                assert np.array_equal(got, w)
            else:
                assert rel(got, w) <= 1e-6
        # the camera and lens words without grad_vertices
        _, gu2, gl2, _, _ = _call(gs, fctx, v, g, gda, feats, gfm, vertices=False)
        if det:
            assert np.array_equal(gu2, gu) and np.array_equal(gl2, gl)
        else:
            assert rel(gu2, gu) <= 1e-6 and rel(gl2, gl) <= 1e-6
    # a colour-only frame: the vertex words of gsb_render_backward
    fctx.set_backward_deterministic(True)
    fctx.render(u)
    gv, _, _, _, _ = _call(gs, fctx, v, g)
    wv = torch.empty_like(v)
    fctx._backward(v.data_ptr(), g.data_ptr(), wv.data_ptr(), None)
    torch.cuda.synchronize()
    assert np.array_equal(gv, wv.cpu().numpy().astype(np.float64))
    fctx.set_backward_deterministic(False)


def test_deterministic_words(gs, fctx):
    torch = _torch()
    vtx, u, cam = _case(gs, "wide")
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    fctx.set_backward(True)
    fctx.set_backward_deterministic(True)
    v = torch.from_numpy(vtx).cuda()
    g = torch.from_numpy(grad_image(u)).cuda()
    outs = []
    for level in (0, 1, 2):
        _render(gs, fctx, u, False, level)
        outs.append(_call(gs, fctx, v, g)[1:3])
        outs.append(_call(gs, fctx, v, g)[1:3])  # a repeated call
    fctx.render(u)  # a re-rendered frame, on a side stream
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        outs.append(_call(gs, fctx, v, g, stream=side)[1:3])
    other = gs.Context(0)  # a fresh context
    try:
        other.upload(vtx)
        other.set_camera_model(cam)
        other.set_backward(True)
        other.set_backward_deterministic(True)
        other.render(u)
        outs.append(_call(gs, other, v, g)[1:3])
    finally:
        other.close()
    for gu, gl in outs[1:]:
        assert np.array_equal(gu, outs[0][0]) and np.array_equal(gl, outs[0][1])
    assert np.abs(outs[0][1]).max() > 0
    fctx.set_backward_deterministic(False)


def test_nothing_visible_and_empty_scene_give_zeros(gs, fctx):
    torch = _torch()
    vtx, u, cam = _case(gs, "c1")
    away = scenes.camera("away")
    fctx.upload(vtx)
    fctx.set_camera_model(gs.fisheye_camera(300.0, 300.0, 159.5, 119.5, max_theta=0.5))
    fctx.set_backward(True)
    fctx.render(away)
    v = torch.from_numpy(vtx).cuda()
    g = torch.ones((away.height, away.width, 4), dtype=torch.float32, device="cuda")
    gv, gu, gl, _, _ = _call(gs, fctx, v, g)
    assert not gv.any() and not gu.any() and not gl.any()
    fctx.upload(np.zeros((0, 60), np.float32))
    fctx.render(away)
    gu = torch.full((40,), float("nan"), device="cuda")
    gl = torch.full((10,), float("nan"), device="cuda")
    # n = 0: vertices is never read, but must not be NULL
    fctx._backward_fisheye(v.data_ptr(), g.data_ptr(), None, None, grad_uniforms_ptr=gu.data_ptr(), grad_lens_ptr=gl.data_ptr())
    torch.cuda.synchronize()
    assert not gu.cpu().numpy().any() and not gl.cpu().numpy().any()


def test_error_cases(gs, fctx):
    torch = _torch()
    vtx, u, cam = _case(gs, "c1")
    v = torch.from_numpy(vtx).cuda()
    g = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    gu = torch.empty(40, dtype=torch.float32, device="cuda")
    gl = torch.empty(10, dtype=torch.float32, device="cuda")
    gv = torch.empty_like(v)
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
    feats = torch.zeros((v.shape[0], 3), dtype=torch.float32, device="cuda")
    gfm = torch.zeros((u.height, u.width, 3), dtype=torch.float32, device="cuda")
    gda = torch.zeros((u.height, u.width, 2), dtype=torch.float32, device="cuda")

    def call(c=None, **kw):
        a = dict(vertices=v.data_ptr(), grad_image=g.data_ptr(), grad_da=None, features=None, channels=0, gfm=None, gv=None,
                 gu=gu.data_ptr(), gl=gl.data_ptr(), gf=None, density=None)
        a.update(kw)
        (c or fctx)._ck(gs.lib.gsb_render_backward_fisheye((c or fctx).h, a["vertices"], a["grad_image"], 0, a["grad_da"], 0,
                                                           a["features"], a["channels"], a["gfm"], 0, a["gv"], a["gu"], a["gl"],
                                                           a["gf"], a["density"], None))

    bad = lambda code, fn, c=None: expect(gs, c or fctx, code, fn, ENTRY)  # noqa: E731
    bad(gs.ERR_NO_SCENE, call)
    fctx.upload(vtx)
    bad(gs.ERR_NO_SCENE, call)  # no frame yet
    fctx.set_backward(True)
    fctx.render(u)  # a pinhole frame
    bad(gs.ERR_INVALID, call)
    fctx.set_camera_model(cam)
    fctx.set_backward(False)
    fctx.render(u)
    bad(gs.ERR_INVALID, call)  # not recorded
    fctx.set_backward(True)
    fctx.render(u, rows=(0, 2))
    bad(gs.ERR_INVALID, call)  # a band
    fctx.render(u)
    call()
    bad(gs.ERR_INVALID, lambda: call(gu=None, gl=None))  # all outputs NULL
    bad(gs.ERR_INVALID, lambda: call(gu=None, gl=None, gv=None, density=dens.data_ptr()))
    bad(gs.ERR_INVALID, lambda: call(features=feats.data_ptr(), channels=3))  # no grad_feature_map
    bad(gs.ERR_INVALID, lambda: call(gfm=gfm.data_ptr()))  # a map without features
    bad(gs.ERR_INVALID, lambda: call(features=feats.data_ptr(), channels=0, gfm=gfm.data_ptr()))
    bad(gs.ERR_INVALID, lambda: call(gf=feats.data_ptr()))  # grad_features without features
    bad(gs.ERR_INVALID, lambda: call(grad_da=gda.data_ptr()))  # not a depth frame
    bad(gs.ERR_INVALID, lambda: call(vertices=None))
    call(features=feats.data_ptr(), channels=3, gfm=gfm.data_ptr(), gf=feats.data_ptr(), gu=None, gl=None)  # features alone
    # a pipelined frame that overflowed its arena (gsb_render_async never regrows; a fresh context holds N = 10 k instances)
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        fresh.set_camera_model(_lens(gs, scenes.camera("inside"), fov_deg=180.0))
        fresh.set_backward(True)
        ui = scenes.camera("inside")
        dev = torch.empty((ui.height, ui.width, 4), dtype=torch.float32, device="cuda")
        fresh.render_into(ui, dev.data_ptr(), gs.FORMAT_RGBA32F, sync=False)
        torch.cuda.synchronize()
        bad(gs.ERR_INVALID, lambda: call(fresh), fresh)
        with pytest.raises(gs.GsbError):
            fresh.stats()  # reports (and clears) the overflow
    finally:
        fresh.close()
    fctx.render(u)
    params, m, s2 = gs.raw_parameters(v), torch.zeros_like(v), torch.zeros_like(v)
    fctx.adam_step(params, m, s2, torch.zeros_like(v), v.clone(), gs.adam_config([0.0] * 6))
    bad(gs.ERR_INVALID, call)  # the scene was stepped after the frame
    fctx.set_sh_storage(True)
    fctx.upload(vtx)
    fctx.render(u)
    bad(gs.ERR_INVALID, call)  # fp16 SH
    fctx.set_sh_storage(False)
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        bad(gs.ERR_INVALID, lambda: call(c0), c0)
    finally:
        grp.close()
    sc = gs.ShardedContext(0, 0, 1, gs.shard_unique_id())
    try:
        bad(gs.ERR_INVALID, lambda: call(sc), sc)
    finally:
        sc.close()


def test_translation_identity_at_full_size(gs):
    import sys
    from pathlib import Path

    torch = _torch()
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    u = bench.cameras(gs, wl)[0]
    ctx = gs.Context(0)
    try:
        ctx.set_tile_cull(1)
        ctx.set_backward(True)
        ctx.set_camera_model(_lens(gs, u, fov_deg=180.0))
        v = torch.from_numpy(bench.make_scene(gs, wl)).cuda()
        ctx.upload(v)
        ctx.render_into(u, torch.empty((u.height, u.width, 4), dtype=torch.float32, device="cuda").data_ptr())
        gi = torch.randn((u.height, u.width, 4), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
        gv, gu, gl, _, _ = _call(gs, ctx, v, gi)
    finally:
        ctx.close()
    gp = gv[:, 0:3]
    res, scale = translation_identity(gp.sum(0), np.abs(gp).sum(0), u, gu[gs.UBO_FLOAT_WORDS])
    print("fisheye translation identity: residual", res, "scale", scale)
    assert np.abs(gu).max() > 0 and np.abs(gl).max() > 0
    assert (np.abs(res) <= 1e-5 * scale).all(), (res, scale)


def test_render_torch_lens_and_ubo(gs, fctx):
    torch = _torch()
    vtx, u, cam = _case(gs, "odd_size")
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    v = torch.from_numpy(vtx).cuda().requires_grad_()
    ubo = torch.tensor(gs.pack_uniforms(u), device="cuda", requires_grad=True)
    lens = gs.lens_tensor(cam, "cuda").requires_grad_()
    with pytest.raises(ValueError):
        gs.render_torch(fctx, v, u, ubo=ubo)  # a fisheye context without lens=
    fctx.set_camera_model(None)  # the lens comes from the tensor, max_theta from fisheye_camera's default
    g = torch.from_numpy(grad_image(u)).cuda()
    img = gs.render_torch(fctx, v, u, ubo=ubo, lens=lens)
    assert fctx.camera is None
    (img * g).sum().backward()
    default = gs.lens_camera(lens, gs.fisheye_camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.k).max_theta)
    fctx.set_camera_model(default)
    fctx.render(u)
    wv, wu, wl, _, _ = _call(gs, fctx, v.detach(), g)
    assert rel(v.grad.cpu().numpy(), wv) <= 1e-6
    assert rel(ubo.grad.cpu().numpy(), wu[gs.UBO_FLOAT_WORDS]) <= 1e-6
    assert rel(lens.grad.cpu().numpy(), wl[1:9]) <= 1e-6
    # the context's own model is kept (and its max_theta used); frozen vertices give the same camera words
    ubo.grad = lens.grad = None
    frozen = v.detach()
    fctx.set_camera_model(cam)
    img = gs.render_torch(fctx, frozen, u, ubo=ubo, lens=lens)
    assert bytes(fctx.camera) == bytes(cam)
    (img * g).sum().backward()
    fctx.render(u)
    _, wu, wl, _, _ = _call(gs, fctx, frozen, g, vertices=False)
    assert rel(ubo.grad.cpu().numpy(), wu[gs.UBO_FLOAT_WORDS]) <= 1e-6 and rel(lens.grad.cpu().numpy(), wl[1:9]) <= 1e-6
    # a lens the setter refuses raises and leaves the model as it was
    bad = lens.detach().clone()
    bad[4] = -0.5
    with pytest.raises(gs.GsbError):
        gs.render_torch(fctx, frozen, u, lens=bad)
    assert bytes(fctx.camera) == bytes(cam)


def _pose_run(gs, ctx, v, u, target, pos0, q0, fov, W, H, pos, q):
    torch = _torch()
    opt = torch.optim.Adam([{"params": [pos], "lr": POSE_LR_POS}, {"params": [q], "lr": POSE_LR_ROT}])
    lens = gs.lens_tensor(ctx.camera, "cuda")
    losses = []
    for _ in range(POSE_STEPS):
        opt.zero_grad()
        ubo = gs.uniforms_torch(pos, q / q.norm(), fov, 0.1, 1000.0, W, H)
        img = gs.render_torch(ctx, v, u, ubo, lens=lens)
        loss = ((img[..., :3] - target) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    with torch.no_grad():
        ubo = gs.uniforms_torch(pos, q / q.norm(), fov, 0.1, 1000.0, W, H)
        final = float(((gs.render_torch(ctx, v, u, ubo, lens=lens)[..., :3] - target) ** 2).sum())
    return losses, final


@pytest.mark.parametrize("fov_deg", [140.0, 180.0])
def test_pose_refinement_through_the_lens(gs, fctx, fov_deg):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    pos0, q0, fov, W, H = [0.0, 0.0, 5.0], [1.0, 0.0, 0.0, 0.0], 45.0, 640, 480
    u = gs.uniforms_from_camera(pos0, q0, fov, 0.1, 1000.0, W, H)
    fctx.set_camera_model(_lens(gs, u, fov_deg=fov_deg, k=(0.01, -0.001, 0.0, 0.0)))
    v = torch.from_numpy(vtx).cuda()
    with torch.no_grad():
        target = gs.render_torch(fctx, v, u)[..., :3].clone()
    pos = torch.tensor([0.03, -0.02, 5.04], dtype=torch.float64, requires_grad=True)
    q = torch.tensor(scenes.quat_axis_angle([0.3, 1.0, 0.2], 1.0), dtype=torch.float64, requires_grad=True)
    e_pos0, e_rot0 = float(np.linalg.norm(pos.detach().numpy() - pos0)), _quat_angle_deg(q.detach().numpy(), np.array(q0))
    losses, final = _pose_run(gs, fctx, v, u, target, pos0, q0, fov, W, H, pos, q)
    e_pos, e_rot = float(np.linalg.norm(pos.detach().numpy() - pos0)), _quat_angle_deg(q.detach().numpy(), np.array(q0))
    print(f"fisheye {fov_deg:.0f} pose refinement: loss {losses[0]:.4g} -> {final:.4g}; translation {100 * e_pos0:.2f} -> "
          f"{100 * e_pos:.2f} cm; rotation {e_rot0:.3f} -> {e_rot:.3f} deg")
    assert final < 0.25 * losses[0], (losses[0], final)
    assert e_pos <= 0.5 * e_pos0 and e_rot <= 0.5 * e_rot0, (e_pos0, e_pos, e_rot0, e_rot)


def test_lens_self_calibration(gs, fctx):
    torch = _torch()
    _, vtx, u = scenes.c1()
    true = _lens(gs, u, fov_deg=150.0, k=(0.02, -0.003, 0.0, 0.0))
    fctx.set_camera_model(true)
    v = torch.from_numpy(vtx).cuda()
    with torch.no_grad():
        target = gs.render_torch(fctx, v, u)[..., :3].clone()
    t0 = gs.lens_tensor(true).double()
    start = t0.clone()
    start[0:2] *= 1.03
    start[2:4] += 4.0
    start[4] += 0.02
    # Adam steps each word by about lr: the leaf is the lens in units of 1 px (fx, fy, cx, cy) and of k_j such that every k
    # word moves theta_d by about the same at the lens's edge (t2^j ~ 2.6^j), which keeps theta_d increasing on the way
    unit = torch.tensor([1.0, 1.0, 1.0, 1.0, 1e-3, 1e-4, 1e-5, 1e-6], dtype=torch.float64)
    delta = torch.zeros(8, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([delta], lr=0.1)

    def err(x):
        d = (x.detach() - t0).abs()
        return [float(d[0:2].max()), float(d[2:4].max()), float(d[4])]

    losses = []
    for _ in range(200):
        opt.zero_grad()
        lens = start + delta * unit
        img = gs.render_torch(fctx, v, u, lens=lens.float())
        loss = ((img[..., :3] - target) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    lens = (start + delta * unit).detach()
    with torch.no_grad():
        final = float(((gs.render_torch(fctx, v, u, lens=lens.float())[..., :3] - target) ** 2).sum())
    e0, e1 = err(start), err(lens)
    print(f"lens self-calibration: loss {losses[0]:.4g} -> {final:.4g}; focal, principal point, k1 error {e0} -> {e1}")
    assert final < 0.25 * losses[0], (losses[0], final)
    for a, b in zip(e0, e1):
        assert b <= 0.5 * a, (e0, e1)
    assert bytes(fctx.camera) == bytes(true)


def test_scene_adam_camera_outputs(gs, fctx):
    from test_gpu_adam import TRAIN_LR

    torch = _torch()
    vtx, u, cam = _case(gs, "c1")
    v0 = torch.from_numpy(vtx).cuda()
    g = torch.from_numpy(grad_image(u)).cuda()
    torch.use_deterministic_algorithms(True)
    try:
        results = {}
        for ask in (False, True):
            for model in (None, cam):
                fctx.set_camera_model(model)
                opt = gs.SceneAdam(fctx, v0, TRAIN_LR)
                opt.render(u)
                gu = torch.empty(40, dtype=torch.float32, device="cuda") if ask else None
                gl = torch.empty(8, dtype=torch.float32, device="cuda") if ask and model is not None else None
                if ask:  # the entry's words for the same frame
                    if model is None:
                        want_u = torch.empty(40, dtype=torch.float32, device="cuda")
                        fctx._backward(opt.vertices.data_ptr(), g.data_ptr(), None, gs._torch_stream_arg(torch.cuda.current_stream()),
                                       grad_uniforms_ptr=want_u.data_ptr())
                        torch.cuda.synchronize()
                        want = (want_u.cpu().numpy(), None)
                    else:
                        _, wu, wl, _, _ = _call(gs, fctx, opt.vertices, g, vertices=False)
                        want = (wu.astype(np.float32), wl[1:9].astype(np.float32))
                if model is None and ask:
                    with pytest.raises(ValueError):
                        opt.step(g, grad_lens=torch.empty(8, dtype=torch.float32, device="cuda"))
                opt.step(g, grad_uniforms=gu, grad_lens=gl)
                torch.cuda.synchronize()
                results[(ask, model is None)] = (opt.grad.cpu().numpy(), opt.vertices.cpu().numpy())
                if ask:
                    assert np.array_equal(gu.cpu().numpy(), want[0])
                    if gl is not None:
                        assert np.array_equal(gl.cpu().numpy(), want[1])
        for pin in (True, False):
            for a, b in zip(results[(False, pin)], results[(True, pin)]):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    finally:
        torch.use_deterministic_algorithms(False)
        fctx.set_camera_model(None)


def test_scene_adam_joint_pose_refinement(gs, fctx):
    """Three fisheye views with perturbed poses: training the scene and the poses together lowers the pose error and ends
    with a lower loss than training the scene with the poses frozen."""
    from test_gpu_adam import POSES, TRAIN_LR

    torch = _torch()
    W, H, fov = 320, 240, 45.0
    u0 = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], fov, 0.1, 1000.0, W, H)
    fctx.set_camera_model(_lens(gs, u0, fov_deg=140.0, k=(0.01, 0.0, 0.0, 0.0)))
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    poses = POSES[:3]
    views = [gs.uniforms_from_camera(p, q, fov, 0.1, 1000.0, W, H) for p, q in poses]
    with torch.no_grad():
        targets = [gs.render_torch(fctx, full, u).clone() for u in views]
    start = full[::2].contiguous()
    rng = np.random.default_rng(11)
    pert = [(np.asarray(p, np.float64) + rng.normal(0, 0.02, 3), np.asarray(q, np.float64)) for p, q in poses]
    g = torch.empty((H, W, 4), dtype=torch.float32, device="cuda")

    def run(refine):
        pos = [torch.tensor(p, requires_grad=refine) for p, _ in pert]
        rot = [torch.tensor(q, requires_grad=refine) for _, q in pert]
        popt = torch.optim.Adam(pos + rot, lr=1e-3) if refine else None
        opt = gs.SceneAdam(fctx, start, TRAIN_LR)
        gu = torch.empty(40, dtype=torch.float32, device="cuda")
        loss = 0.0
        for it in range(240):
            k = it % 3
            ubo = gs.uniforms_torch(pos[k], rot[k] / rot[k].norm(), fov, 0.1, 1000.0, W, H)
            img = opt.render(gs.unpack_uniforms(ubo.detach().cpu().numpy(), W, H))
            loss_k = fctx.image_loss(img, targets[k], 0.2, grad_image=g)
            opt.step(g, grad_uniforms=gu if refine else None)
            if refine:
                ubo.backward(gu[gs.UBO_FLOAT_WORDS].cpu().double())
                popt.step()
                popt.zero_grad()
            if it >= 240 - 3:
                loss += float(loss_k[0])
        err = sum(float(np.linalg.norm(p.detach().numpy() - np.asarray(t[0]))) for p, t in zip(pos, poses))
        return loss, err

    frozen_loss, err0 = run(False)
    loss, err = run(True)
    print(f"joint pose refinement: loss {frozen_loss:.5f} (poses frozen) vs {loss:.5f}; pose error {err0:.4f} -> {err:.4f}")
    assert err < err0 and loss < frozen_loss, (err0, err, frozen_loss, loss)
    fctx.set_camera_model(None)
