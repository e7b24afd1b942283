"""gsb_set_camera_model's fisheye lens on the GPU: frames and gradients against the float64 restatement (tests/fisheye_ref.py)
blended over the frame's own level-0 lists, the frame equalities of the pinhole path within fisheye frames, the pinhole frame
unchanged, the backward following the recorded frame, the error codes and training through the lens."""
import math

import numpy as np
import pytest

import edge_scene
import fisheye_ref
import scenes
from backward_util import GROUPS, expect, grad_image, rel

pytestmark = pytest.mark.gpu

# the fraction of pixels where the fp32 frame and the float64 restatement may take a different side of one of the blend's
# step functions (alpha >= 1/255, the T < 1e-4 break) -- the pixels the pinhole tests flag with the oracle's probes; the
# restatement has no fp32 twin to probe, so they are bounded by count instead
STEP_FRACTION = 2e-3


def _torch():
    import torch

    return torch


@pytest.fixture
def fctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _lens(gs, u, fov_deg=None, k=(0.0, 0.0, 0.0, 0.0), max_theta=None, focal=None):
    """A fisheye over u's frame: focal `focal` (default that of u's pinhole tan_fovx), or the equidistant focal that maps
    fov_deg / 2 to the frame's half width; principal point at the frame's centre pixel."""
    if focal is None:
        focal = (u.width / 2.0) / math.radians(fov_deg / 2.0) if fov_deg else u.width / (2.0 * u.tan_fovx)
    if max_theta is None and fov_deg:
        max_theta = min(math.radians(fov_deg / 2.0) + 0.3, 3.0)
    return gs.fisheye_camera(focal, focal, (u.width - 1) / 2.0, (u.height - 1) / 2.0, k, max_theta)


def _frame_lists(gs, ctx, u, vtx, cam):
    """Render u in debug mode at level 0 and return (image, {"vals", "ranges"}) after checking that every Gaussian's tile
    AABB (GSB_BUF_ATTR) equals the float64 restatement's but for rounding-boundary cases."""
    ctx.set_debug(True)
    ctx.set_tile_cull(0)
    img = ctx.render(u)
    frame = {"vals": ctx.download(gs.BUF_VALS_SORTED), "ranges": ctx.download(gs.BUF_TILE_BOUNDARY)}
    attr = ctx.download(gs.BUF_ATTR)
    ctx.set_debug(False)
    box = fisheye_ref.aabb(vtx, u, cam)
    got = attr["aabb"].astype(np.int64)
    mism = np.any(got != box, axis=1) & (box[:, 0] >= 0)
    assert mism.mean() <= 1e-3 and np.abs(got - box)[mism].max(initial=0) <= 1, (mism.sum(), u.width)
    return img, frame


def _check_frame(img, ref, what):
    err = np.abs(img[..., :3].astype(np.float64) - ref["image"]).max(-1)
    bad = err > 1e-4
    assert bad.mean() <= STEP_FRACTION and err.max() < 0.5, (what, bad.mean(), err.max())


def _edge_vertices():
    return edge_scene.vertices()[0]


CASES = {  # name: (scene, pose, lens arguments)
    "c1": ("c1", "c1", {}),
    "odd_size": ("c1", "odd_size", {"k": (0.02, -0.01, 0.002, 0.0)}),
    "edge": ("edge", "c1", {}),
    "fov90": ("c1", "c1", {"fov_deg": 90.0}),
    "fov180": ("c1", "inside", {"fov_deg": 180.0}),
    "fov200": ("c1", "inside", {"fov_deg": 200.0}),
    "k_nonzero": ("c1", "inside", {"fov_deg": 150.0, "k": (-0.05, 0.004, -0.0002, 0.0)}),
}


def _case(gs, name):
    scene, pose, kw = CASES[name]
    vtx = scenes.c1()[1] if scene == "c1" else _edge_vertices()
    u = scenes.camera(pose)
    return vtx, u, _lens(gs, u, **kw)


# the edge scene's needles (scale ratios to 1e4) and saturated near-plane rows are ill-conditioned between fp32 and float64
# (the pinhole tests hold them to the fp32 oracle instead); here it takes part in the bit-exact equalities below
@pytest.mark.parametrize("name", sorted(set(CASES) - {"edge"}))
def test_frame_matches_float64_reference(gs, fctx, name):
    vtx, u, cam = _case(gs, name)
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    img, frame = _frame_lists(gs, fctx, u, vtx, cam)
    assert frame["vals"].size > 0
    _check_frame(img, fisheye_ref.reference(vtx, u, cam, frame), name)


def _render_all(gs, ctx, u, fmt=None):
    return ctx.render(u, gs.FORMAT_RGBA32F if fmt is None else fmt)


@pytest.mark.parametrize("name", ["c1", "edge", "fov200", "k_nonzero"])
def test_equalities_within_fisheye_frames(gs, oracle, fctx, name):
    vtx, u, cam = _case(gs, name)
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    for aa, bg in ((False, None), (True, [0.2, 0.5, 0.9])):
        fctx.set_antialiased(aa)
        fctx.set_background(bg)
        ref = None
        for timers in (True, False):  # direct launches, then the captured middle graph
            fctx.set_timers(timers)
            for level in (0, 1, 2):
                fctx.set_tile_cull(level)
                img = _render_all(gs, fctx, u)
                if ref is None:
                    ref = img
                assert np.array_equal(img.view(np.uint32), ref.view(np.uint32)), (name, aa, timers, level)
        fctx.set_timers(True)
        fctx.set_tile_cull(0)
        assert np.array_equal(_render_all(gs, fctx, u, gs.FORMAT_RGBA8), oracle.pack_unorm8(ref))
        assert np.array_equal(_render_all(gs, fctx, u, gs.FORMAT_BGRA8), oracle.pack_unorm8(ref, bgra=True))
        tiles_y = (u.height + 15) // 16
        cut = max(1, tiles_y // 3)
        top = fctx.render(u, rows=(0, cut))
        bottom = fctx.render(u, rows=(cut, tiles_y))
        assert np.array_equal(np.concatenate([top, bottom]).view(np.uint32), ref.view(np.uint32))
        if name == "edge":  # FAST's bound does not hold on the 45-degree needles for the pinhole either (DESIGN.md section 2)
            continue
        fctx.set_mode(gs.MODE_FAST)
        fast = _render_all(gs, fctx, u)
        fctx.set_mode(gs.MODE_EXACT)
        err = np.abs(fast - ref).max(-1)  # __expf may flip a step decision on a few pixels, as against the float64 reference
        assert (err > 1e-4).mean() <= STEP_FRACTION and err.max() <= 1e-3, (name, (err > 1e-4).mean(), err.max())
    fctx.set_antialiased(False)
    fctx.set_background(None)


def test_antialiased_opacity_and_background(gs, fctx):
    vtx, u, cam = _case(gs, "fov180")
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    fctx.set_debug(True)
    fctx.render(u)
    plain = fctx.download(gs.BUF_ATTR)
    fctx.set_antialiased(True)
    fctx.render(u)
    aa = fctx.download(gs.BUF_ATTR)
    fctx.set_debug(False)
    live = plain["color_radii"][:, 3] > 0
    assert live.sum() > 1000
    assert np.array_equal(aa["conic_opacity"][live, :3], plain["conic_opacity"][live, :3])
    A, B, C = (plain["conic_opacity"][live, j].astype(np.float64) for j in range(3))
    det_k = A * C - B * B
    a, b, c = C / det_k, -B / det_k, A / det_k  # cov2d + 0.3 I
    comp = np.sqrt(np.maximum(0.0, ((a - 0.3) * (c - 0.3) - b * b) / (a * c - b * b)))
    want = plain["conic_opacity"][live, 3] * comp
    assert np.allclose(aa["conic_opacity"][live, 3], want, rtol=1e-3, atol=1e-6)
    fctx.set_antialiased(False)
    # the background: every pixel moves by T_final * bg
    fctx.set_backward(True)
    black = fctx.render(u)
    fctx.set_background([0.25, 0.5, 1.0])
    over = fctx.render(u)
    fctx.set_background(None)
    empty = (black[..., :3] == 0).all(-1)
    assert empty.any() and np.array_equal(over[empty, :3], np.tile([0.25, 0.5, 1.0], (empty.sum(), 1)).astype(np.float32))
    assert (over[..., :3] >= black[..., :3]).all()


def test_pinhole_frame_is_unaffected(gs, fctx):
    vtx, u, cam = _case(gs, "fov180")
    fctx.upload(vtx)
    base = fctx.render(u)
    for reset in (None, gs.CameraModel(gs.CAMERA_PINHOLE)):
        fctx.set_camera_model(cam)
        fish = fctx.render(u)
        assert not np.array_equal(fish, base)
        fctx.set_camera_model(reset)
        assert np.array_equal(fctx.render(u).view(np.uint32), base.view(np.uint32))


def test_on_axis_matches_pinhole(gs, fctx):
    """Gaussians with r / z < 1e-3: the fisheye with the pinhole's focal and centre differs from the pinhole by
    f (tan(theta) - theta) <= f theta^3 / 3 < 1e-6 px in uv and by O(theta^2) = 1e-6 relative in J, so uv agrees within
    1e-4 px plus a few fp32 roundings of uv, and the conic within 1e-4 of its largest entry (2e-6 from J, the rest for the
    roundings of det's cancellation, which the two cameras' different op sequences take differently)."""
    _, vtx, u = scenes.c1()
    rng = np.random.default_rng(3)
    n = 2000
    v = vtx[:n].copy()
    z = rng.uniform(2.0, 8.0, n)
    ang = rng.uniform(0, 2 * np.pi, n)
    rr = z * rng.uniform(0.0, 9e-4, n)
    # camera (0, 0, 5) looking down -z in world (view z = 5 - p.z): place the Gaussians on its axis
    v[:, 0], v[:, 1], v[:, 2] = rr * np.cos(ang), rr * np.sin(ang), 5.0 - z
    v[:, 4:7] = np.exp(rng.uniform(-4.5, -3.0, (n, 3)))
    fctx.upload(v.astype(np.float32))
    fctx.set_debug(True)
    fctx.render(u)
    pin = fctx.download(gs.BUF_ATTR)
    fctx.set_camera_model(gs.fisheye_camera(u.width / (2 * u.tan_fovx), u.height / (2 * u.tan_fovy), (u.width - 1) / 2,
                                            (u.height - 1) / 2))
    fctx.render(u)
    fish = fctx.download(gs.BUF_ATTR)
    fctx.set_debug(False)
    live = (pin["color_radii"][:, 3] > 0) & (fish["color_radii"][:, 3] > 0)
    assert live.sum() > 0.9 * n
    duv = np.abs(pin["uv"][live].astype(np.float64) - fish["uv"][live])
    assert duv.max() <= 1e-4 + 4 * np.spacing(np.float32(u.width)), duv.max()
    for j in range(3):
        a, b = pin["conic_opacity"][live, j].astype(np.float64), fish["conic_opacity"][live, j].astype(np.float64)
        scale = np.abs(pin["conic_opacity"][live, :3]).max(1)
        assert (np.abs(a - b) <= 1e-4 * scale).all(), j


def test_wide_lens_draws_gaussians_behind_the_camera(gs, fctx):
    u = gs.uniforms_from_camera([0, 0, 0], [1, 0, 0, 0], 60.0, 0.1, 1000.0, 512, 512)
    cam = _lens(gs, u, fov_deg=240.0, max_theta=math.radians(120.0))
    rng = np.random.default_rng(5)
    _, vtx, _ = scenes.c1(n=3000)
    v = vtx.copy()
    # view z < 0 at 100-115 degrees off the axis; the view looks down world -z, so view z = -world z
    th = np.radians(rng.uniform(100, 115, v.shape[0]))
    ph = rng.uniform(0, 2 * np.pi, v.shape[0])
    d = rng.uniform(2, 4, v.shape[0])
    v[:, 0], v[:, 1], v[:, 2] = d * np.sin(th) * np.cos(ph), -d * np.sin(th) * np.sin(ph), -d * np.cos(th)
    fctx.upload(v)
    fctx.set_camera_model(cam)
    fctx.set_debug(True)
    img = fctx.render(u)
    attr = fctx.download(gs.BUF_ATTR)
    fctx.set_debug(False)
    tz = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T @ np.c_[v[:, :3], np.ones(len(v))].T
    assert (tz[2] < 0).all()
    assert (attr["color_radii"][:, 3] > 0).mean() > 0.95
    assert img[..., :3].max() > 0.1


# ---------------------------------------------------------------------------------------------------------------------
# the backward pass
# ---------------------------------------------------------------------------------------------------------------------
def _backward(gs, ctx, vtx, g, density=None):
    torch = _torch()
    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    gi = torch.from_numpy(g).cuda()
    out = torch.full_like(v, float("nan"))
    dens = None if density is None else torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
    ctx._backward(v.data_ptr(), gi.data_ptr(), out.data_ptr(), None,
                  density_ptr=None if dens is None else dens.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.float64), None if dens is None else dens.cpu().numpy()


GRAD_CASES = {"c1": "c1", "odd_size": "odd_size", "inside": "fov180", "wide": "wide"}


def _grad_case(gs, name):
    if name == "wide":  # rows near the axis and near max_theta
        u = gs.uniforms_from_camera([0.2, -0.1, 0.4], scenes.quat_axis_angle([0, 1, 0], 20), 60.0, 0.1, 1000.0, 480, 400)
        return scenes.c1()[1], u, _lens(gs, u, fov_deg=190.0, k=(0.01, -0.002, 0.0, 0.0), max_theta=math.radians(97.0))
    return _case(gs, GRAD_CASES[name])


@pytest.mark.parametrize("name", sorted(GRAD_CASES))
def test_gradient_matches_float64_reference(gs, fctx, name):
    vtx, u, cam = _grad_case(gs, name)
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    fctx.set_backward(True)
    img, frame = _frame_lists(gs, fctx, u, vtx, cam)
    g = grad_image(u)
    ref = fisheye_ref.reference(vtx, u, cam, frame, g)
    _check_frame(img, ref, name)
    keep = ~ref["exclude"]
    assert keep.sum() > 100
    for det in (False, True):
        fctx.set_backward_deterministic(det)
        fctx.set_tile_cull(0)
        fctx.render(u)
        got, _ = _backward(gs, fctx, vtx, g)
        assert np.isfinite(got).all()
        for group, cols in GROUPS.items():
            r = rel(got[keep, cols], ref["grad"][keep, cols])
            assert r <= 1e-3, (name, det, group, r)
        assert not got[:, 3].any()
    fctx.set_backward_deterministic(False)


def test_deterministic_levels_density_and_background_gradient(gs, fctx):
    torch = _torch()
    vtx, u, cam = _grad_case(gs, "wide")
    fctx.upload(vtx)
    fctx.set_camera_model(cam)
    fctx.set_backward(True)
    fctx.set_backward_deterministic(True)
    g = grad_image(u)
    outs = []
    for level in (0, 1, 2):
        fctx.set_tile_cull(level)
        fctx.render(u)
        outs.append(_backward(gs, fctx, vtx, g, density=True))
    for got, dens in outs[1:]:
        assert np.array_equal(got, outs[0][0]) and np.array_equal(dens, outs[0][1])
    fctx.set_tile_cull(0)
    dens = outs[0][1]
    seen = dens[:, 2] > 0
    assert seen.sum() > 100 and (dens[:, 3][seen] > 0).all()
    # the background gradient is sum_p T_final g: T_final from the frame over white minus the frame over black
    fctx.render(u)
    gi = torch.from_numpy(g).cuda()
    got_bg = fctx.background_gradient(gi).cpu().numpy().astype(np.float64)
    fctx.set_background([1.0, 1.0, 1.0])
    white = fctx.render(u)
    fctx.set_background(None)
    black = fctx.render(u)
    T = (white[..., :3].astype(np.float64) - black[..., :3])
    want = (T * g[..., :3]).sum((0, 1))
    assert np.allclose(got_bg, want, rtol=1e-4, atol=1e-2), (got_bg, want)
    fctx.set_backward_deterministic(False)


def test_backward_follows_the_recorded_frame(gs, fctx):
    vtx, u, cam = _case(gs, "fov180")
    fctx.upload(vtx)
    fctx.set_backward(True)
    fctx.set_backward_deterministic(True)
    g = grad_image(u)
    fctx.set_camera_model(cam)
    fctx.render(u)
    want, _ = _backward(gs, fctx, vtx, g)
    fctx.render(u)
    fctx.set_camera_model(None)  # after the frame: the backward still follows the fisheye frame
    got, _ = _backward(gs, fctx, vtx, g)
    assert np.array_equal(got, want)
    fctx.render(u)  # a pinhole frame recorded while a fisheye is set is differentiated as a pinhole frame
    pin, _ = _backward(gs, fctx, vtx, g)
    fctx.set_camera_model(cam)
    assert np.array_equal(_backward(gs, fctx, vtx, g)[0], pin)
    fctx.set_backward_deterministic(False)


def test_error_cases(gs, fctx):
    torch = _torch()
    good = gs.fisheye_camera(300.0, 300.0, 319.5, 239.5, max_theta=1.5)
    assert gs.lib.gsb_set_camera_model(None, good) == gs.ERR_INVALID

    def fish(**kw):
        c = gs.fisheye_camera(300.0, 300.0, 319.5, 239.5, max_theta=1.5)
        for key, val in kw.items():
            if key == "k":
                c.k = (type(c.k))(*val)
            else:
                setattr(c, key, val)
        return c

    bad = [fish(kind=7), fish(fx=0.0), fish(fy=-1.0), fish(fx=float("inf")), fish(cx=float("nan")), fish(cy=float("inf")),
           fish(k=(0.0, float("nan"), 0.0, 0.0)), fish(max_theta=0.0), fish(max_theta=float(np.float32(np.pi))),
           fish(max_theta=-0.5), fish(max_theta=float("nan")),
           fish(k=(-0.5, 0.0, 0.0, 0.0)),                          # d theta_d / d theta = 1 - 1.5 t^2 < 0 past 0.82
           fish(k=(0.0, 0.0, 0.0, -0.1), max_theta=1.4),           # 1 - 0.9 t^8 < 0 past 1.01
           fish(k=(-0.5, 0.1, 0.0, 0.0), max_theta=1.9)]           # 1 - 1.5 t^2 + 0.5 t^4 dips below 0 inside the range
    _, vtx, u = scenes.c1()
    fctx.upload(vtx)
    fctx.set_camera_model(good)
    base = fctx.render(u)
    for c in bad:
        expect(gs, fctx, gs.ERR_INVALID, lambda c=c: fctx.set_camera_model(c), "gsb_set_camera_model")
        assert np.array_equal(fctx.render(u).view(np.uint32), base.view(np.uint32))  # the setting is unchanged
    # the camera gradient refusals, then render_torch's
    fctx.set_backward(True)
    fctx.render(u)
    v = torch.from_numpy(vtx).cuda()
    gi = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    gv, gu = torch.empty_like(v), torch.empty(40, dtype=torch.float32, device="cuda")
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
    expect(gs, fctx, gs.ERR_INVALID, lambda: fctx._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), None,
                                                            grad_uniforms_ptr=gu.data_ptr()), "gsb_render_backward_camera")
    expect(gs, fctx, gs.ERR_INVALID, lambda: fctx._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), None,
                                                            grad_uniforms_ptr=gu.data_ptr(), density_ptr=dens.data_ptr()),
           "gsb_render_backward_density")
    fctx._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), None, density_ptr=dens.data_ptr())  # vertices only: fine
    ubo = torch.tensor(gs.pack_uniforms(u), device="cuda", requires_grad=True)
    with pytest.raises(ValueError):
        gs.render_torch(fctx, v, u, ubo=ubo)
    # sharded contexts and gsb_group ranks have only the pinhole camera
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, lambda: c0.set_camera_model(good), "gsb_set_camera_model")
    finally:
        grp.close()
    sc = gs.ShardedContext(0, 0, 1, gs.shard_unique_id())
    try:
        expect(gs, sc, gs.ERR_INVALID, lambda: sc.set_camera_model(good), "gsb_set_camera_model")
    finally:
        sc.close()


# ---------------------------------------------------------------------------------------------------------------------
# training and full size
# ---------------------------------------------------------------------------------------------------------------------
def _fisheye_views(gs, ctx):
    from test_gpu_adam import _training_setup

    u0 = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 320, 240)
    ctx.set_camera_model(_lens(gs, u0, fov_deg=140.0, k=(0.01, 0.0, 0.0, 0.0)))
    return _training_setup(gs, ctx)


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_scene_adam_fits_from_fisheye_views(gs, fctx, selective):
    from test_gpu_adam import TRAIN_LR, _evaluate

    torch = _torch()
    start, views, targets = _fisheye_views(gs, fctx)
    opt = gs.SceneAdam(fctx, start, TRAIN_LR, selective=selective)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    loss0, dssim0 = _evaluate(gs, fctx, opt, views, targets)
    for it in range(300):
        k = it % 3
        fctx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g)
    loss1, dssim1 = _evaluate(gs, fctx, opt, views, targets)
    print(f"SceneAdam fisheye ({'selective' if selective else 'dense'}): loss {loss0:.5f} -> {loss1:.5f}")
    assert loss1 < 0.8 * loss0 and dssim1 < dssim0


def test_render_torch_fits_from_fisheye_views(gs, fctx):
    torch = _torch()
    _, views, targets = _fisheye_views(gs, fctx)
    fixed = torch.from_numpy(scenes.c1()[1]).cuda()  # the targets' geometry, with the colours to recover perturbed
    dc = (fixed[:, 12:15] * 0.5).requires_grad_()
    optim = torch.optim.Adam([dc], lr=0.02)

    def loss_at(k):
        v = torch.cat([fixed[:, :12], dc, fixed[:, 15:]], 1)
        return gs.image_loss_torch(fctx, gs.render_torch(fctx, v, views[k]), targets[k])

    with torch.no_grad():
        before = sum(float(loss_at(k)) for k in range(len(views)))
    for it in range(150):
        optim.zero_grad()
        loss = loss_at(it % len(views))
        loss.backward()
        optim.step()
    with torch.no_grad():
        after = sum(float(loss_at(k)) for k in range(len(views)))
    print(f"render_torch fisheye: loss {before:.5f} -> {after:.5f}")
    assert after < 0.5 * before


def test_full_size_levels_and_bands_agree(gs):
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    vtx = bench.make_scene(gs, wl)
    u = bench.cameras(gs, wl)[3]
    c = gs.Context(0)
    try:
        c.upload(vtx)
        c.set_camera_model(_lens(gs, u, fov_deg=180.0))
        ref = c.render(u)
        assert c.stats().num_instances > 0
        for level in (1, 2):
            c.set_tile_cull(level)
            assert np.array_equal(c.render(u).view(np.uint32), ref.view(np.uint32)), level
        tiles_y = (u.height + 15) // 16
        parts = [c.render(u, rows=(a, min(tiles_y, a + 30))) for a in range(0, tiles_y, 30)]
        assert np.array_equal(np.concatenate(parts).view(np.uint32), ref.view(np.uint32))
    finally:
        c.close()
