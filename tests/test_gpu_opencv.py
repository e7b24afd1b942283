"""gsb_set_camera_model's OpenCV (radial-tangential) lens on the GPU: frames, tile AABBs and gradients against the float64
restatement (tests/opencv_ref.py) blended over the frame's own level-0 lists, the frame equalities of the pinhole path within
OpenCV frames, the pinhole frame unchanged, k = 0 against the pinhole, the camera and lens gradients of
gsb_render_backward_fisheye, determinism, the error codes, the full-size garden stand-in, and training through the lens."""
import math

import numpy as np
import pytest

import opencv_ref
import scenes
from backward_util import GROUPS, expect, grad_image, rel, translation_identity
from test_gpu_fisheye import STEP_FRACTION, _backward, _check_frame
from test_gpu_fisheye_camera import _call, _render, _upstream

pytestmark = pytest.mark.gpu

UBO_GROUPS = {"camera_position": [0, 1, 2], "view_3x3": [20 + c * 4 + r for c in range(3) for r in range(3)],
              "view_translation": [32, 33, 34]}
LENS_GROUPS = {"focal": [0, 1], "principal_point": [2, 3], "radial": [4, 5], "tangential": [6, 7]}
DEAD_UBO = np.nonzero(~opencv_ref.LIVE_UBO)[0]
PHONE = (-0.12, 0.03, 0.0008, -0.0006)  # a typical phone main camera calibrated as OPENCV


def _torch():
    import torch

    return torch


@pytest.fixture
def octx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _lens(gs, u, k=(0.0, 0.0, 0.0, 0.0), aspect=1.0, shift=(0.0, 0.0), max_theta=None):
    """An OpenCV lens over u's frame: the pinhole's focal (fy = aspect fx), principal point at the frame's centre pixel plus
    `shift` pixels."""
    f = u.width / (2.0 * u.tan_fovx)
    return gs.opencv_camera(f, f * aspect, (u.width - 1) / 2.0 + shift[0], (u.height - 1) / 2.0 + shift[1], k, max_theta)


CASES = {  # name: (pose, lens arguments)
    "c1": ("c1", {}),
    "odd_size": ("odd_size", {"k": PHONE}),
    # from inside the cloud, culled at 60 degrees: past it the barrel polynomial is an extrapolation no calibration covers
    "inside": ("inside", {"k": (-0.28, 0.07, 0.0, 0.0), "max_theta": math.radians(60.0)}),
    "barrel": ("c1", {"k": (-0.28, 0.07, 0.0, 0.0)}),
    "pincushion": ("c1", {"k": (0.12, 0.03, 0.0, 0.0)}),
    "tangential": ("c1", {"k": (-0.05, 0.01, 0.006, -0.008), "aspect": 1.07}),
    "off_centre": ("odd_size", {"k": PHONE, "aspect": 0.93, "shift": (23.7, -17.2)}),
}


def _case(gs, name):
    pose, kw = CASES[name]
    u = scenes.camera(pose)
    return scenes.c1()[1], u, _lens(gs, u, **kw)


def _frame_lists(gs, ctx, u, vtx, cam):
    """Render u in debug mode at level 0 and return (image, {"vals", "ranges"}) after checking that every Gaussian's tile
    AABB (GSB_BUF_ATTR) equals the float64 restatement's but for rounding-boundary cases."""
    ctx.set_debug(True)
    ctx.set_tile_cull(0)
    img = ctx.render(u)
    frame = {"vals": ctx.download(gs.BUF_VALS_SORTED), "ranges": ctx.download(gs.BUF_TILE_BOUNDARY)}
    attr = ctx.download(gs.BUF_ATTR)
    ctx.set_debug(False)
    box = opencv_ref.aabb(vtx, u, cam)
    got = attr["aabb"].astype(np.int64)
    mism = np.any(got != box, axis=1) & (box[:, 0] >= 0)
    assert mism.mean() <= 1e-3 and np.abs(got - box)[mism].max(initial=0) <= 1, (mism.sum(), u.width)
    return img, frame


@pytest.mark.parametrize("name", sorted(CASES))
def test_frame_matches_float64_reference(gs, octx, name):
    vtx, u, cam = _case(gs, name)
    octx.upload(vtx)
    octx.set_camera_model(cam)
    img, frame = _frame_lists(gs, octx, u, vtx, cam)
    assert frame["vals"].size > 0
    ref = opencv_ref.reference(vtx, u, cam, frame)
    _check_frame(img, ref, name)


@pytest.mark.parametrize("name", ["c1", "tangential", "off_centre"])
def test_equalities_within_opencv_frames(gs, oracle, octx, name):
    vtx, u, cam = _case(gs, name)
    octx.upload(vtx)
    octx.set_camera_model(cam)
    for aa, bg in ((False, None), (True, [0.2, 0.5, 0.9])):
        octx.set_antialiased(aa)
        octx.set_background(bg)
        ref = ref_d = None
        for timers in (True, False):  # direct launches, then the captured middle graph
            octx.set_timers(timers)
            for level in (0, 1, 2):
                octx.set_tile_cull(level)
                img = octx.render(u)
                _, da = octx.render_depth(u)
                if ref is None:
                    ref, ref_d = img, da
                assert np.array_equal(img.view(np.uint32), ref.view(np.uint32)), (name, aa, timers, level)
                assert np.array_equal(da.view(np.uint32), ref_d.view(np.uint32)), (name, aa, timers, level)
        octx.set_timers(True)
        octx.set_tile_cull(0)
        assert np.array_equal(octx.render(u, gs.FORMAT_RGBA8), oracle.pack_unorm8(ref))
        assert np.array_equal(octx.render(u, gs.FORMAT_BGRA8), oracle.pack_unorm8(ref, bgra=True))
        tiles_y = (u.height + 15) // 16
        cut = max(1, tiles_y // 3)
        bands = np.concatenate([octx.render(u, rows=(0, cut)), octx.render(u, rows=(cut, tiles_y))])
        assert np.array_equal(bands.view(np.uint32), ref.view(np.uint32))
    octx.set_antialiased(False)
    octx.set_background(None)


def test_depth_is_view_space_z(gs, octx):
    """D = sum z alpha T and A of the frame against the float64 restatement's (the depth key of an OpenCV frame is z)."""
    vtx, u, cam = _case(gs, "tangential")
    octx.upload(vtx)
    octx.set_camera_model(cam)
    _, frame = _frame_lists(gs, octx, u, vtx, cam)
    _, da = octx.render_depth(u)
    ref = opencv_ref.reference(vtx, u, cam, frame)
    err = np.abs(da.astype(np.float64) - ref["depth_alpha"]) / np.maximum(1.0, np.abs(ref["depth_alpha"]))
    bad = err.max(-1) > 1e-4
    assert bad.mean() <= STEP_FRACTION and ref["depth_alpha"][..., 0].max() > 1.0, (bad.mean(), err.max())


def test_pinhole_frame_is_unaffected(gs, octx):
    vtx, u, cam = _case(gs, "barrel")
    octx.upload(vtx)
    base = octx.render(u)
    for reset in (None, gs.CameraModel(gs.CAMERA_PINHOLE)):
        octx.set_camera_model(cam)
        assert not np.array_equal(octx.render(u), base)
        octx.set_camera_model(reset)
        assert np.array_equal(octx.render(u).view(np.uint32), base.view(np.uint32))


def test_k0_matches_pinhole(gs, octx):
    """k = 0 with the pinhole's focal and centre pixel is the pinhole map: where the pinhole's 1.3 tan_fov clamp is inactive
    the records agree to fp32 roundings (the two cameras reach uv and J through different op sequences)."""
    vtx, u, _ = _case(gs, "c1")
    octx.upload(vtx)
    octx.set_debug(True)
    octx.render(u)
    pin = octx.download(gs.BUF_ATTR)
    octx.set_camera_model(_lens(gs, u))
    octx.render(u)
    ocv = octx.download(gs.BUF_ATTR)
    octx.set_debug(False)
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    t = (V @ np.c_[vtx[:, :3], np.ones(len(vtx))].T)[:3].T
    inside = (np.abs(t[:, 0] / t[:, 2]) < 1.29 * u.tan_fovx) & (np.abs(t[:, 1] / t[:, 2]) < 1.29 * u.tan_fovy)
    live = (pin["color_radii"][:, 3] > 0) & (ocv["color_radii"][:, 3] > 0) & inside
    assert live.sum() > 1000
    assert np.array_equal((pin["color_radii"][:, 3] > 0) & inside, (ocv["color_radii"][:, 3] > 0) & inside)
    duv = np.abs(pin["uv"][live].astype(np.float64) - ocv["uv"][live])
    assert duv.max() <= 1e-3, duv.max()
    scale = np.abs(pin["conic_opacity"][live, :3].astype(np.float64)).max(1)
    for j in range(3):
        d = np.abs(pin["conic_opacity"][live, j].astype(np.float64) - ocv["conic_opacity"][live, j])
        assert (d <= 1e-4 * scale).all(), (j, (d / scale).max())


def test_tangential_fold_is_culled(gs, octx):
    """Tangential terms strong enough to fold the map inside max_theta: Gaussians past the fold (det D <= 0) are culled,
    never splatted with a flipped Jacobian."""
    vtx, u, _ = _case(gs, "c1")
    cam = _lens(gs, u, k=(0.0, 0.0, 0.3, -0.25), max_theta=math.radians(60.0))
    octx.upload(vtx)
    octx.set_camera_model(cam)
    octx.set_debug(True)
    octx.render(u)
    attr = octx.download(gs.BUF_ATTR)
    octx.set_debug(False)
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    t = (V @ np.c_[vtx[:, :3], np.ones(len(vtx))].T)[:3].T
    det = opencv_ref.geo(t, cam)["det"]
    live = attr["color_radii"][:, 3] > 0
    folded = (t[:, 2] > 0.2) & (det < -1e-3)
    assert folded.sum() > 10 and not live[folded].any()


# ---------------------------------------------------------------------------------------------------------------------
# the backward pass
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["c1", "odd_size", "inside", "tangential", "off_centre"])
def test_gradient_matches_float64_reference(gs, octx, name):
    vtx, u, cam = _case(gs, name)
    octx.upload(vtx)
    octx.set_camera_model(cam)
    octx.set_backward(True)
    img, frame = _frame_lists(gs, octx, u, vtx, cam)
    g = grad_image(u)
    ref = opencv_ref.reference(vtx, u, cam, frame, g)
    _check_frame(img, ref, name)
    keep = ~ref["exclude"]
    assert keep.sum() > 100
    for det in (False, True):
        octx.set_backward_deterministic(det)
        octx.set_tile_cull(0)
        octx.render(u)
        got, _ = _backward(gs, octx, vtx, g)
        assert np.isfinite(got).all()
        for group, cols in GROUPS.items():
            r = rel(got[keep, cols], ref["grad"][keep, cols])
            assert r <= 1e-3, (name, det, group, r)
        assert not got[:, 3].any()
    octx.set_backward_deterministic(False)


REF_RUNS = [("c1", "colour", False), ("odd_size", "colour", True), ("tangential", "colour", False),
            ("off_centre", "colour", False), ("barrel", "colour", True), ("tangential", "depth", False),
            ("off_centre", "alpha", True), ("tangential", "feature", False)]


@pytest.mark.parametrize("name,kind,aa", REF_RUNS, ids=[f"{n}-{k}-{'aa' if a else 'plain'}" for n, k, a in REF_RUNS])
def test_camera_lens_and_vertex_gradients_match_float64_reference(gs, octx, name, kind, aa):
    torch = _torch()
    vtx, u, cam = _case(gs, name)
    octx.upload(vtx)
    octx.set_camera_model(cam)
    octx.set_antialiased(aa)
    octx.set_backward(True)
    _, frame = _frame_lists(gs, octx, u, vtx, cam)
    steps = opencv_ref.step_pixels(vtx, u, cam, frame, aa)
    assert steps.mean() < 0.05
    gi, gda, feats, gfm = _upstream(u, kind, steps, vtx.shape[0])
    ref = opencv_ref.reference(vtx, u, cam, frame, grad_image=gi, grad_da=gda, features=feats, grad_fm=gfm, antialiased=aa)
    keep = ~ref["exclude"]
    v = torch.from_numpy(vtx).cuda()
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    for det in (False, True):
        octx.set_backward_deterministic(det)
        _render(gs, octx, u, gda is not None)
        gv, gu, gl, _, _ = _call(gs, octx, v, t(gi), t(gda), t(feats), t(gfm))
        for group, words in UBO_GROUPS.items():
            r = rel(gu[words], ref["grad_ubo"][words])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
        for group, words in LENS_GROUPS.items():
            r = rel(gl[1:9][words], ref["grad_lens"][words])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
        assert not gu[DEAD_UBO].any() and gl[0] == 0 and gl[9] == 0
        for group, cols in GROUPS.items():
            r = rel(gv[keep][:, cols], ref["grad"][keep][:, cols])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
    octx.set_backward_deterministic(False)
    octx.set_antialiased(False)


def test_deterministic_words(gs, octx):
    torch = _torch()
    vtx, u, cam = _case(gs, "tangential")
    octx.upload(vtx)
    octx.set_camera_model(cam)
    octx.set_backward(True)
    octx.set_backward_deterministic(True)
    v = torch.from_numpy(vtx).cuda()
    g = torch.from_numpy(grad_image(u)).cuda()
    outs = []
    for level in (0, 1):
        _render(gs, octx, u, False, level)
        outs.append(_call(gs, octx, v, g)[:3])
        outs.append(_call(gs, octx, v, g)[:3])  # a repeated call
    octx.render(u)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        outs.append(_call(gs, octx, v, g, stream=side)[:3])
    other = gs.Context(0)
    try:
        other.upload(vtx)
        other.set_camera_model(cam)
        other.set_backward(True)
        other.set_backward_deterministic(True)
        other.render(u)
        outs.append(_call(gs, other, v, g)[:3])
    finally:
        other.close()
    for got in outs[1:]:
        for a, b in zip(got, outs[0]):
            assert np.array_equal(a, b)
    assert np.abs(outs[0][2]).max() > 0
    octx.set_backward_deterministic(False)


def test_error_cases(gs, octx):
    torch = _torch()
    good = gs.opencv_camera(500.0, 500.0, 319.5, 239.5, PHONE)

    def ocv(**kw):
        c = gs.opencv_camera(500.0, 500.0, 319.5, 239.5, PHONE)
        for key, val in kw.items():
            if key == "k":
                c.k = (type(c.k))(*val)
            else:
                setattr(c, key, val)
        return c

    bad = [ocv(fx=0.0), ocv(fy=-1.0), ocv(fx=float("inf")), ocv(cx=float("nan")), ocv(cy=float("inf")),
           ocv(k=(0.0, float("nan"), 0.0, 0.0)), ocv(k=(0.0, 0.0, float("inf"), 0.0)), ocv(max_theta=0.0),
           ocv(max_theta=float(np.float32(np.pi / 2))), ocv(max_theta=2.0), ocv(max_theta=-0.5), ocv(max_theta=float("nan")),
           ocv(k=(-0.5, 0.0, 0.0, 0.0), max_theta=1.0),     # 1 - 1.5 u: not increasing past u = 2/3 (tan^2 1 = 2.43)
           ocv(k=(0.0, -0.1, 0.0, 0.0), max_theta=1.3),     # 1 - 0.5 u^2 < 0 past u = 1.41
           ocv(k=(-1.0, 0.4, 0.0, 0.0), max_theta=1.2)]     # 1 - 3 u + 2 u^2 dips below 0 at the vertex (u = 0.75) only
    assert opencv_ref.radial_increasing(-1.0, 0.4, 0.5) and not opencv_ref.radial_increasing(-1.0, 0.4, 1.2)
    _, vtx, u = scenes.c1()
    octx.upload(vtx)
    octx.set_camera_model(good)
    base = octx.render(u)
    for c in bad:
        expect(gs, octx, gs.ERR_INVALID, lambda c=c: octx.set_camera_model(c), "gsb_set_camera_model")
        assert np.array_equal(octx.render(u).view(np.uint32), base.view(np.uint32))  # the setting is unchanged
    # the camera gradient refusals of the other entries on an OpenCV frame
    octx.set_backward(True)
    octx.render_depth(u)
    v = torch.from_numpy(vtx).cuda()
    gi = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    gda = torch.zeros((u.height, u.width, 2), dtype=torch.float32, device="cuda")
    gv, gu = torch.empty_like(v), torch.empty(40, dtype=torch.float32, device="cuda")
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
    feats = torch.zeros((v.shape[0], 2), dtype=torch.float32, device="cuda")
    gfm = torch.zeros((u.height, u.width, 2), dtype=torch.float32, device="cuda")
    expect(gs, octx, gs.ERR_INVALID, lambda: octx._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), None,
                                                            grad_uniforms_ptr=gu.data_ptr()), "gsb_render_backward_camera")
    expect(gs, octx, gs.ERR_INVALID, lambda: octx._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), None,
                                                            grad_uniforms_ptr=gu.data_ptr(), density_ptr=dens.data_ptr()),
           "gsb_render_backward_density")
    expect(gs, octx, gs.ERR_INVALID, lambda: octx._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), None,
                                                            grad_uniforms_ptr=gu.data_ptr(), grad_depth_alpha_ptr=gda.data_ptr()),
           "gsb_render_backward_depth")
    expect(gs, octx, gs.ERR_INVALID, lambda: octx.render_backward_features(v.data_ptr(), feats, gfm, gv.data_ptr(), None,
                                                                          grad_image_ptr=gi.data_ptr(),
                                                                          grad_uniforms_ptr=gu.data_ptr()),
           "gsb_render_backward_features")
    octx._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), None, density_ptr=dens.data_ptr())  # vertices only: fine
    ubo = torch.tensor(gs.pack_uniforms(u), device="cuda", requires_grad=True)
    with pytest.raises(ValueError):
        gs.render_torch(octx, v, u, ubo=ubo)
    # a pinhole frame has no lens gradient
    octx.set_camera_model(None)
    octx.render(u)
    gl = torch.empty(10, dtype=torch.float32, device="cuda")
    expect(gs, octx, gs.ERR_INVALID, lambda: octx._backward_fisheye(v.data_ptr(), gi.data_ptr(), None, None,
                                                                    grad_lens_ptr=gl.data_ptr()), "gsb_render_backward_fisheye")
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
# full size
# ---------------------------------------------------------------------------------------------------------------------
def _garden():
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    return bench, wl


def test_full_size_levels_and_bands_agree(gs):
    bench, wl = _garden()
    vtx = bench.make_scene(gs, wl)
    u = bench.cameras(gs, wl)[3]
    c = gs.Context(0)
    try:
        c.upload(vtx)
        c.set_camera_model(_lens(gs, u, k=PHONE))
        ref = c.render(u)
        assert c.stats().num_instances > 0
        for level in (1, 2):
            c.set_tile_cull(level)
            assert np.array_equal(c.render(u).view(np.uint32), ref.view(np.uint32)), level
        tiles_y = (u.height + 15) // 16
        step = -(-tiles_y // 3)  # three bands
        parts = [c.render(u, rows=(a, min(tiles_y, a + step))) for a in range(0, tiles_y, step)]
        assert len(parts) == 3 and np.array_equal(np.concatenate(parts).view(np.uint32), ref.view(np.uint32))
    finally:
        c.close()


def test_translation_identity_at_full_size(gs):
    torch = _torch()
    bench, wl = _garden()
    u = bench.cameras(gs, wl)[0]
    ctx = gs.Context(0)
    try:
        ctx.set_tile_cull(1)
        ctx.set_backward(True)
        ctx.set_camera_model(_lens(gs, u, k=PHONE, shift=(11.0, -7.0)))
        v = torch.from_numpy(bench.make_scene(gs, wl)).cuda()
        ctx.upload(v)
        ctx.render_into(u, torch.empty((u.height, u.width, 4), dtype=torch.float32, device="cuda").data_ptr())
        gi = torch.randn((u.height, u.width, 4), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
        gv, gu, gl, _, _ = _call(gs, ctx, v, gi)
    finally:
        ctx.close()
    gp = gv[:, 0:3]
    res, scale = translation_identity(gp.sum(0), np.abs(gp).sum(0), u, gu[gs.UBO_FLOAT_WORDS])
    print("OpenCV translation identity: residual", res, "scale", scale)
    assert np.abs(gu).max() > 0 and np.abs(gl).max() > 0
    assert (np.abs(res) <= 1e-5 * scale).all(), (res, scale)


# ---------------------------------------------------------------------------------------------------------------------
# training through the lens
# ---------------------------------------------------------------------------------------------------------------------
def test_lens_self_calibration(gs, octx):
    """k1, k2, p1, p2 recovered from zero on a frozen scene, from targets rendered through a known lens."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    # a 75-degree view (the frame's corners lie 43.8 degrees off the axis) so that k2 moves the periphery by pixels; culled at
    # 46 degrees, where every k the optimiser visits keeps r R(r^2) increasing
    u = gs.uniforms_from_camera([0, 0, 6], [1, 0, 0, 0], 75.0, 0.1, 1000.0, 640, 480)
    true = _lens(gs, u, k=(-0.1, 0.02, 0.003, -0.002), shift=(5.0, -3.0), max_theta=math.radians(46.0))
    octx.set_camera_model(true)
    v = torch.from_numpy(vtx).cuda()
    with torch.no_grad():
        target = gs.render_torch(octx, v, u)[..., :3].clone()
    t0 = gs.lens_tensor(true).double()
    # Adam steps each word by about lr: the leaf is k in units that move xd by a similar amount at the frame's edge
    unit = torch.tensor([3e-3, 3e-3, 1e-4, 1e-4], dtype=torch.float64)
    delta = torch.zeros(4, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([delta], lr=0.5)
    losses = []
    for it in range(400):
        if it in (250, 350):
            for group in opt.param_groups:
                group["lr"] *= 0.2
        opt.zero_grad()
        img = gs.render_torch(octx, v, u, lens=torch.cat([t0[:4], delta * unit]).float())
        loss = ((img[..., :3] - target) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    k = (delta * unit).detach()
    with torch.no_grad():
        final = float(((gs.render_torch(octx, v, u, lens=torch.cat([t0[:4], k]).float())[..., :3] - target) ** 2).sum())

    def field(kk):  # the distortion in pixels over a grid of the frame's normalised coordinates
        xn, yn = np.meshgrid(np.linspace(-u.tan_fovx, u.tan_fovx, 33), np.linspace(-u.tan_fovy, u.tan_fovy, 25))
        t = torch.tensor(np.stack([xn.ravel(), yn.ravel(), np.ones(xn.size)], 1))
        return opencv_ref.project(t, (float(t0[0]), float(t0[1]), 0.0, 0.0, [float(x) for x in kk], 0.0)).numpy()

    px0 = np.abs(field(torch.zeros(4)) - field(t0[4:])).max()
    px = np.abs(field(k) - field(t0[4:])).max()
    err = (k - t0[4:]).abs()
    print(f"OpenCV lens self-calibration: loss {losses[0]:.4g} -> {final:.4g}; k {k.tolist()} of {t0[4:].tolist()}; "
          f"distortion error {px0:.2f} -> {px:.3f} px")
    assert final < 0.01 * losses[0], (losses[0], final)
    assert px < 0.02 * px0 and px < 0.5, (px0, px)
    # inside a 44-degree field k2 trades off against k1 along a shallow valley, so it is held to 50 %, the others to 20 %
    assert (err <= torch.tensor([0.2, 0.5, 0.2, 0.2], dtype=torch.float64) * t0[4:].abs()).all(), (k, t0[4:])
    assert bytes(octx.camera) == bytes(true)


def test_scene_adam_fits_distorted_views_better_than_a_pinhole(gs, octx):
    """Targets rendered through a strong barrel lens; the same SceneAdam run through that lens and through a pinhole of equal
    focal, scored by L1 on a held-out view through the lens."""
    from test_gpu_adam import POSES, TRAIN_LR

    torch = _torch()
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = [gs.uniforms_from_camera(p, q, 60.0, 0.1, 1000.0, 320, 240) for p, q in POSES]
    lens = _lens(gs, views[0], k=(-0.3, 0.08, 0.0, 0.0))
    octx.set_camera_model(lens)
    with torch.no_grad():
        targets = [gs.render_torch(octx, full, u).clone() for u in views]
    train, held = list(range(len(views) - 1)), len(views) - 1
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    scores = {}
    for name, cam in (("opencv", lens), ("pinhole", None)):
        start = full[::4].clone()
        start[:, 4:7] *= 1.5
        octx.set_camera_model(cam)
        opt = gs.SceneAdam(octx, start, TRAIN_LR)
        for it in range(300):
            k = train[it % len(train)]
            octx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
            opt.step(g)
        octx.set_camera_model(lens)
        scores[name] = gs.image_metrics(octx, opt.render(views[held]), targets[held])["l1"]
    print(f"held-out L1 through the lens: OpenCV training {scores['opencv']:.5f}, pinhole training {scores['pinhole']:.5f}")
    assert scores["opencv"] < 0.95 * scores["pinhole"], scores
