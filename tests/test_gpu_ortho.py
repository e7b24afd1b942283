"""gsb_set_camera_model's orthographic camera on the GPU: the record words against the fp32 restatement bit for bit and the
frame against the float64 restatement (tests/ortho_ref.py) over the frame's own level-0 lists, the frame equalities of the
pinhole path within orthographic frames, the pinhole frame unchanged, the SH degrees, depth as a height map, the vertex,
camera and lens gradients of the backward entries, determinism, the error codes, the lens 3D filter, the full-size garden
stand-in and pose refinement and training through the camera."""
import math

import numpy as np
import pytest

import edge_scene
import ortho_ref
import scenes
from backward_util import GROUPS, expect, grad_image, rel
from test_gpu_fisheye import STEP_FRACTION, _backward, _check_frame
from test_gpu_fisheye_camera import _call, _render, _upstream

pytestmark = pytest.mark.gpu

VIEW_GROUPS = {"view_3x3": [20 + c * 4 + r for c in range(3) for r in range(3)], "view_translation": [32, 33, 34]}
LENS_GROUPS = {"focal": [0, 1], "principal_point": [2, 3]}
DEAD_UBO = np.nonzero(~ortho_ref.LIVE_UBO)[0]


def _torch():
    import torch

    return torch


@pytest.fixture
def octx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _view(vtx, u):
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    return (V @ np.c_[np.asarray(vtx, np.float64)[:, :3], np.ones(len(vtx))].T)[:3].T


def _ortho(gs, vtx, u, aspect=1.0, shift=(0.0, 0.0)):
    """An orthographic camera over u's pose whose frame holds the middle 90 % of the visible cloud across its width (fy =
    aspect fx), principal point at the frame's centre pixel plus `shift` pixels."""
    t = _view(vtx, u)
    x = np.abs(t[t[:, 2] > 0.2, 0])
    f = 0.5 * u.width / float(np.quantile(x, 0.9))
    return gs.ortho_camera(f, f * aspect, (u.width - 1) / 2.0 + shift[0], (u.height - 1) / 2.0 + shift[1])


CASES = {  # name: (scene, pose, camera arguments)
    "c1": ("c1", "c1", {}),
    "odd_size": ("c1", "odd_size", {"aspect": 1.13}),
    "edge": ("edge", "c1", {}),
    "off_centre": ("c1", "odd_size", {"aspect": 0.93, "shift": (23.7, -17.2)}),
}


def _case(gs, name):
    scene, pose, kw = CASES[name]
    vtx = scenes.c1()[1] if scene == "c1" else edge_scene.vertices()[0]
    u = scenes.camera(pose)
    return vtx, u, _ortho(gs, vtx, u, **kw)


def _frame_lists(gs, ctx, u):
    """Render u in debug mode at level 0: (image, {"vals", "ranges"}, GSB_BUF_ATTR, GSB_BUF_COV3D)."""
    ctx.set_debug(True)
    ctx.set_tile_cull(0)
    img = ctx.render(u)
    frame = {"vals": ctx.download(gs.BUF_VALS_SORTED), "ranges": ctx.download(gs.BUF_TILE_BOUNDARY)}
    attr, cov = ctx.download(gs.BUF_ATTR), ctx.download(gs.BUF_COV3D)
    ctx.set_debug(False)
    return img, frame, attr, cov


def _ulp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("name", sorted(CASES))
def test_records_and_frame_match_restatements(gs, octx, name):
    vtx, u, cam = _case(gs, name)
    octx.upload(vtx)
    octx.set_camera_model(cam)
    img, frame, attr, cov = _frame_lists(gs, octx, u)
    rec = ortho_ref.record32(vtx, cov, u, cam)
    live = attr["color_radii"][:, 3] > 0
    assert np.array_equal(live, rec["kept"]) and live.sum() > 100, (name, live.sum(), rec["kept"].sum())
    assert np.array_equal(attr["uv"][live].view(np.uint32), rec["uv"][live].view(np.uint32))
    assert np.array_equal(attr["conic_opacity"][live, :3].view(np.uint32), rec["conic"][live].view(np.uint32))
    assert np.array_equal(attr["color_radii"][live, 3].view(np.uint32), rec["radii"][live].view(np.uint32))
    assert np.array_equal(attr["aabb"][live].astype(np.int64), rec["aabb"][live])
    assert np.array_equal(attr["depth"][live].view(np.uint32), rec["depth"][live].view(np.uint32))
    col32 = ortho_ref.colour32(vtx[:, 12:60], u.view_mat)
    assert _ulp(attr["color_radii"][live, :3], col32[live]).max() <= 2
    torch = _torch()
    col64, _ = ortho_ref.colour(torch.tensor(vtx.astype(np.float64)),
                                torch.tensor(np.asarray(list(u.view_mat), np.float32).astype(np.float64)))
    assert np.abs(attr["color_radii"][live, :3] - col64.numpy()[live]).max() <= 1e-6
    if name != "edge":  # the edge scene's needles and near-singular footprints: its words above, not a float64 image
        ref = ortho_ref.reference(vtx, u, cam, frame)
        _check_frame(img, ref, name)


@pytest.mark.parametrize("name", ["c1", "off_centre"])
def test_equalities_within_ortho_frames(gs, oracle, octx, name):
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
        assert np.array_equal(octx.render(u, gs.FORMAT_BGRA8), oracle.pack_unorm8(ref, bgra=True))
        tiles_y = (u.height + 15) // 16
        cut = max(1, tiles_y // 3)
        bands = np.concatenate([octx.render(u, rows=(0, cut)), octx.render(u, rows=(cut, tiles_y))])
        assert np.array_equal(bands.view(np.uint32), ref.view(np.uint32))
    octx.set_antialiased(False)
    octx.set_background(None)


def test_depth_is_view_space_z(gs, octx):
    vtx, u, cam = _case(gs, "odd_size")
    octx.upload(vtx)
    octx.set_camera_model(cam)
    _, frame, _, _ = _frame_lists(gs, octx, u)
    _, da = octx.render_depth(u)
    ref = ortho_ref.reference(vtx, u, cam, frame)
    err = np.abs(da.astype(np.float64) - ref["depth_alpha"]) / np.maximum(1.0, np.abs(ref["depth_alpha"]))
    bad = err.max(-1) > 1e-4
    assert bad.mean() <= STEP_FRACTION and ref["depth_alpha"][..., 0].max() > 1.0, (bad.mean(), err.max())


@pytest.mark.parametrize("degree", [0, 1, 2])
def test_sh_degree_equals_zeroed_scene(gs, octx, degree):
    vtx, u, cam = _case(gs, "c1")
    zeroed = vtx.copy()
    zeroed[:, 12 + 3 * (degree + 1) ** 2:60] = 0.0
    octx.set_camera_model(cam)
    for half in (False, True):
        octx.set_sh_storage(half)
        octx.upload(zeroed)
        octx.set_sh_degree(3)
        want = octx.render(u)
        octx.upload(vtx)
        octx.set_sh_degree(degree)
        got = octx.render(u)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (degree, half)
    octx.set_sh_degree(3)


def test_pinhole_frame_is_unaffected(gs, octx):
    vtx, u, cam = _case(gs, "c1")
    octx.upload(vtx)
    base = octx.render(u)
    for reset in (None, gs.CameraModel(gs.CAMERA_PINHOLE)):
        octx.set_camera_model(cam)
        assert not np.array_equal(octx.render(u), base)
        octx.set_camera_model(reset)
        assert np.array_equal(octx.render(u).view(np.uint32), base.view(np.uint32))


def test_height_map_of_a_surface(gs, octx):
    """Gaussians laid on the surface z = h(x, y) (world z up), seen straight down by an orthographic camera at height Z0:
    D / A is the height below the camera plane, Z0 - h.  The blend weighs the nearest of the overlapping discs most, so on a
    slope D / A leans towards the uphill neighbours within a footprint: the stated tolerance is 0.03 + 3 sigma |grad h|
    (sigma = 0.12, the discs' radius) at 99 % of the covered pixels, and 0.05 + 3 sigma |grad h| everywhere."""
    rng = np.random.default_rng(3)
    n = 60_000
    xy = rng.uniform(-10.0, 10.0, (n, 2))

    def h(x, y):
        return 1.5 * np.sin(0.4 * x) * np.cos(0.3 * y) + 0.05 * x

    def slope(x, y):
        return np.hypot(0.6 * np.cos(0.4 * x) * np.cos(0.3 * y) + 0.05, 0.45 * np.sin(0.4 * x) * np.sin(0.3 * y))

    vtx = np.zeros((n, 60), np.float32)  # activated records: position, scale, opacity, rotation (w first), SH
    vtx[:, 0:3] = np.c_[xy, h(xy[:, 0], xy[:, 1])]
    vtx[:, 4:7] = (0.12, 0.12, 0.01)
    vtx[:, 7] = 0.95
    vtx[:, 8] = 1.0
    vtx[:, 12:15] = 0.5
    Z0 = 20.0
    # the identity pose at (0, 0, Z0) looks down -z: view rows x = world x, y = -world y, z = Z0 - world z
    u = gs.uniforms_from_camera([0, 0, Z0], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 512, 512)
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    assert np.allclose(V[2, :3], [0, 0, -1], atol=1e-6) and abs(V[2, 3] - Z0) < 1e-5, V
    f = 512 / 16.0
    octx.upload(vtx)
    octx.set_camera_model(gs.ortho_camera(f, f, 255.5, 255.5))
    _, da = octx.render_depth(u)
    A = da[..., 1].astype(np.float64)
    D = da[..., 0].astype(np.float64) / np.maximum(A, 1e-10)
    jj, ii = np.mgrid[0:512, 0:512]
    inv = np.linalg.inv(V)
    t = np.stack([(ii - 255.5) / f, (jj - 255.5) / f, np.full(ii.shape, Z0)], -1)  # the pixel's ray at depth Z0
    w = t @ inv[:3, :3].T + inv[:3, 3]
    want = Z0 - h(w[..., 0], w[..., 1])
    mask = A > 0.99
    assert mask.mean() > 0.9
    err = np.abs(D - want)[mask]
    bound = 3.0 * 0.12 * slope(w[..., 0], w[..., 1])[mask]
    assert (err <= 0.03 + bound).mean() >= 0.99 and (err <= 0.05 + bound).all(), (np.quantile(err - bound, 0.99), (err - bound).max())


# ---------------------------------------------------------------------------------------------------------------------
# the backward pass
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["c1", "odd_size", "off_centre"])
def test_gradient_matches_float64_reference(gs, octx, name):
    vtx, u, cam = _case(gs, name)
    octx.upload(vtx)
    octx.set_camera_model(cam)
    octx.set_backward(True)
    img, frame, _, _ = _frame_lists(gs, octx, u)
    g = grad_image(u)
    ref = ortho_ref.reference(vtx, u, cam, frame, g)
    _check_frame(img, ref, name)
    keep = ~ref["exclude"]
    assert keep.sum() > 100
    for det in (False, True):
        octx.set_backward_deterministic(det)
        octx.set_tile_cull(0)
        octx.render(u)
        got, dens = _backward(gs, octx, vtx, g, density=True)
        assert np.isfinite(got).all() and dens[:, 2].sum() > 0
        for group, cols in GROUPS.items():  # 2e-3: the fp32 rotation column of off_centre measured 1.03e-3
            r = rel(got[keep][:, cols], ref["grad"][keep][:, cols])
            assert r <= 2e-3, (name, det, group, r)
        assert not got[:, 3].any()
    octx.set_backward_deterministic(False)


REF_RUNS = [("c1", "colour", False), ("odd_size", "colour", True), ("off_centre", "colour", False),
            ("c1", "depth", False), ("off_centre", "alpha", True), ("odd_size", "feature", False)]


@pytest.mark.parametrize("name,kind,aa", REF_RUNS, ids=[f"{n}-{k}-{'aa' if a else 'plain'}" for n, k, a in REF_RUNS])
def test_camera_lens_and_vertex_gradients_match_float64_reference(gs, octx, name, kind, aa):
    torch = _torch()
    vtx, u, cam = _case(gs, name)
    octx.upload(vtx)
    octx.set_camera_model(cam)
    octx.set_antialiased(aa)
    octx.set_backward(True)
    _, frame, _, _ = _frame_lists(gs, octx, u)
    steps = ortho_ref.step_pixels(vtx, u, cam, frame, aa)
    assert steps.mean() < 0.05
    gi, gda, feats, gfm = _upstream(u, kind, steps, vtx.shape[0])
    ref = ortho_ref.reference(vtx, u, cam, frame, grad_image=gi, grad_da=gda, features=feats, grad_fm=gfm, antialiased=aa)
    keep = ~ref["exclude"]
    v = torch.from_numpy(vtx).cuda()
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    for det in (False, True):
        octx.set_backward_deterministic(det)
        _render(gs, octx, u, gda is not None)
        gv, gu, gl, _, _ = _call(gs, octx, v, t(gi), t(gda), t(feats), t(gfm))
        for group, words in VIEW_GROUPS.items():
            r = rel(gu[words], ref["grad_ubo"][words])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
        for group, words in LENS_GROUPS.items():
            r = rel(gl[1:9][words], ref["grad_lens"][words])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
        assert not gu[DEAD_UBO].any() and not gu[0:4].any()  # camera_position exactly 0
        assert not gl[5:9].any() and gl[0] == 0 and gl[9] == 0
        for group, cols in GROUPS.items():
            r = rel(gv[keep][:, cols], ref["grad"][keep][:, cols])
            assert r <= 1e-3, (name, kind, aa, det, group, r)
    octx.set_backward_deterministic(False)
    octx.set_antialiased(False)


def test_deterministic_words(gs, octx):
    torch = _torch()
    vtx, u, cam = _case(gs, "off_centre")
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
        outs.append(_call(gs, octx, v, g)[:3])
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
    good = gs.ortho_camera(50.0, 50.0, 319.5, 239.5)

    def oc(**kw):
        c = gs.ortho_camera(50.0, 50.0, 319.5, 239.5)
        for key, val in kw.items():
            if key == "k":
                c.k = (type(c.k))(*val)
            else:
                setattr(c, key, val)
        return c

    bad = [(oc(fx=0.0), "fx"), (oc(fy=-1.0), "fx"), (oc(fx=float("inf")), "fx"), (oc(fy=float("nan")), "fx"),
           (oc(cx=float("nan")), "cx"), (oc(cy=float("inf")), "cx"), (oc(k=(0.1, 0.0, 0.0, 0.0)), "k[0..3]"),
           (oc(k=(0.0, 0.0, 0.0, -1e-30)), "k[0..3]"), (oc(k=(0.0, float("nan"), 0.0, 0.0)), "k[0..3]"),
           (oc(max_theta=0.5), "max_theta"), (oc(max_theta=float("nan")), "max_theta")]
    _, vtx, u = scenes.c1()
    octx.upload(vtx)
    octx.set_camera_model(good)
    base = octx.render(u)
    for c, field in bad:
        expect(gs, octx, gs.ERR_INVALID, lambda c=c: octx.set_camera_model(c), "gsb_set_camera_model")
        msg = gs.lib.gsb_last_error(octx.h).decode()
        assert field in msg, (field, msg)
        assert np.array_equal(octx.render(u).view(np.uint32), base.view(np.uint32))
    # the camera gradient refusals of the other entries on an orthographic frame
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
    assert "orthographic" in gs.lib.gsb_last_error(octx.h).decode()
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
# the lens 3D filter
# ---------------------------------------------------------------------------------------------------------------------
def _filter_model(vtx, cams, models):
    """gsb_filter3d_variance_lens for orthographic and pinhole cameras in numpy fp32, op for op."""
    p = np.asarray(vtx, np.float32).reshape(-1, 60)[:, :3]
    s = np.full(len(p), np.inf, np.float32)
    for u, m in zip(cams, models):
        vm = np.asarray(list(u.view_mat), np.float32)
        W, H = np.float32(u.width), np.float32(u.height)
        with np.errstate(all="ignore"):
            vx = ((vm[0] * p[:, 0] + vm[4] * p[:, 1]) + vm[8] * p[:, 2]) + vm[12]
            vy = ((vm[1] * p[:, 0] + vm[5] * p[:, 1]) + vm[9] * p[:, 2]) + vm[13]
            vz = ((vm[2] * p[:, 0] + vm[6] * p[:, 1]) + vm[10] * p[:, 2]) + vm[14]
            uu = np.float32(m.fx) * vx + np.float32(m.cx)
            vv = np.float32(m.fy) * vy + np.float32(m.cy)
        seen = (vz > np.float32(0.2)) & (uu >= np.float32(-0.15) * W) & (uu <= np.float32(1.15) * W) \
            & (vv >= np.float32(-0.15) * H) & (vv <= np.float32(1.15) * H)
        sc = np.float32(1.0) / np.fmin(np.float32(m.fx), np.float32(m.fy))
        s = np.where(seen, np.fmin(s, sc), s)
    seen = np.isfinite(s)
    fill = s[seen].max() if seen.any() else np.float32(0)
    s = np.where(seen, s, fill).astype(np.float32)
    return ((s * s) * np.float32(0.2)).astype(np.float32), seen


def test_filter3d_lens_matches_numpy_model(gs, octx):
    torch = _torch()
    vtx, u, cam = _case(gs, "c1")
    u2 = scenes.camera("odd_size")
    cams = [u, u2, u]
    models = [cam, _ortho(gs, vtx, u2, aspect=1.4), gs.ortho_camera(cam.fx * 3.0, cam.fy * 2.0, cam.cx + 40.0, cam.cy)]
    v = torch.from_numpy(vtx).cuda()
    got = octx.filter3d_variance(v, cams, models).cpu().numpy()
    want, seen = _filter_model(vtx, cams, models)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    rev = octx.filter3d_variance(v, cams[::-1], models[::-1]).cpu().numpy()
    assert np.array_equal(rev.view(np.uint32), got.view(np.uint32))
    # mixed with a fisheye and an OpenCV camera: a row the orthographic cameras see only keeps or lowers its scale (the
    # unseen rows take the largest seen scale, which the new cameras may raise)
    assert seen.mean() > 0.5
    mixed = octx.filter3d_variance(v, cams + [u, u], models + [gs.fisheye_camera(300.0, 300.0, 319.5, 239.5, max_theta=1.5),
                                                             gs.opencv_camera(300.0, 300.0, 319.5, 239.5)]).cpu().numpy()
    assert (mixed[seen] <= got[seen]).all() and (mixed[seen] < got[seen]).any()


# ---------------------------------------------------------------------------------------------------------------------
# full size, pose refinement and training
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
        c.set_camera_model(_ortho(gs, vtx[::50], u))
        ref = c.render(u)
        assert c.stats().num_instances > 0
        for level in (1, 2):
            c.set_tile_cull(level)
            assert np.array_equal(c.render(u).view(np.uint32), ref.view(np.uint32)), level
        c.set_tile_cull(0)
        tiles_y = (u.height + 15) // 16
        step = -(-tiles_y // 3)
        parts = [c.render(u, rows=(a, min(tiles_y, a + step))) for a in range(0, tiles_y, step)]
        assert len(parts) == 3 and np.array_equal(np.concatenate(parts).view(np.uint32), ref.view(np.uint32))
    finally:
        c.close()


def test_pose_and_scale_refinement_through_render_torch(gs, octx):
    """x/y translation, rotation and fx, fy from a perturbed start back towards the target through render_torch (translation
    along the view axis is unobservable but for the cull and depth order, so it is not perturbed)."""
    torch = _torch()
    vtx, u, cam = _case(gs, "c1")
    v = torch.from_numpy(vtx).cuda()
    octx.set_camera_model(cam)
    ubo0 = np.asarray(gs.pack_uniforms(u), np.float32)
    lens0 = gs.lens_tensor(cam)
    with torch.no_grad():
        target = gs.render_torch(octx, v, u, ubo=torch.tensor(ubo0, device="cuda"), lens=lens0.cuda()).clone()
    ang = math.radians(1.5)
    R = np.array([[math.cos(ang), -math.sin(ang), 0], [math.sin(ang), math.cos(ang), 0], [0, 0, 1]])
    V = ubo0[20:36].reshape(4, 4).T.astype(np.float64)
    V[:3, :3] = R @ V[:3, :3]
    V[0, 3] += 0.05
    V[1, 3] -= 0.04
    ubo = ubo0.copy()
    ubo[20:36] = V.T.reshape(-1)
    pose = torch.tensor(ubo, device="cuda", requires_grad=True)
    lens = lens0.clone().cuda()
    lens[0] *= 1.04
    lens[1] *= 0.97
    lens.requires_grad_()
    opt = torch.optim.Adam([{"params": [pose], "lr": 2e-3}, {"params": [lens], "lr": 0.5}])
    live = torch.zeros(gs.UBO_FLOATS, dtype=torch.bool, device="cuda")
    live[[20 + c * 4 + r for c in range(4) for r in range(3)]] = True
    first = None
    for _ in range(150):
        opt.zero_grad()
        img = gs.render_torch(octx, v, u, ubo=pose, lens=lens)
        loss = (img[..., :3] - target[..., :3]).abs().mean()
        first = float(loss.detach()) if first is None else first
        loss.backward()
        pose.grad[~live] = 0
        lens.grad[4:] = 0
        opt.step()
    assert float(loss.detach()) < 0.3 * first, (first, float(loss.detach()))
    w = lens.detach().cpu()
    fe = abs(float(w[0]) / float(lens0[0]) - 1.0), abs(float(w[1]) / float(lens0[1]) - 1.0)
    assert fe[0] < 0.5 * 0.04 and fe[1] < 0.5 * 0.03, fe  # at least half of the 4 % and 3 % start errors recovered
    assert not lens.detach()[4:].any()


def test_scene_adam_fits_held_out_ortho_view(gs, octx):
    """SceneAdam trained from orthographic views of a scene brings a held-out orthographic view closer to its target (held-out
    L1 0.103 to 0.082 when measured on an H100)."""
    from test_gpu_adam import POSES, TRAIN_LR

    torch = _torch()
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = [gs.uniforms_from_camera(p, q, 60.0, 0.1, 1000.0, 320, 240) for p, q in POSES]
    cams = [_ortho(gs, vtx, u) for u in views]
    targets = []
    for u, cam in zip(views, cams):
        octx.set_camera_model(cam)
        with torch.no_grad():
            targets.append(gs.render_torch(octx, full, u).clone())
    train, held = list(range(len(views) - 1)), len(views) - 1
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    start = full[::4].clone()
    start[:, 4:7] *= 1.5
    opt = gs.SceneAdam(octx, start, TRAIN_LR)

    def held_out():
        octx.set_camera_model(cams[held])
        return gs.image_metrics(octx, opt.render(views[held]), targets[held])["l1"]

    before = held_out()
    for it in range(300):
        k = train[it % len(train)]
        octx.set_camera_model(cams[k])
        octx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g)
    after = held_out()
    print(f"held-out orthographic L1: {before:.5f} before training, {after:.5f} after")
    assert after < 0.9 * before, (before, after)


def test_headless_viewer_ortho(gs, octx, tmp_path):
    """gs_viewer_headless --ortho renders the frame a context renders through the same camera, and a non-zero k is refused
    with the field named."""
    import subprocess
    from pathlib import Path

    exe = Path(__file__).resolve().parents[1] / "3dgs.cpp_b200" / "gs_viewer_headless"
    rec = gs.synth_records(42, 10_000)
    ply = tmp_path / "c1.ply"
    gs.write_ply(ply, rec)
    pfm = tmp_path / "frame.pfm"
    r = subprocess.run([str(exe), "-w", "640", "-h", "480", "--camera", "0,0,5", "--ortho", "120,120,319.5,239.5", "--float-out",
                        str(pfm), str(ply)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    blob = pfm.read_bytes()
    head = b"PF\n640 480\n-1.0\n"
    assert blob.startswith(head)
    img = np.frombuffer(blob[len(head):], "<f4").reshape(480, 640, 3)[::-1]
    u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 640, 480)
    octx.upload(gs.activate_records(rec))
    octx.set_camera_model(gs.ortho_camera(120.0, 120.0, 319.5, 239.5))
    want = octx.render(u)
    assert np.abs(want[..., :3]).max() > 0 and np.array_equal(img, want[..., :3])
    bad = subprocess.run([str(exe), "--ortho", "120,120,319.5,239.5,0.1", str(ply)], capture_output=True, text=True, timeout=120)
    assert bad.returncode != 0 and "k[0..3]" in bad.stderr, bad.stderr
