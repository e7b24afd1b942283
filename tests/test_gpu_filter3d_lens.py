"""gsb_filter3d_variance_lens / Context.filter3d_variance(lenses=) / SceneAdam(filter_lenses=): the 3D smoothing filter
from cameras that each have their own lens.  PINHOLE and OPENCV words equal the fp32 model of tests/filter3d_lens_ref.py bit
for bit and FISHEYE words lie within its stated bound, at every size and across the camera staging chunks; all-pinhole
cameras of one focal give gsb_filter3d_variance's words; a 200 deg lens sees what no pinhole can; every filtered footprint
keeps lambda_min >= 0.2 px^2 at the camera that resolves it best; the words are reproducible and leave the last frame
alone; and SceneAdam trains through a fisheye and an OpenCV lens with the filter."""
import math
import sys
from pathlib import Path

import numpy as np
import pytest

import filter3d_lens_ref as lr
import scenes
from backward_util import expect, grad_image, render
from test_filter3d_lens_ref import F32_ULPS, _directions, common_focal_c1, lens_for
from test_filter3d_ref import cloud, look_at_poses, uniforms
from test_gpu_adam import POSES, TRAIN_LR, _assert_coherent, _evaluate

pytestmark = pytest.mark.gpu

# FISHEYE words against the fp32 model: both are within F32_ULPS of float64 on rows away from the margins and culls, and
# differ only through atan2 (atan2f is not correctly rounded, nor is numpy's)
FISHEYE_ULPS = 2 * F32_ULPS


def _torch():
    import torch

    return torch


@pytest.fixture
def lctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _rows(xyz):
    torch = _torch()
    v = torch.zeros((xyz.shape[0], 60), dtype=torch.float32)
    v[:, 0:3] = torch.from_numpy(np.ascontiguousarray(xyz, np.float32))
    return v.cuda()


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _views(gs, k, seed, names):
    cams = uniforms(gs, look_at_poses(k, seed=seed))
    return cams, [_lens(gs, u, names[i % len(names)]) for i, u in enumerate(cams)]


def _lens(gs, u, name):
    """lens_for's lenses and two more OpenCV ones: "k0" (no distortion, off-centre) and "barrel"."""
    if name in ("k0", "barrel"):
        fx = u.width / (2.0 * float(u.tan_fovx))
        k = (0.0, 0.0, 0.0, 0.0) if name == "k0" else (-0.28, 0.07, 0.0, 0.0)
        return gs.opencv_camera(fx, fx * 0.97, u.width / 2.0 + 5.5, u.height / 2.0 - 4.0, k)
    return lens_for(gs, u, name)


EXACT = ["pinhole", "k0", "barrel", "phone"]


@pytest.mark.parametrize("n,k,names", [(1, 1, ["phone"]), (1000, 63, ["k0"]), (4097, 64, ["barrel"]), (10_000, 65, EXACT),
                                       (3000, 128, ["phone"]), (3000, 129, EXACT), (2000, 1000, EXACT),
                                       ((1 << 20) + 3, 5, EXACT)])
def test_pinhole_and_opencv_words_equal_the_model(gs, lctx, n, k, names):
    xyz = cloud(n, seed=n + k)
    cams, models = _views(gs, k, k, names)
    got = lctx.filter3d_variance(_rows(xyz), cams, models).cpu().numpy()
    want = lr.variance(xyz, cams, models)
    assert np.array_equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())
    print(f"n = {n}, k = {k}, {'/'.join(names)}: {int(lr.scales(xyz, cams, models)[1].sum())} rows seen")


@pytest.mark.parametrize("n,k,names", [(1, 1, ["fish180"]), (5000, 7, ["fish180"]), (5000, 64, ["fish200"]),
                                       (20_000, 65, ["fish200", "pinhole", "phone", "fish180", "barrel"]),
                                       (3000, 300, ["fish180", "k0", "fish200"])])
def test_fisheye_words_within_the_model_bound(gs, lctx, n, k, names):
    cams, models = _views(gs, k, k + 1, names)
    xyz = cloud(max(n, 64), seed=n)
    xyz = xyz[~lr.borderline(xyz, cams, models)][:n]
    got = lctx.filter3d_variance(_rows(xyz), cams, models).cpu().numpy()
    want = lr.variance(xyz, cams, models)
    worst = int(lr.ulps(got, want).max())
    print(f"n = {xyz.shape[0]}, k = {k}, {'/'.join(names)}: within {worst} ulp of the fp32 model")
    assert worst <= FISHEYE_ULPS


def test_single_lens_for_every_camera(gs, lctx):
    xyz = cloud(4000, seed=1)
    cams = uniforms(gs, look_at_poses(9, seed=1))
    lens = _lens(gs, cams[0], "phone")
    got = lctx.filter3d_variance(_rows(xyz), cams, lens).cpu().numpy()
    assert np.array_equal(_bits(got), _bits(lr.variance(xyz, cams, [lens] * 9)))


def _garden():
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    return bench, bench.WORKLOADS["garden-standin"]


def test_common_focal_pinholes_equal_the_pinhole_entry(gs, lctx):
    """c1's poses at one focal, and bench.py's garden poses (focal_x == focal_y in fp32): gsb_filter3d_variance's words."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    cams = common_focal_c1(gs)
    for xyz in (vtx[:, 0:3], cloud(50_000, seed=3)):
        v = _rows(xyz)
        want = lctx.filter3d_variance(v, cams).cpu()
        for lenses in (gs.CameraModel(), [gs.CameraModel()] * len(cams)):
            assert torch.equal(want.view(torch.int32), lctx.filter3d_variance(v, cams, lenses).cpu().view(torch.int32))
    bench, wl = _garden()
    gv = torch.from_numpy(bench.make_scene(gs, wl)).cuda()
    gcams = bench.cameras(gs, wl)
    assert len({lr.pinhole_focal(u) for u in gcams}) == 1
    assert all(np.float32(u.width) / (np.float32(2) * np.float32(u.tan_fovx)) == lr.pinhole_focal(u) for u in gcams)
    want = lctx.filter3d_variance(gv, gcams)
    got = lctx.filter3d_variance(gv, gcams, gs.CameraModel())
    assert torch.equal(want.view(torch.int32), got.view(torch.int32))


def test_wide_lens_sees_past_90_degrees(gs, lctx):
    """Rows at 92-99 deg off the axis of a 200 deg lens are seen (their own variance, no fill); through a pinhole of the same
    focal the same rows are unseen and take the fill."""
    u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 60.0, 0.1, 1000.0, 640, 480)
    wide = lens_for(gs, u, "fish200")
    V = np.array(u.view_mat, np.float64).reshape(4, 4)
    R, tr = V[:3, :3], V[3, :3]
    t = np.concatenate([_directions(math.radians(a), 12) * r for a in (92, 95, 99) for r in (0.5, 2.0, 7.0)]
                       + [_directions(math.radians(20), 12) * 3.0])
    xyz = ((t - tr) @ np.linalg.inv(R)).astype(np.float32)
    back = np.arange(xyz.shape[0]) < xyz.shape[0] - 12
    s, seen = lr.scales(xyz, [u], [wide])
    assert seen.all()
    got = lctx.filter3d_variance(_rows(xyz), [u], wide).cpu().numpy()
    assert int(lr.ulps(got, lr.variance(xyz, [u], [wide])).max()) <= FISHEYE_ULPS
    assert len(set(_bits(got[back]).tolist())) > 3  # the rows' own scales, not one fill value
    f = wide.fx
    pin = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], math.degrees(2 * math.atan(640 / (2 * f))), 0.1, 1000.0, 640, 480)
    assert not lr.scales(xyz[back], [pin], None)[1].any()
    p = lctx.filter3d_variance(_rows(xyz), [pin], gs.CameraModel()).cpu().numpy()
    assert np.array_equal(_bits(p), _bits(lr.variance(xyz, [pin], None)))
    assert len(set(_bits(p[back]).tolist())) == 1 and p[back][0] == p[~back].max()


@pytest.mark.parametrize("names", [["phone"], ["fish180"], ["barrel", "fish200", "pinhole"]])
def test_footprint_bound_at_the_attaining_camera(gs, lctx, names):
    """Every seen survivor of the filtered records, rendered through the lens of the camera that attains its scale, has an
    undilated 2D covariance (from GSB_BUF_ATTR's conic) with lambda_min >= 0.2 px^2 (1 - 1e-5), less the fp32 rounding of
    inverting the conic (1e-5 (lambda_max + 0.3))."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    cams = [gs.uniforms_from_camera(p, q, 50.0, 0.1, 1000.0, 320, 240) for p, q, *_ in scenes.CAMERAS.values()]
    models = [_lens(gs, u, names[i % len(names)]) for i, u in enumerate(cams)]
    v = torch.from_numpy(vtx).cuda()
    var = lctx.filter3d_variance(v, cams, models)
    lctx.upload(gs.apply_filter_3d(v, var).contiguous())
    lctx.set_debug(True)
    s_min, _ = lr.scales(vtx[:, 0:3], cams, models)
    checked = 0
    for u, m in zip(cams, models):
        s_c, seen_c = lr.camera_scale(vtx[:, 0:3], u, m)
        attains = seen_c & (s_c == s_min)
        lctx.set_camera_model(m if m.kind != gs.CAMERA_PINHOLE else None)
        lctx.render(u)
        attr = lctx.download(gs.BUF_ATTR)
        live = (attr["magic"] != 0) & attains
        a, b, c = (attr["conic_opacity"][live][:, j].astype(np.float64) for j in range(3))
        det = a * c - b * b
        m00, m01, m11 = c / det - 0.3, -b / det, a / det - 0.3
        mid, rad = 0.5 * (m00 + m11), np.sqrt(0.25 * (m00 - m11) ** 2 + m01 * m01)
        lam_min, lam_max = mid - rad, mid + rad
        assert bool((lam_min >= 0.2 * (1 - 1e-5) - 1e-5 * (lam_max + 0.3)).all()), float(lam_min.min())
        checked += int(live.sum())
    lctx.set_camera_model(None)
    assert checked > 500
    print(f"{'/'.join(names)}: {checked} survivors checked at their attaining camera")


def test_reproducible_over_calls_streams_contexts_and_orders(gs, lctx):
    torch = _torch()
    v = _rows(cloud(50_000, seed=3))
    cams, models = _views(gs, 100, 3, ["fish200", "phone", "pinhole", "fish180"])
    first = lctx.filter3d_variance(v, cams, models).cpu()
    assert torch.equal(first.view(torch.int32), lctx.filter3d_variance(v, cams, models).cpu().view(torch.int32))
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        other = lctx.filter3d_variance(v, cams, models)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int32), other.cpu().view(torch.int32))
    fresh = gs.Context(0)  # never had a scene
    try:
        assert torch.equal(first.view(torch.int32), fresh.filter3d_variance(v, cams, models).cpu().view(torch.int32))
    finally:
        fresh.close()
    perm = np.random.default_rng(7).permutation(len(cams))
    permuted = lctx.filter3d_variance(v, [cams[i] for i in perm], [models[i] for i in perm]).cpu()
    assert torch.equal(first.view(torch.int32), permuted.view(torch.int32))


def test_leaves_scene_and_last_frame_alone(gs, lctx):
    torch = _torch()
    _, vtx, u = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    gi = torch.from_numpy(grad_image(u)).cuda()
    other = _rows(cloud(20_000, seed=9))
    cams, models = _views(gs, 8, 9, ["fish200", "phone"])
    lctx.upload(vtx)
    lctx.set_backward_deterministic(True)

    def frame_and_grad(between):
        render(lctx, u)
        torch.cuda.synchronize()
        if between:
            lctx.filter3d_variance(other, cams, models)
        gv = torch.empty_like(v)
        lctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr())
        torch.cuda.synchronize()
        return gv.cpu(), lctx.render(u)

    g0, f0 = frame_and_grad(False)
    g1, f1 = frame_and_grad(True)
    assert torch.equal(g0.view(torch.int32), g1.view(torch.int32))
    assert np.array_equal(f0.view(np.uint32), f1.view(np.uint32))
    assert lctx.num_gaussians == vtx.shape[0]


def test_error_cases(gs, lctx):
    torch = _torch()
    v = _rows(cloud(100, seed=1))
    out = torch.empty(100, dtype=torch.float32, device="cuda")
    c1 = [scenes.camera(k) for k in scenes.CAMERAS]
    good = (gs.Uniforms * 2)(*c1[:2])
    lens = [_lens(gs, c1[0], "phone"), _lens(gs, c1[1], "fish200")]
    goodm = (gs.CameraModel * 2)(*lens)
    entry = "gsb_filter3d_variance_lens"

    def raw(c, vp=v.data_ptr(), n=100, cams=good, models=goodm, k=2, op=out.data_ptr()):
        return lambda: c._ck(gs.lib.gsb_filter3d_variance_lens(c.h, vp, n, cams, models, k, op, None))

    assert gs.lib.gsb_filter3d_variance_lens(None, v.data_ptr(), 100, good, goodm, 2, out.data_ptr(), None) == gs.ERR_INVALID
    raw(lctx)()  # needs no scene
    expect(gs, lctx, gs.ERR_INVALID, raw(lctx, k=0), entry)
    expect(gs, lctx, gs.ERR_INVALID, raw(lctx, cams=None), entry)
    expect(gs, lctx, gs.ERR_INVALID, raw(lctx, models=None), entry)
    expect(gs, lctx, gs.ERR_INVALID, raw(lctx, vp=None), entry)
    expect(gs, lctx, gs.ERR_INVALID, raw(lctx, op=None), entry)
    expect(gs, lctx, gs.ERR_INVALID, raw(lctx, vp=v.data_ptr() + 4), entry)
    expect(gs, lctx, gs.ERR_INVALID, raw(lctx, op=out.data_ptr() + 2), entry)
    for field, value in (("width", 0), ("height", 0)):
        bad = (gs.Uniforms * 2)(*c1[:2])
        setattr(bad[1], field, value)
        expect(gs, lctx, gs.ERR_INVALID, raw(lctx, cams=bad), entry)
    # a lens camera's tan_fov is not read; a pinhole camera's is checked
    bad = (gs.Uniforms * 2)(*c1[:2])
    bad[1].tan_fovx = float("nan")
    raw(lctx, cams=bad)()
    pin = (gs.CameraModel * 2)(lens[0], gs.CameraModel())
    for field, value in (("tan_fovx", 0.0), ("tan_fovx", -1.0), ("tan_fovy", float("inf")), ("tan_fovy", float("nan"))):
        bad = (gs.Uniforms * 2)(*c1[:2])
        setattr(bad[1], field, value)
        expect(gs, lctx, gs.ERR_INVALID, raw(lctx, cams=bad, models=pin), entry)
    # every lens gsb_set_camera_model refuses is refused here, and the setter still refuses it with its own message
    refused = []
    for field, value in (("kind", 7), ("fx", 0.0), ("fy", float("inf")), ("cx", float("nan")), ("max_theta", 0.0),
                         ("max_theta", 3.2)):
        m = gs.fisheye_camera(300.0, 300.0, 160.0, 120.0)
        setattr(m, field, value)
        refused.append(m)
    refused.append(gs.fisheye_camera(300.0, 300.0, 160.0, 120.0, (-0.4, 0.0, 0.0, 0.0), 3.0))  # theta_d not increasing
    refused.append(gs.opencv_camera(300.0, 300.0, 160.0, 120.0, (0.0, 0.0, 0.0, 0.0), 1.6))  # max_theta >= pi / 2
    refused.append(gs.opencv_camera(300.0, 300.0, 160.0, 120.0, (-0.5, 0.0, 0.0, 0.0), 1.2))  # r R(r^2) not increasing
    for m in refused:
        expect(gs, lctx, gs.ERR_INVALID, raw(lctx, models=(gs.CameraModel * 2)(lens[0], m)), entry)
        expect(gs, lctx, gs.ERR_INVALID, lambda: lctx.set_camera_model(m), "gsb_set_camera_model: ")
    assert lctx.camera is None or lctx.camera.kind == gs.CAMERA_PINHOLE
    raw(lctx, vp=None, n=0, op=None)()  # n = 0
    with pytest.raises(ValueError):
        lctx.filter3d_variance(v, c1[:2], lens[:1])
    with pytest.raises(ValueError):
        lctx.filter3d_variance(v, c1[:2], [lens[0], "fisheye"])
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, raw(c0), entry)
    finally:
        grp.close()


# ---- SceneAdam with the filter through a lens ----

def _lens_training(gs, ctx, name, every=4):
    """(start, views, targets, lens): c1 rendered through one lens (the context's camera model) from POSES."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = [gs.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 320, 240) for p, q in POSES]
    lens = lens_for(gs, views[0], name)
    ctx.set_camera_model(lens)
    with torch.no_grad():
        targets = [gs.render_torch(ctx, full, u).clone() for u in views]
    start = full[::every].clone()
    start[:, 4:7] *= 1.5
    return start, views, targets, lens


@pytest.mark.parametrize("name", ["fish180", "phone"])
def test_scene_adam_with_lens_filter_fits(gs, lctx, name):
    torch = _torch()
    start, views, targets, lens = _lens_training(gs, lctx, name)
    opt = gs.SceneAdam(lctx, start, TRAIN_LR, filter_cameras=views, filter_lenses=lens)
    want = lctx.filter3d_variance(opt.params, views, lens)
    assert torch.equal(opt.variance.view(torch.int32), want.view(torch.int32))
    assert not torch.equal(opt.variance, lctx.filter3d_variance(opt.params, views))  # the lens is not the UBO's pinhole
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    loss0, dssim0 = _evaluate(gs, lctx, opt, views, targets)
    for it in range(300):
        k = it % 3
        lctx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g)
        if it % 100 == 99:
            before = opt.variance.clone()
            opt.update_filter_3d()
            again = lctx.filter3d_variance(opt.params, views, lens)
            assert torch.equal(opt.variance.view(torch.int32), again.view(torch.int32))
            assert not torch.equal(before, opt.variance)
    loss1, dssim1 = _evaluate(gs, lctx, opt, views, targets)
    print(f"SceneAdam {name} with the lens filter: loss {loss0:.5f} -> {loss1:.5f}, 1 - SSIM {dssim0:.5f} -> {dssim1:.5f}")
    assert loss1 < 0.8 * loss0 and dssim1 < dssim0
    lctx.set_camera_model(None)  # _assert_coherent's fresh context renders through the pinhole
    _assert_coherent(gs, lctx, opt.vertices, views)


def test_densify_refilters_through_the_lens(gs, lctx):
    torch = _torch()
    start, views, targets, lens = _lens_training(gs, lctx, "fish180", every=8)
    opt = gs.SceneAdam(lctx, start, TRAIN_LR, filter_cameras=views, filter_lenses=lens)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    dens = torch.zeros((start.shape[0], 4), dtype=torch.float32, device="cuda")
    for it in range(30):
        k = it % 3
        lctx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g, density=dens)
    torch.cuda.synchronize()
    thr = float(torch.quantile((dens[:, 0] / dens[:, 2].clamp(min=1))[dens[:, 2] > 0], 0.8))
    opt.densify(dens, grad_threshold=thr, scene_extent=2.0, min_opacity=0.05, generator=torch.Generator(device="cuda").manual_seed(1))
    n = opt.vertices.shape[0]
    assert opt.variance.shape == (n,) and n != start.shape[0]
    assert torch.equal(opt.variance.view(torch.int32), lctx.filter3d_variance(opt.params, views, lens).view(torch.int32))
    torch.testing.assert_close(opt.vertices, gs.apply_filter_3d(gs.activate_parameters(opt.params), opt.variance),
                               rtol=1e-6, atol=1e-7)
    opt.render(views[0])
    opt.step(g)
    lctx.set_camera_model(None)


def test_baked_ply_renders_the_resident_scene_through_the_lens(gs, lctx, tmp_path):
    torch = _torch()
    start, views, targets, lens = _lens_training(gs, lctx, "phone")
    opt = gs.SceneAdam(lctx, start, TRAIN_LR, filter_cameras=views, filter_lenses=[lens] * len(views))
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    for it in range(60):
        lctx.image_loss(opt.render(views[it % 3]), targets[it % 3], 0.2, grad_image=g)
        opt.step(g)
    torch.cuda.synchronize()
    path = tmp_path / "filtered_lens.ply"
    gs.write_ply(path, gs.ply_records(gs.raw_parameters(opt.vertices.double())))
    loaded = gs.load_ply(path)
    fresh = gs.Context(0)
    try:
        fresh.set_camera_model(lens)
        fresh.upload(loaded)
        for u in views:
            diff = np.abs(opt.render(u).cpu().numpy() - fresh.render(u))
            off = float((diff > 1e-4).mean())
            print(f"baked PLY through the lens: pixels off by more than 1e-4: {off:.2e}, largest {float(diff.max()):.2e}")
            assert off <= 1e-3 and float(diff.max()) <= 2.0 / 255
    finally:
        fresh.close()
        lctx.set_camera_model(None)
