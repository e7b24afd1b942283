"""gsb_filter3d_variance / gsb_adam_step_filter3d / SceneAdam(filter_cameras=...): Mip-Splatting's 3D smoothing filter.
The variance equals the numpy fp32 restatement (tests/filter3d_ref.py) bit for bit, at every size and across the camera
staging chunks, is reproducible and leaves the last frame alone; the filtered step matches the float64 reference, reduces
to gsb_adam_step at zero variance and leaves a scene that renders what an upload renders; the filtered records keep every
footprint above the filter's bound; and SceneAdam trains with the filter, densifies, refuses 3DGS-MCMC and exports a PLY
that renders as the resident scene."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

import adam_ref
import edge_scene
import filter3d_ref as fr
import scenes
from backward_util import expect, grad_image, render
from test_filter3d_ref import cloud, look_at_poses, uniforms
from test_gpu_adam import LR, POSES, SIX, TRAIN_LR, _assert_coherent, _check_against_ref, _evaluate, _frame_grad, _start

pytestmark = pytest.mark.gpu

C1_CAMERAS = [scenes.camera(k) for k in scenes.CAMERAS]


def _torch():
    import torch

    return torch


@pytest.fixture
def fctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _rows(xyz):
    """(n, 60) float32 CUDA records with the given positions (the other columns are never read by the variance)."""
    torch = _torch()
    v = torch.zeros((xyz.shape[0], 60), dtype=torch.float32)
    v[:, 0:3] = torch.from_numpy(np.ascontiguousarray(xyz, np.float32))
    return v.cuda()


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("n,k", [(1, 1), (1000, 63), (4097, 64), (10_000, 65), (3000, 128), (3000, 129), (2000, 1000),
                                 ((1 << 20) + 3, 5)])
def test_variance_matches_restatement_bitwise(gs, fctx, n, k):
    xyz = cloud(n, seed=n + k)
    cams = uniforms(gs, look_at_poses(k, seed=k))
    got = fctx.filter3d_variance(_rows(xyz), cams).cpu().numpy()
    want = fr.variance_f32(xyz, cams)
    assert np.array_equal(_bits(got), _bits(want)), int((_bits(got) != _bits(want)).sum())
    print(f"n = {n}, k = {k}: {int(fr.depth_f32(xyz, cams)[1].sum())} rows seen")


def test_variance_c1_and_edge_cameras(gs, fctx):
    _, vtx, _ = scenes.c1()
    assert np.array_equal(_bits(fctx.filter3d_variance(_rows(vtx[:, 0:3]), C1_CAMERAS).cpu()), _bits(fr.variance_f32(vtx[:, 0:3], C1_CAMERAS)))
    ev = edge_scene.vertices()[0]
    cams = [edge_scene.camera(c) for c in edge_scene.CAMERAS]
    assert np.array_equal(_bits(fctx.filter3d_variance(_rows(ev[:, 0:3]), cams).cpu()), _bits(fr.variance_f32(ev[:, 0:3], cams)))


def _garden():
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    return bench, bench.WORKLOADS["garden-standin"]


def test_full_size_garden_standin(gs, fctx):
    """bench.py's 8 cameras: every row against the restatement; 300 orbit cameras: a sample of rows (unseen rows against
    the largest variance, which is the fill's)."""
    torch = _torch()
    bench, wl = _garden()
    vtx = bench.make_scene(gs, wl)
    v = torch.from_numpy(vtx).cuda()
    cams = bench.cameras(gs, wl)
    got = fctx.filter3d_variance(v, cams).cpu().numpy()
    assert np.array_equal(_bits(got), _bits(fr.variance_f32(vtx[:, 0:3], cams)))
    orbit = uniforms(gs, look_at_poses(300, seed=5, radius=(8.0, 20.0)))
    got = fctx.filter3d_variance(v, orbit).cpu().numpy()
    rows = np.random.default_rng(0).choice(vtx.shape[0], 100_000, replace=False)
    d, seen = fr.depth_f32(vtx[rows, 0:3], orbit)
    t = d[seen] / fr.focal_f32(orbit)
    assert np.array_equal(_bits(got[rows[seen]]), _bits((t * t) * np.float32(0.2)))
    assert np.array_equal(_bits(got[rows[~seen]]), _bits(np.full(int((~seen).sum()), got.max(), np.float32)))
    print(f"garden stand-in, 300 cameras: {int(seen.sum())} of the 100000 sampled rows seen")


def test_no_row_seen_gives_zeros(gs, fctx):
    _, vtx, _ = scenes.c1()
    got = fctx.filter3d_variance(_rows(vtx[:, 0:3]), [scenes.camera("away")]).cpu()
    assert not bool(got.view(_torch().int32).any())


def test_reproducible_over_calls_streams_and_contexts(gs, fctx):
    torch = _torch()
    xyz = cloud(50_000, seed=3)
    v = _rows(xyz)
    cams = uniforms(gs, look_at_poses(100, seed=3))
    first = fctx.filter3d_variance(v, cams).cpu()
    assert torch.equal(first.view(torch.int32), fctx.filter3d_variance(v, cams).cpu().view(torch.int32))
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        other = fctx.filter3d_variance(v, cams)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int32), other.cpu().view(torch.int32))
    fresh = gs.Context(0)  # never had a scene
    try:
        assert torch.equal(first.view(torch.int32), fresh.filter3d_variance(v, cams).cpu().view(torch.int32))
    finally:
        fresh.close()


def test_leaves_scene_and_last_frame_alone(gs, fctx):
    """Deterministic backward: the gradient of the last frame, the next frame and the scene size are the same words with
    and without a gsb_filter3d_variance in between."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    gi = torch.from_numpy(grad_image(u)).cuda()
    other = _rows(cloud(20_000, seed=9))
    fctx.upload(vtx)
    fctx.set_backward_deterministic(True)

    def frame_and_grad(between):
        render(fctx, u)
        torch.cuda.synchronize()
        if between:
            fctx.filter3d_variance(other, C1_CAMERAS)
        gv = torch.empty_like(v)
        fctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr())
        torch.cuda.synchronize()
        return gv.cpu(), fctx.render(u)

    g0, f0 = frame_and_grad(False)
    g1, f1 = frame_and_grad(True)
    assert torch.equal(g0.view(torch.int32), g1.view(torch.int32))
    assert np.array_equal(f0.view(np.uint32), f1.view(np.uint32))
    assert fctx.num_gaussians == vtx.shape[0]


def test_variance_error_cases(gs, fctx):
    torch = _torch()
    v = _rows(cloud(100, seed=1))
    out = torch.empty(100, dtype=torch.float32, device="cuda")
    good = (gs.Uniforms * 2)(*C1_CAMERAS[:2])
    entry = "gsb_filter3d_variance"

    def raw(c, vp=v.data_ptr(), n=100, cams=good, k=2, op=out.data_ptr()):
        return lambda: c._ck(gs.lib.gsb_filter3d_variance(c.h, vp, n, cams, k, op, None))

    assert gs.lib.gsb_filter3d_variance(None, v.data_ptr(), 100, good, 2, out.data_ptr(), None) == gs.ERR_INVALID
    raw(fctx)()  # needs no scene
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, k=0), entry)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, cams=None), entry)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, vp=None), entry)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, op=None), entry)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, vp=v.data_ptr() + 4), entry)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, op=out.data_ptr() + 2), entry)
    for field, value in (("width", 0), ("height", 0), ("tan_fovx", 0.0), ("tan_fovx", -1.0), ("tan_fovy", float("inf")),
                         ("tan_fovy", float("nan"))):
        bad = (gs.Uniforms * 2)(*C1_CAMERAS[:2])
        setattr(bad[1], field, value)
        expect(gs, fctx, gs.ERR_INVALID, raw(fctx, cams=bad), entry)
    raw(fctx, vp=None, n=0, op=None)()  # n = 0
    with pytest.raises(ValueError):
        fctx.filter3d_variance(v, [])
    with pytest.raises(ValueError):
        fctx.filter3d_variance(v[:, :59].contiguous(), C1_CAMERAS)
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, raw(c0), entry)
    finally:
        grp.close()


# ---- the filtered Adam step ----

def _filtered_start(gs, ctx, vtx, cams=C1_CAMERAS):
    """(params, exp_avg, exp_avg_sq, variance, filtered records) of _start's raw parameters, the filtered records uploaded."""
    torch = _torch()
    p, m, s = _start(gs, vtx)
    var = ctx.filter3d_variance(p, cams)
    v = gs.apply_filter_3d(gs.activate_parameters(p), var).contiguous()
    ctx.upload(v)
    return p, m, s, var, v


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
@pytest.mark.parametrize("cam", ("c1", "odd_size", "inside"))
def test_one_step_matches_reference(gs, fctx, cam, selective):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    p, m, s, var, v = _filtered_start(gs, fctx, vtx)
    gv, surv = _frame_grad(fctx, v, scenes.camera(cam))
    cfg = gs.adam_config(LR, step=3, selective=selective)
    ref = fr.step(p.cpu(), m.cpu(), s.cpu(), gv.cpu(), cfg, var.cpu(), surv.cpu() if selective else None)
    out = v.clone()
    fctx.adam_step(p, m, s, gv, out, cfg, variance=var)
    torch.cuda.synchronize()
    rows = surv.cpu() if selective else torch.ones(v.shape[0], dtype=torch.bool)
    assert 100 < int(surv.sum()) < v.shape[0]
    _check_against_ref(f"{cam} {'selective' if selective else 'dense'} filtered step", (p, m, s, out), ref, rows, 1e-6)


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_twenty_steps_track_reference(gs, fctx, selective):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    p, m, s, var, v = _filtered_start(gs, fctx, vtx)
    P, M, S = p.cpu().double(), m.cpu().double(), s.cpu().double()
    names = ("c1", "odd_size", "inside")
    for t in range(1, 21):
        gv, surv = _frame_grad(fctx, v, scenes.camera(names[t % 3]), seed=t)
        cfg = gs.adam_config(LR, step=t, selective=selective)
        P, M, S, V = fr.step(P, M, S, gv.cpu(), cfg, var.cpu(), surv.cpu() if selective else None)
        fctx.adam_step(p, m, s, gv, v, cfg, variance=var)
    torch.cuda.synchronize()
    rows = torch.ones(v.shape[0], dtype=torch.bool)
    _check_against_ref(f"{'selective' if selective else 'dense'} 20 filtered steps", (p, m, s, v), (P, M, S, V), rows, 1e-5)


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_zero_filter_is_the_plain_step(gs, fctx, selective):
    """Every word of the five arrays and of the scene equals gsb_adam_step's, except that -0 may become +0."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    v0 = torch.from_numpy(vtx).cuda()
    p0, m0, s0 = _start(gs, vtx)
    fctx.upload(v0)
    gv, _ = _frame_grad(fctx, v0, u)
    zero = torch.zeros(v0.shape[0], dtype=torch.float32, device="cuda")
    cfg = gs.adam_config(LR, step=2, selective=selective)
    results = []
    for variance in (None, zero):
        fctx.upload(v0)
        render(fctx, u)
        p, m, s, v = p0.clone(), m0.clone(), s0.clone(), v0.clone()
        torch.cuda.synchronize()
        fctx.adam_step(p, m, s, gv, v, cfg, variance=variance)
        torch.cuda.synchronize()
        results.append([p, m, s, v, torch.from_numpy(fctx.download(gs.BUF_COV3D)).cuda()])
    for a, b in zip(*results):
        same = (a.view(torch.int32) == b.view(torch.int32)) | ((a == 0) & (b == 0))
        assert bool(same.all()), int((~same).sum())


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_resident_scene_equals_upload(gs, fctx, selective):
    """6 cameras x EXACT / FAST x tile-cull levels 0, 1, 2, after a filtered step."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    p, m, s, var, v = _filtered_start(gs, fctx, vtx)
    gv, _ = _frame_grad(fctx, v, u)
    fctx.set_backward(True)
    render(fctx, u)
    fctx.adam_step(p, m, s, gv, v, gs.adam_config(LR, step=1, selective=selective), variance=var)
    _assert_coherent(gs, fctx, v, SIX)


def test_selective_touches_exactly_the_survivors(gs, fctx):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    p, m, s, var, v = _filtered_start(gs, fctx, vtx)
    gv, surv = _frame_grad(fctx, v, scenes.camera("inside"))
    before = [t.clone() for t in (p, m, s, v)]
    cov0 = fctx.download(gs.BUF_COV3D)
    fctx.adam_step(p, m, s, gv, v, gs.adam_config(LR, step=1, selective=True), variance=var)
    torch.cuda.synchronize()
    cov1 = fctx.download(gs.BUF_COV3D)
    changed = torch.zeros(v.shape[0], dtype=torch.bool, device="cuda")
    for a, b in zip((p, m, s, v), before):
        changed |= (a.view(torch.int32) != b.view(torch.int32)).any(1)
        assert torch.equal(a[~surv].view(torch.int32), b[~surv].view(torch.int32))
    out = (~surv).cpu().numpy()
    assert np.array_equal(cov1[out].view(np.uint32), cov0[out].view(np.uint32))
    assert torch.equal(changed, surv)


def test_step_agrees_with_autograd_through_apply_filter_3d(gs, fctx):
    """The raw-parameter gradient autograd takes through apply_filter_3d(activate(x), v) in fp32, fed to Adam, gives the
    fused step's parameters to fp32 rounding."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    p, m, s, var, v = _filtered_start(gs, fctx, vtx)
    gv, _ = _frame_grad(fctx, v, u)
    x = p.clone().requires_grad_()
    (gs.apply_filter_3d(_activate_torch(x), var) * gv).sum().backward()
    cfg = gs.adam_config(LR, step=1)
    P, M, S = adam_ref.adam_update(p.cpu(), m.cpu(), s.cpu(), x.grad.cpu(), list(cfg.lr), cfg.beta1, cfg.beta2, cfg.eps,
                                   cfg.bias_correction1, cfg.bias_correction2_sqrt)
    fctx.adam_step(p, m, s, gv, v, cfg, variance=var)
    torch.cuda.synchronize()
    _check_against_ref("autograd through apply_filter_3d", (p, m, s, v), (P, M, S, fr.activate(P, var.cpu())),
                       torch.ones(v.shape[0], dtype=torch.bool), 1e-6)


def _activate_torch(x):
    """adam_ref.activate in differentiable torch ops of the tensor's own dtype."""
    torch = _torch()
    q = x[:, 8:12]
    return torch.cat([x[:, 0:3], torch.ones_like(x[:, 3:4]), x[:, 4:7].exp(), torch.sigmoid(x[:, 7:8]),
                      q / q.norm(dim=1, keepdim=True), x[:, 12:60]], 1)


def test_step_error_cases(gs, fctx):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    p, m, s = _start(gs, vtx)
    gv = torch.zeros_like(v)
    out = torch.empty_like(v)
    var = torch.zeros(v.shape[0], dtype=torch.float32, device="cuda")
    cfg = gs.adam_config(LR)
    entry = "gsb_adam_step_filter3d"

    def raw(c, vp=var.data_ptr(), config=cfg):
        return lambda: c._ck(gs.lib.gsb_adam_step_filter3d(c.h, p.data_ptr(), m.data_ptr(), s.data_ptr(), gv.data_ptr(),
                                                           out.data_ptr(), vp, ctypes.byref(config), None))

    assert gs.lib.gsb_adam_step_filter3d(None, p.data_ptr(), m.data_ptr(), s.data_ptr(), gv.data_ptr(), out.data_ptr(),
                                         var.data_ptr(), ctypes.byref(cfg), None) == gs.ERR_INVALID
    expect(gs, fctx, gs.ERR_NO_SCENE, raw(fctx), entry)
    fctx.upload(vtx)
    raw(fctx)()
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, vp=None), entry)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, vp=var.data_ptr() + 2), entry)
    bad = gs.adam_config(LR)
    bad.beta1 = 1.0
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, config=bad), entry)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx, config=gs.adam_config(LR, selective=True)), entry)  # no frame since the step
    with pytest.raises(ValueError):
        fctx.adam_step(p, m, s, gv, out, cfg, variance=var[:-1])
    with pytest.raises(ValueError):
        fctx.adam_step(p, m, s, gv, out, cfg, variance=var.double())
    fctx.set_sh_storage(True)
    fctx.upload(vtx)
    expect(gs, fctx, gs.ERR_INVALID, raw(fctx), entry)
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, raw(c0), entry)
    finally:
        grp.close()


# ---- the footprint bound ----

@pytest.mark.parametrize("scene", ["c1", "edge"])
def test_footprint_bound_on_the_frames(gs, fctx, scene):
    """Every seen survivor's undilated 2D covariance (GSB_BUF_ATTR conics of debug frames of the filtered records) has
    lambda_min >= 0.2 (min(f_x, f_y) d / (f v_z))^2 at every training camera, up to fp32 rounding."""
    torch = _torch()
    if scene == "c1":
        vtx, cams = scenes.c1()[1], C1_CAMERAS
    else:
        vtx, cams = edge_scene.vertices()[0], [edge_scene.camera(c) for c in edge_scene.CAMERAS]
    v = torch.from_numpy(vtx).cuda()
    var = fctx.filter3d_variance(v, cams)
    filt = gs.apply_filter_3d(v, var).contiguous()
    fctx.upload(filt)
    fctx.set_debug(True)
    d, seen = fr.depth_f32(vtx[:, 0:3], cams)
    d = np.where(seen, d, d[seen].max())
    f = fr.focal_f32(cams)
    checked = 0
    for u in cams:
        fctx.render(u)
        attr = fctx.download(gs.BUF_ATTR)
        _, seen_c = fr.depth_f32(vtx[:, 0:3], [u])
        live = (attr["magic"] != 0) & seen_c
        slack, lam_max, bound = fr.footprint_slack(attr["conic_opacity"][live][:, 0:3], attr["depth"][live], d[live], f, u)
        assert bool((slack >= -(1e-4 * bound + 1e-5 * (lam_max + 0.3))).all())
        checked += int(live.sum())
    assert checked > 100
    print(f"{scene}: {checked} (camera, survivor) pairs within the bound")


# ---- SceneAdam with the filter ----

def _training_setup(gs, ctx, every=4):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = [gs.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 320, 240) for p, q in POSES]
    with torch.no_grad():
        targets = [gs.render_torch(ctx, full, u).clone() for u in views]
    start = full[::every].clone()
    start[:, 4:7] *= 1.5
    return start, views, targets


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_scene_adam_with_filter_fits(gs, fctx, selective):
    torch = _torch()
    start, views, targets = _training_setup(gs, fctx)
    opt = gs.SceneAdam(fctx, start, TRAIN_LR, selective=selective, filter_cameras=views)
    assert torch.equal(opt.variance.view(torch.int32), fctx.filter3d_variance(opt.params, views).view(torch.int32))
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    loss0, dssim0 = _evaluate(gs, fctx, opt, views, targets)
    for it in range(300):
        k = it % 3
        fctx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g)
        if it % 100 == 99:
            opt.update_filter_3d()
    loss1, dssim1 = _evaluate(gs, fctx, opt, views, targets)
    print(f"filtered SceneAdam {'selective' if selective else 'dense'}: loss {loss0:.5f} -> {loss1:.5f}, "
          f"1 - SSIM {dssim0:.5f} -> {dssim1:.5f}")
    assert loss1 < loss0 and dssim1 < dssim0
    _assert_coherent(gs, fctx, opt.vertices, views)


def test_densify_decides_unfiltered_and_refilters(gs, fctx):
    torch = _torch()
    start, views, targets = _training_setup(gs, fctx, every=8)
    opt = gs.SceneAdam(fctx, start, TRAIN_LR, filter_cameras=views)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    dens = torch.zeros((start.shape[0], 4), dtype=torch.float32, device="cuda")
    for it in range(30):
        k = it % 3
        fctx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g, density=dens)
    torch.cuda.synchronize()
    thr = float(torch.quantile((dens[:, 0] / dens[:, 2].clamp(min=1))[dens[:, 2] > 0], 0.8))
    kw = dict(grad_threshold=thr, scene_extent=2.0, min_opacity=0.05)
    unfiltered = gs.activate_parameters(opt.params)
    want, want_src = gs.densify_and_prune(unfiltered, dens, generator=torch.Generator(device="cuda").manual_seed(1), **kw)
    source = opt.densify(dens, generator=torch.Generator(device="cuda").manual_seed(1), **kw)
    assert torch.equal(source, want_src) and torch.equal(opt.params[:, 0:3], want[:, 0:3])
    n = opt.vertices.shape[0]
    assert opt.variance.shape == (n,) and n > start.shape[0] // 2
    assert torch.equal(opt.variance.view(torch.int32), fctx.filter3d_variance(opt.params, views).view(torch.int32))
    torch.testing.assert_close(opt.vertices, gs.apply_filter_3d(want, opt.variance), rtol=1e-6, atol=1e-7)
    _assert_coherent(gs, fctx, opt.vertices, views)
    opt.render(views[0])
    opt.step(g)  # the step after densify runs on the new rows' filter


def test_mcmc_refused_with_filter(gs, fctx):
    torch = _torch()
    start, views, _ = _training_setup(gs, fctx)
    opt = gs.SceneAdam(fctx, start, TRAIN_LR, filter_cameras=views)
    with pytest.raises(ValueError):
        opt.inject_noise()
    with pytest.raises(ValueError):
        opt.relocate(start.shape[0] * 2)


def test_baked_ply_renders_the_resident_scene(gs, fctx, tmp_path):
    """write_ply(ply_records(raw_parameters(vertices))) bakes the filter in: the loaded records are within 4 ulp of the
    filtered records, and a plain context renders them within 1e-4 of the resident scene, but for the few pixels where
    such an ulp moves a Gaussian's alpha across the blend's 1/255 cut."""
    torch = _torch()
    start, views, targets = _training_setup(gs, fctx)
    opt = gs.SceneAdam(fctx, start, TRAIN_LR, filter_cameras=views)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    for it in range(60):
        fctx.image_loss(opt.render(views[it % 3]), targets[it % 3], 0.2, grad_image=g)
        opt.step(g)
    torch.cuda.synchronize()
    path = tmp_path / "filtered.ply"
    gs.write_ply(path, gs.ply_records(gs.raw_parameters(opt.vertices.double())))
    loaded = gs.load_ply(path)
    dev = opt.vertices.cpu().numpy()
    cols = np.r_[0:3, 4:60]

    def ordered(a):  # float32 bits as integers in the order of the values (-0 == +0)
        i = np.ascontiguousarray(a).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)

    ulp = int(np.abs(ordered(loaded[:, cols]) - ordered(dev[:, cols])).max())
    assert ulp <= 4, ulp
    fresh = gs.Context(0)
    try:
        fresh.upload(loaded)
        for u in views:
            diff = np.abs(opt.render(u).cpu().numpy() - fresh.render(u))
            off = float((diff > 1e-4).mean())
            print(f"baked PLY: {ulp} ulp at most; pixels off by more than 1e-4: {off:.2e}, largest {float(diff.max()):.2e}")
            assert off <= 1e-3 and float(diff.max()) <= 2.0 / 255
    finally:
        fresh.close()


def test_render_torch_with_apply_filter_3d_trains(gs, fctx):
    torch = _torch()
    start, views, targets = _training_setup(gs, fctx)
    var = fctx.filter3d_variance(start, views)
    raw = gs.raw_parameters(start).requires_grad_()
    opt = torch.optim.Adam([raw], lr=2e-3, eps=1e-15)

    def loss_of(k):
        return gs.image_loss_torch(fctx, gs.render_torch(fctx, gs.apply_filter_3d(_activate_torch(raw), var), views[k]),
                                   targets[k], 0.2)

    with torch.no_grad():
        loss0 = sum(float(loss_of(k)) for k in range(3))
    for it in range(150):
        opt.zero_grad()
        loss_of(it % 3).backward()
        opt.step()
    with torch.no_grad():
        loss1 = sum(float(loss_of(k)) for k in range(3))
    print(f"render_torch + apply_filter_3d: loss {loss0:.5f} -> {loss1:.5f}")
    assert loss1 < loss0
