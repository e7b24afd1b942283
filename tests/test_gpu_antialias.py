"""gsb_set_antialiased: frames against the anti-aliased oracle (tests/aa_ref.py) bit for bit, the backward pass against the
float64 reference of the compensated function, and training and zoom-out with the mode on."""
import functools
import sys
from pathlib import Path

import numpy as np
import pytest

import aa_ref
import edge_scene
import scale_scene
import scenes
from backward_util import CAMERA_GROUPS, DEAD, GROUPS, expect, grad_image, rel, translation_identity
from test_gpu_backward_camera import camera_scene
from test_gpu_backward_regimes import _check_density, _check_vertices

pytestmark = pytest.mark.gpu

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
EPS = float(np.finfo(np.float32).eps)


def _torch():
    import torch

    return torch


@pytest.fixture
def actx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _oracle_aa(oracle, vtx, u, mode, rows=None):
    oracle.set_exp_mode(mode)
    try:
        return aa_ref.oracle_frame(vtx, oracle.cov3d(vtx), u, rows)
    finally:
        oracle.set_exp_mode(0)


def _scene(name):
    if name == "edge":
        return edge_scene.vertices()[0], edge_scene.camera("axis")
    if name == "scale":
        return scale_scene.vertices()[0], scale_scene.camera("axis")
    if name == "subpixel":
        return subpixel_scene(), scenes.camera("c1")
    _, vtx, _ = scenes.c1()
    return vtx, scenes.camera(name)


@pytest.mark.parametrize("cam", sorted(scenes.CAMERAS) + ["edge", "scale", "subpixel"])
def test_frames_match_the_antialiased_oracle(gs, oracle, actx, cam):
    """Levels 0/1/2 x direct launches (timers on) and graph replay x float and BGRA8: bit-exact vs the anti-aliased oracle
    (shared-definition exp); FAST within 1e-4 on the c1 scene, away from the pixels whose alpha < 1/255 or T < 1e-4 test
    sits on its threshold (a few ulp of exp may flip them, as for the plain frame); GSB_BUF_ATTR's opacity is the compensated one bit for bit; switching the
    mode off again gives the plain frame bit for bit."""
    vtx, u = _scene(cam)
    oracle.set_exp_mode(1)
    try:
        ref, steps = aa_ref.oracle_frame_probed(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)
    actx.upload(vtx)
    actx.set_mode(gs.MODE_EXACT)
    actx.set_tile_cull(0)
    plain = actx.render(u)
    actx.set_antialiased(True)
    for level in (0, 1, 2):
        actx.set_tile_cull(level)
        for timers in (True, False, False):
            actx.set_timers(timers)
            assert np.array_equal(actx.render(u), ref["rgba"]), (cam, level, timers)
        assert np.array_equal(actx.render(u, gs.FORMAT_BGRA8), oracle.pack_unorm8(ref["rgba"], bgra=True)), (cam, level)
        st = actx.stats()
        if level == 0:
            assert st.num_instances == ref["m"], cam
        else:
            assert st.num_instances_aabb == ref["m"], cam
        if cam in scenes.CAMERAS:  # FAST: within 1e-4 away from the step pixels (not on 45-degree needles, DESIGN.md section 2)
            actx.set_mode(gs.MODE_FAST)
            assert np.abs(actx.render(u) - ref["rgba"])[~steps].max() <= 1e-4, (cam, level)
            actx.set_mode(gs.MODE_EXACT)
    actx.set_timers(True)
    actx.set_tile_cull(0)
    actx.set_debug(True)
    try:
        actx.render(u)
        attr = actx.download(gs.BUF_ATTR)
    finally:
        actx.set_debug(False)
    assert attr["conic_opacity"].tobytes() == ref["attr"]["conic_opacity"].tobytes(), cam
    actx.set_antialiased(False)
    assert np.array_equal(actx.render(u), plain), cam


def test_full_size_bands_match_the_antialiased_oracle(gs, oracle):
    """bench.py's garden stand-in (5.8 M Gaussians, 3200 x 1400): three tile-row bands at level 1, bit-exact vs the
    anti-aliased oracle (mode 1)."""
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    vtx = bench.make_scene(gs, wl)
    u = bench.cameras(gs, wl)[3]
    tiles_y = (u.height + 15) // 16
    c = gs.Context(0)
    try:
        c.upload(vtx)
        c.set_tile_cull(1)
        c.set_antialiased(True)
        for rows in ((0, 1), (tiles_y // 2, tiles_y // 2 + 1), (tiles_y - 1, tiles_y)):
            ref = _oracle_aa(oracle, vtx, u, 1, rows)
            sl = slice(rows[0] * 16, min(u.height, rows[1] * 16))
            assert ref["m"] > 0
            assert np.array_equal(c.render(u, gs.FORMAT_RGBA32F, rows=rows), ref["rgba"][sl]), rows
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------
def _backward(gs, vtx, u, g, level=0, deterministic=False, density=False, camera=False, flip_after=False):
    """An anti-aliased frame of u on a fresh context and its backward: (grad_vertices, density or None, grad_uniforms or
    None) on the host, float32.  flip_after: switch the mode off between the frame and the backward call."""
    torch = _torch()
    ctx = gs.Context(0)
    try:
        ctx.upload(vtx)
        ctx.set_tile_cull(level)
        ctx.set_backward(True)
        ctx.set_backward_deterministic(deterministic)
        ctx.set_antialiased(True)
        ctx.render(u)
        if flip_after:
            ctx.set_antialiased(False)
        v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
        gi = torch.from_numpy(g).cuda()
        gv = torch.full_like(v, float("nan"))
        dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if density else None
        gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda") if camera else None
        ctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), grad_uniforms_ptr=gu.data_ptr() if camera else None,
                            density_ptr=dens.data_ptr() if density else None)
        torch.cuda.synchronize()
    finally:
        ctx.close()
    return tuple(None if t is None else t.cpu().numpy() for t in (gv, dens, gu))


def ill_conditioned(vtx, u, frame):
    """Survivors whose fp32 comp cannot resolve its float64 value to 1e-4 relative: comp^2 = det0 / det with det0 a
    cancelling difference (edge-on flat Gaussians, whose comp is near 0).  There fp32 and float64 take different values of
    a steep function, so the opacity gradient and the comp share of the cov2d gradient are ill-posed at fp32 resolution."""
    import oracle

    c00, c01, c10, c11, _ = (x.astype(np.float64) for x in aa_ref.cov2d_f32(vtx, oracle.cov3d(vtx), u))
    with np.errstate(all="ignore"):
        det = (c00 + 0.3) * (c11 + 0.3) - c10 * c01
        r = (c00 * c11 - c10 * c01) / det
        noise = 4 * EPS * (np.abs(c00 * c11) + np.abs(c10 * c01)) / det
        bad = ~(noise <= 1e-4 * np.abs(r))
    return bad & (frame["attr"]["color_radii"][:, 3] != 0) & (frame["comp"] > 0)


@functools.lru_cache(maxsize=None)
def _case(scene, cam, camera_grad=False):
    """(vtx, u, frame, g, ref, keep, sets) of the anti-aliased frame: the oracle's lists (libm exp), a seeded upstream
    gradient zero on the step-probed pixels, aa_ref's float64 reference, and the rows it keeps."""
    import oracle

    sets_of = None
    if scene == "c1":
        vtx = camera_scene() if camera_grad else scenes.c1()[1]
        u = scenes.camera(cam)
    elif scene == "subpixel":
        vtx, u = subpixel_scene(), scenes.camera(cam)
        sets_of = lambda f, keep: {f"comp_{lo}_{hi}": keep & (f["comp"] >= lo) & (f["comp"] < hi)  # noqa: E731
                                   for lo, hi in SUBPIXEL_COMP_BANDS}
    elif scene == "edge":
        vtx, masks, _ = edge_scene.vertices("backward")
        u = edge_scene.camera(cam)
        sets_of = lambda f, keep: {k: keep & m & (f["attr"]["color_radii"][:, 3] != 0) for k, m in masks.items()}  # noqa: E731
    else:
        vtx, masks, _, _ = scale_scene.vertices()
        u = scale_scene.camera(cam)
        sets_of = lambda f, keep: {k: keep & m for k, m in scale_scene.groups_at(masks, f).items()}  # noqa: E731
    oracle.set_exp_mode(0)
    frame, steps = aa_ref.oracle_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    ref = aa_ref.reference(vtx, u, frame, g, camera=camera_grad)
    keep = ~ref["exclude"] & ~ill_conditioned(vtx, u, frame)
    # a set is checked where the reference has a gradient (the test names the sets that must be among them)
    sets = {} if sets_of is None else {k: s for k, s in sets_of(frame, keep).items() if (np.abs(ref["grad"][s]).sum(1) > 0).any()}
    return vtx, u, frame, g, ref, keep, sets


# Sub-pixel Gaussians that stay visible: sigma about 0.3-0.9 px at c1's camera (comp about 0.2-0.75) and opacity 0.73-0.98,
# so alpha clears 1/255 on their centre pixels.  scale_scene's rows at the 0.3 floor are far smaller (comp ~ 0): under the
# mode they fall below 1/255 on every pixel and have no gradient to compare.
SUBPIXEL_COMP_BANDS = ((0.2, 0.4), (0.4, 0.6), (0.6, 0.8))


@functools.lru_cache(maxsize=None)
def subpixel_scene(n=20_000):
    import oracle

    p = oracle.synth_params(half_extent=(2.0, 1.5, 1.0), log_scale_min=float(np.log(0.002)),
                            log_scale_max=float(np.log(0.006)), opacity_min=1.0, opacity_max=4.0)
    return oracle.load_records(oracle.synth_records(11, n, p))


# the named sets of each scene whose gradients are checked per Gaussian on their own (at least one row with a gradient each)
REQUIRED_SETS = {
    "scale": {"backdrop", "needle", "far", "near"},  # plus at least one band of the huge rows, asserted below
    "edge": {"plane", "big", "ident", "dup", "opacity"},
    "subpixel": {f"comp_{lo}_{hi}" for lo, hi in SUBPIXEL_COMP_BANDS},
}


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_gradient_matches_float64_reference(gs, cam):
    vtx, u, frame, g, ref, keep, _ = _case("c1", cam)
    assert keep.sum() > 100
    for level in (0, 1):
        gv, dens, _ = _backward(gs, vtx, u, g, level=level, density=True)
        assert np.isfinite(gv).all() and not gv[:, 3].any()
        for name, cols in GROUPS.items():
            r = rel(gv[keep, cols].astype(np.float64), ref["grad"][keep, cols])
            assert r <= 1e-3, (cam, level, name, r)
        dref = aa_ref.density_reference(vtx, u, frame, g)
        for c in (0, 1):
            assert rel(dens[keep, c].astype(np.float64), dref["density"][keep, c]) <= 1e-3, (cam, level, c)
        assert np.array_equal(dens[:, 2], dref["survivor"].astype(np.float32)), cam
        assert np.array_equal(dens[:, 3].view(np.uint32), dref["radii"].astype(np.float32).view(np.uint32)), cam


@pytest.mark.parametrize("scene,cam", [("scale", c) for c in scale_scene.CAMERAS] + [("edge", c) for c in edge_scene.BACKWARD_CAMERAS]
                         + [("subpixel", "c1")])
def test_gradient_on_the_scale_edge_and_subpixel_scenes(gs, scene, cam):
    """Needles and edge-on discs (comp 0 or near it), huge Gaussians, and visible sub-pixel Gaussians with comp in 0.2-0.8,
    where the compensation's share of the chain rule is largest: per group and per Gaussian, each named set on its own,
    with the per-group tolerances of test_gpu_backward_scale.py."""
    vtx, u, frame, g, ref, keep, sets = _case(scene, cam)
    surv = frame["attr"]["color_radii"][:, 3] != 0
    print(scene, cam, "survivors", int(surv.sum()), "comp == 0:", int((surv & (frame["comp"] == 0)).sum()),
          "comp < 0.5:", int((surv & (frame["comp"] < 0.5)).sum()), "ill-conditioned:", int((surv & ~keep).sum()),
          "sets:", {k: int(v.sum()) for k, v in sets.items()})
    assert REQUIRED_SETS[scene] <= set(sets), (scene, cam, sorted(sets))
    if scene == "scale":
        assert any(k.startswith("huge") for k in sets), (cam, sorted(sets))
    if scene == "subpixel":
        assert all(sets[k].sum() >= 100 for k in REQUIRED_SETS[scene]), {k: int(v.sum()) for k, v in sets.items()}
    for level in (0, 1):
        for det in (False, True):
            gv, dens, _ = _backward(gs, vtx, u, g, level=level, deterministic=det, density=True)
            _check_vertices(gv.astype(np.float64), ref["grad"], keep, sets, (scene, cam, level, det), set_atol=True, min_rows=1)
            zero = surv & (frame["comp"] == 0)
            assert not gv[zero, 7].any()  # d opacity = d(o comp) comp = 0 where comp = 0
    dref = aa_ref.density_reference(vtx, u, frame, g)
    _check_density(dens.astype(np.float64), dref, keep, (scene, cam))


@pytest.mark.parametrize("cam", ["c1", "odd_size"])
def test_camera_gradient_matches_float64_reference(gs, cam):
    vtx, u, frame, g, ref, keep, _ = _case("c1", cam, camera_grad=True)
    assert not ref["exclude"].any()
    want = np.zeros(40)
    want[gs.UBO_FLOAT_WORDS] = ref["grad_ubo"]
    for level in (0, 1):
        _, _, got = _backward(gs, vtx, u, g, level=level, camera=True)
        got = got.astype(np.float64)
        assert np.isfinite(got).all() and not got[DEAD].any()
        for name, idx in CAMERA_GROUPS.items():
            r = rel(got[idx], want[idx])
            assert r <= 1e-3, (cam, level, name, r)


def test_translation_identity_at_full_size(gs):
    """The camera-side terms of the translation identity equal the summed position gradient with the mode on."""
    import bench

    torch = _torch()
    wl = bench.WORKLOADS["garden-standin"]
    u = bench.cameras(gs, wl)[0]
    ctx = gs.Context(0)
    try:
        ctx.set_tile_cull(1)
        ctx.set_backward(True)
        ctx.set_antialiased(True)
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
    assert np.abs(g38).max() > 0
    assert (np.abs(res) <= 1e-5 * scale).all(), (res, scale)


def test_deterministic_is_reproducible_and_level_independent(gs):
    vtx, u, _, g, _, _, _ = _case("c1", "c1")
    runs = [_backward(gs, vtx, u, g, level=lv, deterministic=True, density=True, camera=True) for lv in (0, 0, 1, 2)]
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert a.tobytes() == b.tobytes()


def _plain_backward(gs, vtx, u, g, flip_after):
    """The deterministic gradient of a plain frame; flip_after: the mode is switched on between the frame and the backward."""
    torch = _torch()
    c = gs.Context(0)
    try:
        c.upload(vtx)
        c.set_backward(True)
        c.set_backward_deterministic(True)
        c.render(u)
        if flip_after:
            c.set_antialiased(True)
        v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
        gi = torch.from_numpy(g).cuda()
        out = torch.full_like(v, float("nan"))
        c.render_backward(v.data_ptr(), gi.data_ptr(), out.data_ptr())
        torch.cuda.synchronize()
        return out.cpu().numpy()
    finally:
        c.close()


@pytest.mark.parametrize("scene", ["c1", "subpixel"])
def test_backward_follows_the_frames_setting(gs, scene):
    """A backward after the switch is flipped differentiates the frame as it was rendered, bit for bit (deterministic
    mode), in both directions: an anti-aliased frame with the switch turned off, and a plain frame with it turned on."""
    vtx, u, _, g, _, _, _ = _case(scene, "c1")
    want = _backward(gs, vtx, u, g, deterministic=True)[0]
    got = _backward(gs, vtx, u, g, deterministic=True, flip_after=True)[0]
    assert got.tobytes() == want.tobytes()
    plain = _plain_backward(gs, vtx, u, g, flip_after=False)
    assert _plain_backward(gs, vtx, u, g, flip_after=True).tobytes() == plain.tobytes()
    assert plain.tobytes() != want.tobytes()  # the two settings give different gradients, so the checks can tell them apart


def test_error_cases(gs, actx):
    assert gs.lib.gsb_set_antialiased(None, 1) == gs.ERR_INVALID
    assert gs.lib.gsb_set_antialiased(actx.h, 1) == gs.OK and gs.lib.gsb_set_antialiased(actx.h, 0) == gs.OK
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, lambda: c0.set_antialiased(True), "gsb_set_antialiased")
    finally:
        grp.close()
    # a gsb_create_sharded context: this process as the only rank of a world of one
    sc = gs.ShardedContext(0, 0, 1, gs.shard_unique_id())
    try:
        expect(gs, sc, gs.ERR_INVALID, lambda: sc.set_antialiased(True), "gsb_set_antialiased")
        assert gs.lib.gsb_set_antialiased(sc.h, 0) == gs.ERR_INVALID
    finally:
        sc.close()


# ---------------------------------------------------------------------------------------------------------------------
# training and zoom-out
# ---------------------------------------------------------------------------------------------------------------------
def test_scene_adam_fit_lowers_loss_and_dssim(gs, actx):
    from test_gpu_adam import TRAIN_LR, _evaluate, _training_setup

    torch = _torch()
    actx.set_antialiased(True)
    start, views, targets = _training_setup(gs, actx)
    opt = gs.SceneAdam(actx, start, TRAIN_LR, selective=True)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    loss0, dssim0 = _evaluate(gs, actx, opt, views, targets)
    for it in range(300):
        k = it % 3
        actx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g)
    loss1, dssim1 = _evaluate(gs, actx, opt, views, targets)
    print(f"SceneAdam antialiased: loss {loss0:.5f} -> {loss1:.5f}, 1 - SSIM {dssim0:.5f} -> {dssim1:.5f}")
    assert loss1 < loss0 and dssim1 < dssim0


def test_zoom_out_is_closer_to_the_box_average(gs, oracle, actx):
    """test_antialias_ref.py's zoom-out comparison on the GPU: the frames equal the oracle's, so the distances do too."""
    from test_antialias_ref import zoom_case

    W, H = 640, 480
    p = oracle.synth_params(half_extent=(2.0, 1.5, 1.0), log_scale_min=float(np.log(0.0015)),
                            log_scale_max=float(np.log(0.0045)), opacity_min=-3.0, opacity_max=1.0)
    vtx = oracle.load_records(oracle.synth_records(7, 200_000, p))
    actx.upload(vtx)
    d = {}
    for aa in (False, True):
        actx.set_antialiased(aa)
        big, small = (actx.render(gs.uniforms_from_camera([0, 0, 6], [1, 0, 0, 0], 45.0, 0.1, 1000.0, w, h))[..., :3]
                      .astype(np.float64) for w, h in ((W, H), (W // 4, H // 4)))
        box = big.reshape(H // 4, 4, W // 4, 4, 3).mean((1, 3))
        d[aa] = float(np.abs(small - box).mean())
        oracle.set_exp_mode(1)
        try:
            small_ref, box_ref = zoom_case(oracle, aa)
        finally:
            oracle.set_exp_mode(0)
        assert np.array_equal(small, small_ref) and np.array_equal(box, box_ref), aa
    print(f"GPU zoom-out mean L1: plain {d[False]:.5f}, antialiased {d[True]:.5f}")
    assert d[True] < 0.5 * d[False], d
