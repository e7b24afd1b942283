"""gsb_set_background / gsb_background_gradient: frames against the oracle composited over the background (tests/bg_ref.py) bit
for bit, the backward pass against the float64 reference with the T_final * bg term, dL/d(background), and training with a
fixed, a random and a learned background."""
import math
import sys
from pathlib import Path

import numpy as np
import pytest

import bg_ref
import edge_scene
import scenes
from backward_util import GROUPS, expect, grad_image, rel

pytestmark = pytest.mark.gpu

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
BACKGROUNDS = [(1.0, 1.0, 1.0), (0.25, 0.5, 0.75), (-0.5, 2.0, 0.1), (0.0, 0.0, 0.0)]
EPS = float(np.finfo(np.float32).eps)


def _torch():
    import torch

    return torch


@pytest.fixture
def bctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _scene(name):
    if name == "edge":
        return edge_scene.vertices()[0], edge_scene.camera("axis")
    _, vtx, _ = scenes.c1()
    return vtx, scenes.camera(name)


def _oracle_bg(oracle, vtx, u, bg, antialiased=False, rows=None):
    oracle.set_exp_mode(1)
    try:
        return bg_ref.oracle_frame(vtx, oracle.cov3d(vtx), u, bg, antialiased=antialiased, rows=rows)
    finally:
        oracle.set_exp_mode(0)


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside", "edge"])
def test_frames_match_the_composited_oracle(gs, oracle, bctx, cam):
    """Levels 0/1/2 x direct launches and graph replay x RGBA32F / RGBA8 / BGRA8, recorded frames too: bit-exact vs the oracle
    composited over bg; FAST within 1e-4 off the step pixels; bg = 0 and set-then-reset give the default frame bit for bit."""
    vtx, u = _scene(cam)
    bctx.upload(vtx)
    bctx.set_mode(gs.MODE_EXACT)
    plain = bctx.render(u)
    oracle.set_exp_mode(1)
    try:
        _, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)
    for bg in BACKGROUNDS:
        ref = _oracle_bg(oracle, vtx, u, bg)
        bctx.set_background(bg)
        for level in (0, 1, 2):
            bctx.set_tile_cull(level)
            for timers in (True, False, False):
                bctx.set_timers(timers)
                assert np.array_equal(bctx.render(u), ref["rgba"]), (cam, bg, level, timers)
            bctx.set_timers(True)
            assert np.array_equal(bctx.render(u, gs.FORMAT_RGBA8), oracle.pack_unorm8(ref["rgba"])), (cam, bg, level)
            assert np.array_equal(bctx.render(u, gs.FORMAT_BGRA8), oracle.pack_unorm8(ref["rgba"], bgra=True)), (cam, bg, level)
            bctx.set_backward(True)  # the recording instantiations
            assert np.array_equal(bctx.render(u), ref["rgba"]), (cam, bg, level, "recorded")
            bctx.set_backward(False)
            if cam != "edge":
                bctx.set_mode(gs.MODE_FAST)
                assert np.abs(bctx.render(u) - ref["rgba"])[~steps].max() <= 1e-4 * max(1.0, max(map(abs, bg))), (cam, bg, level)
                bctx.set_mode(gs.MODE_EXACT)
        bctx.set_tile_cull(0)
        if bg == (0.0, 0.0, 0.0):
            assert np.array_equal(bctx.render(u), plain)
    bctx.set_background((-0.0, 0.0, -0.0))
    assert np.array_equal(bctx.render(u), plain)
    bctx.set_background(None)
    assert np.array_equal(bctx.render(u), plain)


def test_bands_match_the_composited_oracle(gs, oracle, bctx):
    vtx, u = _scene("odd_size")
    bctx.upload(vtx)
    bctx.set_background((0.25, 0.5, 0.75))
    tiles_y = (u.height + 15) // 16
    for rows in ((0, 1), (tiles_y // 2, tiles_y // 2 + 2), (tiles_y - 1, tiles_y)):
        ref = _oracle_bg(oracle, vtx, u, (0.25, 0.5, 0.75), rows=rows)
        sl = slice(rows[0] * 16, min(u.height, rows[1] * 16))
        assert np.array_equal(bctx.render(u, rows=rows), ref["rgba"][sl]), rows


def test_empty_scene_is_the_background(gs, bctx):
    u = scenes.camera("odd_size")
    bctx.upload(np.zeros((0, 60), np.float32))
    for bg in BACKGROUNDS[:3]:
        bctx.set_background(bg)
        img = bctx.render(u)
        assert np.array_equal(img[..., :3], np.broadcast_to(np.float32(bg), img[..., :3].shape)) and (img[..., 3] == 1).all()


def test_group_ranks_equal_the_single_gpu_frame(gs, oracle):
    vtx, u = _scene("c1")
    bg = (-0.5, 2.0, 0.1)
    ref = _oracle_bg(oracle, vtx, u, bg)
    for world in (1, 2, 3):
        grp = gs.Group([0] * world)
        try:
            for r in range(world):
                grp.context(r).set_background(bg)
            grp.upload(vtx)
            assert np.array_equal(grp.render(u), ref["rgba"]), world
        finally:
            grp.close()


def test_background_with_antialiasing_equals_the_composed_references(gs, oracle, bctx):
    vtx, u = _scene("c1")
    bg = (0.25, 0.5, 0.75)
    ref = _oracle_bg(oracle, vtx, u, bg, antialiased=True)
    bctx.upload(vtx)
    bctx.set_antialiased(True)
    bctx.set_background(bg)
    for level in (0, 1, 2):
        bctx.set_tile_cull(level)
        assert np.array_equal(bctx.render(u), ref["rgba"]), level


# ---------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------
def _backward(gs, vtx, u, g, bg, level=0, deterministic=False, density=False, flip_to=None):
    """A frame of u over bg on a fresh context and its backward: (grad_vertices, density or None, grad_background) on the
    host.  flip_to: set this background between the frame and the backward call."""
    torch = _torch()
    ctx = gs.Context(0)
    try:
        ctx.upload(vtx)
        ctx.set_tile_cull(level)
        ctx.set_backward(True)
        ctx.set_backward_deterministic(deterministic)
        ctx.set_background(bg)
        ctx.render(u)
        if flip_to is not None:
            ctx.set_background(flip_to)
        v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
        gi = torch.from_numpy(g).cuda()
        gv = torch.full_like(v, float("nan"))
        dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if density else None
        ctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), density_ptr=dens.data_ptr() if density else None)
        gb = ctx.background_gradient(gi)
        torch.cuda.synchronize()
    finally:
        ctx.close()
    return gv.cpu().numpy(), None if dens is None else dens.cpu().numpy(), gb.cpu().numpy()


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
@pytest.mark.parametrize("bg", BACKGROUNDS[:3])
def test_gradient_matches_float64_reference(gs, oracle, cam, bg):
    vtx, u = _scene(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    ref = bg_ref.reference(vtx, u, frame, bg, g)
    keep = ~ref["exclude"]
    dref = bg_ref.density_reference(vtx, u, frame, bg, g)
    assert keep.sum() > 100
    for level in (0, 1):
        gv, dens, _ = _backward(gs, vtx, u, g, bg, level=level, density=True)
        assert np.isfinite(gv).all()
        for name, cols in GROUPS.items():
            r = rel(gv[keep, cols].astype(np.float64), ref["grad"][keep, cols])
            assert r <= 1e-3, (cam, bg, level, name, r)
        for c in (0, 1):
            assert rel(dens[keep, c].astype(np.float64), dref["density"][keep, c]) <= 1e-3, (cam, bg, level, c)
        assert np.array_equal(dens[:, 2], dref["survivor"].astype(np.float32))


def test_gradient_on_the_edge_scene(gs, oracle):
    """Breaks, 0.99 clamps, opacity edges and empty tiles: the per-group comparison of the edge scene's backward tests."""
    from test_gpu_backward_regimes import _check_vertices

    vtx, masks, _ = edge_scene.vertices("backward")
    u = edge_scene.camera("axis")
    bg = (-0.5, 2.0, 0.1)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    ref = bg_ref.reference(vtx, u, frame, bg, g)
    keep = ~ref["exclude"]
    sets = {k: keep & m & (frame["attr"]["color_radii"][:, 3] != 0) for k, m in masks.items()}
    sets = {k: s for k, s in sets.items() if (np.abs(ref["grad"][s]).sum(1) > 0).any()}
    for det in (False, True):
        gv, _, _ = _backward(gs, vtx, u, g, bg, deterministic=det)
        _check_vertices(gv.astype(np.float64), ref["grad"], keep, sets, ("edge", det), set_atol=True, min_rows=1)


def test_deterministic_follows_the_frame_and_zero_is_the_default_path(gs):
    vtx, u = _scene("c1")
    g = grad_image(u)
    bg = (0.25, 0.5, 0.75)
    runs = [_backward(gs, vtx, u, g, bg, level=lv, deterministic=True, density=True) for lv in (0, 0, 1)]
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert a.tobytes() == b.tobytes()
    # the backward follows the frame's colour, not the setting at the time of the call
    flipped = _backward(gs, vtx, u, g, bg, deterministic=True, density=True, flip_to=(0.0, 0.0, 0.0))
    assert all(a.tobytes() == b.tobytes() for a, b in zip(runs[0], flipped))
    black = _backward(gs, vtx, u, g, (0.0, 0.0, 0.0), deterministic=True, density=True)
    assert black[0].tobytes() != runs[0][0].tobytes()
    # bg = 0 is the default path: the same words as a context that never set a background
    torch = _torch()
    c = gs.Context(0)
    try:
        c.upload(vtx)
        c.set_backward(True)
        c.set_backward_deterministic(True)
        c.render(u)
        v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
        gi = torch.from_numpy(g).cuda()
        gv = torch.full_like(v, float("nan"))
        dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
        c.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), density_ptr=dens.data_ptr())
        torch.cuda.synchronize()
        assert gv.cpu().numpy().tobytes() == black[0].tobytes() and dens.cpu().numpy().tobytes() == black[1].tobytes()
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# gsb_background_gradient
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", ["c1", "odd_size", "edge"])
def test_background_gradient_is_the_sum_of_t_times_g(gs, oracle, cam):
    """Within 1 fp32 ulp + 1e-9 sum |T g| of math.fsum over the oracle's T; bit-identical over calls, streams, a fresh
    context, levels 0 and 1, both deterministic settings and the frame's own background."""
    torch = _torch()
    vtx, u = _scene(cam)
    T = _oracle_bg(oracle, vtx, u, (0.0, 0.0, 0.0))["T"].astype(np.float64)
    g = grad_image(u)
    want = np.array([math.fsum((T * g[..., c].astype(np.float64)).ravel()) for c in range(3)])
    scale = np.abs(T[..., None] * g[..., :3].astype(np.float64)).sum((0, 1))
    gi = torch.from_numpy(g).cuda()
    words = set()
    for level in (0, 1):
        for det in (False, True):
            for bg in ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)):
                c = gs.Context(0)
                try:
                    c.upload(vtx)
                    c.set_tile_cull(level)
                    c.set_backward(True)
                    c.set_backward_deterministic(det)
                    c.set_background(bg)
                    c.render(u)
                    s = torch.cuda.Stream()
                    outs = [c.background_gradient(gi), c.background_gradient(gi, s)]
                    torch.cuda.synchronize()
                    for o in outs:
                        words.add(o.cpu().numpy().tobytes())
                finally:
                    c.close()
    assert len(words) == 1, cam
    got = np.frombuffer(next(iter(words)), np.float32).astype(np.float64)
    tol = np.abs(want) * EPS + 1e-9 * scale
    assert (np.abs(got - want) <= tol).all(), (cam, got, want)


def test_background_gradient_of_an_empty_scene_is_the_sum_of_g(gs, bctx):
    torch = _torch()
    u = scenes.camera("odd_size")
    bctx.upload(np.zeros((0, 60), np.float32))
    bctx.set_backward(True)
    bctx.render(u)
    g = grad_image(u)
    got = bctx.background_gradient(torch.from_numpy(g).cuda()).cpu().numpy().astype(np.float64)
    want = np.array([math.fsum(g[..., c].astype(np.float64).ravel()) for c in range(3)])
    assert (np.abs(got - want) <= np.abs(want) * EPS + 1e-9 * np.abs(g[..., :3]).sum((0, 1))).all()


def test_error_cases(gs, bctx):
    torch = _torch()
    lib = gs.lib
    import ctypes

    three = (ctypes.c_float * 3)(0.0, 0.0, 0.0)
    assert lib.gsb_set_background(None, three) == gs.ERR_INVALID
    for bad in ((float("nan"), 0, 0), (0, float("inf"), 0), (0, 0, -float("inf"))):
        expect(gs, bctx, gs.ERR_INVALID, lambda: bctx.set_background(bad), "gsb_set_background")
    u = scenes.camera("odd_size")
    g = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    out = torch.empty(3, dtype=torch.float32, device="cuda")
    assert lib.gsb_background_gradient(None, g.data_ptr(), 0, out.data_ptr(), None) == gs.ERR_INVALID
    e = "gsb_background_gradient"
    expect(gs, bctx, gs.ERR_NO_SCENE, lambda: bctx.background_gradient(g), e)
    _, vtx, _ = scenes.c1()
    bctx.upload(vtx)
    expect(gs, bctx, gs.ERR_NO_SCENE, lambda: bctx.background_gradient(g), e)  # no frame yet
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID, lambda: bctx.background_gradient(g), e)  # not recorded
    bctx.set_backward(True)
    bctx.render(u, rows=(0, 1))
    expect(gs, bctx, gs.ERR_INVALID, lambda: bctx.background_gradient(g), e)  # a band
    bctx.render(u)
    assert lib.gsb_background_gradient(bctx.h, None, 0, out.data_ptr(), None) == gs.ERR_INVALID
    assert lib.gsb_background_gradient(bctx.h, g.data_ptr(), 0, None, None) == gs.ERR_INVALID
    assert lib.gsb_background_gradient(bctx.h, g.data_ptr(), 8, out.data_ptr(), None) == gs.ERR_INVALID  # pitch < row
    assert lib.gsb_background_gradient(bctx.h, g.data_ptr(), u.width * 16 + 4, out.data_ptr(), None) == gs.ERR_INVALID
    bctx.upload(vtx)
    expect(gs, bctx, gs.ERR_INVALID, lambda: bctx.background_gradient(g), e)  # scene changed after the frame
    sc = gs.ShardedContext(0, 0, 1, gs.shard_unique_id())
    try:
        sc.set_background((1.0, 1.0, 1.0))  # accepted: the blend is shared
        expect(gs, sc, gs.ERR_INVALID, lambda: sc.background_gradient(g), e)
    finally:
        sc.close()


# ---------------------------------------------------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------------------------------------------------
def test_learned_background_reaches_the_targets(gs, bctx):
    """A frozen scene, a learned background from 0 through render_torch (only the background requires grad): it converges
    to the colour the target was rendered over."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 320, 240)
    v = torch.from_numpy(vtx).cuda()
    want = torch.tensor([0.8, 0.3, 0.55], device="cuda")
    with torch.no_grad():
        target = gs.render_torch(bctx, v, u, background=want).clone()
    bg = torch.zeros(3, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([bg], lr=0.05)
    for _ in range(300):
        opt.zero_grad()
        img = gs.render_torch(bctx, v, u, background=bg)
        loss = ((img[..., :3] - target[..., :3]) ** 2).mean()
        loss.backward()
        opt.step()
    print("learned background", bg.detach().cpu().numpy(), "target", want.cpu().numpy())
    assert (bg.detach() - want).abs().max().item() <= 1e-3


def _object_setup(gs, bctx):
    """Distant views of the c1 scene and their RGBA targets: colour over black and alpha = 1 - the frame's T_final (from the frame
    over white minus the frame over black)."""
    from test_gpu_adam import POSES

    torch = _torch()
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    # three times as far as test_gpu_adam's poses: the scene covers the middle of the frame and leaves empty space around it
    views = [gs.uniforms_from_camera([3.0 * x for x in p], q, 45.0, 0.1, 1000.0, 320, 240) for p, q in POSES]
    targets = []
    with torch.no_grad():
        for u in views:
            black = gs.render_torch(bctx, full, u).clone()
            white = gs.render_torch(bctx, full, u, background=torch.ones(3, device="cuda")).clone()
            rgba = black.clone()
            rgba[..., 3] = 1.0 - (white[..., 0] - black[..., 0])
            targets.append(rgba)
    start = full[::4].clone()
    start[:, 4:7] *= 1.5
    return start, views, targets


def _psnr(gs, ctx, opt, views, targets, bg):
    ms = []
    for u, t in zip(views, targets):
        opt.background = list(bg)
        ctx.set_background(bg)
        ms.append(gs.image_metrics(ctx, ctx._render_whole_frame(u, opt.vertices.device), gs.composite_target(t, bg))["psnr"])
    return sum(ms) / len(ms)


def test_scene_adam_white_background_and_random_background(gs, bctx):
    """SceneAdam over white on white-composited targets beats the same run over black; with random_background the trained
    scene matches both the black and the white composite."""
    from test_gpu_adam import TRAIN_LR

    torch = _torch()
    start, views, targets = _object_setup(gs, bctx)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    white = [gs.composite_target(t, (1.0, 1.0, 1.0)) for t in targets]
    res = {}
    for name, bg in (("white", (1.0, 1.0, 1.0)), ("black", (0.0, 0.0, 0.0))):
        opt = gs.SceneAdam(bctx, start, TRAIN_LR, background=bg)
        for it in range(300):
            k = it % 3
            bctx.image_loss(opt.render(views[k]), white[k], 0.2, grad_image=g)
            opt.step(g)
        bctx.set_background(bg)
        res[name] = sum(gs.image_metrics(bctx, opt.render(u), w)["psnr"] for u, w in zip(views, white)) / len(views)
    print(f"PSNR vs the white composite: trained over white {res['white']:.2f} dB, over black {res['black']:.2f} dB")
    # measured on an H100: 28.47 dB over white vs 14.07 dB over black (the black run must paint the white itself)
    assert res["white"] > res["black"] + 10.0, res
    opt = gs.SceneAdam(bctx, start, TRAIN_LR, random_background=True, seed=1)
    for it in range(300):
        k = it % 3
        img = opt.render(views[k])
        assert opt.background is not None and all(0.0 <= x < 1.0 for x in opt.background)
        bctx.image_loss(img, gs.composite_target(targets[k], opt.background), 0.2, grad_image=g)
        opt.step(g)
    p_black, p_white = (_psnr(gs, bctx, opt, views, targets, bg) for bg in ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)))
    print(f"random background: PSNR over black {p_black:.2f} dB, over white {p_white:.2f} dB")
    bctx.set_background(None)
    assert p_black > 24.0 and p_white > 24.0, (p_black, p_white)  # measured on an H100: 27.09 and 27.01 dB
