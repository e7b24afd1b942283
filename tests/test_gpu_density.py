"""gsb_render_backward_density / render_torch(..., density=) / densify_and_prune: the per-Gaussian statistics of adaptive
density control match the float64 reference (tests/grad_ref.py) and the oracle's survivors and radii, accumulate over
frames, leave the gradients of the other two entries unchanged, and let a sparse scene grow while it trains."""
import numpy as np
import pytest

import grad_ref
import scenes
from backward_util import expect, grad_image, rel, render

pytestmark = pytest.mark.gpu

ENTRY = "gsb_render_backward_density"  # what its error messages start with
REF_CAMERAS = ("c1", "odd_size", "inside")


@pytest.fixture
def bctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _density_backward(ctx, vtx, g, density=None, vertices=True, camera=False):
    """gsb_render_backward_density of the context's last frame: (density, grad_vertices or None, grad_uniforms or None), the
    density accumulated into `density` (a CUDA tensor) or into a zeroed buffer."""
    import torch

    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    gi = torch.from_numpy(g).cuda()
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if density is None else density
    gv = torch.full_like(v, float("nan")) if vertices else None
    gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda") if camera else None
    ctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr() if vertices else None,
                        grad_uniforms_ptr=gu.data_ptr() if camera else None, density_ptr=dens.data_ptr())
    torch.cuda.synchronize()

    def host(t):
        return None if t is None else t.cpu().numpy().astype(np.float64)

    return host(dens), host(gv), host(gu)


def _frame_density(ctx, vtx, u, g, level=0, mode=0):
    render(ctx, u, level, mode)
    return _density_backward(ctx, vtx, g)[0]


def _same_stats(a, b, tol):
    assert rel(a[:, 0], b[:, 0]) <= tol and rel(a[:, 1], b[:, 1]) <= tol
    assert np.array_equal(a[:, 2], b[:, 2]) and np.array_equal(a[:, 3], b[:, 3])


@pytest.mark.parametrize("cam", REF_CAMERAS)
def test_density_matches_float64_reference(oracle, bctx, cam):
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    ref = grad_ref.density_reference(vtx, u, frame, g)
    keep = ~grad_ref.reference(vtx, u, frame, g)["exclude"]
    bctx.upload(vtx)
    got = _frame_density(bctx, vtx, u, g)
    assert np.isfinite(got).all()
    assert keep.sum() > 100 and got[keep, 0].max() > 0
    for c in (0, 1):
        r = rel(got[keep, c], ref["density"][keep, c])
        assert r <= 1e-3, (cam, c, r)
    assert np.array_equal(got[:, 2], ref["survivor"].astype(np.float64))
    assert np.array_equal(got[:, 3].astype(np.float32).view(np.uint32), ref["radii"].astype(np.float32).view(np.uint32))


def test_density_accumulates_over_frames(gs, bctx):
    import torch

    _, vtx, _ = scenes.c1()
    n = vtx.shape[0]
    frames = []
    for i, cam in enumerate(REF_CAMERAS):
        u = scenes.camera(cam)
        frames.append((u, grad_image(u, np.zeros((u.height, u.width), bool), seed=i)))
    single = []
    for u, g in frames:  # each frame alone, each on a fresh context
        c = gs.Context(0)
        try:
            c.upload(vtx)
            single.append(_frame_density(c, vtx, u, g))
        finally:
            c.close()
    acc = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
    bctx.upload(vtx)
    for u, g in frames:  # one context, one buffer: its abs scratch must be back at zero after every call
        render(bctx, u)
        _density_backward(bctx, vtx, g, density=acc)
    got = acc.cpu().numpy().astype(np.float64)
    want01 = sum(s[:, :2] for s in single)
    assert rel(got[:, 0], want01[:, 0]) <= 1e-6 and rel(got[:, 1], want01[:, 1]) <= 1e-6
    assert np.array_equal(got[:, 2], sum(s[:, 2] for s in single))
    assert got[:, 2].max() == 3
    assert np.array_equal(got[:, 3], np.maximum.reduce([s[:, 3] for s in single]))


def test_gradient_outputs_are_the_other_entries(bctx):
    import torch

    _, vtx, u = scenes.c1()
    g = grad_image(u, np.zeros((u.height, u.width), bool))
    bctx.upload(vtx)
    render(bctx, u)
    v = torch.from_numpy(vtx).cuda()
    gi = torch.from_numpy(g).cuda()
    want_v = torch.empty_like(v)
    bctx.render_backward(v.data_ptr(), gi.data_ptr(), want_v.data_ptr())
    cam_v, want_u = torch.empty_like(v), torch.empty(40, dtype=torch.float32, device="cuda")
    bctx.render_backward(v.data_ptr(), gi.data_ptr(), cam_v.data_ptr(), grad_uniforms_ptr=want_u.data_ptr())
    torch.cuda.synchronize()
    want_v, want_u = want_v.cpu().numpy().astype(np.float64), want_u.cpu().numpy().astype(np.float64)
    assert np.abs(want_v).max() > 0 and np.abs(want_u).max() > 0
    d_both, gv, gu = _density_backward(bctx, vtx, g, vertices=True, camera=True)
    assert rel(gv, want_v) <= 1e-6 and rel(gu, want_u) <= 1e-6
    d_v, gv, gu = _density_backward(bctx, vtx, g, vertices=True, camera=False)
    assert gu is None and rel(gv, want_v) <= 1e-6
    d_u, gv, gu = _density_backward(bctx, vtx, g, vertices=False, camera=True)
    assert gv is None and rel(gu, want_u) <= 1e-6
    for d in (d_v, d_u):
        _same_stats(d, d_both, 1e-6)


def test_levels_agree(bctx):
    _, vtx, u = scenes.c1()
    g = grad_image(u, np.zeros((u.height, u.width), bool))
    bctx.upload(vtx)
    d0 = _frame_density(bctx, vtx, u, g, level=0)
    d1 = _frame_density(bctx, vtx, u, g, level=1)
    d2 = _frame_density(bctx, vtx, u, g, level=2)  # falls back to level 1 while recording
    assert d0[:, 0].max() > 0
    _same_stats(d1, d0, 1e-6)
    _same_stats(d2, d0, 1e-6)


def test_fast_mode_close_to_exact(oracle, bctx):
    _, vtx, u = scenes.c1()
    oracle.set_exp_mode(0)
    _, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    bctx.upload(vtx)
    de = _frame_density(bctx, vtx, u, g, mode=0)
    df = _frame_density(bctx, vtx, u, g, mode=1)
    _same_stats(df, de, 1e-3)


def test_nothing_visible_leaves_the_buffer_zero(bctx):
    _, vtx, _ = scenes.c1()
    u = scenes.camera("away")
    bctx.upload(vtx)
    got = _frame_density(bctx, vtx, u, np.ones((u.height, u.width, 4), np.float32))
    assert not got.any()


def test_error_cases(gs, bctx):
    import torch

    _, vtx, u = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    gi = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    out = torch.empty_like(v)
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")

    def raw(c, gv, gu, d):
        return lambda: c._ck(gs.lib.gsb_render_backward_density(c.h, v.data_ptr(), gi.data_ptr(), 0, gv, gu, d, None))

    def bw(c):
        return raw(c, out.data_ptr(), None, dens.data_ptr())

    expect(gs, bctx, gs.ERR_NO_SCENE, bw(bctx), ENTRY)  # nothing uploaded
    bctx.upload(vtx)
    expect(gs, bctx, gs.ERR_NO_SCENE, bw(bctx), ENTRY)  # no frame yet
    bctx.set_backward(False)
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx), ENTRY)  # switch off
    bctx.set_backward(True)
    bctx.render(u, rows=(0, 2))
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx), ENTRY)  # a band
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID, raw(bctx, out.data_ptr(), None, None), ENTRY)  # a NULL density
    expect(gs, bctx, gs.ERR_INVALID, raw(bctx, None, None, dens.data_ptr()), ENTRY)  # no gradient output
    bw(bctx)()  # the whole frame: fine
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


def test_full_size_counts_every_survivor(gs):
    """On bench.py's garden stand-in (5.8 M Gaussians): one view per survivor of the frame, every value finite."""
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
        nv = ctx.stats().num_visible
        gi = torch.randn((u.height, u.width, 4), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
        dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
        gu = torch.empty(40, dtype=torch.float32, device="cuda")
        ctx.render_backward(v.data_ptr(), gi.data_ptr(), None, grad_uniforms_ptr=gu.data_ptr(), density_ptr=dens.data_ptr())
        torch.cuda.synchronize()
        count = int(dens[:, 2].double().sum())
        finite = bool(torch.isfinite(dens).all())
        seen = dens[:, 2] > 0
        radius_ok = bool((dens[seen, 3] >= 1).all()) and not dens[~seen].any()
        grad_ok = bool((dens[:, 1] >= dens[:, 0] * (1 - 1e-5)).all())
    finally:
        ctx.close()
    print("full size: num_visible", nv, "views counted", count)
    assert nv > 0 and count == nv
    assert finite and radius_ok and grad_ok


def test_render_torch_density_equals_the_context_call(gs, bctx):
    import torch

    _, vtx, u = scenes.c1()
    g = torch.from_numpy(grad_image(u, np.zeros((u.height, u.width), bool))).cuda()
    v = torch.from_numpy(vtx).cuda().requires_grad_()
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
    img = gs.render_torch(bctx, v, u, density=dens)
    (img * g).sum().backward()
    got = dens.cpu().numpy().astype(np.float64)
    want, want_v, _ = _density_backward(bctx, vtx, g.cpu().numpy())  # the same frame, again, into a zeroed buffer
    assert got[:, 0].max() > 0
    _same_stats(got, want, 1e-6)
    assert rel(v.grad.cpu().numpy().astype(np.float64), want_v) <= 1e-6
    with pytest.raises(ValueError):
        gs.render_torch(bctx, v, u, density=torch.zeros((3, 4), device="cuda"))


# training with density control: Adam step sizes, steps, when to densify, and the gradient quantile that densifies
TRAIN_STEPS, DENSIFY_EVERY, DENSIFY_UNTIL, DENSIFY_QUANTILE = 600, 100, 300, 0.8
TRAIN_LR = {"pos": 1e-3, "log_scale": 5e-3, "logit_opacity": 5e-2, "dc": 1e-2}


def _train(gs, ctx, start, views, targets, densify):
    """Adam on position, log scale, opacity logit and SH DC of the activated records `start`, over the summed-squares loss of
    the views, densifying and pruning every DENSIFY_EVERY steps up to DENSIFY_UNTIL when `densify`.  Returns (final loss, n)."""
    import torch

    def split_params(vtx):
        return {"pos": vtx[:, 0:3].clone(), "log_scale": vtx[:, 4:7].log(), "logit_opacity": torch.logit(vtx[:, 7:8].clamp(1e-6, 1 - 1e-6)),
                "dc": vtx[:, 12:15].clone()}

    def assemble(p, frozen):
        return torch.cat([p["pos"], frozen[:, 3:4], p["log_scale"].exp(), torch.sigmoid(p["logit_opacity"]), frozen[:, 8:12], p["dc"],
                          frozen[:, 15:]], 1)

    def make_opt(p):
        return torch.optim.Adam([{"params": [p[k]], "lr": TRAIN_LR[k]} for k in TRAIN_LR])

    frozen = start.clone()
    params = {k: t.requires_grad_() for k, t in split_params(start).items()}
    opt = make_opt(params)
    density = torch.zeros((start.shape[0], 4), dtype=torch.float32, device="cuda")

    def loss_of(grad):
        total = 0.0
        for u, t in zip(views, targets):
            img = gs.render_torch(ctx, assemble(params, frozen), u, density=density if grad else None)
            loss = ((img[..., :3] - t) ** 2).sum()
            if grad:
                loss.backward()  # before the next view's frame replaces this one on the context
            total += float(loss.detach())
        return total

    for step in range(1, TRAIN_STEPS + 1):
        opt.zero_grad()
        loss_of(grad=True)
        opt.step()
        if densify and step % DENSIFY_EVERY == 0 and step <= DENSIFY_UNTIL:
            with torch.no_grad():
                cur = assemble(params, frozen)
                avg = density[:, 0] / density[:, 2].clamp(min=1)
                thr = float(torch.quantile(avg[density[:, 2] > 0], DENSIFY_QUANTILE))
                new, src = gs.densify_and_prune(cur, density, grad_threshold=thr, scene_extent=10.0)
            # the optimizer state follows its rows through `src`; new rows start from their source's moments
            old = [params[k] for k in TRAIN_LR]
            frozen = frozen[src]
            params = {k: t.requires_grad_() for k, t in split_params(new).items()}
            new_opt = make_opt(params)
            for o, k in zip(old, TRAIN_LR):
                st = opt.state.get(o)
                if st:
                    new_opt.state[params[k]] = {"step": st["step"].clone(), "exp_avg": st["exp_avg"][src].clone(),
                                                "exp_avg_sq": st["exp_avg_sq"][src].clone()}
            opt = new_opt
            density = torch.zeros((new.shape[0], 4), dtype=torch.float32, device="cuda")
    with torch.no_grad():
        final = loss_of(grad=False)
    return final, frozen.shape[0]


def test_training_with_density_control(gs, bctx):
    """From every 8th Gaussian of c1 with scales x 1.5, fit c1's frames from three poses: with densify_and_prune the scene
    grows and ends at a lower loss than the same run without it."""
    import torch

    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    poses = [([0, 0, 5], [1, 0, 0, 0]), ([0.6, 0.1, 5.2], scenes.quat_axis_angle([0, 1, 0], 6)),
             ([-0.5, -0.3, 4.8], scenes.quat_axis_angle([1, 0, 0], -5))]
    views = [gs.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 320, 240) for p, q in poses]
    with torch.no_grad():
        targets = [gs.render_torch(bctx, full, u)[..., :3].clone() for u in views]
    start = full[::8].clone()
    start[:, 4:7] *= 1.5
    torch.manual_seed(0)
    plain, n_plain = _train(gs, bctx, start, views, targets, densify=False)
    torch.manual_seed(0)
    dense, n_dense = _train(gs, bctx, start, views, targets, densify=True)
    print(f"training {TRAIN_STEPS} steps from {start.shape[0]} Gaussians: without density control loss {plain:.4g} (n = {n_plain}); "
          f"with densify_and_prune loss {dense:.4g} (n = {n_dense})")
    assert n_plain == start.shape[0]
    assert n_dense > start.shape[0]
    assert dense < plain, (dense, plain)
