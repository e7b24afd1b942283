"""gsb_adam_step / Context.adam_step / SceneAdam: one fused Adam step of the resident scene matches the float64 reference
(tests/adam_ref.py) on real frame gradients, dense and selective; the selective step touches exactly the frame's survivors;
the scene it leaves renders bit for bit what an upload of its records renders, with the captured graph kept; its outputs are
bit-reproducible; every invalid call is refused; and SceneAdam trains, tracks the torch path and densifies."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

import adam_ref
import scenes
from adam_ref import GROUPS
from backward_util import expect, grad_image, rel, render

pytestmark = pytest.mark.gpu

ENTRY = "gsb_adam_step"  # what its error messages start with
REF_CAMERAS = ("c1", "odd_size", "inside")
LR = [1.6e-3, 5e-3, 5e-2, 1e-3, 2.5e-3, 1.25e-4]  # position, scale, opacity, rotation, SH DC, SH rest


def _torch():
    import torch

    return torch


@pytest.fixture
def actx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _start(gs, vtx, seed=0):
    """Raw parameters of the records (quaternions scaled to norm 1.7, so 1 / |q| matters) and non-zero seeded moments, as
    float32 CUDA tensors: (params, exp_avg, exp_avg_sq)."""
    torch = _torch()
    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    p = gs.raw_parameters(v)
    p[:, 8:12] *= 1.7
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = torch.randn(v.shape, generator=g, device="cuda") * 1e-3
    s = torch.randn(v.shape, generator=g, device="cuda").square() * 1e-6
    m[:, 3] = 0.0
    s[:, 3] = 0.0
    return p, m, s


def _frame_grad(ctx, vertices, u, seed=7, level=0, mode=0):
    """Render u on ctx (recorded) and run gsb_render_backward_density on it: (grad_vertices, survivor mask), on the GPU.
    The frame and the backward run on the context's stream, the steps on torch's: the device is synchronised in between."""
    torch = _torch()
    torch.cuda.synchronize()
    render(ctx, u, level, mode)
    gi = torch.from_numpy(grad_image(u, np.zeros((u.height, u.width), bool), seed=seed)).cuda()
    gv = torch.empty_like(vertices)
    dens = torch.zeros((vertices.shape[0], 4), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.render_backward(vertices.data_ptr(), gi.data_ptr(), gv.data_ptr(), density_ptr=dens.data_ptr())
    torch.cuda.synchronize()
    return gv, dens[:, 2] > 0


def _group_errors(got, want, rows):
    return {name: rel(got[rows][:, cols], want[rows][:, cols]) for name, cols in GROUPS.items()}


def _check_against_ref(label, gpu, ref, rows, tol):
    """gpu = (params, exp_avg, exp_avg_sq, vertices) CUDA tensors; ref = adam_ref's float64 results: per group rel L2 <= tol."""
    worst = {}
    for what, a, b in zip(("params", "exp_avg", "exp_avg_sq", "vertices"), gpu, ref):
        errs = _group_errors(a.double().cpu(), b, rows)
        worst[what] = max(errs.values())
        assert all(e <= tol for e in errs.values()), (label, what, errs)
    print(f"{label}: worst relative L2 per array {worst}")


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
@pytest.mark.parametrize("cam", REF_CAMERAS)
def test_one_step_matches_reference(gs, actx, cam, selective):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    p, m, s = _start(gs, vtx)
    v = torch.from_numpy(vtx).cuda()
    actx.upload(v)
    gv, surv = _frame_grad(actx, v, u)
    cfg = gs.adam_config(LR, step=3, selective=selective)
    ref = adam_ref.step(p.cpu(), m.cpu(), s.cpu(), gv.cpu(), cfg, surv.cpu() if selective else None)
    out = torch.empty_like(v)
    actx.adam_step(p, m, s, gv, out, cfg)
    torch.cuda.synchronize()
    rows = surv.cpu() if selective else torch.ones(v.shape[0], dtype=torch.bool)
    assert 100 < int(surv.sum()) < v.shape[0]
    _check_against_ref(f"{cam} {'selective' if selective else 'dense'} one step", (p, m, s, out), ref, rows, 1e-6)
    assert bool((out[rows.cuda(), 3] == 1).all())


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_twenty_steps_track_reference(gs, actx, selective):
    """Both sides take the GPU's gradients of the frames the stepped scene renders, 20 steps, alternating three cameras."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    p, m, s = _start(gs, vtx)
    v = torch.from_numpy(vtx).cuda()
    actx.upload(v)
    P, M, S = p.cpu().double(), m.cpu().double(), s.cpu().double()
    for t in range(1, 21):
        gv, surv = _frame_grad(actx, v, scenes.camera(REF_CAMERAS[t % 3]), seed=t)
        cfg = gs.adam_config(LR, step=t, selective=selective)
        P, M, S, V = adam_ref.step(P, M, S, gv.cpu(), cfg, surv.cpu() if selective else None)
        actx.adam_step(p, m, s, gv, v, cfg)
    torch.cuda.synchronize()
    # rows no frame kept keep their uploaded records, which the reference's activation of their raw parameters equals to
    # within rounding
    rows = torch.ones(v.shape[0], dtype=torch.bool)
    _check_against_ref(f"{'selective' if selective else 'dense'} 20 steps", (p, m, s, v), (P, M, S, V), rows, 1e-5)


def test_selective_touches_exactly_the_survivors(gs, actx):
    torch = _torch()
    _, vtx, _ = scenes.c1()
    u = scenes.camera("inside")
    p, m, s = _start(gs, vtx)
    v = torch.from_numpy(vtx).cuda()
    actx.upload(v)
    gv, surv = _frame_grad(actx, v, u)
    before = [t.clone() for t in (p, m, s, v)]
    cov0 = actx.download(gs.BUF_COV3D)
    actx.adam_step(p, m, s, gv, v, gs.adam_config(LR, step=1, selective=True))
    torch.cuda.synchronize()
    cov1 = actx.download(gs.BUF_COV3D)
    changed = torch.zeros(v.shape[0], dtype=torch.bool, device="cuda")
    for a, b in zip((p, m, s, v), before):
        changed |= (a.view(torch.int32) != b.view(torch.int32)).any(1)
    out = ~surv
    for a, b in zip((p, m, s, v), before):
        assert torch.equal(a[out].view(torch.int32), b[out].view(torch.int32))
    assert np.array_equal(cov1[out.cpu().numpy()].view(np.uint32), cov0[out.cpu().numpy()].view(np.uint32))
    assert torch.equal(changed, surv)  # the moments are non-zero, so every updated row changes
    print(f"selective: {int(surv.sum())} of {v.shape[0]} rows updated")


def _frames(gs, ctx, cams):
    """Frames of every camera in EXACT and FAST mode at tile-cull levels 0, 1 and 2, as host arrays."""
    out = []
    for mode in (gs.MODE_EXACT, gs.MODE_FAST):
        ctx.set_mode(mode)
        for level in (0, 1, 2):
            ctx.set_tile_cull(level)
            out.extend(ctx.render(u) for u in cams)
    return out


def _assert_coherent(gs, ctx, vertices, cams):
    """ctx's resident scene renders what a fresh upload of `vertices` renders, bit for bit, and holds the same Sigma."""
    torch = _torch()
    torch.cuda.synchronize()
    fresh = gs.Context(0)
    try:
        fresh.set_backward(True)  # as on ctx: tile-cull level 2 falls back to 1
        fresh.upload(vertices.cpu().numpy())
        assert np.array_equal(ctx.download(gs.BUF_COV3D).view(np.uint32), fresh.download(gs.BUF_COV3D).view(np.uint32))
        for a, b in zip(_frames(gs, ctx, cams), _frames(gs, fresh, cams)):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    finally:
        fresh.close()


SIX = [scenes.camera(k) for k in scenes.CAMERAS]


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_resident_scene_equals_upload(gs, actx, selective):
    torch = _torch()
    _, vtx, u = scenes.c1()
    opt = gs.SceneAdam(actx, torch.from_numpy(vtx).cuda(), LR, selective=selective)
    g = torch.from_numpy(grad_image(u, np.zeros((u.height, u.width), bool))).cuda()
    opt.render(u)
    opt.step(g)
    _assert_coherent(gs, actx, opt.vertices, SIX)
    # after densify_and_prune and one more step
    dens = torch.zeros((opt.vertices.shape[0], 4), dtype=torch.float32, device="cuda")
    opt.render(u)
    opt.step(g, density=dens)
    thr = float(torch.quantile((dens[:, 0] / dens[:, 2].clamp(min=1))[dens[:, 2] > 0], 0.8))
    n0 = opt.vertices.shape[0]
    opt.densify(dens, grad_threshold=thr, scene_extent=10.0, generator=torch.Generator(device="cuda").manual_seed(0))
    assert opt.vertices.shape[0] != n0
    opt.render(u)
    opt.step(g)
    _assert_coherent(gs, actx, opt.vertices, SIX)


def test_full_size_selective_step_equals_upload(gs):
    torch = _torch()
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    u = bench.cameras(gs, wl)[0]
    ctx = gs.Context(0)
    try:
        ctx.set_tile_cull(1)
        opt = gs.SceneAdam(ctx, torch.from_numpy(bench.make_scene(gs, wl)).cuda(), LR, selective=True)
        opt.render(u)
        gi = torch.randn((u.height, u.width, 4), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
        before = opt.params.clone()
        opt.step(gi)
        torch.cuda.synchronize()
        updated = int((opt.params != before).any(1).sum())
        nv = ctx.stats().num_visible
        fresh = gs.Context(0)
        try:
            fresh.set_tile_cull(1)
            fresh.set_backward(True)
            fresh.upload(opt.vertices)
            assert np.array_equal(ctx.download(gs.BUF_COV3D).view(np.uint32), fresh.download(gs.BUF_COV3D).view(np.uint32))
            a = opt.render(u)
            b = torch.empty_like(a)
            fresh.render_into(u, b.data_ptr())
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        finally:
            fresh.close()
    finally:
        ctx.close()
    print(f"full size: {updated} rows updated, N_v of the frame {nv}")
    assert 0 < updated <= nv


def test_step_keeps_the_captured_graph(gs, actx):
    """With timers and debug off the frame after a step replays the middle-of-frame graph captured before it; that frame
    equals the same frame rendered without graphs, bit for bit."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    actx.set_timers(False)
    opt = gs.SceneAdam(actx, torch.from_numpy(vtx).cuda(), LR, selective=True)
    g = torch.from_numpy(grad_image(u, np.zeros((u.height, u.width), bool))).cuda()
    for _ in range(3):
        opt.render(u)
        opt.step(g)
    with_graph = opt.render(u).cpu().numpy()
    actx.set_graph(False)
    without = opt.render(u).cpu().numpy()
    assert np.array_equal(with_graph.view(np.uint32), without.view(np.uint32))


def test_outputs_are_bit_reproducible(gs):
    """The same step on two contexts, on torch's default stream and on a side stream, twice: identical outputs and Sigma."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    v0 = torch.from_numpy(vtx).cuda()
    p0, m0, s0 = _start(gs, vtx)
    c = gs.Context(0)
    try:
        c.upload(v0)
        gv, _ = _frame_grad(c, v0, u)  # one gradient, the same input to every step below
    finally:
        c.close()
    cfg = gs.adam_config(LR, step=2, selective=True)
    side = torch.cuda.Stream()
    results = []
    for _run in range(2):
        for use_side in (False, True):
            c = gs.Context(0)
            try:
                c.upload(v0)
                render(c, u)
                p, m, s, v = p0.clone(), m0.clone(), s0.clone(), v0.clone()
                torch.cuda.synchronize()
                if use_side:
                    with torch.cuda.stream(side):
                        c.adam_step(p, m, s, gv, v, cfg)
                else:
                    c.adam_step(p, m, s, gv, v, cfg)
                torch.cuda.synchronize()
                results.append([t.cpu().view(torch.int32) for t in (p, m, s, v)] +
                               [torch.from_numpy(c.download(gs.BUF_COV3D).view(np.int32))])
            finally:
                c.close()
    for r in results[1:]:
        for a, b in zip(results[0], r):
            assert torch.equal(a, b)


def test_error_cases(gs, actx):
    torch = _torch()
    _, vtx, u = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    p, m, s = _start(gs, vtx)
    gv = torch.zeros_like(v)
    out = torch.empty_like(v)
    good = gs.adam_config(LR)

    def raw(c, cfg=good, params=p, selective=None):
        if selective is not None:
            cfg = gs.adam_config(LR, selective=selective)
        ptr = None if params is None else params.data_ptr()
        return lambda: c._ck(gs.lib.gsb_adam_step(c.h, ptr, m.data_ptr(), s.data_ptr(), gv.data_ptr(), out.data_ptr(),
                                                  None if cfg is None else ctypes.byref(cfg), None))

    assert gs.lib.gsb_adam_step(None, p.data_ptr(), m.data_ptr(), s.data_ptr(), gv.data_ptr(), out.data_ptr(), ctypes.byref(good),
                                None) == gs.ERR_INVALID
    expect(gs, actx, gs.ERR_NO_SCENE, raw(actx), ENTRY)  # nothing uploaded
    actx.upload(vtx)
    raw(actx)()  # dense: needs no frame
    expect(gs, actx, gs.ERR_INVALID, raw(actx, params=None), ENTRY)
    expect(gs, actx, gs.ERR_INVALID, raw(actx, cfg=None), ENTRY)
    for field, value in (("beta1", 1.0), ("beta2", -0.1), ("beta1", float("nan")), ("eps", -1e-8), ("eps", float("nan")),
                         ("bias_correction1", 0.0), ("bias_correction1", 1.5), ("bias_correction2_sqrt", 0.0),
                         ("selective", 2)):
        cfg = gs.adam_config(LR)
        setattr(cfg, field, value)
        expect(gs, actx, gs.ERR_INVALID, raw(actx, cfg), ENTRY)
    for bad_lr in (-1e-3, float("nan")):
        cfg = gs.adam_config(LR)
        cfg.lr[3] = bad_lr
        expect(gs, actx, gs.ERR_INVALID, raw(actx, cfg), ENTRY)
    expect(gs, actx, gs.ERR_INVALID, raw(actx, selective=True), ENTRY)  # no frame since the upload
    actx.set_backward(False)
    actx.render(u)
    expect(gs, actx, gs.ERR_INVALID, raw(actx, selective=True), ENTRY)  # not recorded
    actx.set_backward(True)
    actx.render(u, rows=(0, 2))
    expect(gs, actx, gs.ERR_INVALID, raw(actx, selective=True), ENTRY)  # a band
    actx.render(u)
    raw(actx, selective=True)()  # a recorded whole frame: fine
    expect(gs, actx, gs.ERR_INVALID, raw(actx, selective=True), ENTRY)  # a second selective step on the same frame
    actx.render(u)
    raw(actx)()  # a dense step
    expect(gs, actx, gs.ERR_INVALID, raw(actx, selective=True), ENTRY)  # ... also ends the frame
    gi = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    expect(gs, actx, gs.ERR_INVALID, lambda: actx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr()),
           "gsb_render_backward")  # a backward after a step
    with pytest.raises(ValueError):
        actx.adam_step(p[:-1], m, s, gv, out, good)
    with pytest.raises(ValueError):
        actx.adam_step(p, m, s, gv.double(), out, good)
    with pytest.raises(ValueError):
        actx.adam_step(p, m, s, gv.t().contiguous().t(), out, good)
    # a pipelined frame that overflowed its arena (gsb_render_async never regrows; a fresh context holds N = 10 k instances)
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        fresh.set_backward(True)
        ui = scenes.camera("inside")
        dev = torch.empty((ui.height, ui.width, 4), dtype=torch.float32, device="cuda")
        fresh.render_into(ui, dev.data_ptr(), gs.FORMAT_RGBA32F, sync=False)
        torch.cuda.synchronize()
        expect(gs, fresh, gs.ERR_INVALID, raw(fresh, selective=True), ENTRY)
        with pytest.raises(gs.GsbError):
            fresh.stats()  # reports (and clears) the overflow
    finally:
        fresh.close()
    # fp16 SH storage
    actx.set_sh_storage(True)
    actx.upload(vtx)
    expect(gs, actx, gs.ERR_INVALID, raw(actx), ENTRY)
    # a sharded context (two ranks on one GPU)
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, raw(c0), ENTRY)
    finally:
        grp.close()


# training: c1's frames from three poses, from every 4th Gaussian with scales x 1.5 (tests/test_gpu_loss.py's sparse start)
POSES = [([0, 0, 5], [1, 0, 0, 0]), ([0.6, 0.1, 5.2], scenes.quat_axis_angle([0, 1, 0], 6)),
         ([-0.5, -0.3, 4.8], scenes.quat_axis_angle([1, 0, 0], -5))]
TRAIN_LR = [1e-3, 5e-3, 5e-2, 1e-3, 1e-2, 5e-4]


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


def _evaluate(gs, ctx, opt, views, targets):
    ms = [gs.image_metrics(ctx, opt.render(u), t) for u, t in zip(views, targets)]
    return (sum(0.8 * m["l1"] + 0.2 * (1 - m["ssim"]) for m in ms) / len(ms), sum(1 - m["ssim"] for m in ms) / len(ms))


@pytest.mark.parametrize("selective", [False, True], ids=["dense", "selective"])
def test_scene_adam_fit_lowers_loss_and_dssim(gs, actx, selective):
    torch = _torch()
    start, views, targets = _training_setup(gs, actx)
    opt = gs.SceneAdam(actx, start, TRAIN_LR, selective=selective)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    loss0, dssim0 = _evaluate(gs, actx, opt, views, targets)
    for it in range(300):
        k = it % 3
        actx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g)
    loss1, dssim1 = _evaluate(gs, actx, opt, views, targets)
    print(f"SceneAdam {'selective' if selective else 'dense'}: loss {loss0:.5f} -> {loss1:.5f}, 1 - SSIM {dssim0:.5f} -> {dssim1:.5f}")
    assert loss1 < loss0 and dssim1 < dssim0


# per-group relative L2 between dense SceneAdam and the torch path after 5 steps, about 5x what an H100 gives (DESIGN.md
# section 12: 7.8e-8, 7.9e-8, 6.1e-6, 1.6e-7, 2.3e-6, 7.6e-7); both paths are deterministic here
TRACK_TOL = {"position": 5e-7, "scale": 5e-7, "opacity": 3e-5, "rotation": 1e-6, "sh_dc": 1e-5, "sh_rest": 4e-6}


def test_dense_scene_adam_tracks_the_torch_path(gs, actx):
    torch = _torch()
    start, views, targets = _training_setup(gs, actx)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)  # no atomics in either backward pass: only the paths differ
    try:
        raw = gs.raw_parameters(start)
        leaves = {name: raw[:, cols].clone().contiguous().requires_grad_() for name, cols in GROUPS.items()}
        opt_t = torch.optim.Adam([{"params": [t], "lr": TRAIN_LR[k]} for k, t in enumerate(leaves.values())], eps=1e-15, fused=True)
        col3 = start[:, 3:4]

        def assemble():
            q = leaves["rotation"]
            return torch.cat([leaves["position"], col3, leaves["scale"].exp(), torch.sigmoid(leaves["opacity"]),
                              q / q.norm(dim=1, keepdim=True), leaves["sh_dc"], leaves["sh_rest"]], 1)

        for it in range(5):
            opt_t.zero_grad()
            k = it % 3
            gs.image_loss_torch(actx, gs.render_torch(actx, assemble(), views[k]), targets[k], 0.2).backward()
            opt_t.step()
        want = torch.cat([leaves[n].detach() if n != "position" else torch.cat([leaves[n].detach(), col3], 1)
                          for n in GROUPS], 1)
        opt = gs.SceneAdam(actx, start, TRAIN_LR, eps=1e-15, selective=False)
        g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
        for it in range(5):
            k = it % 3
            actx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
            opt.step(g)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    rows = torch.ones(start.shape[0], dtype=torch.bool)
    errs = _group_errors(opt.params.double().cpu(), want.double().cpu(), rows)
    print(f"dense SceneAdam vs torch path after 5 steps, relative L2 per group: {errs}")
    assert all(errs[k] <= TRACK_TOL[k] for k in GROUPS), errs


def test_training_with_densify(gs, actx):
    """From every 8th Gaussian with scales x 1.5: densifying every 100 steps up to 300 grows the scene while the loss drops."""
    torch = _torch()
    torch.manual_seed(0)
    start, views, targets = _training_setup(gs, actx, every=8)
    opt = gs.SceneAdam(actx, start, TRAIN_LR, selective=True)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    dens = torch.zeros((start.shape[0], 4), dtype=torch.float32, device="cuda")
    loss0, _ = _evaluate(gs, actx, opt, views, targets)
    for it in range(1, 601):
        k = it % 3
        actx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g, density=dens)
        if it % 100 == 0 and it <= 300:
            avg = dens[:, 0] / dens[:, 2].clamp(min=1)
            thr = float(torch.quantile(avg[dens[:, 2] > 0], 0.8))
            opt.densify(dens, grad_threshold=thr, scene_extent=10.0)
            dens = torch.zeros((opt.vertices.shape[0], 4), dtype=torch.float32, device="cuda")
    loss1, _ = _evaluate(gs, actx, opt, views, targets)
    print(f"SceneAdam with densify: n {start.shape[0]} -> {opt.vertices.shape[0]}, loss {loss0:.5f} -> {loss1:.5f}")
    assert opt.vertices.shape[0] > start.shape[0]
    assert loss1 < loss0
