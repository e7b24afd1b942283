"""gsb_render_features / gsb_render_backward_features / gsb_adam_step_features: the map against the fp32 restatement of the
oracle's blend bit for bit (tests/features_ref.py) and against the image and gsb_render_depth's D, the gradients against the
float64 reference, the deterministic mode, every error code, the Adam step against torch, and training a label field."""
import numpy as np
import pytest

import edge_scene
import features_ref
import scenes
from backward_util import CAMERA_GROUPS, GROUPS, expect, grad_image, rel

pytestmark = pytest.mark.gpu

ENTRY = "gsb_render_backward_features"
GEOMETRY = {k: GROUPS[k] for k in ("position", "scale", "opacity", "rotation")}


def _torch():
    import torch

    return torch


@pytest.fixture
def fctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _scene(name):
    if name == "edge":
        return edge_scene.vertices("backward")[0], edge_scene.camera("axis")
    if name == "scale":
        import scale_scene

        return scale_scene.vertices()[0], scale_scene.camera("axis")
    return scenes.c1()[1], scenes.camera(name)


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


def _features(n, c, seed=11):
    return np.random.default_rng(seed).uniform(-1, 1, (n, c)).astype(np.float32)


def _fmap(ctx, F):
    torch = _torch()
    out = ctx.render_features(torch.from_numpy(np.ascontiguousarray(F)).cuda())
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _backward(ctx, vtx, F, gfm, gi=None, density=False, camera=False, stream=None, vertices=True, features=True):
    """gsb_render_backward_features of the last frame: (grad_vertices, grad_features, density, 40 camera words), None for
    what was not asked."""
    torch = _torch()
    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    f = torch.from_numpy(np.ascontiguousarray(F, np.float32)).cuda()
    g = torch.from_numpy(np.ascontiguousarray(gfm, np.float32)).cuda()
    gim = None if gi is None else torch.from_numpy(np.ascontiguousarray(gi, np.float32)).cuda()
    gv = torch.full_like(v, float("nan")) if vertices else None
    gf = torch.full_like(f, float("nan")) if features else None
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if density else None
    gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda") if camera else None
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    ctx.render_backward_features(v.data_ptr(), f, g, grad_vertices_ptr=ptr(gv), grad_features_ptr=ptr(gf), grad_image_ptr=ptr(gim),
                                 grad_uniforms_ptr=ptr(gu), density_ptr=ptr(dens), stream=stream)
    torch.cuda.synchronize()
    host = lambda t: None if t is None else t.cpu().numpy()  # noqa: E731
    return host(gv), host(gf), host(dens), host(gu)


# ---------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("channels", [1, 3, 32, 33, 128])
def test_map_bit_exact(gs, oracle, fctx, channels):
    """EXACT, levels 0 and 1: the map equals the fp32 restatement bit for bit, on c1 and odd_size."""
    for cam in ("c1", "odd_size"):
        vtx, u = _scene(cam)
        F = _features(vtx.shape[0], channels)
        oracle.set_exp_mode(1)
        try:
            frame = oracle.render_frame(vtx, oracle.cov3d(vtx), u)
        finally:
            oracle.set_exp_mode(0)
        ref = features_ref.blend32(frame, u.width, u.height, F)
        fctx.upload(vtx)
        fctx.set_backward(True)
        for level in (0, 1):
            fctx.set_tile_cull(level)
            fctx.render(u)
            assert _same(_fmap(fctx, F), ref), (cam, channels, level)


@pytest.mark.parametrize("case", ["plain", "aa", "fisheye"])
def test_colour_and_depth_features_give_image_and_depth(gs, fctx, case):
    """Features set to the frame's own colours (GSB_BUF_ATTR) give the image's RGB, set to its depth keys gsb_render_depth's
    D, bit for bit, in EXACT and FAST."""
    vtx, u = _scene("c1")
    fctx.upload(vtx)
    if case == "aa":
        fctx.set_antialiased(True)
    if case == "fisheye":
        from test_gpu_fisheye import _lens

        fctx.set_camera_model(_lens(gs, u, fov_deg=200.0, k=(0.05, -0.01, 0.0, 0.0)))
    fctx.set_backward(True)
    fctx.set_debug(True)
    for mode in (gs.MODE_EXACT, gs.MODE_FAST):
        fctx.set_mode(mode)
        img, da = fctx.render_depth(u)
        attr = fctx.download(gs.BUF_ATTR)
        col = np.nan_to_num(attr["color_radii"][:, :3].astype(np.float32))
        dep = np.nan_to_num(attr["depth"].astype(np.float32))[:, None]
        assert _same(_fmap(fctx, col), img[..., :3]), (case, mode)
        assert _same(_fmap(fctx, dep)[..., 0], da[..., 0]), (case, mode)


def test_culled_rows_and_recorded_state(gs, fctx):
    """NaN rows of Gaussians in no list leave the map finite; a feature call leaves the deterministic backward's words alone."""
    vtx, u = _scene("c1")
    fctx.upload(vtx)
    fctx.set_backward(True)
    fctx.set_debug(True)
    fctx.render(u)
    listed = np.zeros(vtx.shape[0], bool)
    listed[np.unique(fctx.download(gs.BUF_VALS_SORTED)[: fctx.stats().num_instances])] = True
    F = _features(vtx.shape[0], 16)
    F[~listed] = np.nan
    assert (~listed).any() and np.isfinite(_fmap(fctx, F)).all()
    fctx.set_backward_deterministic(True)
    F = np.nan_to_num(F)
    gfm = np.random.default_rng(2).standard_normal((u.height, u.width, 16)).astype(np.float32)
    before = _backward(fctx, vtx, F, gfm, gi=grad_image(u), density=True)
    _fmap(fctx, F)
    after = _backward(fctx, vtx, F, gfm, gi=grad_image(u), density=True)
    for a, b in zip(before[:3], after[:3]):
        assert _same(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside", "edge", "scale"])
def test_gradient_matches_float64_reference(gs, oracle, fctx, cam):
    vtx, u = _scene(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    C = 20
    F = _features(vtx.shape[0], C)
    gi = grad_image(u, steps)
    gfm = np.random.default_rng(5).standard_normal((u.height, u.width, C)).astype(np.float32)
    gfm[steps] = 0.0
    ref = features_ref.reference(vtx, u, frame, F, gi, gfm, camera=True)
    keep = ~ref["exclude"]
    ref40 = np.zeros(40)
    ref40[:36], ref40[38:] = ref["grad_ubo"][:36], ref["grad_ubo"][36:]
    tol = 2e-3 if cam in ("edge", "scale") else 1e-3
    fctx.upload(vtx)
    fctx.set_backward(True)
    for det in (False, True):
        fctx.set_backward_deterministic(det)
        fctx.render(u)
        gv, gf, _, gu = _backward(fctx, vtx, F, gfm, gi, camera=True)
        assert np.isfinite(gv).all() and np.isfinite(gf).all() and not gv[:, 3].any()
        for name, cols in GROUPS.items():
            assert rel(gv[keep, cols], ref["grad"][keep, cols]) <= tol, (cam, det, name)
        assert rel(gf[keep], ref["grad_features"][keep]) <= tol, (cam, det)
        for name, words in CAMERA_GROUPS.items():
            assert rel(gu[words], ref40[words]) <= tol, (cam, det, name)


def _plain_density_backward(ctx, vtx, gi):
    torch = _torch()
    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    g = torch.from_numpy(gi).cuda()
    gv = torch.full_like(v, float("nan"))
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
    ctx._backward(v.data_ptr(), g.data_ptr(), gv.data_ptr(), None, density_ptr=dens.data_ptr())
    torch.cuda.synchronize()
    return gv.cpu().numpy(), dens.cpu().numpy()


def _equal_up_to_zero_sign(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(np.where(a == 0, np.float32(0), a).view(np.uint32), np.where(b == 0, np.float32(0), b).view(np.uint32))


def test_zero_feature_gradient_and_colour_features(gs, fctx):
    """A zero feature gradient gives gsb_render_backward_density's words (det) and density column 0 / 2-3 as there; features
    set to the colours with g_feat = g_image and no image gradient give the colour-only geometry gradient."""
    vtx, u = _scene("c1")
    vtx = vtx.copy()
    vtx[:, 15:60] = 0.0  # degree-0 colours: no view-direction term, which the feature path does not have
    gi = grad_image(u)
    fctx.upload(vtx)
    fctx.set_backward(True)
    fctx.set_debug(True)
    for det in (True, False):
        fctx.set_backward_deterministic(det)
        fctx.render(u)
        gv0, d0 = _plain_density_backward(fctx, vtx, gi)
        F = _features(vtx.shape[0], 5)
        gv1, gf1, d1, _ = _backward(fctx, vtx, F, np.zeros((u.height, u.width, 5), np.float32), gi, density=True)
        if det:
            assert _equal_up_to_zero_sign(gv0, gv1) and _equal_up_to_zero_sign(d0, d1)
        else:
            assert rel(gv1, gv0) <= 1e-6 and rel(d1, d0) <= 1e-6
        assert not gf1.any()
        attr = fctx.download(gs.BUF_ATTR)
        col = np.nan_to_num(attr["color_radii"][:, :3].astype(np.float32))
        gfm = np.ascontiguousarray(gi[..., :3])
        gv2, _, d2, _ = _backward(fctx, vtx, col, gfm, None, density=True, features=False)
        for name, cols in GEOMETRY.items():
            assert rel(gv2[:, cols], gv0[:, cols]) <= 1e-6, (det, name)
        assert rel(d2[:, 0], d0[:, 0]) <= 1e-6 and _same(d2[:, 2:], d0[:, 2:])
        assert (d2[:, 1] >= d0[:, 1] * (1 - 1e-6)).all()


def test_deterministic_matrix(gs, fctx):
    """Five calls, a side stream, a larger arena, a fresh context and levels 0 / 1 give the same words; within 1e-6 of atomic."""
    torch = _torch()
    vtx, u = _scene("c1")
    F = _features(vtx.shape[0], 37)
    gfm = np.random.default_rng(9).standard_normal((u.height, u.width, 37)).astype(np.float32)
    gi = grad_image(u)
    fctx.upload(vtx)
    fctx.set_backward(True)
    fctx.set_backward_deterministic(True)
    runs = []
    for level in (0, 1):
        fctx.set_tile_cull(level)
        fctx.render(u)
        for _ in range(5 if level == 0 else 1):
            runs.append(_backward(fctx, vtx, F, gfm, gi, density=True, camera=True))
    runs.append(_backward(fctx, vtx, F, gfm, gi, density=True, camera=True, stream=torch.cuda.Stream()))
    fctx.reserve(4 * fctx.stats().num_instances)
    fctx.render(u)
    runs.append(_backward(fctx, vtx, F, gfm, gi, density=True, camera=True))
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        fresh.set_backward(True)
        fresh.set_backward_deterministic(True)
        fresh.render(u)
        runs.append(_backward(fresh, vtx, F, gfm, gi, density=True, camera=True))
    finally:
        fresh.close()
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert _same(a, b)
    fctx.set_backward_deterministic(False)
    fctx.render(u)
    atomic = _backward(fctx, vtx, F, gfm, gi, density=True, camera=True)
    for a, b in zip(atomic, runs[0]):
        assert rel(a.astype(np.float64), b.astype(np.float64)) <= 1e-6


def test_error_codes(gs, fctx):
    torch = _torch()
    vtx, u = _scene("odd_size")
    n, C = vtx.shape[0], 4
    v = torch.from_numpy(vtx).cuda()
    f = torch.zeros((n, C), dtype=torch.float32, device="cuda")
    gv, gf = torch.empty_like(v), torch.empty_like(f)
    fm = torch.empty((u.height, u.width + 1, C), dtype=torch.float32, device="cuda")
    lib, INV = gs.lib, gs.ERR_INVALID

    def rf(fp=f.data_ptr(), c=C, mp=fm.data_ptr(), pitch=0):
        fctx._ck(lib.gsb_render_features(fctx.h, fp, c, mp, pitch, None))

    def bw(vp=v.data_ptr(), fp=f.data_ptr(), c=C, gfmp=fm.data_ptr(), pitch=0, gvp=gv.data_ptr(), gup=None, gfp=gf.data_ptr(),
           gdp=None, dens=None):
        fctx._ck(lib.gsb_render_backward_features(fctx.h, vp, None, 0, gdp, 0, fp, c, gfmp, pitch, gvp, gup, gfp, dens, None))

    assert lib.gsb_render_features(None, f.data_ptr(), C, fm.data_ptr(), 0, None) == INV
    expect(gs, fctx, gs.ERR_NO_SCENE, lambda: rf())
    fctx.upload(vtx)
    expect(gs, fctx, gs.ERR_NO_SCENE, lambda: rf(), "gsb_render_features")  # no frame yet
    fctx.render(u)
    expect(gs, fctx, INV, lambda: rf(), "gsb_render_features")  # not recorded
    expect(gs, fctx, INV, lambda: bw(), ENTRY)
    fctx.set_backward(True)
    fctx.render(u)
    for bad in (dict(fp=None), dict(mp=None), dict(c=0), dict(c=129), dict(pitch=u.width * C * 4 - 4),
                dict(pitch=u.width * C * 4 + 2), dict(mp=fm.data_ptr() + 2, pitch=(u.width + 1) * C * 4)):
        expect(gs, fctx, INV, lambda: rf(**bad), "gsb_render_features")
    rf(pitch=(u.width + 1) * C * 4)  # a padded pitch is fine
    for bad in (dict(vp=None), dict(fp=None), dict(gfmp=None), dict(gvp=None, gfp=None), dict(c=0), dict(c=129),
                dict(pitch=u.width * C * 4 - 4), dict(gfp=gf.data_ptr() + 2), dict(gdp=fm.data_ptr()),
                dict(gvp=None, dens=gv.data_ptr())):
        expect(gs, fctx, INV, lambda: bw(**bad), ENTRY)
    bw(gvp=None)  # features only
    bw(gfp=None)  # geometry only
    fctx.upload(vtx)
    expect(gs, fctx, INV, lambda: rf(), "gsb_render_features")  # the scene changed after the frame
    cfg = gs.AdamConfig()
    cfg.beta1, cfg.beta2, cfg.eps, cfg.bias_correction1, cfg.bias_correction2_sqrt, cfg.selective = 0.9, 0.999, 1e-15, 1.0, 1.0, 1
    st = lambda lr=0.1, c=C: fctx._ck(lib.gsb_adam_step_features(fctx.h, f.data_ptr(), f.data_ptr(), f.data_ptr(),  # noqa: E731
                                                                 gf.data_ptr(), c, lr, gs.C.byref(cfg), None))
    expect(gs, fctx, INV, lambda: st(), "gsb_adam_step_features")  # selective without a valid frame
    cfg.selective = 0
    expect(gs, fctx, INV, lambda: st(lr=-1.0), "gsb_adam_step_features")
    expect(gs, fctx, INV, lambda: st(c=0), "gsb_adam_step_features")
    assert lib.gsb_adam_step_features(None, f.data_ptr(), f.data_ptr(), f.data_ptr(), gf.data_ptr(), C, 0.1, gs.C.byref(cfg), None) == INV
    assert lib.gsb_render_backward_features(None, v.data_ptr(), None, 0, None, 0, f.data_ptr(), C, fm.data_ptr(), 0, gv.data_ptr(),
                                            None, gf.data_ptr(), None, None) == INV


def test_error_codes_of_the_frame(gs, fctx):
    """A band frame, an overflowed frame, fp16 SH (backward only), a fisheye frame with grad_uniforms and sharded contexts."""
    torch = _torch()
    vtx, u = _scene("c1")
    n, C = vtx.shape[0], 3
    v = torch.from_numpy(vtx).cuda()
    f = torch.zeros((n, C), dtype=torch.float32, device="cuda")
    gv, gf = torch.empty_like(v), torch.empty_like(f)
    lib, INV = gs.lib, gs.ERR_INVALID

    def rf(ctx, hw=(u.height, u.width)):
        fm = torch.empty((hw[0], hw[1], C), dtype=torch.float32, device="cuda")
        return lambda: ctx._ck(lib.gsb_render_features(ctx.h, f.data_ptr(), C, fm.data_ptr(), 0, None))

    def bw(ctx, hw=(u.height, u.width), gup=None):
        fm = torch.zeros((hw[0], hw[1], C), dtype=torch.float32, device="cuda")
        return lambda: ctx._ck(lib.gsb_render_backward_features(ctx.h, v.data_ptr(), None, 0, None, 0, f.data_ptr(), C, fm.data_ptr(), 0,
                                                                gv.data_ptr(), gup, gf.data_ptr(), None, None))

    fctx.upload(vtx)
    fctx.set_backward(True)
    fctx.render(u, rows=(0, 1))  # a band
    expect(gs, fctx, INV, rf(fctx), "gsb_render_features")
    expect(gs, fctx, INV, bw(fctx), ENTRY)
    # a pipelined frame that overflowed its arena (gsb_render_async never regrows; a fresh context holds N = 10 k instances)
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        fresh.set_backward(True)
        ui = scenes.camera("inside")
        dev = torch.empty((ui.height, ui.width, 4), dtype=torch.float32, device="cuda")
        fresh.render_into(ui, dev.data_ptr(), gs.FORMAT_RGBA32F, sync=False)
        torch.cuda.synchronize()
        expect(gs, fresh, INV, rf(fresh, (ui.height, ui.width)), "gsb_render_features")
        expect(gs, fresh, INV, bw(fresh, (ui.height, ui.width)), ENTRY)
        with pytest.raises(gs.GsbError):
            fresh.stats()  # reports (and clears) the overflow
    finally:
        fresh.close()
    # a fisheye frame has no camera gradient
    from test_gpu_fisheye import _lens

    fctx.set_camera_model(_lens(gs, u, fov_deg=120.0))
    fctx.render(u)
    gu = torch.empty(40, dtype=torch.float32, device="cuda")
    expect(gs, fctx, INV, bw(fctx, gup=gu.data_ptr()), ENTRY)
    bw(fctx)()
    fctx.set_camera_model(None)
    # fp16 SH storage: the map is defined, the backward is not
    fctx.set_sh_storage(True)
    fctx.upload(vtx)
    fctx.render(u)
    rf(fctx)()
    expect(gs, fctx, INV, bw(fctx), ENTRY)
    # a sharded context (two ranks on one GPU)
    grp = gs.Group([0, 0])
    try:
        grp.upload(vtx)
        c0 = grp.context(0)
        expect(gs, c0, INV, rf(c0), "gsb_render_features")
        expect(gs, c0, INV, bw(c0), ENTRY)
        cfg = gs.AdamConfig()
        cfg.beta1, cfg.beta2, cfg.bias_correction1, cfg.bias_correction2_sqrt = 0.9, 0.999, 1.0, 1.0
        expect(gs, c0, INV, lambda: c0._ck(lib.gsb_adam_step_features(c0.h, f.data_ptr(), f.data_ptr(), f.data_ptr(), gf.data_ptr(), C,
                                                                      0.1, gs.C.byref(cfg), None)), "gsb_adam_step_features")
    finally:
        grp.close()


# ---------------------------------------------------------------------------------------------------------------------
# Adam and training
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("selective", [False, True])
def test_adam_matches_torch(gs, fctx, selective):
    torch = _torch()
    vtx, u = _scene("c1")
    n, C = vtx.shape[0], 6
    fctx.upload(vtx)
    fctx.set_backward(True)
    fctx.set_debug(True)
    fctx.render(u)
    survivors = np.zeros(n, bool)
    survivors[np.unique(fctx.download(gs.BUF_VALS_SORTED)[: fctx.stats().num_instances])] = True
    rows = torch.from_numpy(survivors).cuda() if selective else torch.ones(n, dtype=torch.bool, device="cuda")
    x0 = torch.from_numpy(_features(n, C)).cuda()
    x, m, v = x0.clone(), torch.zeros_like(x0), torch.zeros_like(x0)
    ref = x0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=0.01, betas=(0.9, 0.999), eps=1e-15)
    gen = torch.Generator(device="cuda").manual_seed(1)
    cfg = gs.AdamConfig()
    cfg.beta1, cfg.beta2, cfg.eps, cfg.selective = 0.9, 0.999, 1e-15, int(selective)
    for step in range(1, 21):
        g = torch.randn(x0.shape, generator=gen, device="cuda")
        cfg.bias_correction1, cfg.bias_correction2_sqrt = 1 - 0.9 ** step, (1 - 0.999 ** step) ** 0.5
        fctx.adam_step_features(x, m, v, g, 0.01, cfg)
        ref.grad = torch.where(rows[:, None], g, torch.zeros_like(g))
        opt.step()
    torch.cuda.synchronize()
    assert rel(x[rows], ref.detach()[rows]) <= 1e-6
    if selective:
        assert _same(x[~rows].cpu().numpy(), x0[~rows].cpu().numpy())
        assert not m[~rows].any() and (m[rows] != 0).any()


def test_label_field_training(gs, fctx):
    """Geometry frozen, 16-channel features from zero, MSE of feature maps of 8 views against the maps of a one-hot labelling
    of the Gaussians by spatial region: the held-out view's argmax accuracy over pixels with A > 0.5 rises from chance."""
    torch = _torch()
    vtx, _ = _scene("c1")
    n, C = vtx.shape[0], 16
    pos = vtx[:, :3]
    lab = (np.digitize(pos[:, 0], np.quantile(pos[:, 0], [0.25, 0.5, 0.75])) * 4 +
           np.digitize(pos[:, 1], np.quantile(pos[:, 1], [0.25, 0.5, 0.75])))
    onehot = torch.from_numpy(np.eye(C, dtype=np.float32)[lab]).cuda()
    views = []  # 9 views of the cloud from within +-20 degrees about the y axis, at 160 x 120; the last is held out
    for k in range(9):
        deg = -20.0 + 40.0 * ((k * 4) % 9) / 8.0
        a = np.radians(deg)
        views.append(gs.uniforms_from_camera([5 * np.sin(a), 0, 5 * np.cos(a)], scenes.quat_axis_angle([0, 1, 0], deg), 45.0,
                                             0.1, 1000.0, 160, 120))
    v = torch.from_numpy(vtx).cuda()
    feat = torch.zeros((n, C), dtype=torch.float32, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([feat], lr=0.05)

    def accuracy(u):
        with torch.no_grad():
            img, da, fmap = gs.render_torch(fctx, v, u, depth=True, features=feat)
            _, _, target = gs.render_torch(fctx, v, u, depth=True, features=onehot)
            mask = da[..., 1] > 0.5
            return float((fmap.argmax(-1) == target.argmax(-1))[mask].float().mean())

    held = views[-1]
    before = accuracy(held)
    for it in range(STEPS):
        u = views[it % 8]
        with torch.no_grad():
            _, target = gs.render_torch(fctx, v, u, features=onehot)
        _, fmap = gs.render_torch(fctx, v, u, features=feat)
        loss = ((fmap - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    after = accuracy(held)
    print(f"label field: held-out accuracy {before:.3f} -> {after:.3f} after {STEPS} steps")
    assert after >= ACCURACY > before


STEPS, ACCURACY = 200, 0.95  # one H100 run: 0.000 -> 0.997 (zero features pick label 0 everywhere)


def test_render_torch_composes(gs, fctx):
    """features= with depth=True, ubo= and density=: every output and input gradient is finite and the density rows grow."""
    torch = _torch()
    vtx, u = _scene("c1")
    v = torch.from_numpy(vtx).cuda().requires_grad_(True)
    f = torch.from_numpy(_features(vtx.shape[0], 7)).cuda().requires_grad_(True)
    ubo = torch.tensor(gs.pack_uniforms(u), dtype=torch.float32, device="cuda", requires_grad=True)
    dens = torch.zeros((vtx.shape[0], 4), dtype=torch.float32, device="cuda")
    img, da, fmap = gs.render_torch(fctx, v, u, ubo=ubo, density=dens, depth=True, features=f)
    assert fmap.shape == (u.height, u.width, 7)
    (img[..., :3].sum() + da.sum() + (fmap ** 2).sum()).backward()
    assert torch.isfinite(v.grad).all() and torch.isfinite(f.grad).all() and (f.grad != 0).any()
    assert torch.isfinite(ubo.grad).all() and (ubo.grad != 0).any()
    assert dens[:, 2].max() == 1


def test_scene_adam_keeps_feature_rows_aligned(gs, fctx):
    """SceneAdam(features=): render(features=True) and step(grad_feature_map=) train the features; densify() gathers their
    rows by `source` (split children with zero moments) and relocate() copies / appends them with zero moments."""
    torch = _torch()
    vtx, _ = _scene("c1")
    u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 160, 120)
    n, C = vtx.shape[0], 4
    ident = torch.arange(n, dtype=torch.float32, device="cuda")[:, None].repeat(1, C)  # row i holds i: its origin
    opt = gs.SceneAdam(fctx, torch.from_numpy(vtx).cuda(), [1e-4, 1e-3, 1e-2, 1e-3, 1e-3, 1e-4], features=ident, feature_lr=0.0)
    img, fmap = opt.render(u, features=True)
    assert fmap.shape == (u.height, u.width, C)
    gfm = torch.randn(fmap.shape, device="cuda")
    dens = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
    opt.step(torch.zeros_like(img), density=dens, grad_feature_map=gfm)
    assert torch.equal(opt.features, ident)  # lr 0: unchanged, moments filled
    assert (opt.feature_exp_avg != 0).any() and (opt.grad_features != 0).any()
    m_before, v_before = opt.feature_exp_avg.clone(), opt.vertices.clone()
    source = opt.densify(dens, grad_threshold=0.0, scene_extent=5.0)
    assert opt.features.shape == (opt.vertices.shape[0], C) and opt.feature_exp_avg.shape == opt.features.shape
    assert torch.equal(opt.features, ident[source])
    child = (opt.vertices[:, 4:7] != v_before[source, 4:7]).any(1)
    assert torch.equal(opt.feature_exp_avg[~child], m_before[source][~child]) and not opt.feature_exp_avg[child].any()
    # relocation: dead rows take their sources' features with zero moments; growth appends features[src]
    opt2 = gs.SceneAdam(fctx, torch.from_numpy(vtx).cuda(), [1e-4, 1e-3, 1e-2, 1e-3, 1e-3, 1e-4], features=ident, feature_lr=0.0)
    opt2.vertices[: n // 10, 7] = 0.001  # dead
    opt2.feature_exp_avg.fill_(1.0)
    gen = torch.Generator().manual_seed(0)
    n_rel, k = opt2.relocate(int(n * 1.05), generator=gen)
    assert n_rel == n // 10 and k > 0 and opt2.features.shape == (n + k, C)
    f = opt2.features[:, 0]
    assert torch.equal(opt2.features, f[:, None].repeat(1, C))  # whole rows were copied
    dead = torch.arange(n, device="cuda") < n // 10
    assert (f[:n][dead] >= n // 10).all() and torch.equal(f[:n][~dead], ident[:, 0][~dead])
    assert not opt2.feature_exp_avg[:n][dead].any() and (opt2.feature_exp_avg[:n][~dead] == 1).all()
    assert not opt2.feature_exp_avg[n:].any()
    # the appended rows are copies of their sources: each holds a live row's feature
    assert (f[n:] >= n // 10).all()
