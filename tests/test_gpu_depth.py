"""gsb_render_depth / gsb_render_backward_depth: (D, A) against the fp32 restatement of the oracle's blend bit for bit
(tests/depth_ref.py), the gradients against the float64 reference for colour, depth and alpha upstream gradients, the
deterministic mode, every error code, and training with depth and mask losses through render_torch and SceneAdam."""
import math

import numpy as np
import pytest

import aa_ref
import depth_ref
import edge_scene
import scenes
from backward_util import CAMERA_GROUPS, DEAD, GROUPS, expect, grad_image, rel

pytestmark = pytest.mark.gpu

ENTRY = "gsb_render_backward_depth"


def _torch():
    import torch

    return torch


@pytest.fixture
def dctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _scene(name):
    if name == "edge":
        return edge_scene.vertices()[0], edge_scene.camera("axis")
    return scenes.c1()[1], scenes.camera(name)


def _oracle32(oracle, vtx, u, antialiased=False, rows=None):
    """The oracle's frame at exp mode 1 and its (D, A) from depth_ref.blend32."""
    oracle.set_exp_mode(1)
    try:
        f = aa_ref.oracle_frame(vtx, oracle.cov3d(vtx), u, rows) if antialiased else oracle.render_frame(vtx, oracle.cov3d(vtx), u, rows)
    finally:
        oracle.set_exp_mode(0)
    return f, depth_ref.depth_alpha32(f, u, rows)


def _steps(oracle, vtx, u):
    oracle.set_exp_mode(1)
    try:
        return oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)[1]
    finally:
        oracle.set_exp_mode(0)


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", ["c1", "odd_size", "edge"])
def test_depth_alpha_bit_exact(gs, oracle, dctx, cam):
    """Levels 0/1/2 x direct launches and graph replay x RGBA32F / BGRA8, recorded frames too: (D, A) equal the fp32
    restatement bit for bit and the image equals gsb_render's; FAST within 1e-4 off the step pixels."""
    vtx, u = _scene(cam)
    f, ref = _oracle32(oracle, vtx, u)
    dctx.upload(vtx)
    for level in (0, 1, 2):
        dctx.set_tile_cull(level)
        for timers in (True, False, False):
            dctx.set_timers(timers)
            img, da = dctx.render_depth(u)
            assert _same(da, ref), (cam, level, timers)
            assert _same(img, f["rgba"]) and _same(img, dctx.render(u)), (cam, level, timers)
        dctx.set_timers(True)
        img8, da = dctx.render_depth(u, gs.FORMAT_BGRA8)
        assert _same(da, ref) and np.array_equal(img8, oracle.pack_unorm8(f["rgba"], bgra=True)), (cam, level)
        dctx.set_backward(True)
        img, da = dctx.render_depth(u)
        assert _same(da, ref) and _same(img, f["rgba"]), (cam, level, "recorded")
        dctx.set_backward(False)
        if cam != "edge":  # the edge scene's needles exceed FAST's bound on the colour too
            steps = _steps(oracle, vtx, u)
            dctx.set_mode(gs.MODE_FAST)
            _, da = dctx.render_depth(u)
            dctx.set_mode(gs.MODE_EXACT)
            err = np.abs(da.astype(np.float64) - ref) / np.maximum(1.0, np.abs(ref))
            assert err[~steps].max() <= 1e-4, (cam, level, err[~steps].max())
    assert (ref[..., 1] <= 1.0).all() and (ref[..., 0] >= 0).all()


def test_bands(gs, oracle, dctx):
    vtx, u = _scene("odd_size")
    dctx.upload(vtx)
    tiles_y = (u.height + 15) // 16
    for rows in ((0, 1), (tiles_y // 2, tiles_y // 2 + 2), (tiles_y - 1, tiles_y)):
        f, ref = _oracle32(oracle, vtx, u, rows=rows)
        img, da = dctx.render_depth(u, rows=rows)
        sl = slice(rows[0] * 16, min(u.height, rows[1] * 16))
        assert _same(da, ref) and _same(img, f["rgba"][sl]), rows


def test_antialiased_background_and_alpha_is_one_minus_t(gs, oracle, dctx):
    """The AA frame's (D, A) equal the restatement of aa_ref's oracle frame; a background changes the image only; A is 1 - the T
    gsb_background_gradient sums."""
    torch = _torch()
    vtx, u = _scene("c1")
    dctx.upload(vtx)
    dctx.set_antialiased(True)
    _, ref = _oracle32(oracle, vtx, u, antialiased=True)
    for level in (0, 1, 2):
        dctx.set_tile_cull(level)
        assert _same(dctx.render_depth(u)[1], ref), level
    dctx.set_antialiased(False)
    dctx.set_tile_cull(0)
    _, plain = dctx.render_depth(u)
    dctx.set_background((0.25, 0.5, 0.75))
    dctx.set_backward(True)
    img, da = dctx.render_depth(u)
    assert _same(da, plain) and _same(img, dctx.render(u))
    dctx.render_depth(u)
    g = grad_image(u)
    gb = dctx.background_gradient(torch.from_numpy(g).cuda()).cpu().numpy().astype(np.float64)
    want = ((1.0 - da[..., 1].astype(np.float64))[..., None] * g[..., :3]).sum((0, 1))
    assert np.abs(gb - want).max() <= 1e-5 * np.abs(g[..., :3]).sum(), (gb, want)


def test_empty_pixels_and_scene(gs, dctx):
    u = scenes.camera("odd_size")
    dctx.upload(np.zeros((0, 60), np.float32))
    _, da = dctx.render_depth(u)
    assert not da.any()


def test_host_pinned_and_device_outputs_agree(gs, dctx):
    torch = _torch()
    vtx, u = _scene("c1")
    dctx.upload(vtx)
    _, host = dctx.render_depth(u)
    img = torch.empty((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    pitch = u.width * 8 + 64  # a padded pitch
    buf = torch.full((u.height, pitch // 4), float("nan"), dtype=torch.float32, device="cuda")
    dctx._ck(gs.lib.gsb_render_depth(dctx.h, gs.C.byref(u), 0, gs.ALL_ROWS, img.data_ptr(), 0, gs.MEM_DEVICE, gs.FORMAT_RGBA32F,
                                     buf.data_ptr(), pitch, None))
    torch.cuda.synchronize()
    dev = buf[:, : u.width * 2].reshape(u.height, u.width, 2).cpu().numpy()
    assert _same(dev, host)
    pinned = torch.empty((u.height, u.width, 2), dtype=torch.float32).pin_memory()
    imgh = np.empty((u.height, u.width, 4), np.float32)
    dctx._ck(gs.lib.gsb_render_depth(dctx.h, gs.C.byref(u), 0, gs.ALL_ROWS, imgh.ctypes.data, 0, gs.MEM_HOST, gs.FORMAT_RGBA32F,
                                     pinned.data_ptr(), 0, None))
    assert _same(pinned.numpy(), host)


FISHEYE = {"fov90": ("c1", 90.0, (0.0, 0.0, 0.0, 0.0)), "fov200": ("inside", 200.0, (0.0, 0.0, 0.0, 0.0)),
           "k_nonzero": ("inside", 150.0, (-0.05, 0.004, -0.0002, 0.0))}


def _fisheye_case(gs, name):
    from test_gpu_fisheye import _lens

    pose, fov, k = FISHEYE[name]
    u = scenes.camera(pose)
    return scenes.c1()[1], u, _lens(gs, u, fov_deg=fov, k=k)


def _fisheye_lists(gs, ctx, u, vtx, cam):
    from test_gpu_fisheye import _frame_lists

    return _frame_lists(gs, ctx, u, vtx, cam)[1]


@pytest.mark.parametrize("name", sorted(FISHEYE))
def test_fisheye_depth_is_the_distance(gs, dctx, name):
    vtx, u, cam = _fisheye_case(gs, name)
    dctx.upload(vtx)
    dctx.set_camera_model(cam)
    frame = _fisheye_lists(gs, dctx, u, vtx, cam)
    _, da = dctx.render_depth(u)
    ref = depth_ref.reference(vtx, u, frame, pre=depth_ref.fisheye(cam))["values"]
    err = np.abs(da.astype(np.float64) - ref[..., 3:]) / np.maximum(1.0, np.abs(ref[..., 3:]))
    bad = err.max(-1) > 1e-4
    assert bad.mean() <= 5e-3 and err.max() < 0.5, (name, bad.mean(), err.max())
    assert da[..., 0].max() > 0


# ---------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------
def _upstream(u, kind, steps=None):
    """(grad_image or None, grad_da) of an upstream `kind`: colour, depth, alpha or mixed; zero on the step pixels."""
    gi = grad_image(u, steps, seed=7)
    gda = np.random.default_rng(11).standard_normal((u.height, u.width, 2)).astype(np.float32)
    if steps is not None:
        gda[steps] = 0.0
    if kind == "colour":
        gda[:] = 0.0
    elif kind == "depth":
        gi, gda[..., 1] = None, 0.0
    elif kind == "alpha":
        gi, gda[..., 0] = None, 0.0
    return gi, gda


def _depth_backward(ctx, vtx, gi, gda, density=False, camera=False, stream=None):
    """gsb_render_backward_depth of the last frame: (grad_vertices, density or None, 40 camera words or None) on the host."""
    torch = _torch()
    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    g = None if gi is None else torch.from_numpy(np.ascontiguousarray(gi)).cuda()
    gd = torch.from_numpy(np.ascontiguousarray(gda)).cuda()
    gv = torch.full_like(v, float("nan"))
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if density else None
    gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda") if camera else None
    ctx._backward(v.data_ptr(), None if g is None else g.data_ptr(), gv.data_ptr(), stream,
                  grad_uniforms_ptr=None if gu is None else gu.data_ptr(), density_ptr=None if dens is None else dens.data_ptr(),
                  grad_depth_alpha_ptr=gd.data_ptr())
    torch.cuda.synchronize()
    return (gv.cpu().numpy().astype(np.float64), None if dens is None else dens.cpu().numpy(),
            None if gu is None else gu.cpu().numpy().astype(np.float64))


def _check_groups(got, ref, keep, what, tol=1e-3):
    assert np.isfinite(got).all(), what
    for name, cols in GROUPS.items():
        r = rel(got[keep, cols], ref["grad"][keep, cols])
        assert r <= tol, (what, name, r)
    assert not got[:, 3].any()


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
@pytest.mark.parametrize("kind", ["colour", "depth", "alpha", "mixed"])
def test_gradient_matches_float64_reference(gs, oracle, dctx, cam, kind):
    vtx, u = _scene(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    gi, gda = _upstream(u, kind, steps)
    ref = depth_ref.reference(vtx, u, frame, gi, gda)
    keep = ~ref["exclude"]
    assert keep.sum() > 100
    dctx.upload(vtx)
    dctx.set_backward(True)
    for det in (False, True):
        dctx.set_backward_deterministic(det)
        for level in (0, 1):
            dctx.set_tile_cull(level)
            dctx.render_depth(u)
            got, _, _ = _depth_backward(dctx, vtx, gi, gda)
            _check_groups(got, ref, keep, (cam, kind, det, level))


@pytest.mark.parametrize("scene", ["edge", "scale"])
def test_gradient_on_edge_and_scale_scenes(gs, oracle, dctx, scene):
    if scene == "edge":
        vtx, u = edge_scene.vertices("backward")[0], edge_scene.camera("axis")
    else:
        import scale_scene

        vtx, u = scale_scene.vertices()[0], scale_scene.camera("axis")
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    gi, gda = _upstream(u, "mixed", steps)
    ref = depth_ref.reference(vtx, u, frame, gi, gda)
    keep = ~ref["exclude"]
    dctx.upload(vtx)
    dctx.set_backward(True)
    for det in (False, True):
        dctx.set_backward_deterministic(det)
        dctx.render_depth(u)
        got, _, _ = _depth_backward(dctx, vtx, gi, gda)
        _check_groups(got, ref, keep, (scene, det), tol=2e-3)


def test_background_and_antialiased_frames(gs, oracle, dctx):
    vtx, u = _scene("c1")
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    gi, gda = _upstream(u, "mixed", steps)
    bg = (0.25, 0.5, 0.75)
    dctx.upload(vtx)
    dctx.set_backward(True)
    cases = [("bg", depth_ref.reference(vtx, u, frame, gi, gda, bg=bg)),
             ("aa", depth_ref.reference(vtx, u, aa_ref.oracle_frame(vtx, oracle.cov3d(vtx), u), gi, gda, pre=depth_ref.pinhole(True)))]
    for what, ref in cases:
        dctx.set_background(bg if what == "bg" else None)
        dctx.set_antialiased(what == "aa")
        for det in (False, True):
            dctx.set_backward_deterministic(det)
            dctx.render_depth(u)
            got, _, _ = _depth_backward(dctx, vtx, gi, gda)
            _check_groups(got, ref, ~ref["exclude"], (what, det))


def test_fisheye_vertex_gradient(gs, dctx):
    vtx, u, cam = _fisheye_case(gs, "fov200")
    dctx.upload(vtx)
    dctx.set_camera_model(cam)
    dctx.set_backward(True)
    frame = _fisheye_lists(gs, dctx, u, vtx, cam)
    gi, gda = _upstream(u, "mixed")
    ref = depth_ref.reference(vtx, u, frame, gi, gda, pre=depth_ref.fisheye(cam))
    keep = ~ref["exclude"]
    for det in (False, True):
        dctx.set_backward_deterministic(det)
        dctx.set_tile_cull(0)
        dctx.render_depth(u)
        got, _, _ = _depth_backward(dctx, vtx, gi, gda)
        _check_groups(got, ref, keep, ("fisheye", det))


def test_camera_gradient_and_density(gs, oracle, dctx):
    """dL/d(UBO) including view row 2, for depth-only and mixed upstream gradients, and the density columns."""
    from test_gpu_backward_camera import camera_scene

    vtx = camera_scene()
    u = scenes.camera("c1")
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    dctx.upload(vtx)
    dctx.set_backward(True)
    for kind in ("depth", "mixed"):
        gi, gda = _upstream(u, kind, steps)
        ref = depth_ref.reference(vtx, u, frame, gi, gda, camera=True)
        ref40 = np.zeros(40)
        ref40[:36], ref40[38:] = ref["grad_ubo"][:36], ref["grad_ubo"][36:]
        dctx.render_depth(u)
        _, dens, gu = _depth_backward(dctx, vtx, gi, gda, density=True, camera=True)
        for name, words in CAMERA_GROUPS.items():
            assert rel(gu[words], ref40[words]) <= 1e-3, (kind, name, gu[words], ref40[words])
        row2 = [20 + c * 4 + 2 for c in range(4)]
        assert np.abs(ref40[row2]).max() > 0 and rel(gu[row2], ref40[row2]) <= 1e-3, kind
        assert not gu[DEAD].any()
        # density column 0: |dL/duv| in NDC units, with the depth and alpha terms (grad_ref's statistics of the 5-channel blend)
        assert np.isfinite(dens).all() and (dens[:, 2] <= 1).all() and dens[:, 0].max() > 0


# ---------------------------------------------------------------------------------------------------------------------
# deterministic mode, unchanged entries, errors
# ---------------------------------------------------------------------------------------------------------------------
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


def test_deterministic_words(gs, dctx):
    torch = _torch()
    vtx, u = _scene("c1")
    gi, gda = _upstream(u, "mixed")
    dctx.upload(vtx)
    dctx.set_backward(True)
    dctx.set_backward_deterministic(True)
    # zero depth and alpha gradients: gsb_render_backward_density's words
    dctx.render(u)
    gv0, d0 = _plain_density_backward(dctx, vtx, gi)
    dctx.render_depth(u)
    gv1, d1, _ = _depth_backward(dctx, vtx, gi, np.zeros_like(gda), density=True)
    assert _equal_up_to_zero_sign(gv0, gv1) and _equal_up_to_zero_sign(d0, d1)
    # levels 0 and 1, repeated calls, a side stream, a fresh context
    runs = []
    for level in (0, 1):
        dctx.set_tile_cull(level)
        dctx.render_depth(u)
        runs.append(_depth_backward(dctx, vtx, gi, gda, density=True))
        runs.append(_depth_backward(dctx, vtx, gi, gda, density=True))
    side = torch.cuda.Stream()
    runs.append(_depth_backward(dctx, vtx, gi, gda, density=True, stream=gs.stream_ptr(side)))
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        fresh.set_backward(True)
        fresh.set_backward_deterministic(True)
        fresh.render_depth(u)
        runs.append(_depth_backward(fresh, vtx, gi, gda, density=True))
    finally:
        fresh.close()
    for r in runs[1:]:
        assert _same(r[0].astype(np.float32), runs[0][0].astype(np.float32)) and _same(r[1], runs[0][1])


def test_depth_frame_leaves_the_other_entries_alone(gs, dctx):
    torch = _torch()
    vtx, u = _scene("odd_size")
    gi = grad_image(u)
    dctx.upload(vtx)
    dctx.set_backward(True)
    dctx.set_backward_deterministic(True)
    dctx.set_background((0.25, 0.5, 0.75))
    out = []
    for depth in (False, True):
        if depth:
            dctx.render_depth(u)
        else:
            dctx.render(u)
        gv, dens = _plain_density_backward(dctx, vtx, gi)
        gb = dctx.background_gradient(torch.from_numpy(gi).cuda()).cpu().numpy()
        out.append((gv, dens, gb))
    assert all(_same(a, b) for a, b in zip(*out))


def test_error_codes(gs, dctx):
    torch = _torch()
    vtx, u = _scene("odd_size")
    v = torch.from_numpy(vtx).cuda()
    gv = torch.empty_like(v)
    gi = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    gd = torch.zeros((u.height, u.width, 2), dtype=torch.float32, device="cuda")
    img = np.empty((u.height, u.width, 4), np.float32)
    da = np.empty((u.height, u.width + 1, 2), np.float32)
    lib, INV = gs.lib, gs.ERR_INVALID

    def rd(depth_ptr, pitch=0, ctx=dctx):
        ctx._ck(lib.gsb_render_depth(ctx.h, gs.C.byref(u), 0, gs.ALL_ROWS, img.ctypes.data, 0, gs.MEM_HOST, gs.FORMAT_RGBA32F,
                                     depth_ptr, pitch, None))

    def bw(vp=v.data_ptr(), gip=gi.data_ptr(), gdp=gd.data_ptr(), dpitch=0, gvp=gv.data_ptr(), gup=None):
        dctx._ck(lib.gsb_render_backward_depth(dctx.h, vp, gip, 0, gdp, dpitch, gvp, gup, None, None))

    expect(gs, dctx, gs.ERR_NO_SCENE, lambda: rd(da.ctypes.data))
    dctx.upload(vtx)
    expect(gs, dctx, INV, lambda: rd(None), "gsb_render_depth")
    expect(gs, dctx, INV, lambda: rd(da.ctypes.data, u.width * 8 - 8), "gsb_render_depth")
    expect(gs, dctx, INV, lambda: rd(da.ctypes.data, u.width * 8 + 4), "gsb_render_depth")
    expect(gs, dctx, INV, lambda: rd(da.ctypes.data + 4, (u.width + 1) * 8), "gsb_render_depth")
    rd(da.ctypes.data, (u.width + 1) * 8)  # a padded pitch is fine
    # the backward: no recorded frame, then a frame without depth
    expect(gs, dctx, INV, lambda: bw(), ENTRY)
    dctx.set_backward(True)
    dctx.render(u)
    expect(gs, dctx, INV, lambda: bw(), ENTRY)
    dctx.render_depth(u)
    bw()
    bw(gip=None)  # no colour gradient
    expect(gs, dctx, INV, lambda: bw(vp=None), ENTRY)
    expect(gs, dctx, INV, lambda: bw(gdp=None), ENTRY)
    expect(gs, dctx, INV, lambda: bw(gvp=None), ENTRY)
    expect(gs, dctx, INV, lambda: bw(dpitch=u.width * 8 - 8), ENTRY)
    expect(gs, dctx, INV, lambda: bw(dpitch=u.width * 8 + 4), ENTRY)
    expect(gs, dctx, INV, lambda: bw(gdp=gd.data_ptr() + 4), ENTRY)
    dctx.render_depth(u, rows=(0, 1))  # a band
    expect(gs, dctx, INV, lambda: bw(), ENTRY)
    dctx.render_depth(u)
    dctx.upload(vtx)  # the scene changed after the frame
    expect(gs, dctx, INV, lambda: bw(), ENTRY)
    # a fisheye frame has no camera gradient
    from test_gpu_fisheye import _lens

    dctx.set_camera_model(_lens(gs, u, fov_deg=120.0))
    dctx.render_depth(u)
    gu = torch.empty(40, dtype=torch.float32, device="cuda")
    expect(gs, dctx, INV, lambda: bw(gup=gu.data_ptr()), ENTRY)
    bw()
    # group ranks
    grp = gs.Group([0, 0])
    try:
        grp.upload(vtx)
        rank = grp.context(0)
        with pytest.raises(gs.GsbError) as ei:
            rd(da.ctypes.data, (u.width + 1) * 8, ctx=rank)
        assert ei.value.code == INV
    finally:
        grp.close()


# ---------------------------------------------------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------------------------------------------------
def test_render_torch_depth_autograd(gs, oracle, dctx):
    """render_torch(depth=True) through autograd: a loss on image, D / A and 1 / (D / A) gives the float64 chain rule."""
    torch = _torch()
    vtx, u = _scene("odd_size")
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    v = torch.from_numpy(vtx).cuda().requires_grad_()
    img, da = gs.render_torch(dctx, v, u, depth=True)
    assert img.shape == (u.height, u.width, 4) and da.shape == (u.height, u.width, 2)
    mask = torch.from_numpy(~steps).cuda()
    w = torch.from_numpy(np.random.default_rng(3).standard_normal((u.height, u.width)).astype(np.float32)).cuda() * mask
    ed = da[..., 0] / da[..., 1].clamp_min(1e-10)
    inv = 1.0 / ed.clamp_min(1e-3)
    hit = (da[..., 1] > 0.5) & mask
    loss = (img[..., :3].sum(-1) * w).sum() + (ed * w * hit).sum() + (inv * w * hit).sum()
    loss.backward()
    # the same loss's upstream gradients, fed to the float64 reference
    with torch.no_grad():
        d_, a_ = da[..., 0].double(), da[..., 1].double()
        wd, h = w.double(), hit.double()
        ac = a_.clamp_min(1e-10)
        e = d_ / ac
        ge = wd * h - wd * h / e.clamp_min(1e-3) ** 2 * (e > 1e-3).double()
        gD = ge / ac
        gA = -ge * d_ / ac ** 2 * (a_ > 1e-10).double()
    gi = np.zeros((u.height, u.width, 4), np.float32)
    gi[..., :3] = w.cpu().numpy()[..., None]
    gda = np.stack([gD.cpu().numpy(), gA.cpu().numpy()], -1).astype(np.float32)
    ref = depth_ref.reference(vtx, u, frame, gi, gda)
    _check_groups(v.grad.double().cpu().numpy(), ref, ~ref["exclude"], "render_torch", tol=2e-3)


def _depth_views(gs, distance=1.0):
    """test_gpu_adam's poses at 160 x 120, `distance` times as far from the scene."""
    from test_gpu_adam import POSES

    return [gs.uniforms_from_camera([distance * x for x in p], q, 45.0, 0.1, 1000.0, 160, 120) for p, q in POSES]


def test_expected_depth_loss_lowers_held_out_depth_error(gs, dctx):
    """An image + expected-depth loss trains a perturbed scene to a lower held-out depth error than the image loss alone."""
    torch = _torch()
    from test_gpu_adam import TRAIN_LR

    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = _depth_views(gs)
    train, held = views[:-1], views[-1:]
    with torch.no_grad():
        targets = [tuple(t.clone() for t in gs.render_torch(dctx, full, u, depth=True)) for u in views]
    start = full[::4].clone()
    start[:, 0:3] += 0.05 * torch.randn(start[:, 0:3].shape, generator=torch.Generator().manual_seed(0)).cuda()
    res = {}
    for name, lam in (("image", 0.0), ("image+depth", 0.5)):
        opt = gs.SceneAdam(dctx, start, TRAIN_LR)
        g = torch.empty((120, 160, 4), dtype=torch.float32, device="cuda")
        for it in range(200):
            k = it % len(train)
            img, da = opt.render(train[k], depth=True)
            dctx.image_loss(img, targets[k][0], 0.2, grad_image=g)
            da = da.detach().requires_grad_()
            tda = targets[k][1]
            m = (tda[..., 1] > 0.5).float()
            ed = da[..., 0] / da[..., 1].clamp_min(1e-10)
            loss = lam * ((ed - tda[..., 0] / tda[..., 1].clamp_min(1e-10)).abs() * m).sum() / m.sum().clamp_min(1.0)
            loss.backward()
            opt.step(g, grad_depth_alpha=da.grad)
        errs = []
        for u, (_, tda) in zip(held, targets[-1:]):
            _, da = opt.render(u, depth=True)
            m = (tda[..., 1] > 0.5) & (da[..., 1] > 0.5)
            ed, te = da[..., 0] / da[..., 1], tda[..., 0] / tda[..., 1]
            errs.append(float((ed - te)[m].abs().mean()))
        res[name] = sum(errs) / len(errs)
    print(f"held-out expected-depth error: image only {res['image']:.4f}, image + depth {res['image+depth']:.4f}")
    assert res["image+depth"] < res["image"], res


def test_mask_loss_removes_off_object_alpha(gs, dctx):
    """An object capture: a mask loss on A drives the alpha outside the object's mask below the run without it."""
    torch = _torch()
    from test_gpu_adam import TRAIN_LR

    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = _depth_views(gs, 3.0)  # the object covers the middle of the frame and leaves empty space around it
    with torch.no_grad():
        targets = [tuple(t.clone() for t in gs.render_torch(dctx, full, u, depth=True)) for u in views]
    # floaters the black background hides: black copies of some Gaussians pushed outside the object, at opacity 0.5
    gen = torch.Generator().manual_seed(1)
    floaters = full[torch.randperm(full.shape[0], generator=gen)[:300].cuda()].clone()
    floaters[:, 0:3] += 1.5 * torch.randn(floaters[:, 0:3].shape, generator=gen).cuda()
    floaters[:, 7] = 0.5
    floaters[:, 12:60] = 0.0
    floaters[:, 12:15] = -0.5 / 0.28209479177387814  # SH DC of colour 0
    start = torch.cat([full[::4], floaters])
    res = {}
    for name, lam in (("image", 0.0), ("image+mask", 1.0)):
        opt = gs.SceneAdam(dctx, start, TRAIN_LR)
        g = torch.empty((120, 160, 4), dtype=torch.float32, device="cuda")
        for it in range(150):
            k = it % len(views)
            img, da = opt.render(views[k], depth=True)
            dctx.image_loss(img, targets[k][0], 0.2, grad_image=g)
            mask = (targets[k][1][..., 1] > 0.5).float()
            gda = torch.zeros_like(da)
            gda[..., 1] = lam * 2.0 * (da[..., 1] - mask) / mask.numel()
            opt.step(g, grad_depth_alpha=gda)
        off = []
        for u, (_, tda) in zip(views, targets):
            _, da = opt.render(u, depth=True)
            outside = tda[..., 1] < 1e-3
            assert outside.any()
            off.append(float(da[..., 1][outside].mean()))
        res[name] = sum(off) / len(off)
    print(f"mean off-object alpha: image only {res['image']:.4f}, image + mask {res['image+mask']:.4f}")
    assert res["image+mask"] < res["image"], res


@pytest.mark.parametrize("selective", [False, True])
def test_scene_adam_with_depth_gradient(gs, dctx, selective):
    """SceneAdam.step(grad_depth_alpha=) equals a step from the gradient gsb_render_backward_depth gives, and refuses a depth
    gradient after a frame without depth."""
    torch = _torch()
    from test_gpu_adam import TRAIN_LR

    vtx, u = _scene("odd_size")
    v = torch.from_numpy(vtx).cuda()
    gi, gda = _upstream(u, "mixed")
    opt = gs.SceneAdam(dctx, v, TRAIN_LR, selective=selective)
    img, da = opt.render(u, depth=True)
    opt.step(torch.from_numpy(gi).cuda(), grad_depth_alpha=torch.from_numpy(gda).cuda())
    torch.cuda.synchronize()
    other = gs.Context(0)
    try:
        other.upload(vtx)
        other.set_backward(True)
        other.render_depth(u)
        want, _, _ = _depth_backward(other, vtx, gi, gda)
    finally:
        other.close()
    assert rel(opt.grad.double().cpu().numpy(), want) <= 1e-6
    assert not torch.equal(opt.vertices, v)
    opt.render(u)
    with pytest.raises(ValueError):
        opt.step(torch.from_numpy(gi).cuda(), grad_depth_alpha=torch.from_numpy(gda).cuda())
    opt.render(u, depth=True)
    opt.step(None, grad_depth_alpha=torch.from_numpy(gda).cuda())  # depth alone
