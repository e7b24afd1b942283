"""gsb_bilagrid_apply / gsb_bilagrid_backward / bilateral_grid_torch: the bilateral-grid colour correction and its gradients
against the float64 reference (tests/bilagrid_ref.py; its F.grid_sample form in float64, which the CPU tests tie to the explicit
numpy slice within 1e-12), the identity grid bit for bit, bitwise reproducibility, every error code, the untouched last frame,
and two training fits."""
import ctypes as C

import numpy as np
import pytest

import bilagrid_ref as br
import scenes

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (5, 3), (17, 31), (641, 479), (3200, 1400)]  # W x H
SHAPES = [(2, 2, 2), (16, 16, 8), (5, 9, 3), (64, 64, 16)]  # X, Y, L


def _torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def bctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _dev(a):
    torch = _torch()
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _grid(shape, spread, seed=7):
    return _dev(br.random_grid(shape, spread, seed).astype(np.float32))


def _reference(img, grid, g_out=None):
    """float64 (out, d image, d grid) through the grid_sample form at the definition's fp32 coordinates."""
    torch = _torch()
    ti = img.detach().double().requires_grad_()
    tg = grid.detach().double().requires_grad_()
    out = br.torch_path(ti, tg, coords32=True)
    if g_out is None:
        return out.detach(), None, None
    (out[..., :3] * g_out[..., :3].double()).sum().backward()
    return out.detach(), ti.grad, tg.grad


def _near_plane(img, L, tol=1e-6):
    """Pixels whose luma lies within tol of a z node plane or a clamp (the slice's kinks)."""
    return _dev(br.node_distance(img.cpu().numpy(), L) < tol)


def _rel(a, b):
    return float((a.double() - b).norm() / max(float(b.norm()), 1e-300))


def _check_forward(bctx, img, grid, what):
    torch = _torch()
    out = bctx.bilagrid_apply(img, grid)
    ref, _, _ = _reference(img, grid)
    torch.cuda.synchronize()
    err = ((out[..., :3].double() - ref[..., :3]).abs() / ref[..., :3].abs().clamp(min=1.0)).max()
    assert float(err) <= 1e-5, (what, float(err))
    assert torch.equal(out[..., 3], img[..., 3]), what


@pytest.mark.parametrize("spread", [0.05, 1.0], ids=["near", "far"])
@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_forward_matches_reference(bctx, size, shape, spread):
    w, h = size
    _check_forward(bctx, _dev(br.random_image(w, h, seed=w + h)), _grid(shape, spread), (size, shape, spread))


def _c1_frames(gs):
    _, vtx, _ = scenes.c1()
    c = gs.Context(0)
    try:
        c.upload(vtx)
        u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 320, 240)
        plain = c.render(u)
        c.set_background((0.25, 0.5, 1.5))  # a learned colour may leave [0, 1]
        over = c.render(u)
    finally:
        c.close()
    return plain, over


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_forward_on_rendered_frames(gs, bctx, shape):
    for name, frame in zip(("c1", "background"), _c1_frames(gs)):
        _check_forward(bctx, _dev(frame), _grid(shape, 0.3), (name, shape))


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_identity_grid_returns_the_image(gs, bctx, shape):
    torch = _torch()
    X, Y, L = shape
    grid = gs.identity_bilateral_grids(1, shape, device="cuda")[0]
    for img in (_dev(br.random_image(641, 479, seed=1, lo=-3.0, hi=4.0)), _dev(_c1_frames(gs)[0])):
        img[0, 0, :3] = -0.0
        out = bctx.bilagrid_apply(img, grid)
        torch.cuda.synchronize()
        # == treats -0 and +0 as equal, the one difference allowed; A is copied word for word
        assert bool((out[..., :3] == img[..., :3]).all())
        assert torch.equal(out[..., 3].view(torch.int32), img[..., 3].view(torch.int32))


def _backward(bctx, img, grid, g, want_image=True, want_grid=True, stream=None):
    torch = _torch()
    gi = torch.full(img.shape, float("nan"), device="cuda") if want_image else None
    gg = torch.full(grid.shape, float("nan"), device="cuda") if want_grid else None
    bctx.bilagrid_backward(img, grid, g, gi, gg, stream=stream)
    torch.cuda.synchronize()
    return gi, gg


BW_CASES = [((5, 3), (2, 2, 2)), ((17, 31), (5, 9, 3)), ((641, 479), (16, 16, 8)), ((641, 479), (64, 64, 16)),
            ((3200, 1400), (16, 16, 8)), ((1, 1), (16, 16, 8))]


@pytest.mark.parametrize("spread", [0.05, 1.0], ids=["near", "far"])
@pytest.mark.parametrize("size,shape", BW_CASES, ids=[f"{w}x{h}-{'x'.join(map(str, s))}" for (w, h), s in BW_CASES])
def test_backward_matches_reference(bctx, size, shape, spread):
    torch = _torch()
    w, h = size
    img = _dev(br.random_image(w, h, seed=3 * w + h))
    grid = _grid(shape, spread)
    g = torch.randn((h, w, 4), generator=torch.Generator(device="cuda").manual_seed(w), device="cuda")
    gi, gg = _backward(bctx, img, grid, g)
    _, ri, rg = _reference(img, grid, g)
    assert bool((gi[..., 3] == 0).all())
    keep = ~_near_plane(img, shape[2])
    for c in range(3):
        a, b = gi[..., c][keep], ri[..., c][keep]
        assert _rel(a, b) <= 1e-5, (c, _rel(a, b))
        assert float((a.double() - b).abs().max()) <= 1e-5 * float(b.abs().max()), c
    for k in range(12):
        assert _rel(gg[k], rg[k]) <= 1e-5, (k, _rel(gg[k], rg[k]))
        assert float((gg[k].double() - rg[k]).abs().max()) <= 1e-5 * float(rg[k].abs().max()), k


def test_backward_on_a_rendered_frame(gs, bctx):
    torch = _torch()
    img = _dev(_c1_frames(gs)[1])
    grid = _grid((16, 16, 8), 0.3)
    g = torch.randn(img.shape, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    gi, gg = _backward(bctx, img, grid, g)
    _, ri, rg = _reference(img, grid, g)
    keep = ~_near_plane(img, 8)
    assert _rel(gi[..., :3][keep], ri[..., :3][keep]) <= 1e-5
    assert _rel(gg, rg) <= 1e-5


def test_null_combinations_and_reproducibility(gs, bctx):
    torch = _torch()
    w, h = 641, 479
    img = _dev(br.random_image(w, h, seed=9))
    grid = _grid((16, 16, 8), 0.5)
    g = torch.randn((h, w, 4), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    gi, gg = _backward(bctx, img, grid, g)
    out = bctx.bilagrid_apply(img, grid)
    only_i, _ = _backward(bctx, img, grid, g, want_grid=False)
    _, only_g = _backward(bctx, img, grid, g, want_image=False)
    assert torch.equal(gi, only_i) and torch.equal(gg, only_g)
    for _ in range(3):
        a, b = _backward(bctx, img, grid, g)
        assert torch.equal(a, gi) and torch.equal(b, gg)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        a, b = _backward(bctx, img, grid, g, stream=side)
        o = bctx.bilagrid_apply(img, grid)
    side.synchronize()
    assert torch.equal(a, gi) and torch.equal(b, gg) and torch.equal(o, out)
    fresh = gs.Context(0)
    try:
        a, b = _backward(fresh, img, grid, g)
        assert torch.equal(a, gi) and torch.equal(b, gg) and torch.equal(fresh.bilagrid_apply(img, grid), out)
    finally:
        fresh.close()
    # padded rows: views of wider buffers
    wide = lambda t: torch.full((h, w + 3, 4), float("nan"), device="cuda")  # noqa: E731
    pi, pg, pgi, po = wide(0), wide(0), wide(0), wide(0)
    pi[:, :w] = img
    pg[:, :w] = g
    bctx.bilagrid_backward(pi[:, :w], grid, pg[:, :w], pgi[:, :w], b)
    bctx.bilagrid_apply(pi[:, :w], grid, po[:, :w])
    torch.cuda.synchronize()
    assert torch.equal(pgi[:, :w], gi) and torch.equal(b, gg) and torch.equal(po[:, :w], out)
    assert bool(pgi[:, w:].isnan().all()) and bool(po[:, w:].isnan().all())


def test_error_codes_and_the_last_frame(gs):
    torch = _torch()
    lib = gs.lib
    c = gs.Context(0)
    try:
        _, vtx, _ = scenes.c1()
        v = torch.from_numpy(vtx).cuda()
        c.upload(vtx)
        c.set_backward(True)
        u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 64, 48)
        frame = c._render_whole_frame(u, v.device)
        g_frame = torch.randn(frame.shape, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")
        before = torch.empty_like(v)
        torch.cuda.synchronize()
        c.render_backward(v.data_ptr(), g_frame.data_ptr(), before.data_ptr())

        W, H = 8, 4
        img = torch.rand((H, W, 4), device="cuda")
        grid = gs.identity_bilateral_grids(1, (4, 4, 4), device="cuda")[0]
        out = torch.empty_like(img)
        go = torch.rand_like(img)
        gi = torch.empty_like(img)
        gg = torch.empty_like(grid)
        buf = torch.zeros(4096, device="cuda")
        P = 16 * W
        ok = dict(ctx=c.h, W=W, H=H, image=img.data_ptr(), ip=P, grid=grid.data_ptr(), X=4, Y=4, L=4, out=out.data_ptr(), op=P)

        def apply(**kw):
            a = {**ok, **kw}
            return lib.gsb_bilagrid_apply(a["ctx"], a["W"], a["H"], a["image"], a["ip"], a["grid"], a["X"], a["Y"], a["L"],
                                          a["out"], a["op"], None)

        okb = {**ok, "go": go.data_ptr(), "gop": P, "gi": gi.data_ptr(), "gip": P, "gg": gg.data_ptr()}

        def backward(**kw):
            a = {**okb, **kw}
            return lib.gsb_bilagrid_backward(a["ctx"], a["W"], a["H"], a["image"], a["ip"], a["grid"], a["X"], a["Y"], a["L"],
                                             a["go"], a["gop"], a["gi"], a["gip"], a["gg"], None)

        assert apply() == gs.OK and backward() == gs.OK
        assert backward(gi=None) == gs.OK and backward(gg=None) == gs.OK
        common = [dict(ctx=None), dict(image=None), dict(grid=None), dict(W=0), dict(H=0), dict(X=1), dict(Y=65), dict(L=1),
                  dict(L=65), dict(ip=P - 16), dict(ip=0), dict(image=img.data_ptr() + 4), dict(ip=P + 4),
                  dict(grid=buf.data_ptr() + 2)]
        for bad in common + [dict(out=None), dict(op=P - 16), dict(out=out.data_ptr() + 8), dict(op=P + 8)]:
            assert apply(**bad) == gs.ERR_INVALID, bad
        for bad in common + [dict(go=None), dict(gi=None, gg=None), dict(gop=P - 16), dict(go=go.data_ptr() + 4),
                             dict(gop=P + 4), dict(gip=P - 16), dict(gi=gi.data_ptr() + 4), dict(gip=P + 8),
                             dict(gg=buf.data_ptr() + 2)]:
            assert backward(**bad) == gs.ERR_INVALID, bad
        assert backward(gi=None, gip=0) == gs.OK  # grad_image's pitch is not read without it
        for bad_grid in (grid[:, :, :, :3], grid.double(), grid.unsqueeze(0), torch.ones((12, 4, 4, 65), device="cuda"),
                         grid.cpu()):
            with pytest.raises(ValueError):
                c.bilagrid_apply(img, bad_grid)
        with pytest.raises(ValueError):
            c.bilagrid_apply(img[..., :3], grid)
        with pytest.raises(ValueError):
            c.bilagrid_backward(img, grid, go)
        with pytest.raises(ValueError):
            c.bilagrid_backward(img, grid, go, grad_grid=gg[:, :2])

        after = torch.empty_like(v)
        torch.cuda.synchronize()
        c.render_backward(v.data_ptr(), g_frame.data_ptr(), after.data_ptr())
        torch.cuda.synchronize()
        assert torch.equal(before, after)
    finally:
        c.close()


def test_torch_path(gs, bctx):
    torch = _torch()
    w, h = 641, 479
    img0 = _dev(br.random_image(w, h, seed=4))
    grids = torch.nn.Parameter(_grid((16, 16, 8), 0.3).unsqueeze(0).repeat(2, 1, 1, 1, 1).contiguous())
    target = torch.rand((h, w, 4), generator=torch.Generator(device="cuda").manual_seed(0), device="cuda")

    def run(fn):
        grids.grad = None
        img = img0.clone().requires_grad_()
        out = fn(img, grids[1])
        ((out - target)[..., :3].square().sum() + out[..., 3].sum()).backward()
        return out.detach(), img.grad, grids.grad.clone()

    ours = run(lambda i, g: gs.bilateral_grid_torch(bctx, i, g))
    again = run(lambda i, g: gs.bilateral_grid_torch(bctx, i, g))
    ref = run(br.torch_path)
    assert all(torch.equal(a, b) for a, b in zip(ours, again))
    assert bool((ours[2][0] == 0).all())  # autograd's indexing backward: only grids[1] gets a gradient
    assert _rel(ours[0], ref[0].double()) <= 1e-6
    keep = ~_near_plane(img0, 8)
    assert _rel(ours[1][keep], ref[1][keep].double()) <= 1e-5
    assert _rel(ours[2], ref[2].double()) <= 1e-5


def test_fit_a_gain_and_white_balance_field(gs, bctx):
    """A frozen render as the image, its copy under a smooth gain and white balance as the target: the grid alone, from
    identity, fits the difference."""
    torch = _torch()
    frame, _ = _c1_frames(gs)
    img = _dev(frame)
    h, w = img.shape[:2]
    gain = 0.75 + 0.5 * torch.linspace(0, 1, w, device="cuda")[None, :, None] * torch.ones((h, 1, 1), device="cuda")
    wb = torch.tensor([1.15, 1.0, 0.8], device="cuda")
    target = img.clone()
    target[..., :3] = img[..., :3] * gain * wb
    grids = torch.nn.Parameter(gs.identity_bilateral_grids(1, device="cuda"))
    opt = torch.optim.Adam([grids], lr=0.01, eps=1e-15)

    def loss_of():
        return gs.image_loss_torch(bctx, gs.bilateral_grid_torch(bctx, img, grids[0]), target)

    loss0 = float(loss_of())
    for _ in range(300):
        loss = loss_of()
        opt.zero_grad()
        loss.backward()
        opt.step()
    loss1 = float(loss_of())
    print(f"grid fit: loss {loss0:.5f} -> {loss1:.5f}")
    assert loss1 < 0.1 * loss0 and loss1 < 5e-3, (loss0, loss1)


def test_scene_adam_with_per_view_exposure(gs, bctx):
    """Two views whose targets differ by an exposure: SceneAdam with a grid per view reaches a lower loss than without."""
    from test_gpu_adam import POSES, TRAIN_LR

    torch = _torch()
    _, vtx, _ = scenes.c1()
    full = torch.from_numpy(vtx).cuda()
    views = [gs.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 320, 240) for p, q in POSES[:2]]
    with torch.no_grad():
        targets = [gs.render_torch(bctx, full, u).clone() for u in views]
    for t, e in zip(targets, (0.6, 1.4)):
        t[..., :3] *= e
    start = full[::4].clone()
    start[:, 4:7] *= 1.5
    final = {}
    for use_grids in (False, True):
        opt = gs.SceneAdam(bctx, start, TRAIN_LR)
        grids = torch.nn.Parameter(gs.identity_bilateral_grids(2, device="cuda"))
        grid_opt = torch.optim.Adam([grids], lr=5e-3, eps=1e-15)
        for it in range(300):
            i = it % 2
            img = opt.render(views[i]).requires_grad_()
            out = gs.bilateral_grid_torch(bctx, img, grids[i]) if use_grids else img
            loss = gs.image_loss_torch(bctx, out, targets[i])
            if use_grids:
                loss = loss + 10.0 * gs.bilateral_grid_tv(grids)
            loss.backward()
            opt.step(img.grad)
            if use_grids:
                grid_opt.step()
                grid_opt.zero_grad()
        with torch.no_grad():
            total = 0.0
            for i, u in enumerate(views):
                img = opt.render(u)
                out = gs.bilateral_grid_torch(bctx, img, grids[i]) if use_grids else img
                total += float(gs.image_loss_torch(bctx, out, targets[i]))
        final[use_grids] = total / 2
    print(f"per-view exposure: loss without grids {final[False]:.5f}, with grids {final[True]:.5f}")
    assert final[True] < final[False], final
