"""gsb_set_backward / gsb_render_backward / gs_b200.render_torch: the recording forward leaves the image bit-identical, and
the gradient of a frame matches the float64 restatement of the forward (tests/grad_ref.py)."""
import numpy as np
import pytest

import grad_ref
import scenes
from backward_util import GROUPS, expect, grad_image, rel, render

pytestmark = pytest.mark.gpu

@pytest.fixture
def bctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _backward(ctx, vtx, g):
    import torch

    v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
    gi = torch.from_numpy(g).cuda()
    out = torch.full_like(v, float("nan"))
    ctx.render_backward(v.data_ptr(), gi.data_ptr(), out.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.float64)


def _frame_grad(ctx, vtx, u, g, level=0, mode=0):
    render(ctx, u, level, mode)
    return _backward(ctx, vtx, g)


@pytest.mark.parametrize("cam", sorted(scenes.CAMERAS))
def test_recording_frame_is_bit_identical(gs, bctx, cam):
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    bctx.upload(vtx)
    for level in (0, 1, 2):
        bctx.set_tile_cull(level)
        for mode in (gs.MODE_EXACT, gs.MODE_FAST):
            bctx.set_mode(mode)
            for fmt in (gs.FORMAT_RGBA32F, gs.FORMAT_BGRA8):
                bctx.set_backward(False)
                plain = bctx.render(u, fmt)
                bctx.set_backward(True)
                rec = bctx.render(u, fmt)
                assert np.array_equal(plain.view(np.uint8), rec.view(np.uint8)), (cam, level, mode, fmt)


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_gradient_matches_float64_reference(oracle, bctx, cam):
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    ref = grad_ref.reference(vtx, u, frame, g)
    bctx.upload(vtx)
    got = _frame_grad(bctx, vtx, u, g)
    assert np.isfinite(got).all()
    keep = ~ref["exclude"]
    assert keep.sum() > 100
    for name, cols in GROUPS.items():
        r = rel(got[keep, cols], ref["grad"][keep, cols])
        assert r <= 1e-3, (cam, name, r)
    assert not got[:, 3].any()  # position.w


def test_levels_0_and_1_agree(bctx):
    _, vtx, u = scenes.c1()
    g = grad_image(u, np.zeros((u.height, u.width), bool))
    bctx.upload(vtx)
    g0 = _frame_grad(bctx, vtx, u, g, level=0)
    g1 = _frame_grad(bctx, vtx, u, g, level=1)
    g2 = _frame_grad(bctx, vtx, u, g, level=2)  # falls back to level 1 while recording
    assert rel(g1, g0) <= 1e-6
    assert rel(g2, g0) <= 1e-6


def test_fast_mode_close_to_exact(oracle, bctx):
    _, vtx, u = scenes.c1()
    oracle.set_exp_mode(0)
    _, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    bctx.upload(vtx)
    ge = _frame_grad(bctx, vtx, u, g, mode=0)
    gf = _frame_grad(bctx, vtx, u, g, mode=1)
    assert rel(gf, ge) <= 1e-3


def test_nothing_visible_gives_zero(bctx):
    _, vtx, _ = scenes.c1()
    u = scenes.camera("away")
    bctx.upload(vtx)
    got = _frame_grad(bctx, vtx, u, np.ones((u.height, u.width, 4), np.float32))
    assert not got.any()


def test_error_cases(gs, bctx):
    import torch

    _, vtx, u = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    gi = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    out = torch.empty_like(v)

    def bw(c):
        return lambda: c.render_backward(v.data_ptr(), gi.data_ptr(), out.data_ptr())

    expect(gs, bctx, gs.ERR_NO_SCENE, bw(bctx))  # nothing uploaded
    bctx.upload(vtx)
    expect(gs, bctx, gs.ERR_NO_SCENE, bw(bctx))  # no frame yet
    bctx.set_backward(False)
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx))  # switch off
    bctx.set_backward(True)
    bctx.render(u, rows=(0, 2))
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx))  # a band
    bctx.render(u)
    bctx.render_backward(v.data_ptr(), gi.data_ptr(), out.data_ptr())  # the whole frame: fine
    bctx.upload(vtx)
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx))  # uploaded again after the frame
    # a pipelined frame that overflowed its arena (gsb_render_async never regrows; a fresh context holds N = 10 k instances)
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        fresh.set_backward(True)
        ui = scenes.camera("inside")
        dev = torch.empty((ui.height, ui.width, 4), dtype=torch.float32, device="cuda")
        fresh.render_into(ui, dev.data_ptr(), gs.FORMAT_RGBA32F, sync=False)
        torch.cuda.synchronize()
        expect(gs, fresh, gs.ERR_INVALID, bw(fresh))
        with pytest.raises(gs.GsbError):
            fresh.stats()  # reports (and clears) the overflow
    finally:
        fresh.close()
    # fp16 SH storage
    bctx.set_sh_storage(True)
    bctx.upload(vtx)
    bctx.render(u)
    expect(gs, bctx, gs.ERR_INVALID, bw(bctx))
    # a sharded context (two ranks on one GPU)
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        expect(gs, c0, gs.ERR_INVALID, lambda: c0.set_backward(True))
        expect(gs, c0, gs.ERR_INVALID, bw(c0))
    finally:
        grp.close()


def test_render_torch_fits_a_perturbed_scene(gs, bctx):
    import torch

    _, vtx, u = scenes.c1()
    base = torch.from_numpy(vtx).cuda()
    target = gs.render_torch(bctx, base, u).detach()
    gen = torch.Generator(device="cpu").manual_seed(3)
    n = vtx.shape[0]
    noise = torch.zeros((n, 60))
    noise[:, 0:3] = 0.003 * torch.randn(n, 3, generator=gen)
    noise[:, 7] = 0.05 * torch.randn(n, generator=gen)
    noise[:, 12:15] = 0.1 * torch.randn(n, 3, generator=gen)
    start = base + noise.cuda()
    start[:, 7] = start[:, 7].clamp(0.02, 1.0)
    # one parameter tensor per perturbed group, each with its own step size
    pos = start[:, 0:3].clone().requires_grad_()
    opa = start[:, 7:8].clone().requires_grad_()
    dc = start[:, 12:15].clone().requires_grad_()
    opt = torch.optim.Adam([{"params": [pos], "lr": 3e-4}, {"params": [opa], "lr": 3e-3}, {"params": [dc], "lr": 5e-3}])

    def scene():
        return torch.cat([pos, start[:, 3:7], opa, start[:, 8:12], dc, start[:, 15:]], 1)

    losses = []
    for _ in range(50):
        opt.zero_grad()
        img = gs.render_torch(bctx, scene(), u)
        loss = ((img[..., :3] - target[..., :3]) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    with torch.no_grad():
        final = float(((gs.render_torch(bctx, scene(), u)[..., :3] - target[..., :3]) ** 2).sum())
    print("render_torch fit: initial loss", losses[0], "final", final)
    assert final < 0.5 * losses[0], (losses[0], final)
    # a frame rendered between forward and backward makes backward refuse
    img = gs.render_torch(bctx, scene(), u)
    bctx.render(u)
    with pytest.raises(RuntimeError):
        img.sum().backward()


def test_render_torch_gradient_is_ordered_on_torchs_stream(gs, bctx):
    """autograd's dL/dvertices, read by torch right after backward on its default stream, is the whole gradient."""
    import torch

    _, vtx, u = scenes.c1()
    g = grad_image(u, np.zeros((u.height, u.width), bool))
    v = torch.from_numpy(vtx).cuda().requires_grad_()
    img = gs.render_torch(bctx, v, u)
    (img * torch.from_numpy(g).cuda()).sum().backward()
    got = v.grad.cpu().numpy().astype(np.float64)
    want = _backward(bctx, vtx, g)  # the same frame, differentiated again and synchronised
    assert np.abs(want).max() > 0
    assert rel(got, want) <= 1e-6
