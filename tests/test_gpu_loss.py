"""gsb_image_loss / image_loss_torch / image_metrics: the fused L1 + D-SSIM loss and its gradient match the float64
reference (tests/loss_ref.py) from 1 x 1 to the bench frame, on rendered frames, noise, flat and saturated images, float32 and
RGBA8 targets and lambda in {0, 0.2, 1}; they are bit-reproducible across calls, streams, pitches and contexts; every
invalid argument is refused; and the loss drives gsb_render_backward and render_torch."""
import sys
from pathlib import Path

import numpy as np
import pytest

import loss_ref
import scenes
from backward_util import rel

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (3, 2), (11, 11), (16, 16), (17, 33), (320, 240), (641, 479)]  # W x H


def _torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def lctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _inputs(kind, w, h, seed=0):
    """(image, target) (H, W, 4) float32 of one input kind."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 1, (h, w, 4)).astype(np.float32)
    y = rng.uniform(0, 1, (h, w, 4)).astype(np.float32)
    if kind == "flat":  # large constant regions: sigma exactly 0 inside them, and x == y on some of them
        x[: h // 2], y[: h // 2] = 0.25, 0.625
        x[:, : w // 3], y[:, : w // 3] = 0.5, 0.5
    elif kind == "saturated":  # many values exactly 0 or 1 on both sides, x == y on a share of pixels
        x = np.clip(rng.normal(0.5, 0.8, (h, w, 4)), 0, 1).astype(np.float32)
        y = np.clip(rng.normal(0.5, 0.8, (h, w, 4)), 0, 1).astype(np.float32)
    return x, y


def _render_pair(gs, w, h):
    """c1's scene rendered at w x h from its camera and from a nearby pose."""
    _, vtx, _ = scenes.c1()
    c = gs.Context(0)
    try:
        c.upload(vtx)
        a = c.render(gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, w, h))
        b = c.render(gs.uniforms_from_camera([0.15, -0.05, 5.1], scenes.quat_axis_angle([0, 1, 0], 2), 45.0, 0.1, 1000.0, w, h))
    finally:
        c.close()
    return a, b


def _run(lctx, image, target, lam, grad=True):
    """gsb_image_loss of host or device (H, W, 4) arrays: (result as 4 floats, gradient (H, W, 4) float64 or None)."""
    torch = _torch()
    x = torch.as_tensor(image).cuda()
    y = torch.as_tensor(target).cuda()
    g = torch.full(x.shape, float("nan"), dtype=torch.float32, device="cuda") if grad else None
    r = lctx.image_loss(x, y, lam, g)
    torch.cuda.synchronize()
    return r.cpu().numpy(), None if g is None else g.cpu().numpy().astype(np.float64)


def _check(lctx, image, target, lam, device="cpu", what=""):
    got, grad = _run(lctx, image, target, lam)
    ref = loss_ref.reference(image, target, lam, device=device)
    loss, l1, ssim, mse = got
    assert abs(l1 - ref["l1"]) <= 1e-6 * ref["l1"], (what, l1, ref["l1"])
    assert abs(mse - ref["mse"]) <= 1e-6 * ref["mse"], (what, mse, ref["mse"])
    assert abs(ssim - ref["ssim"]) <= 1e-5, (what, ssim, ref["ssim"])
    assert abs(loss - ref["loss"]) <= 1e-5, (what, loss, ref["loss"])
    assert np.all(grad[..., 3] == 0)
    assert rel(grad[..., :3], ref["grad"][..., :3]) <= 1e-4, (what, rel(grad[..., :3], ref["grad"][..., :3]))
    # the L1 term's sign on every value: what is left of the gradient once the reference's SSIM term is taken away
    x = loss_ref.as_chw(image).permute(1, 2, 0).numpy()
    y = loss_ref.as_chw(target).permute(1, 2, 0).numpy()
    sign = np.sign(x - y)
    lam32 = float(np.float32(lam))
    n = sign.size
    if lam32 < 1:
        k = (1 - lam32) / n
        ssim_part = ref["grad"][..., :3] - k * sign
        assert np.array_equal(np.rint((grad[..., :3] - ssim_part) / k), sign), what
    if lam32 == 0:  # the L1 term alone: exactly its float32 coefficient times the sign
        assert np.array_equal(grad[..., :3], np.float32(1.0 / n) * sign), what
    return got, grad


@pytest.mark.parametrize("kind", ["noise", "flat", "saturated"])
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_matches_reference(lctx, size, kind):
    w, h = size
    x, y = _inputs(kind, w, h)
    _check(lctx, x, y, 0.2, what=(size, kind))


@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("size", [(3, 2), (17, 33), (320, 240)], ids=["3x2", "17x33", "320x240"])
def test_rgba8_target_and_lambda(lctx, size, lam):
    w, h = size
    x, _ = _inputs("noise", w, h, seed=1)
    t = np.random.default_rng(2).integers(0, 256, (h, w, 4), dtype=np.uint8)
    t[: h // 2, : w // 2] = np.clip(np.rint(x[: h // 2, : w // 2] * 255), 0, 255).astype(np.uint8)  # near-equal values
    _check(lctx, x, t, lam, what=(size, lam, "rgba8"))
    y = t.astype(np.float32) / np.float32(255.0)  # the same target as float32: the same words
    a, ga = _run(lctx, x, t, lam)
    b, gb = _run(lctx, x, y, lam)
    assert np.array_equal(a, b) and np.array_equal(ga, gb)


@pytest.mark.parametrize("size", [(320, 240), (641, 479)], ids=["320x240", "641x479"])
def test_rendered_frames(gs, lctx, size):
    a, b = _render_pair(gs, *size)
    assert np.abs(a - b)[..., :3].max() > 0.05
    for lam in (0.0, 0.2, 1.0):
        _check(lctx, a, b, lam, what=(size, lam))


@pytest.fixture(scope="module")
def garden_pair(gs):
    """bench.py's garden stand-in (5.8 M Gaussians, 3200 x 1400) rendered from its first camera and from the next one of
    the orbit, as device tensors."""
    torch = _torch()
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    cams = bench.cameras(gs, wl)
    c = gs.Context(0)
    try:
        c.upload(bench.make_scene(gs, wl))
        out = []
        for u in cams[:2]:
            t = torch.empty((u.height, u.width, 4), dtype=torch.float32, device="cuda")
            c.render_into(u, t.data_ptr())
            out.append(t)
    finally:
        c.close()
    yield out
    torch.cuda.empty_cache()


def test_bench_frame(lctx, garden_pair):
    a, b = garden_pair
    got, _ = _check(lctx, a, b, 0.2, device="cuda", what="garden 3200x1400")
    print("garden 3200x1400: loss %.6f L1 %.6f SSIM %.6f MSE %.6g" % tuple(got))


def test_metrics_only_gives_the_same_words(lctx):
    x, y = _inputs("noise", 641, 479, seed=3)
    with_grad, _ = _run(lctx, x, y, 0.2)
    without, none = _run(lctx, x, y, 0.2, grad=False)
    assert none is None and np.array_equal(with_grad.view(np.uint64), without.view(np.uint64))


def test_bit_reproducible(gs, lctx):
    """The same result and gradient words on repeated calls, on a torch side stream, with padded pitches and on a fresh
    context."""
    torch = _torch()
    w, h = 641, 479
    xn, yn = _inputs("noise", w, h, seed=4)
    x, y = torch.from_numpy(xn).cuda(), torch.from_numpy(yn).cuda()

    def once(c, x, y, stream=None, pad=0):
        g = torch.full((h, w + pad, 4), float("nan"), dtype=torch.float32, device="cuda")[:, :w]
        r = c.image_loss(x, y, 0.2, g, stream=stream)
        torch.cuda.synchronize()
        return r.cpu().numpy().view(np.uint64), g.cpu().numpy().view(np.uint32)

    base = once(lctx, x, y)
    runs = [once(lctx, x, y) for _ in range(3)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(once(lctx, x, y, stream=side))
    runs.append(once(lctx, x, y, stream=side))
    xp = torch.full((h, w + 3, 4), 7.0, device="cuda")[:, :w]
    yp = torch.full((h, w + 5, 4), -7.0, device="cuda")[:, :w]
    xp.copy_(x)
    yp.copy_(y)
    assert xp.stride(0) != 4 * w and yp.stride(0) != 4 * w
    runs.append(once(lctx, xp, yp, pad=2))
    fresh = gs.Context(0)
    try:
        runs.append(once(fresh, x, y))
    finally:
        fresh.close()
    for r in runs:
        assert np.array_equal(r[0], base[0]) and np.array_equal(r[1], base[1])


def test_invalid_arguments(gs, lctx):
    torch = _torch()
    lib, C = gs.lib, gs.C
    w, h = 40, 20
    x = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    y8 = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
    g = torch.zeros_like(x)
    res = torch.zeros(4, dtype=torch.float64, device="cuda")
    X, Y, Y8, G, R = x.data_ptr(), x.data_ptr(), y8.data_ptr(), g.data_ptr(), res.data_ptr()
    row = w * 16

    def call(ctx=lctx.h, W=w, H=h, img=X, ip=0, tgt=Y, tp=0, fmt=gs.FORMAT_RGBA32F, lam=0.2, grad=G, gp=0, out=R):
        return lib.gsb_image_loss(ctx, W, H, img, ip, tgt, tp, fmt, lam, grad, gp, out, None)

    assert call() == gs.OK and call(grad=None) == gs.OK and call(tgt=Y8, fmt=gs.FORMAT_RGBA8) == gs.OK
    assert call(ip=row + 16, tp=row + 32, gp=row + 48, H=h // 2) == gs.OK  # padded rows inside the buffers
    bad = {
        "null ctx": dict(ctx=None), "null image": dict(img=None), "null target": dict(tgt=None), "null result": dict(out=None),
        "W = 0": dict(W=0), "H = 0": dict(H=0), "lambda < 0": dict(lam=-0.01), "lambda > 1": dict(lam=1.01),
        "lambda NaN": dict(lam=float("nan")), "BGRA8 target": dict(tgt=Y8, fmt=gs.FORMAT_BGRA8), "format 7": dict(fmt=7),
        "image pitch": dict(ip=row - 16), "target pitch": dict(tp=row - 16), "rgba8 pitch": dict(tgt=Y8, fmt=gs.FORMAT_RGBA8, tp=w * 4 - 4),
        "grad pitch": dict(gp=row - 16), "image misaligned": dict(img=X + 4), "image pitch misaligned": dict(ip=row + 4),
        "target misaligned": dict(tgt=Y + 8), "target pitch misaligned": dict(tp=row + 8),
        "rgba8 misaligned": dict(tgt=Y8 + 2, fmt=gs.FORMAT_RGBA8), "rgba8 pitch misaligned": dict(tgt=Y8, fmt=gs.FORMAT_RGBA8, tp=w * 4 + 2),
        "grad misaligned": dict(grad=G + 4), "grad pitch misaligned": dict(gp=row + 4), "result misaligned": dict(out=R + 4),
    }
    for what, kw in bad.items():
        assert call(**kw) == gs.ERR_INVALID, what
        if "ctx" not in kw:
            assert lib.gsb_last_error(lctx.h).decode().startswith("gsb_image_loss"), what
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        lctx.image_loss(x, y8[:, :-1])
    with pytest.raises(ValueError):
        lctx.image_loss(x, y8.to(torch.int32))
    with pytest.raises(ValueError):
        lctx.image_loss(x.cpu(), y8)
    with pytest.raises(ValueError):
        gs.image_loss_torch(lctx, x[..., :3], y8)
    with pytest.raises(ValueError):
        gs.image_loss_torch(lctx, x.double(), y8)


def _c1_frame(gs, ctx):
    """c1 on ctx, a recorded RGBA32F frame of it as a device tensor, and the device vertices."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    ctx.upload(vtx)
    ctx.set_backward(True)
    img = torch.empty((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    ctx.render_into(u, img.data_ptr())
    return u, img, torch.from_numpy(vtx).cuda()


def test_loss_between_frame_and_backward(gs):
    """render (recording) -> gsb_image_loss -> gsb_render_backward succeeds and gives the gradient of the same sequence
    without the loss call."""
    torch = _torch()
    c = gs.Context(0)
    try:
        c.set_backward_deterministic(True)
        u, img, v = _c1_frame(gs, c)
        target, _ = _render_pair(gs, u.width, u.height)
        t = torch.from_numpy(target).cuda()
        g = torch.empty_like(img)
        c.image_loss(img, t, 0.2, g)
        torch.cuda.synchronize()  # the loss ran on torch's stream, the backward runs on the context's own
        after = torch.empty_like(v)
        c.render_backward(v.data_ptr(), g.data_ptr(), after.data_ptr())
        c.render_into(u, img.data_ptr())  # the same frame again, backward without the loss call in between
        plain = torch.empty_like(v)
        c.render_backward(v.data_ptr(), g.data_ptr(), plain.data_ptr())
        torch.cuda.synchronize()
        assert float(after.abs().max()) > 0
        assert torch.equal(after, plain)
    finally:
        c.close()


def test_render_torch_gradient(gs):
    """image_loss_torch(render_torch(...)).backward() gives gsb_render_backward's gradient of the float64 reference's d loss /
    d image; two passes under torch's deterministic mode are bit-identical."""
    torch = _torch()
    c = gs.Context(0)
    try:
        _, vtx, u = scenes.c1()
        t = torch.from_numpy(_render_pair(gs, u.width, u.height)[1]).cuda()
        v = torch.from_numpy(vtx).cuda().requires_grad_()
        img = gs.render_torch(c, v, u)
        loss = gs.image_loss_torch(c, img, t)
        assert loss.dtype == torch.float32 and loss.dim() == 0
        loss.backward()
        got = v.grad.clone()
        ref = loss_ref.reference(img.detach().cpu().numpy(), t.cpu().numpy(), 0.2)
        assert abs(float(loss) - ref["loss"]) <= 1e-5
        gi = torch.from_numpy(ref["grad"].astype(np.float32)).cuda()
        want = torch.empty_like(v)
        torch.cuda.synchronize()  # the context's own stream is not ordered with torch's
        c.render_backward(v.detach().data_ptr(), gi.data_ptr(), want.data_ptr())
        torch.cuda.synchronize()
        assert rel(got, want) <= 1e-4, rel(got, want)
        assert float(got.abs().max()) > 0

        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)
        try:
            passes = []
            for _ in range(2):
                v.grad = None
                loss = gs.image_loss_torch(c, gs.render_torch(c, v, u), t)
                loss.backward()
                passes.append((loss.detach().clone(), v.grad.clone()))
        finally:
            torch.use_deterministic_algorithms(prev)
        assert torch.equal(passes[0][0], passes[1][0]) and torch.equal(passes[0][1], passes[1][1])

        with torch.no_grad():  # no gradient wanted: the loss alone, the same value
            assert torch.equal(gs.image_loss_torch(c, gs.render_torch(c, v, u), t), passes[0][0])
        m = gs.image_metrics(c, img.detach(), t)
        assert abs(m["l1"] - ref["l1"]) <= 1e-6 * ref["l1"] and abs(m["ssim"] - ref["ssim"]) <= 1e-5
        assert abs(m["psnr"] + 10 * np.log10(ref["mse"])) <= 1e-4
    finally:
        c.close()


def test_fit_lowers_loss_and_dssim(gs):
    """Adam on position, log scale, opacity logit and SH DC of a sparse start, fitting c1's frames from three poses with
    image_loss_torch: both the loss and 1 - SSIM go down."""
    torch = _torch()
    c = gs.Context(0)
    try:
        _, vtx, _ = scenes.c1()
        full = torch.from_numpy(vtx).cuda()
        poses = [([0, 0, 5], [1, 0, 0, 0]), ([0.6, 0.1, 5.2], scenes.quat_axis_angle([0, 1, 0], 6)),
                 ([-0.5, -0.3, 4.8], scenes.quat_axis_angle([1, 0, 0], -5))]
        views = [gs.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 320, 240) for p, q in poses]
        with torch.no_grad():
            targets = [gs.render_torch(c, full, u).clone() for u in views]
        start = full[::4].clone()
        start[:, 4:7] *= 1.5
        frozen = start.clone()
        params = {"pos": start[:, 0:3].clone(), "log_scale": start[:, 4:7].log(),
                  "logit_opacity": torch.logit(start[:, 7:8].clamp(1e-6, 1 - 1e-6)), "dc": start[:, 12:15].clone()}
        lr = {"pos": 1e-3, "log_scale": 5e-3, "logit_opacity": 5e-2, "dc": 1e-2}
        for p in params.values():
            p.requires_grad_()
        opt = torch.optim.Adam([{"params": [params[k]], "lr": lr[k]} for k in lr])

        def assemble():
            return torch.cat([params["pos"], frozen[:, 3:4], params["log_scale"].exp(), torch.sigmoid(params["logit_opacity"]),
                              frozen[:, 8:12], params["dc"], frozen[:, 15:]], 1)

        def evaluate():
            with torch.no_grad():
                ms = [gs.image_metrics(c, gs.render_torch(c, assemble(), u), t) for u, t in zip(views, targets)]
            return (sum(0.8 * m["l1"] + 0.2 * (1 - m["ssim"]) for m in ms) / len(ms), sum(1 - m["ssim"] for m in ms) / len(ms))

        loss0, dssim0 = evaluate()
        for _ in range(150):
            opt.zero_grad()
            for u, t in zip(views, targets):
                gs.image_loss_torch(c, gs.render_torch(c, assemble(), u), t).backward()  # before the next frame
            opt.step()
        loss1, dssim1 = evaluate()
        print(f"fit: loss {loss0:.5f} -> {loss1:.5f}, 1 - SSIM {dssim0:.5f} -> {dssim1:.5f}")
        assert loss1 < loss0 and dssim1 < dssim0
    finally:
        c.close()
