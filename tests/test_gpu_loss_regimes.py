"""gsb_image_loss against the float64 reference (tests/loss_ref.py) on the frames training produces rather than uniform
noise: flat regions at the values of sky, backgrounds and saturated areas, whole-frame and inside noise, exact and with
1e-3 / 1e-4 noise; values outside [0, 1]; rendered frames of the edge, stress and scale scenes; sizes around the 11-tap
window and the 32 x 16 tile, 1 x N and N x 1 strips; padded pitches and RGBA8 targets; and the full-size garden stand-in
with a flat sky band.  Besides the whole-frame tolerances of tests/test_gpu_loss.py every gradient value is checked:
|g - g_ref| <= 2e-4 max |g_ref|.  The kernels are also pinned to the numpy model of their arithmetic (tests/loss_model.py).

In fp32, sigma^2 = E[x^2] - mu^2 over a flat window leaves a rounding residue of one sign that C2 = 9e-4 magnifies; the
flat-region cases here fail by up to 6e-5 in SSIM with moments accumulated in fp32."""
import sys
from pathlib import Path

import numpy as np
import pytest

import edge_scene
import loss_model
import loss_ref
import scale_scene
import stress_scene
from backward_util import rel

pytestmark = pytest.mark.gpu

LAM = 0.2
FLAT_PAIRS = [(0.0, 0.02), (0.02, 0.0), (0.93, 0.95), (1.0, 0.99), (0.7, 0.72), (1.0, 1.0)]  # x vs y
FLAT_NOISE = [0.0, 1e-3, 1e-4]
FLAT_W, FLAT_H = 128, 96
GEOMETRY = [5, 6, 10, 11, 12, 31, 32, 33, 47, 48, 49]  # around the 11-tap window and the 32 x 16 tile
STRIPS = [1, 2, 7, 11, 31, 33, 100, 517, 1000]
PIXEL_TOL = 2e-4  # of max |g_ref|, on every RGB value


def _torch():
    import torch

    return torch


# ---- inputs: (H, W, 4) float32 image and target; the A channel holds values the loss must ignore


def _frame(rng, w, h, lo=0.0, hi=1.0):
    x = rng.uniform(lo, hi, (h, w, 4)).astype(np.float32)
    x[..., 3] = rng.uniform(-5, 5, (h, w)).astype(np.float32)
    return x


def flat_case(a, b, noise, where, seed=0):
    """x = a and y = b over the whole frame ("frame") or over a block that crosses tile seams inside uniform noise
    ("region"), each plus its own uniform noise of amplitude `noise` on the flat part."""
    rng = np.random.default_rng(seed)
    x, y = _frame(rng, FLAT_W, FLAT_H), _frame(rng, FLAT_W, FLAT_H)
    sel = (slice(None), slice(None)) if where == "frame" else (slice(13, 77), slice(21, 107))
    shape = x[sel][..., :3].shape
    x[sel + (slice(0, 3),)] = (a + noise * rng.uniform(-1, 1, shape)).astype(np.float32)
    y[sel + (slice(0, 3),)] = (b + noise * rng.uniform(-1, 1, shape)).astype(np.float32)
    return x, y


def out_of_range_case(kind, seed=0):
    """Values a render leaves [0, 1] with: uniform in [-0.3, 2.5] ("wide"), near-flat at 1.8 over the whole frame
    ("near_flat_1.8": 1.85 +- 1e-3 vs 1.8 +- 1e-3), or a flat 1.8 block inside the wide noise ("flat_1.8_in_wide")."""
    rng = np.random.default_rng(seed)
    x, y = _frame(rng, FLAT_W, FLAT_H, -0.3, 2.5), _frame(rng, FLAT_W, FLAT_H, -0.3, 2.5)
    if kind == "near_flat_1.8":
        x[..., :3] = (1.85 + 1e-3 * rng.uniform(-1, 1, x[..., :3].shape)).astype(np.float32)
        y[..., :3] = (1.8 + 1e-3 * rng.uniform(-1, 1, y[..., :3].shape)).astype(np.float32)
    elif kind == "flat_1.8_in_wide":
        x[20:70, 10:90, :3], y[20:70, 10:90, :3] = 1.8, 1.81
    return x, y


def mixed_case(w, h, seed=0):
    """Uniform noise with a flat 0.93 vs 0.95 left half and a flat 1 vs 0.99 top third: flat regions that meet the noise
    and each other at every tile seam the frame has."""
    rng = np.random.default_rng(seed)
    x, y = _frame(rng, w, h), _frame(rng, w, h)
    x[:, : (w + 1) // 2, :3], y[:, : (w + 1) // 2, :3] = 0.93, 0.95
    x[: (h + 2) // 3, :, :3], y[: (h + 2) // 3, :, :3] = 1.0, 0.99
    return x, y


# ---- running and checking


@pytest.fixture(scope="module")
def lctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def run(lctx, image, target, lam=LAM, pads=(0, 0, 0)):
    """gsb_image_loss of host or device (H, W, 4) arrays, with (image, target, grad) rows padded by `pads` pixels:
    (loss, L1, SSIM, MSE) as floats and the gradient as an (H, W, 4) float64 array."""
    torch = _torch()
    x, y = torch.as_tensor(image).cuda(), torch.as_tensor(target).cuda()
    h, w = x.shape[:2]

    def padded(t, p, fill):
        if p == 0:
            return t
        out = torch.full((h, w + p, 4), fill, dtype=t.dtype, device="cuda")[:, :w]
        out.copy_(t)
        return out

    x, y = padded(x, pads[0], 7.0), padded(y, pads[1], 200 if y.dtype == torch.uint8 else -7.0)
    g = padded(torch.full((h, w, 4), float("nan"), device="cuda"), pads[2], float("nan"))
    r = lctx.image_loss(x, y, lam, g)
    torch.cuda.synchronize()
    return [float(v) for v in r.cpu()], g.cpu().numpy().astype(np.float64)


def check(got, grad, ref, what=""):
    """The tolerances of tests/test_gpu_loss.py (L1, MSE <= 1e-6 relative; SSIM, loss <= 1e-5; gradient <= 1e-4 relative
    L2) and on every RGB value |g - g_ref| <= 2e-4 max |g_ref| + 1e-12 / N.  The 1e-12 / N only matters where x == y
    everywhere: there the reference's gradient is 0 up to float64 rounding (S has its maximum at x = y).  Returns the
    deviations."""
    loss, l1, ssim, mse = got
    g, r = grad[..., :3], ref["grad"][..., :3]
    n = r.size
    dev = {"l1": abs(l1 - ref["l1"]), "mse": abs(mse - ref["mse"]), "ssim": abs(ssim - ref["ssim"]),
           "loss": abs(loss - ref["loss"]), "grad_linf": float(np.abs(g - r).max() / max(np.abs(r).max(), 1e-300))}
    assert dev["l1"] <= 1e-6 * ref["l1"], (what, dev)
    assert dev["mse"] <= 1e-6 * ref["mse"], (what, dev)
    assert dev["ssim"] <= 1e-5 and dev["loss"] <= 1e-5, (what, dev, ssim, ref["ssim"])
    assert np.all(grad[..., 3] == 0), what
    assert np.all(np.abs(g - r) <= PIXEL_TOL * np.abs(r).max() + 1e-12 / n), (what, dev)
    if np.abs(r).max() > 1e-9 / n:
        dev["grad_rel_l2"] = rel(g, r)
        assert dev["grad_rel_l2"] <= 1e-4, (what, dev)
    return dev


def run_and_check(lctx, image, target, what="", device="cpu", lam=LAM, pads=(0, 0, 0)):
    got, grad = run(lctx, image, target, lam, pads)
    return check(got, grad, loss_ref.reference(image, target, lam, device=device), what)


# ---- flat regions, values outside [0, 1]


@pytest.mark.parametrize("where", ["frame", "region"])
@pytest.mark.parametrize("noise", FLAT_NOISE, ids=["exact", "noise1e-3", "noise1e-4"])
@pytest.mark.parametrize("pair", FLAT_PAIRS, ids=[f"{a}_vs_{b}" for a, b in FLAT_PAIRS])
def test_flat_regions(lctx, pair, noise, where):
    x, y = flat_case(*pair, noise, where)
    dev = run_and_check(lctx, x, y, (pair, noise, where))
    print(f"{pair} noise {noise} {where}: {dev}")


@pytest.mark.parametrize("kind", ["wide", "near_flat_1.8", "flat_1.8_in_wide"])
def test_out_of_range_values(lctx, kind):
    x, y = out_of_range_case(kind)
    for lam in (0.2, 1.0):
        dev = run_and_check(lctx, x, y, (kind, lam), lam=lam)
        print(f"{kind} lambda {lam}: {dev}")


# ---- rendered frames: black backgrounds, saturated colours, negative G / B, huge flat footprints

# name -> (scene module, its camera's pose as (pos, quat, fov), W, H); the scale scene uses the edge scene's cameras
RENDERED = {"edge_axis": (edge_scene, edge_scene.CAMERA_POSES["axis"][:3], 1280, 720),
            "stress_odd": (stress_scene, stress_scene.CAMERA_POSES["odd_size_near"][:3], 333, 217),
            "scale_axis": (scale_scene, edge_scene.CAMERA_POSES["axis"][:3], 160, 120),
            "scale_rotated": (scale_scene, edge_scene.CAMERA_POSES["rotated_odd"][:3], 333, 217)}


def _scene_vertices(mod):
    v = mod.vertices()
    return v[0] if isinstance(v, tuple) else v


@pytest.fixture(scope="module")
def rendered(gs):
    """name -> (frame, frame from a nearby pose, frame of a perturbed-SH copy), host arrays."""
    out = {}
    c = gs.Context(0)
    try:
        for name, (mod, (pos, q, fov), w, h) in RENDERED.items():
            vtx = _scene_vertices(mod)
            u = gs.uniforms_from_camera(pos, q, fov, 0.1, 1000.0, w, h)
            near = gs.uniforms_from_camera(np.asarray(pos, np.float64) + [0.01, -0.006, 0.004], q, fov, 0.1, 1000.0, w, h)
            c.upload(vtx)
            a, b = c.render(u), c.render(near)
            sh = vtx.copy()
            sh[:, 12:60] += (0.05 * np.random.default_rng(3).standard_normal(sh[:, 12:60].shape)).astype(np.float32)
            c.upload(sh)
            out[name] = (a, b, c.render(u))
    finally:
        c.close()
    return out


@pytest.mark.parametrize("target", ["nearby_pose", "perturbed_sh"])
@pytest.mark.parametrize("name", list(RENDERED))
def test_rendered_frames(lctx, rendered, name, target):
    a, b, s = rendered[name]
    t = b if target == "nearby_pose" else s
    rgb = a[..., :3]
    assert np.abs(a - t)[..., :3].max() > 0.01
    print(f"{name}: {np.mean(rgb == 0):.2f} of values 0, {np.mean(rgb > 1):.3f} above 1, {np.mean(rgb < 0):.3f} below 0")
    dev = run_and_check(lctx, a, t, (name, target), device="cuda")
    print(f"{name} vs {target}: {dev}")


# ---- geometry: sizes around the window and the tile, strips, pitches, RGBA8


@pytest.mark.parametrize("w", GEOMETRY)
def test_sizes_around_window_and_tile(lctx, w):
    for h in GEOMETRY:
        x, y = mixed_case(w, h, seed=w * 100 + h)
        run_and_check(lctx, x, y, (w, h))


@pytest.mark.parametrize("n", STRIPS)
def test_strips(lctx, n):
    for w, h in ((n, 1), (1, n)):
        x, y = mixed_case(w, h, seed=n)
        run_and_check(lctx, x, y, (w, h))


@pytest.mark.parametrize("pads", [(1, 0, 0), (0, 3, 0), (0, 0, 2), (5, 2, 7)], ids=lambda p: "pad_%d_%d_%d" % p)
def test_padded_pitches(lctx, pads):
    """Padded rows against the reference, and word for word against the tight call."""
    x, y = mixed_case(333, 217, seed=5)
    got, grad = run(lctx, x, y, pads=pads)
    check(got, grad, loss_ref.reference(x, y, LAM))
    tight = run(lctx, x, y)
    assert got == tight[0] and np.array_equal(grad, tight[1])


@pytest.mark.parametrize("pad", [0, 1, 6])
def test_rgba8_targets(lctx, pad):
    """A UNORM8 target with flat regions (237 / 255 ~ 0.93, 255 and 0) and a near-equal image, tight and padded."""
    rng = np.random.default_rng(11)
    w, h = 333, 217
    x = _frame(rng, w, h)
    t = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    t[:80, :200, :3], x[:80, :200, :3] = 237, 0.95
    t[80:, 100:250, :3], x[80:, 100:250, :3] = 255, np.float32(0.99)
    t[150:, :60, :3] = 0
    x[150:, :60, :3] = (0.02 + 1e-3 * rng.uniform(-1, 1, x[150:, :60, :3].shape)).astype(np.float32)
    got, grad = run(lctx, x, t, pads=(0, pad, 0))
    dev = check(got, grad, loss_ref.reference(x, t, LAM), ("rgba8", pad))
    print(f"rgba8 pad {pad}: {dev}")


# ---- the kernels against the model of their arithmetic


@pytest.mark.parametrize("case", ["flat_0.93_region", "near_flat_1.8", "mixed_333x217", "wide"])
def test_kernels_match_the_model(lctx, case):
    """Result words within 1e-12 and every gradient value within 2^-20 max |g| (16 float32 ulp at the largest value) of
    tests/loss_model.py, which runs the same formulas in float64 with A, B, C rounded to float32 as the kernels store them:
    only the order of the float64 sums differs."""
    x, y = {"flat_0.93_region": lambda: flat_case(0.93, 0.95, 1e-4, "region"),
            "near_flat_1.8": lambda: out_of_range_case("near_flat_1.8"),
            "mixed_333x217": lambda: mixed_case(333, 217, seed=9),
            "wide": lambda: out_of_range_case("wide")}[case]()
    got, grad = run(lctx, x, y)
    m = loss_model.model(x, y, LAM)
    for k, v in zip(("loss", "l1", "ssim", "mse"), got):
        assert abs(v - m[k]) <= 1e-12, (case, k, v, m[k])
    worst = float(np.abs(grad - m["grad"]).max() / np.abs(m["grad"]).max())
    print(f"{case}: kernel vs model, largest gradient deviation {worst:.3g} of max |g|")
    assert worst <= 2.0 ** -20, (case, worst)


# ---- full size


@pytest.fixture(scope="module")
def garden_with_sky(gs):
    """bench.py's garden stand-in (3200 x 1400) from its first two cameras, with a flat synthetic sky band over the top
    300 rows: 0.93 +- 1e-4 in the frame vs 0.95 in the target."""
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
    gen = torch.Generator(device="cuda").manual_seed(0)
    a, b = out
    a[:300, :, :3] = 0.93 + 1e-4 * (2 * torch.rand(a[:300, :, :3].shape, generator=gen, device="cuda") - 1)
    b[:300, :, :3] = 0.95
    yield a, b
    torch.cuda.empty_cache()


def test_full_size_with_sky(lctx, garden_with_sky):
    a, b = garden_with_sky
    dev = run_and_check(lctx, a, b, "garden 3200x1400 with sky", device="cuda")
    print(f"garden 3200x1400 with a flat sky band: {dev}")
