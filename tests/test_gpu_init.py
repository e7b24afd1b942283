"""gsb_init_from_points / Context.init_from_points: every output word against numpy fp32 -- the scale column against the
exact 3-nearest-neighbour reference (tests/init_ref.py) on small and adversarial clouds, leaf and level boundaries, the
bench's 1 M clouds and the full-size garden stand-in -- reproducibility over calls, streams and contexts, the context's scene
and last frame left alone, every error code, and a scene trained from points alone that round-trips through a .ply."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

import init_ref
import scenes
from backward_util import expect, grad_image, render
from init_ref import BENCH_CLOUDS, SMALL_CLOUDS

pytestmark = pytest.mark.gpu

ENTRY = "gsb_init_from_points"
SH_C0 = np.float32(0.28209479177387814)


def _torch():
    import torch

    return torch


@pytest.fixture
def ictx(gs):
    c = gs.Context(0)
    yield c
    c.close()


def _colours(n, seed=0):
    return np.random.default_rng(seed).uniform(-0.2, 1.2, (n, 3)).astype(np.float32)  # not clamped: outside [0, 1] too


def _init(ctx, xyz, rgb, opacity=0.1):
    torch = _torch()
    out = ctx.init_from_points(torch.from_numpy(xyz).cuda(), torch.from_numpy(rgb).cuda(), opacity)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _expected_rest(xyz, rgb, opacity):
    """Every column but the scale, in numpy fp32."""
    n = xyz.shape[0]
    want = np.zeros((n, 60), np.float32)
    want[:, 0:3] = xyz
    want[:, 3] = 1.0
    want[:, 7] = np.float32(opacity)
    want[:, 8] = 1.0
    want[:, 12:15] = (rgb - np.float32(0.5)) / SH_C0
    return want


def _check(label, out, xyz, rgb, opacity=0.1, D=None):
    want = _expected_rest(xyz, rgb, opacity)
    s = init_ref.scale_from_d(init_ref.d_ref(xyz) if D is None else D)
    want[:, 4:7] = s[:, None]
    bad = (out.view(np.uint32) != want.view(np.uint32)).any(1)
    assert not bad.any(), (label, int(bad.sum()), np.flatnonzero(bad)[:10], out[bad][:3, 4], want[bad][:3, 4])


@pytest.mark.parametrize("name", list(SMALL_CLOUDS))
def test_small_clouds_bit_exact(ictx, name):
    xyz = SMALL_CLOUDS[name]()
    rgb = _colours(xyz.shape[0])
    _check(name, _init(ictx, xyz, rgb), xyz, rgb)


@pytest.mark.parametrize("n", [31, 32, 33, 1023, 1024, 1025, 32769])
def test_leaf_and_level_boundaries(ictx, n):
    for cloud in (init_ref.uniform(n, n), init_ref.heavy_tailed(n, n)):
        rgb = _colours(n, 1)
        _check(f"n={n}", _init(ictx, cloud, rgb, 0.25), cloud, rgb, 0.25)


@pytest.mark.parametrize("name", list(BENCH_CLOUDS))
def test_bench_clouds_bit_exact(ictx, name):
    xyz = BENCH_CLOUDS[name]()
    rgb = _colours(xyz.shape[0], 2)
    _check(name, _init(ictx, xyz, rgb), xyz, rgb)


def _garden_positions(gs):
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    return np.ascontiguousarray(bench.make_scene(gs, bench.WORKLOADS["garden-standin"])[:, 0:3])


def test_full_size_garden_standin(gs, ictx):
    """5.8 M points; a seeded sample of 100 k rows is checked against the tree of all of them."""
    from scipy.spatial import cKDTree

    xyz = _garden_positions(gs)
    rgb = _colours(xyz.shape[0], 3)
    out = _init(ictx, xyz, rgb)
    rows = np.sort(np.random.default_rng(0).choice(xyz.shape[0], 100_000, replace=False))
    D = init_ref.d_ref(xyz, rows, tree=cKDTree(xyz.astype(np.float64)))
    _check("garden sample", out[rows], xyz[rows], rgb[rows], D=D)


def test_uint8_colours_and_opacity(gs, ictx):
    torch = _torch()
    xyz = init_ref.uniform(5000, 4)
    rgb8 = np.random.default_rng(5).integers(0, 256, (5000, 3)).astype(np.uint8)
    c8 = torch.from_numpy(rgb8).cuda()
    out = ictx.init_from_points(torch.from_numpy(xyz).cuda(), c8, opacity=0.5).cpu().numpy()
    _check("uint8", out, xyz, (c8.to(torch.float32) / 255).cpu().numpy(), 0.5)  # v / 255 as torch computes it


def test_reproducible_over_calls_streams_and_contexts(gs, ictx):
    torch = _torch()
    xyz = init_ref.heavy_tailed(200_000, 6)
    rgb = _colours(xyz.shape[0], 6)
    x, c = torch.from_numpy(xyz).cuda(), torch.from_numpy(rgb).cuda()
    first = ictx.init_from_points(x, c)  # a context with no scene
    assert ictx.num_gaussians == 0
    runs = [ictx.init_from_points(x, c) for _ in range(3)]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        runs.append(ictx.init_from_points(x, c))
    fresh = gs.Context(0)
    try:
        runs.append(fresh.init_from_points(x, c))
    finally:
        fresh.close()
    torch.cuda.synchronize()
    for r in runs:
        assert torch.equal(r.view(torch.int32), first.view(torch.int32))


def test_leaves_scene_and_last_frame_alone(gs, ictx):
    """Deterministic backward: the gradient of the last frame, the next frame and the scene size are the same words with
    and without a gsb_init_from_points in between."""
    torch = _torch()
    _, vtx, u = scenes.c1()
    v = torch.from_numpy(vtx).cuda()
    gi = torch.from_numpy(grad_image(u)).cuda()
    xyz, rgb = torch.from_numpy(init_ref.uniform(50_000, 7)).cuda(), torch.from_numpy(_colours(50_000, 7)).cuda()
    ictx.upload(vtx)
    ictx.set_backward_deterministic(True)

    def frame_and_grad(init_between):
        render(ictx, u)
        torch.cuda.synchronize()
        if init_between:
            ictx.init_from_points(xyz, rgb)
        gv = torch.empty_like(v)
        ictx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr())
        torch.cuda.synchronize()
        return gv.cpu(), ictx.render(u)

    g0, f0 = frame_and_grad(False)
    g1, f1 = frame_and_grad(True)
    assert torch.equal(g0.view(torch.int32), g1.view(torch.int32))
    assert np.array_equal(f0.view(np.uint32), f1.view(np.uint32))
    assert ictx.num_gaussians == vtx.shape[0]


def test_error_cases(gs, ictx):
    torch = _torch()
    n = 100
    xyz = torch.from_numpy(init_ref.uniform(n, 8)).cuda()
    rgb = torch.from_numpy(_colours(n, 8)).cuda()
    out = torch.full((n, 60), 7.0, device="cuda")

    def raw(c, x=xyz, r=rgb, count=n, opacity=0.1, o=out, offset=0):
        ptr = lambda t: None if t is None else t.data_ptr() + offset
        return lambda: c._ck(gs.lib.gsb_init_from_points(c.h, ptr(x), ptr(r), count, opacity, ptr(o), None))

    assert gs.lib.gsb_init_from_points(None, xyz.data_ptr(), rgb.data_ptr(), n, 0.1, out.data_ptr(), None) == gs.ERR_INVALID
    raw(ictx, x=None, r=None, o=None, count=0)()  # n == 0: nothing to do
    for kw in ({"x": None}, {"r": None}, {"o": None}, {"offset": 2}, {"count": 1 << 30}, {"opacity": 0.0},
               {"opacity": 1.0}, {"opacity": -0.5}, {"opacity": float("nan")}):
        expect(gs, ictx, gs.ERR_INVALID, raw(ictx, **kw), ENTRY)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    for bad in (float("nan"), float("inf"), -float("inf")):
        x = xyz.clone()
        x[37, 1] = bad
        expect(gs, ictx, gs.ERR_INVALID, raw(ictx, x=x), ENTRY)
        torch.cuda.synchronize()
        assert bool((out == 7.0).all())  # nothing written
    with pytest.raises(ValueError):
        ictx.init_from_points(xyz[:, :2], rgb)
    with pytest.raises(ValueError):
        ictx.init_from_points(xyz, rgb[:-1])
    with pytest.raises(ValueError):
        ictx.init_from_points(xyz.double(), rgb)
    with pytest.raises(ValueError):
        ictx.init_from_points(xyz, rgb.to(torch.int32))
    with pytest.raises(ValueError):
        ictx.init_from_points(xyz.cpu(), rgb)
    assert ictx.init_from_points(xyz[:0], rgb[:0]).shape == (0, 60)


def test_training_from_points_and_ply_round_trip(gs, ictx, tmp_path):
    """c1's positions (every 4th Gaussian) with their DC colours, through init_from_points into SceneAdam: 300 steps on
    the three poses of test_gpu_adam.py's training set-up lower the loss and 1 - SSIM; the trained scene saved with
    write_ply(ply_records(params)) loads back as activate_records of the same records, and within 4 ulp of opt.vertices."""
    torch = _torch()
    from test_gpu_adam import TRAIN_LR, _evaluate, _training_setup

    _, views, targets = _training_setup(gs, ictx)
    _, vtx, _ = scenes.c1()
    sub = vtx[::4]
    xyz = np.ascontiguousarray(sub[:, 0:3])
    rgb = np.clip(sub[:, 12:15] * SH_C0 + np.float32(0.5), 0.0, 1.0).astype(np.float32)
    start = ictx.init_from_points(torch.from_numpy(xyz).cuda(), torch.from_numpy(rgb).cuda())
    opt = gs.SceneAdam(ictx, start, TRAIN_LR, selective=True)
    g = torch.empty((240, 320, 4), dtype=torch.float32, device="cuda")
    loss0, dssim0 = _evaluate(gs, ictx, opt, views, targets)
    for it in range(300):
        k = it % 3
        ictx.image_loss(opt.render(views[k]), targets[k], 0.2, grad_image=g)
        opt.step(g)
    loss1, dssim1 = _evaluate(gs, ictx, opt, views, targets)
    print(f"trained from {xyz.shape[0]} points: loss {loss0:.5f} -> {loss1:.5f}, 1 - SSIM {dssim0:.5f} -> {dssim1:.5f}")
    assert loss1 < loss0 and dssim1 < dssim0
    torch.cuda.synchronize()
    rec = gs.ply_records(opt.params)
    path = tmp_path / "trained.ply"
    gs.write_ply(path, rec)
    loaded = gs.load_ply(path)
    assert np.array_equal(loaded.view(np.uint32), gs.activate_records(rec).view(np.uint32))
    dev = opt.vertices.cpu().numpy()
    cols = np.r_[0:3, 4:60]
    def ordered(a):  # float32 bits as integers in the order of the values (-0 == +0)
        i = a.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)

    ulp = np.abs(ordered(loaded[:, cols]) - ordered(dev[:, cols]))
    worst = {name: int(ulp[:, [list(cols).index(c) for c in cs]].max())
             for name, cs in (("position", range(0, 3)), ("scale", range(4, 7)), ("opacity", [7]),
                              ("rotation", range(8, 12)), ("sh", range(12, 60)))}
    print(f"loaded .ply vs opt.vertices, largest deviation per column group in ulp: {worst}")
    assert max(worst.values()) <= 4, worst
