"""The references of the background colour (tests/bg_ref.py): the oracle's blend restated for its final transmittance, and
grad_ref's float64 function with the T_final * bg term.  CPU only."""
import math

import numpy as np
import pytest
import torch

import bg_ref
import edge_scene
import grad_ref
import scenes
from backward_util import grad_image

EPS = float(np.finfo(np.float32).eps)
BACKGROUNDS = [(1.0, 1.0, 1.0), (0.25, 0.5, 0.75), (-0.5, 2.0, 0.1)]


def _scene(name):
    if name == "edge":
        return edge_scene.vertices()[0], edge_scene.camera("axis")
    _, vtx, _ = scenes.c1()
    return vtx, scenes.camera(name)


def _frame(oracle, vtx, u, mode=1):
    oracle.set_exp_mode(mode)
    try:
        return oracle.render_frame(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)


def test_fmaf_and_exp_restate_the_oracle(oracle):
    """bg_ref's fmaf is correctly rounded (checked against exact rationals) and exp_shared is gso_exp_shared bit for bit."""
    from fractions import Fraction

    rng = np.random.default_rng(3)
    a, b, c = (rng.standard_normal(2000).astype(np.float32) for _ in range(3))
    got = bg_ref.fmaf(a, b, c)
    for i in range(0, 2000, 7):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        cand = [np.nextafter(got[i], np.float32(-np.inf)), got[i], np.nextafter(got[i], np.float32(np.inf))]
        err = [abs(Fraction(float(x)) - exact) for x in cand]
        assert err[1] <= min(err), i
    x = np.concatenate([-np.geomspace(1e-8, 90, 3000), [0.0, -0.0, -87.0, -87.5]]).astype(np.float32)
    want = np.array([oracle.exp_shared(float(v)) for v in x], np.float32)
    assert np.array_equal(bg_ref.exp_shared(x).view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside", "edge"])
def test_transmittance_restates_the_oracle_and_agrees_with_float64(oracle, cam):
    """The restated blend reproduces the oracle's image bit for bit (checked inside with_transmittance), so its T is the
    oracle's; T lies within fp32 bounds of grad_ref's float64 product away from the step pixels."""
    vtx, u = _scene(cam)
    f = bg_ref.with_transmittance(_frame(oracle, vtx, u), u)
    T = f["T"]
    assert (T < 1).any() and (T >= 0).all() and (T <= 1).all()
    oracle.set_exp_mode(1)
    try:
        _, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)
    if cam != "edge":  # the edge scene's saturated pixels carry T through long chains near the 1e-4 break: bit-exactness only
        T64 = bg_ref.transmittance64(vtx, u, f)
        d = np.abs(T.astype(np.float64) - T64)[~steps]
        assert d.max() <= 1e-4, d.max()
    # the background composite of the oracle's frame: bg where no entry reaches, c + T bg elsewhere
    for bg in BACKGROUNDS:
        out = bg_ref.composite(f["rgba"], T, bg)
        assert np.array_equal(out[T == 1][:, :3] - f["rgba"][T == 1][:, :3], np.broadcast_to(np.float32(bg), out[T == 1][:, :3].shape))


def test_zero_background_is_grad_ref_bit_for_bit(oracle):
    vtx, u = _scene("c1")
    f = _frame(oracle, vtx, u, 0)
    g = grad_image(u)
    plain = grad_ref.reference(vtx, u, f, g)
    zero = bg_ref.reference(vtx, u, f, (0.0, 0.0, 0.0), g)
    assert plain["image"].tobytes() == zero["image"].tobytes()
    assert plain["grad"].tobytes() == zero["grad"].tobytes()


@pytest.mark.parametrize("bg", BACKGROUNDS)
def test_float64_image_matches_the_fp32_composite(oracle, bg):
    vtx, u = _scene("c1")
    oracle.set_exp_mode(1)
    try:
        f = bg_ref.oracle_frame(vtx, oracle.cov3d(vtx), u, bg)
        _, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)
    ref = bg_ref.reference(vtx, u, f, bg)
    d = np.abs(ref["image"] - f["rgba"][..., :3].astype(np.float64))[~steps]
    assert d.max() <= 1e-4 * max(1.0, max(abs(x) for x in bg)), d.max()


def test_gradcheck_vertices_camera_and_background():
    """Finite differences of the float64 reference over a few vertices, two camera leaves and a background leaf."""
    import oracle as o

    _, vtx, _ = scenes.c1(n=300, seed=5)
    u = o.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 48, 32)
    f = o.render_frame(vtx, o.cov3d(vtx), u)
    used = np.unique(f["vals"].astype(np.int64))[:6]
    g = torch.tensor(grad_image(u)[..., :3], dtype=torch.float64)

    def loss(rows, bg, cam):
        v = torch.tensor(np.asarray(vtx, np.float64))
        v = v.index_put((torch.tensor(used),), rows)
        frame_patch, _ = bg_ref._background(bg)
        out = torch.zeros((u.height, u.width, 3), dtype=torch.float64)
        with frame_patch:
            uv, conic, op, col, _ = grad_ref.preprocess(v[torch.tensor(np.unique(f["vals"].astype(np.int64)))], u, cam)
            _, _, local = grad_ref.survivors(vtx, f)
            for tl in grad_ref.tiles(u, f, local):
                rgb = grad_ref.blend_tile(uv[tl.idx], conic[tl.idx], op[tl.idx], col[tl.idx], tl.fx, tl.fy)[0]
                out = out.index_put((torch.tensor(tl.py), torch.tensor(tl.px)), rgb)
        empty = torch.tensor(bg_ref._empty_tile_pixels(u, f))
        out = torch.where(empty[..., None], bg[None, None, :].expand_as(out), out)
        return (out * g).sum()

    rows = torch.tensor(np.asarray(vtx, np.float64)[used][:, [0, 1, 2, 7]], requires_grad=True)
    bg = torch.tensor([0.25, 0.5, 0.75], dtype=torch.float64, requires_grad=True)
    cam = grad_ref.camera_leaves(u)

    def fn(r, b, tx, ty):
        full = torch.tensor(np.asarray(vtx, np.float64)[used]).clone()
        full[:, [0, 1, 2, 7]] = r
        c = dict(cam)
        c["tan_fovx"], c["tan_fovy"] = tx, ty
        return loss(full, b, c)

    assert torch.autograd.gradcheck(fn, (rows, bg, cam["tan_fovx"], cam["tan_fovy"]), eps=1e-6, atol=1e-5, rtol=1e-4)


def test_background_gradient_is_the_sum_of_t_times_g(oracle):
    """dL/dbg of the float64 reference (autograd through the tiles plus the empty tiles' pixels) equals sum_p T g, and
    math.fsum of the oracle's fp32 T times g agrees with it to fp32 resolution."""
    vtx, u = _scene("odd_size")
    f = bg_ref.with_transmittance(_frame(oracle, vtx, u), u)
    g = grad_image(u)
    bg = torch.tensor([0.25, 0.5, 0.75], dtype=torch.float64, requires_grad=True)
    bg_ref.reference(vtx, u, f, bg, g)
    empty = bg_ref._empty_tile_pixels(u, f)
    total = bg.grad.numpy() + np.asarray(g, np.float64)[empty][:, :3].sum(0)
    T64 = bg_ref.transmittance64(vtx, u, f)
    want = bg_ref.grad_background(T64, g)
    assert np.allclose(total, want, rtol=1e-12, atol=1e-9)
    fs = np.array([math.fsum((f["T"].astype(np.float64) * np.asarray(g, np.float64)[..., c]).ravel()) for c in range(3)])
    scale = np.abs(f["T"][..., None].astype(np.float64) * np.asarray(g, np.float64)[..., :3]).sum((0, 1))
    assert (np.abs(fs - want) <= 1e-4 * scale).all(), (fs, want)
