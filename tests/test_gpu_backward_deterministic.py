"""gsb_set_backward_deterministic / render_torch under torch.use_deterministic_algorithms: with the switch on, the three
backward entries give the same output words on every call -- same frame, re-rendered frame, fresh context, another stream,
another arena capacity -- and at tile-cull levels 0, 1 and 2, and they stay within 1e-6 of the atomic path."""
import sys
from pathlib import Path

import numpy as np
import pytest

import scenes
from backward_util import CAMERA_GROUPS, DEAD, GROUPS, grad_image, rel

pytestmark = pytest.mark.gpu

# entry -> (grad_vertices, grad_uniforms, density): gsb_render_backward, gsb_render_backward_camera, gsb_render_backward_density
ENTRIES = {"plain": (True, False, False), "camera": (True, True, False), "density": (True, True, True)}


def _torch():
    import torch

    return torch


def _grad_image(u):
    return _torch().from_numpy(grad_image(u)).cuda()


def _backward(ctx, v, gi, entry, stream=None):
    """One backward of the context's last frame through `entry`; the outputs stay on the device."""
    torch = _torch()
    want_v, want_u, want_d = ENTRIES[entry]
    gv = torch.full_like(v, float("nan")) if want_v else None
    gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda") if want_u else None
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if want_d else None
    torch.cuda.synchronize()  # the outputs' fills are complete before the call, whichever stream it runs on
    ctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr() if want_v else None, stream=stream,
                        grad_uniforms_ptr=gu.data_ptr() if want_u else None, density_ptr=dens.data_ptr() if want_d else None)
    torch.cuda.synchronize()
    return {k: t for k, t in (("vertices", gv), ("uniforms", gu), ("density", dens)) if t is not None}


def _same_words(a, b):
    """Bit-for-bit equality of two output sets (compared as int32 words on the device)."""
    torch = _torch()
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k


def _frame(ctx, u, level, mode):
    ctx.set_mode(mode)
    ctx.set_tile_cull(level)
    ctx.set_backward(True)
    ctx.render_into(u, _torch().empty((u.height, u.width, 4), dtype=_torch().float32, device="cuda").data_ptr())


def _new_ctx(gs, v, deterministic=True):
    c = gs.Context(0)
    c.upload(v)
    c.set_backward(True)
    c.set_backward_deterministic(deterministic)
    return c


@pytest.fixture(scope="module")
def garden(gs):
    """bench.py's garden stand-in (5.8 M Gaussians) on the device and its first camera: per-tile lists of thousands of
    entries, far longer than one batch of the reverse walk."""
    torch = _torch()
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    v = torch.from_numpy(bench.make_scene(gs, wl)).cuda()
    yield v, bench.cameras(gs, wl)[0], 1
    del v
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def c1(gs):
    _, vtx, u = scenes.c1()
    return _torch().from_numpy(vtx).cuda(), u, 0


@pytest.mark.parametrize("mode", [0, 1], ids=["exact", "fast"])
@pytest.mark.parametrize("scene", ["c1", "garden"])
def test_repeatable_bit_for_bit(gs, request, scene, mode):
    torch = _torch()
    v, u, level = request.getfixturevalue(scene)
    gi = _grad_image(u)
    ctx = _new_ctx(gs, v)
    side = torch.cuda.Stream()
    try:
        _frame(ctx, u, level, mode)
        first = {e: _backward(ctx, v, gi, e) for e in ENTRIES}
        assert first["plain"]["vertices"].abs().max() > 0 and first["density"]["density"][:, 2].max() > 0
        for e in ENTRIES:
            for _ in range(4):  # five calls on the same frame
                _same_words(_backward(ctx, v, gi, e), first[e])
            _same_words(_backward(ctx, v, gi, e, stream=side), first[e])  # a torch side stream
        _frame(ctx, u, level, mode)  # the same camera rendered again
        for e in ENTRIES:
            _same_words(_backward(ctx, v, gi, e), first[e])
        ctx.reserve(4 * max(ctx.stats().num_instances, 1 << 20))  # a larger arena (the frame has to be rendered again)
        _frame(ctx, u, level, mode)
        for e in ENTRIES:
            _same_words(_backward(ctx, v, gi, e), first[e])
    finally:
        ctx.close()
    fresh = _new_ctx(gs, v)
    try:
        _frame(fresh, u, level, mode)
        for e in ENTRIES:
            _same_words(_backward(fresh, v, gi, e), first[e])
    finally:
        fresh.close()


def test_output_combinations(gs, c1):
    """The camera gradient does not depend on whether grad_vertices is wanted, nor the density columns on which gradient
    outputs are given."""
    torch = _torch()
    v, u, _ = c1
    gi = _grad_image(u)
    ctx = _new_ctx(gs, v)
    try:
        _frame(ctx, u, 0, 0)
        full = _backward(ctx, v, gi, "density")

        def call(fn, gv, gu, dens):
            torch.cuda.synchronize()
            ctx._ck(fn(ctx.h, v.data_ptr(), gi.data_ptr(), 0, gv, gu, dens, None) if dens is not None else
                    fn(ctx.h, v.data_ptr(), gi.data_ptr(), 0, gv, gu, None))
            torch.cuda.synchronize()

        gu = torch.empty(40, dtype=torch.float32, device="cuda")
        call(gs.lib.gsb_render_backward_camera, None, gu.data_ptr(), None)  # frozen scene
        assert torch.equal(gu.view(torch.int32), full["uniforms"].view(torch.int32))
        for with_v, with_u in ((True, False), (False, True), (True, True)):
            gv = torch.empty_like(v)
            gu = torch.empty(40, dtype=torch.float32, device="cuda")
            dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
            call(gs.lib.gsb_render_backward_density, gv.data_ptr() if with_v else None, gu.data_ptr() if with_u else None,
                 dens.data_ptr())
            assert torch.equal(dens.view(torch.int32), full["density"].view(torch.int32)), (with_v, with_u)
            if with_v:
                assert torch.equal(gv.view(torch.int32), full["vertices"].view(torch.int32))
            if with_u:
                assert torch.equal(gu.view(torch.int32), full["uniforms"].view(torch.int32))
    finally:
        ctx.close()


@pytest.mark.parametrize("cam", list(scenes.CAMERAS))
def test_levels_bit_for_bit(gs, c1, cam):
    v, _, _ = c1
    u = scenes.camera(cam)
    gi = _grad_image(u)
    ctx = _new_ctx(gs, v)
    try:
        out = []
        for level in (0, 1, 2):  # 2 falls back to 1 while recording
            _frame(ctx, u, level, 0)
            out.append(_backward(ctx, v, gi, "density"))
        for o in out[1:]:
            _same_words(o, out[0])
    finally:
        ctx.close()


@pytest.mark.parametrize("mode", [0, 1], ids=["exact", "fast"])
@pytest.mark.parametrize("scene", ["c1", "garden"])
def test_close_to_the_atomic_path(gs, request, scene, mode):
    torch = _torch()
    v, u, level = request.getfixturevalue(scene)
    gi = _grad_image(u)
    ctx = _new_ctx(gs, v)
    try:
        _frame(ctx, u, level, mode)
        det = _backward(ctx, v, gi, "density")
        ctx.set_backward_deterministic(False)
        atom = _backward(ctx, v, gi, "density")
    finally:
        ctx.close()
    for name, s in GROUPS.items():
        assert atom["vertices"][:, s].abs().max() > 0, name
        r = rel(det["vertices"][:, s], atom["vertices"][:, s])
        assert r <= 1e-6, (name, r)
    for name, s in CAMERA_GROUPS.items():
        r = rel(det["uniforms"][s], atom["uniforms"][s])
        assert r <= 1e-6, (name, r)
    assert not det["uniforms"][DEAD].any() and not atom["uniforms"][DEAD].any()
    for c in (0, 1):
        r = rel(det["density"][:, c], atom["density"][:, c])
        assert r <= 1e-6, (c, r)
    for c in (2, 3):
        assert torch.equal(det["density"][:, c], atom["density"][:, c]), c


def test_nothing_visible_and_empty_scene(gs, c1):
    torch = _torch()
    v, _, _ = c1
    u = scenes.camera("away")
    ctx = _new_ctx(gs, v)
    try:
        _frame(ctx, u, 0, 0)
        out = _backward(ctx, v, torch.ones((u.height, u.width, 4), dtype=torch.float32, device="cuda"), "density")
        assert not out["vertices"].any() and not out["uniforms"].any() and not out["density"].any()
    finally:
        ctx.close()
    empty = torch.zeros((1, 60), dtype=torch.float32, device="cuda")  # a valid pointer to n = 0 records
    ctx = gs.Context(0)
    try:
        ctx.upload(np.zeros((0, 60), np.float32))
        ctx.set_backward(True)
        ctx.set_backward_deterministic(True)
        u = scenes.camera("c1")
        _frame(ctx, u, 0, 0)
        gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda")
        ctx.render_backward(empty.data_ptr(), _grad_image(u).data_ptr(), None, grad_uniforms_ptr=gu.data_ptr())
        torch.cuda.synchronize()
        assert not gu.any()
    finally:
        ctx.close()


def test_standalone_sort_leaves_the_frame_alone(gs, c1):
    """gsb_sort_pairs32 of unrelated pairs between a recorded frame and its deterministic backward changes no output word:
    the sort keeps its own control words and pair count, so the backward still groups the frame's whole instance list."""
    torch = _torch()
    v, u, _ = c1
    gi = _grad_image(u)
    ctx = _new_ctx(gs, v)
    try:
        _frame(ctx, u, 0, 0)
        want = _backward(ctx, v, gi, "plain")
        m = ctx.stats().num_instances // 3  # well below the frame's M: no read past the arena whatever the sort does
        assert m >= 16
        keys = torch.randint(0, 1 << 16, (m,), dtype=torch.int32, device="cuda")
        vals = torch.arange(m, dtype=torch.int32, device="cuda")
        keys_tmp, vals_tmp = torch.empty_like(keys), torch.empty_like(vals)
        torch.cuda.synchronize()  # the sort runs on the context's stream
        ctx.sort_pairs32(keys.data_ptr(), vals.data_ptr(), keys_tmp.data_ptr(), vals_tmp.data_ptr(), m, 16)
        assert bool((keys[1:] >= keys[:-1]).all())
        _same_words(_backward(ctx, v, gi, "plain"), want)
    finally:
        ctx.close()


def test_switch_error_codes(gs):
    assert gs.lib.gsb_set_backward_deterministic(None, 1) == gs.ERR_INVALID
    grp = gs.Group([0, 0])
    try:
        c0 = grp.context(0)
        with pytest.raises(gs.GsbError) as ei:
            c0.set_backward_deterministic(True)
        assert ei.value.code == gs.ERR_INVALID
        assert gs.lib.gsb_last_error(c0.h).decode().startswith("gsb_set_backward_deterministic")
    finally:
        grp.close()
    ctx = gs.Context(0)
    try:
        ctx.set_backward_deterministic(True)  # before any scene or frame: fine
        ctx.set_backward_deterministic(False)
    finally:
        ctx.close()


def _torch_pass(gs, ctx, vtx, u, g):
    torch = _torch()
    v = vtx.clone().requires_grad_()
    ubo = torch.from_numpy(gs.pack_uniforms(u)).cuda().requires_grad_()
    dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
    img = gs.render_torch(ctx, v, u, ubo, density=dens)
    (img * g).sum().backward()
    torch.cuda.synchronize()
    return {"vertices": v.grad, "uniforms": ubo.grad, "density": dens}


def test_render_torch_honours_deterministic_mode(gs, c1):
    torch = _torch()
    v, u, _ = c1
    g = _grad_image(u)
    ctx = gs.Context(0)
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        try:
            a = _torch_pass(gs, ctx, v, u, g)
            b = _torch_pass(gs, ctx, v, u, g)
        finally:
            torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
        assert a["vertices"].abs().max() > 0 and a["uniforms"].abs().max() > 0
        _same_words(a, b)
        # the switch follows torch's setting: outside deterministic mode the result is the atomic path's
        c = _torch_pass(gs, ctx, v, u, g)
        want = _backward(ctx, v, g, "density")  # the same frame again: the context's switch is off now
        assert rel(c["vertices"], want["vertices"]) <= 1e-6
        assert rel(c["density"][:, :2], want["density"][:, :2]) <= 1e-6
        assert torch.equal(c["density"][:, 2:], want["density"][:, 2:])
        # and inside it, the deterministic words of gsb_render_backward_density
        ctx.set_backward_deterministic(True)
        want = _backward(ctx, v, g, "density")
        assert torch.equal(want["vertices"].view(torch.int32), a["vertices"].view(torch.int32))
        assert torch.equal(want["density"].view(torch.int32), a["density"].view(torch.int32))
    finally:
        ctx.close()
