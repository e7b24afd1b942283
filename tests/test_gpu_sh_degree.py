"""gsb_set_sh_degree through the C ABI: a frame at degree d is, bit for bit, the degree-3 frame of the scene with the bands
above d zeroed (Z_d), and so the oracle's frame of Z_d; every backward entry at degree d gives the deterministic words of Z_d
at degree 3 except the zeroed coefficients, whose gradient is 0; Adam leaves those bands as they are; render_torch and
SceneAdam follow the degree; the viewer's --sh-degree; every error code."""
import json
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import edge_scene
import scenes
import sh_degree_ref
from backward_util import GROUPS, expect, grad_image, rel

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
TRAIN_LR = [1e-3, 5e-3, 5e-2, 1e-3, 1e-2, 5e-4]


def _torch():
    import torch

    return torch


def zero_bands(vtx, d):
    z = np.array(vtx, np.float32, copy=True)
    z[:, 12 + 3 * (d + 1) ** 2:60] = 0.0
    return z


def live_cols(d):
    return 12 + 3 * (d + 1) ** 2


def _scene(name):
    if name == "edge":
        return edge_scene.vertices()[0], edge_scene.camera("axis")
    _, vtx, _ = scenes.c1()
    return vtx, scenes.camera(name)


def _oracle(oracle, vtx, u, rows=None):
    oracle.set_exp_mode(1)
    try:
        return oracle.render_frame(vtx, oracle.cov3d(vtx), u, rows=rows)
    finally:
        oracle.set_exp_mode(0)


@pytest.fixture
def sctx(gs):
    c = gs.Context(0)
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# frames
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", ["c1", "odd_size", "edge"])
def test_frames_equal_the_oracle_of_the_zeroed_scene(gs, oracle, sctx, cam):
    """Levels 0/1/2 x direct / graph replay x RGBA32F / BGRA8, recorded frames and GSB_BUF_ATTR: degree d of S is the
    oracle's frame of Z_d and the product's degree-3 frame of Z_d; degree 3, set-and-reset and a fresh context give the
    default frame."""
    vtx, u = _scene(cam)
    sctx.upload(vtx)
    plain = sctx.render(u)
    for d in (0, 1, 2):
        z = zero_bands(vtx, d)
        ref = _oracle(oracle, z, u)["rgba"]
        sctx.set_sh_degree(d)
        for level in (0, 1, 2):
            sctx.set_tile_cull(level)
            for timers in (True, False, False):
                sctx.set_timers(timers)
                assert np.array_equal(sctx.render(u), ref), (cam, d, level, timers)
            sctx.set_timers(True)
            assert np.array_equal(sctx.render(u, gs.FORMAT_BGRA8), oracle.pack_unorm8(ref, bgra=True)), (cam, d, level)
            sctx.set_backward(True)
            assert np.array_equal(sctx.render(u), ref), (cam, d, level, "recorded")
            sctx.set_backward(False)
        sctx.set_tile_cull(0)
        sctx.set_debug(True)
        sctx.render(u)
        attr = sctx.download(gs.BUF_ATTR).tobytes()
        zc = gs.Context(0)
        try:
            zc.upload(z)
            zc.set_debug(True)
            assert np.array_equal(zc.render(u), ref)
            assert zc.download(gs.BUF_ATTR).tobytes() == attr, (cam, d)
        finally:
            zc.close()
        sctx.set_debug(False)
    sctx.set_sh_degree(3)
    assert np.array_equal(sctx.render(u), plain)
    fresh = gs.Context(0)
    try:
        fresh.upload(vtx)
        assert np.array_equal(fresh.render(u), plain)
    finally:
        fresh.close()
    if cam != "edge":
        assert not np.array_equal(_oracle(oracle, zero_bands(vtx, 0), u)["rgba"], plain)  # the degree is visible


def test_bands_aa_background_and_depth(gs, oracle, sctx):
    """Bands against the oracle of Z_d; with AA and a background on, and through gsb_render_depth's (D, A): S at d equals
    Z_d at 3 under the same settings."""
    vtx, u = _scene("odd_size")
    tiles_y = (u.height + 15) // 16
    sctx.upload(vtx)
    for d in (0, 1, 2):
        z = zero_bands(vtx, d)
        sctx.set_sh_degree(d)
        for rows in ((0, 1), (tiles_y // 2, tiles_y // 2 + 2), (tiles_y - 1, tiles_y)):
            sl = slice(rows[0] * 16, min(u.height, rows[1] * 16))
            assert np.array_equal(sctx.render(u, rows=rows), _oracle(oracle, z, u, rows=rows)["rgba"][sl]), (d, rows)
    zc = gs.Context(0)
    try:
        for c in (sctx, zc):
            c.set_antialiased(True)
            c.set_background((0.25, 0.5, 0.75))
        for d in (0, 1, 2):
            sctx.upload(vtx)
            sctx.set_sh_degree(d)
            zc.upload(zero_bands(vtx, d))
            a, b = sctx.render_depth(u), zc.render_depth(u)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), d
    finally:
        zc.close()


def _lenses(gs, u):
    f = 0.35 * u.width
    return {"fisheye": gs.fisheye_camera(f, f, (u.width - 1) / 2.0, (u.height - 1) / 2.0, (0.05, -0.01, 0.002, 0.0),
                                         max_theta=math.pi / 2),
            "opencv": gs.opencv_camera(1.2 * f, 1.2 * f, (u.width - 1) / 2.0 + 3.0, (u.height - 1) / 2.0 - 2.0,
                                       (-0.1, 0.02, 0.001, -0.001))}


@pytest.mark.parametrize("lens", ["fisheye", "opencv"])
def test_lens_frames_equal_the_zeroed_scene(gs, sctx, lens):
    vtx, u = _scene("c1")
    zc = gs.Context(0)
    try:
        for c in (sctx, zc):
            c.set_camera_model(_lenses(gs, u)[lens])
        sctx.upload(vtx)
        for d in (0, 1, 2):
            sctx.set_sh_degree(d)
            zc.upload(zero_bands(vtx, d))
            for level in (0, 1):
                for c in (sctx, zc):
                    c.set_tile_cull(level)
                a = sctx.render(u)
                assert np.array_equal(a, zc.render(u)), (lens, d, level)
                assert np.array_equal(sctx.render(u, gs.FORMAT_BGRA8), zc.render(u, gs.FORMAT_BGRA8)), (lens, d, level)
    finally:
        zc.close()


def test_fp16_storage_equals_the_zeroed_scene(gs, sctx):
    vtx, u = _scene("odd_size")
    zc = gs.Context(0)
    try:
        for c in (sctx, zc):
            c.set_sh_storage(True)
        sctx.upload(vtx)
        for d in (0, 1, 2):
            sctx.set_sh_degree(d)
            zc.upload(zero_bands(vtx, d))
            assert np.array_equal(sctx.render(u), zc.render(u)), d
    finally:
        zc.close()


def test_fullsize_garden_bands(gs, oracle):
    """The 5.8 M garden stand-in at degrees 0 and 1, three bands of tile rows against the oracle of Z_d."""
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    vtx = bench.make_scene(gs, wl)
    u = bench.cameras(gs, wl)[3]
    tiles_y = (u.height + 15) // 16
    c = gs.Context(0)
    try:
        c.upload(vtx)
        cov = oracle.cov3d(vtx)  # the covariances do not depend on the SH
        for d in (0, 1):
            z = zero_bands(vtx, d)
            c.set_sh_degree(d)
            for rows in ((0, 1), (tiles_y // 2, tiles_y // 2 + 1), (tiles_y - 1, tiles_y)):
                sl = slice(rows[0] * 16, min(u.height, rows[1] * 16))
                oracle.set_exp_mode(1)
                try:
                    ref = oracle.render_frame(z, cov, u, rows=rows)["rgba"][sl]
                finally:
                    oracle.set_exp_mode(0)
                assert np.array_equal(c.render(u, rows=rows), ref), (d, rows)
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# gradients
# ---------------------------------------------------------------------------------------------------------------------
ENTRIES = ["plain", "camera", "density", "depth", "features", "fisheye", "opencv"]


def _grads(gs, vtx, u, g, d, entry, deterministic=True, flip_to=None):
    """One frame of vtx at degree d on a fresh context and the backward entry's outputs, as host arrays by name."""
    torch = _torch()
    c = gs.Context(0)
    try:
        if entry in ("fisheye", "opencv"):
            c.set_camera_model(_lenses(gs, u)[entry])
        c.upload(vtx)
        c.set_backward(True)
        c.set_backward_deterministic(deterministic)
        c.set_sh_degree(d)
        v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
        gi = torch.from_numpy(g).cuda()
        gv = torch.full_like(v, float("nan"))
        out = {"grad": gv}
        feats = None
        if entry == "depth":
            c.render_depth(u)
        else:
            c.render(u)
        if entry == "features":
            feats = torch.from_numpy(np.random.default_rng(3).standard_normal((v.shape[0], 5)).astype(np.float32)).cuda()
            c.render_features(feats)
        if flip_to is not None:
            c.set_sh_degree(flip_to)
        s = gs._torch_stream_arg(torch.cuda.current_stream())
        if entry == "plain":
            c.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr())
        elif entry == "camera":
            gu = out["ubo"] = torch.zeros(40, dtype=torch.float32, device="cuda")
            c.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), grad_uniforms_ptr=gu.data_ptr())
        elif entry == "density":
            dens = out["density"] = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
            c.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), density_ptr=dens.data_ptr())
        elif entry == "depth":
            gda = torch.from_numpy(np.random.default_rng(4).standard_normal((u.height, u.width, 2)).astype(np.float32)).cuda()
            gu = out["ubo"] = torch.zeros(40, dtype=torch.float32, device="cuda")
            c._backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), s, grad_uniforms_ptr=gu.data_ptr(),
                        grad_depth_alpha_ptr=gda.data_ptr())
        elif entry == "features":
            gfm = torch.from_numpy(np.random.default_rng(5).standard_normal((u.height, u.width, 5)).astype(np.float32)).cuda()
            gf = out["features"] = torch.zeros_like(feats)
            gu = out["ubo"] = torch.zeros(40, dtype=torch.float32, device="cuda")
            c.render_backward_features(v.data_ptr(), feats, gfm, grad_vertices_ptr=gv.data_ptr(), grad_features_ptr=gf.data_ptr(),
                                       grad_image_ptr=gi.data_ptr(), grad_uniforms_ptr=gu.data_ptr())
        else:
            gu = out["ubo"] = torch.zeros(40, dtype=torch.float32, device="cuda")
            gl = out["lens"] = torch.zeros(10, dtype=torch.float32, device="cuda")
            dens = out["density"] = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda")
            c._backward_fisheye(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), s, grad_uniforms_ptr=gu.data_ptr(),
                                grad_lens_ptr=gl.data_ptr(), density_ptr=dens.data_ptr())
        torch.cuda.synchronize()
        return {k: t.cpu().numpy() for k, t in out.items()}
    finally:
        c.close()


def _words(a):
    return (np.asarray(a, np.float32) + np.float32(0.0)).tobytes()  # -0 -> +0


@pytest.mark.parametrize("entry", ENTRIES)
def test_deterministic_words_equal_the_zeroed_scene(gs, entry):
    vtx, u = _scene("c1")
    g = grad_image(u)
    for d in (0, 1, 2):
        z = zero_bands(vtx, d)
        got = _grads(gs, vtx, u, g, d, entry)
        want = _grads(gs, z, u, g, 3, entry)
        k = live_cols(d)
        assert np.isfinite(got["grad"]).all()
        assert _words(got["grad"][:, :k]) == _words(want["grad"][:, :k]), (entry, d)
        assert not got["grad"][:, k:].any(), (entry, d)
        assert np.abs(want["grad"][:, k:]).max() > 0, (entry, d)
        for name in got:
            if name != "grad":
                assert _words(got[name]) == _words(want[name]), (entry, d, name)


def test_backward_follows_the_recorded_degree(gs):
    vtx, u = _scene("c1")
    g = grad_image(u)
    for entry in ("camera", "opencv"):
        for d, flip in ((0, 3), (1, 0), (3, 2)):
            a = _grads(gs, vtx, u, g, d, entry)
            b = _grads(gs, vtx, u, g, d, entry, flip_to=flip)
            assert all(a[k].tobytes() == b[k].tobytes() for k in a), (entry, d, flip)


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_atomic_gradient_matches_float64_reference(gs, oracle, cam):
    vtx, u = _scene(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    for d in (0, 1, 2):
        ref = sh_degree_ref.reference(vtx, u, frame, g, sh_degree=d)
        keep = ~ref["exclude"]
        assert keep.sum() > 100
        gv = _grads(gs, vtx, u, g, d, "plain", deterministic=False)["grad"]
        k = live_cols(d)
        assert not gv[:, k:].any()
        for name, cols in GROUPS.items():
            if name == "sh_rest":
                cols = slice(15, k)
                if k == 15:
                    continue
            r = rel(gv[keep, cols].astype(np.float64), ref["grad"][keep, cols])
            assert r <= 1e-3, (cam, d, name, r)


# ---------------------------------------------------------------------------------------------------------------------
# Adam, render_torch, SceneAdam
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("selective", [False, True])
def test_adam_step_leaves_the_dropped_bands(gs, sctx, selective):
    torch = _torch()
    vtx, u = _scene("c1")
    for d in (0, 1, 2):
        v = torch.from_numpy(vtx).cuda()
        opt = gs.SceneAdam(sctx, v, TRAIN_LR, selective=selective, sh_degree=d)
        p0 = opt.params.clone()
        img = opt.render(u)
        gi = torch.from_numpy(grad_image(u)).cuda()
        opt.step(gi)
        torch.cuda.synchronize()
        k = live_cols(d)
        assert opt.params[:, k:].cpu().numpy().tobytes() == p0[:, k:].cpu().numpy().tobytes(), (selective, d)
        assert not opt.exp_avg[:, k:].any() and not opt.exp_avg_sq[:, k:].any()
        assert opt.vertices[:, k:].cpu().numpy().tobytes() == v[:, k:].cpu().numpy().tobytes()
        assert not torch.equal(opt.params[:, 12:k], p0[:, 12:k])  # the live bands move
        # the resident scene is an upload of the records
        resident = sctx.render(u)
        fresh = gs.Context(0)
        try:
            fresh.upload(opt.vertices.cpu().numpy())
            fresh.set_sh_degree(d)
            assert np.array_equal(resident, fresh.render(u)), (selective, d)
        finally:
            fresh.close()
        assert img.shape == (u.height, u.width, 4)


def test_render_torch_gradients_and_restore(gs, sctx):
    torch = _torch()
    vtx, u = _scene("c1")
    g = grad_image(u)
    for d in (0, 1, 2):
        sctx.set_sh_degree(3)
        runs = []
        with torch.enable_grad():
            torch.use_deterministic_algorithms(True)
            try:
                for _ in range(2):
                    v = torch.from_numpy(vtx).cuda().requires_grad_()
                    img = gs.render_torch(sctx, v, u, sh_degree=d)
                    (img * torch.from_numpy(g).cuda()).sum().backward()
                    runs.append(v.grad.cpu().numpy())
            finally:
                torch.use_deterministic_algorithms(False)
        assert sctx.sh_degree == 3
        assert np.array_equal(sctx.render(u), _oracle_free_frame(gs, vtx, u))  # the context is back at degree 3
        assert runs[0].tobytes() == runs[1].tobytes()
        want = _grads(gs, vtx, u, g, d, "plain")["grad"]
        assert runs[0].tobytes() == want.tobytes(), d
        # None uses the context's setting
        sctx.set_sh_degree(d)
        v = torch.from_numpy(vtx).cuda().requires_grad_()
        img = gs.render_torch(sctx, v, u)
        assert np.array_equal(img.detach().cpu().numpy(), _oracle_free_frame(gs, zero_bands(vtx, d), u))


def _oracle_free_frame(gs, vtx, u):
    c = gs.Context(0)
    try:
        c.upload(vtx)
        return c.render(u)
    finally:
        c.close()


def test_scene_adam_degree_schedule(gs, sctx):
    """sh_degree = min(it // K, 3) on c1's views: the loss falls, and each band is bit-identical to its start until its
    degree arrives and moves after."""
    torch = _torch()
    _, vtx, _ = scenes.c1()
    views = [gs.uniforms_from_camera([dx, dy, 5.0], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 160, 120)
             for dx, dy in ((0.0, 0.0), (0.4, 0.0), (0.0, 0.4), (-0.4, -0.2))]
    tgt = gs.Context(0)
    try:
        tgt.upload(vtx)
        targets = [torch.from_numpy(tgt.render(w)).cuda() for w in views]
    finally:
        tgt.close()
    start = vtx.copy()
    start[:, 0:3] += np.random.default_rng(1).normal(0.0, 0.05, (vtx.shape[0], 3)).astype(np.float32)
    start[:, 12:60] *= 0.5
    opt = gs.SceneAdam(sctx, torch.from_numpy(start).cuda(), TRAIN_LR, selective=False)
    p0 = opt.params.clone()
    K = 10
    bands = {1: slice(15, 24), 2: slice(24, 39), 3: slice(39, 60)}
    losses = []
    for it in range(4 * K):
        opt.sh_degree = min(it // K, 3)
        w = it % len(views)
        img = opt.render(views[w])
        gi = torch.empty_like(img)
        losses.append(float(sctx.image_loss(img, targets[w], 0.2, grad_image=gi)[0]))
        opt.step(gi)
        torch.cuda.synchronize()
        for b, cols in bands.items():
            same = torch.equal(opt.params[:, cols], p0[:, cols])
            assert same == (opt.sh_degree < b), (it, b)
    assert np.mean(losses[-4:]) < np.mean(losses[:4]), losses


# ---------------------------------------------------------------------------------------------------------------------
# errors and the viewer
# ---------------------------------------------------------------------------------------------------------------------
def test_error_cases(gs, sctx):
    lib = gs.lib
    assert lib.gsb_set_sh_degree(None, 1) == gs.ERR_INVALID
    for bad in (-1, 4):
        assert lib.gsb_set_sh_degree(sctx.h, bad) == gs.ERR_INVALID
        assert gs.lib.gsb_last_error(sctx.h).decode().startswith("gsb_set_sh_degree")
        with pytest.raises(ValueError):
            sctx.set_sh_degree(bad)
    with pytest.raises(ValueError):
        sctx.set_sh_degree(1.5)
    for ok in (0, 1, 2, 3):
        assert lib.gsb_set_sh_degree(sctx.h, ok) == gs.OK
    sc = gs.ShardedContext(0, 0, 1, gs.shard_unique_id())
    try:
        expect(gs, sc, gs.ERR_INVALID, lambda: sc.set_sh_degree(1), "gsb_set_sh_degree")
        assert lib.gsb_set_sh_degree(sc.h, 3) == gs.ERR_INVALID
    finally:
        sc.close()
    grp = gs.Group([0])
    try:
        r0 = grp.context(0)
        expect(gs, r0, gs.ERR_INVALID, lambda: r0.set_sh_degree(0), "gsb_set_sh_degree")
    finally:
        grp.close()


def test_headless_viewer_sh_degree(gs, tmp_path):
    exe = ROOT / "3dgs.cpp_b200" / "gs_viewer_headless"
    rec = gs.synth_records(42, 10_000)
    ply = tmp_path / "c1.ply"
    gs.write_ply(ply, rec)
    pfm = tmp_path / "frame.pfm"
    r = subprocess.run([str(exe), "-w", "640", "-h", "480", "--camera", "0,0,5", "--sh-degree", "1", "--float-out", str(pfm), str(ply)],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert json.loads(r.stdout.strip().splitlines()[-1])["gaussians"] == 10_000
    blob = pfm.read_bytes()
    head = b"PF\n640 480\n-1.0\n"
    assert blob.startswith(head)
    img = np.frombuffer(blob[len(head):], "<f4").reshape(480, 640, 3)[::-1]
    u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 640, 480)
    want = _oracle_free_frame(gs, zero_bands(gs.activate_records(rec), 1), u)
    assert np.array_equal(img, want[..., :3])
    bad = subprocess.run([str(exe), "--sh-degree", "4", str(ply)], capture_output=True, text=True, timeout=120)
    assert bad.returncode != 0
