"""The backward pass against the float64 references where the reverse walk is most likely to go wrong, and which scenes.c1()
never reaches: the stress scene of tests/stress_scene.py (per-tile lists of ~1 000 entries walked over several batches,
pixels that break deep in their list, alpha clamped at 0.99, red clamped at 0, the 1.3 tan_fov clamp; test_stress_coverage.py
pins that it reaches them) and a band of tile rows of the full-size garden stand-in.

Every comparison is per Gaussian as well as per group: for each Gaussian i the reference keeps and each group,
||got_i - ref_i|| <= RTOL ||ref_i|| + ATOL_FRAC * (99th percentile of ||ref_j|| over the Gaussians with a gradient), so an
error confined to a few dozen Gaussians cannot hide under the norm of the whole frame."""
import functools
import sys
from pathlib import Path

import numpy as np
import pytest

import grad_ref
import stress_scene
from backward_util import CAMERA_GROUPS, DEAD, GROUPS, grad_image, rel

pytestmark = pytest.mark.gpu

# Measured on an H100 80GB HBM3 (700 W limit), over all Gaussians of both paths and levels: the largest ||got_i - ref_i|| is
# 3.3e-4 ||ref_i|| among the rows above a tenth of the 99th percentile, and 2.1e-4 x the 99th percentile among all rows
# (the stress scene's position and scale, the garden band's density column 0).  With these two the largest
# error / tolerance is 0.068: 15x headroom.
RTOL = 1e-3
ATOL_FRAC = 1e-3
PATHS = {"atomic": False, "deterministic": True}
BAND_ROWS = 1  # tile rows of the garden stand-in's band, in the middle of the frame


def _torch():
    import torch

    return torch


def _atol(ref, rows, cols):
    """ATOL_FRAC x the 99th percentile of the per-Gaussian norms of ref[:, cols] over the rows whose norm is non-zero."""
    r = np.linalg.norm(ref[rows][:, cols].reshape(int(rows.sum()), -1), axis=1)
    return ATOL_FRAC * float(np.percentile(r[r > 0], 99))


def _row_ratio(got, ref, rows, cols, atol):
    """max over the Gaussians `rows` of ||got_i - ref_i|| / (RTOL ||ref_i|| + atol): the check holds where it is <= 1."""
    k = int(rows.sum())
    r = np.linalg.norm(ref[rows][:, cols].reshape(k, -1), axis=1)
    d = np.linalg.norm((got[rows][:, cols] - ref[rows][:, cols]).reshape(k, -1), axis=1)
    return float((d / (RTOL * r + atol)).max()) if k else 0.0


def _check_vertices(got, ref, keep, sets, what, set_atol=False, min_rows=10):
    """The per-group norm check over `keep` at 1e-3, the per-Gaussian check over `keep`, and both again over each named
    subset of `keep` in `sets` (name -> bool mask), each of which must hold min_rows Gaussians with a gradient.  The per-Gaussian
    check's absolute tolerance comes from the rows of `keep`, or with set_atol=True from each set's own rows: a set whose
    gradients are all far below the others' (sub-pixel or huge Gaussians) is then held to its own scale."""
    assert np.isfinite(got).all(), what
    assert not got[:, 3].any(), what  # position.w
    worst = {}
    for name, cols in GROUPS.items():
        atol = _atol(ref, keep, cols)
        r = rel(got[keep, cols], ref[keep, cols])
        assert r <= 1e-3, (what, name, r)
        worst[name] = _row_ratio(got, ref, keep, cols, atol)
        for sname, rows in sets.items():
            live = np.linalg.norm(ref[rows][:, cols]) > 0
            if live:
                rs = rel(got[rows][:, cols], ref[rows][:, cols])
                assert rs <= 1e-3, (what, sname, name, rs)
            tol = _atol(ref, rows, cols) if set_atol and live else atol
            worst[f"{sname}/{name}"] = _row_ratio(got, ref, rows, cols, tol)
    print(what, "max per-Gaussian error / tolerance:", {k: f"{v:.3g}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= 1.0, (what, k, v)
    for sname, rows in sets.items():
        assert (np.abs(ref[rows]).sum(1) > 0).sum() >= min_rows, (what, sname)


def _check_density(got, ref, keep, what):
    """Columns 0-1 per Gaussian over `keep` with the same form of tolerance, and as a norm at 1e-3."""
    assert np.isfinite(got).all(), what
    worst = {}
    for c in (0, 1):
        want = ref["density"][:, c:c + 1]
        r = rel(got[keep, c], want[keep, 0])
        assert r <= 1e-3, (what, c, r)
        worst[c] = _row_ratio(got[:, c:c + 1], want, keep, slice(0, 1), _atol(want, keep, slice(0, 1)))
    print(what, "density: max per-Gaussian error / tolerance:", {k: f"{v:.3g}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= 1.0, (what, k, v)


def _backward(gs, vtx, u, g, level=0, deterministic=False, mode=0, density=False, camera=False):
    """One frame of u on a fresh context and its backward: (grad_vertices, density or None, grad_uniforms or None) on the
    host, in float32."""
    torch = _torch()
    ctx = gs.Context(0)
    try:
        ctx.upload(vtx)
        ctx.set_mode(mode)
        ctx.set_tile_cull(level)
        ctx.set_backward(True)
        ctx.set_backward_deterministic(deterministic)
        ctx.render(u)
        v = torch.from_numpy(np.ascontiguousarray(vtx, np.float32)).cuda()
        gi = torch.from_numpy(g).cuda()
        gv = torch.full_like(v, float("nan"))
        dens = torch.zeros((v.shape[0], 4), dtype=torch.float32, device="cuda") if density else None
        gu = torch.full((40,), float("nan"), dtype=torch.float32, device="cuda") if camera else None
        ctx.render_backward(v.data_ptr(), gi.data_ptr(), gv.data_ptr(), grad_uniforms_ptr=gu.data_ptr() if camera else None,
                            density_ptr=dens.data_ptr() if density else None)
        torch.cuda.synchronize()
    finally:
        ctx.close()

    def host(t):
        return None if t is None else t.cpu().numpy()

    return host(gv), host(dens), host(gu)


@pytest.fixture(scope="module")
def stress(oracle):
    """stress_scene.vertices() and, computed once per camera on first use, its oracle frame, upstream gradient (zero on the
    step-probed pixels) and references."""
    vtx = stress_scene.vertices()

    @functools.lru_cache(maxsize=None)
    def at(cam):
        u = stress_scene.camera(cam)
        oracle.set_exp_mode(0)
        frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
        g = grad_image(u, steps)
        ref = grad_ref.reference(vtx, u, frame, g)
        keep = ~ref["exclude"]
        survivor = frame["attr"]["color_radii"][:, 3] != 0
        sets = {"clamped_alpha": keep & stress_scene.walk_coverage(vtx, u, frame, g)["clamped"],
                "red_below_0": keep & survivor & (stress_scene.red(vtx, u) < 0),
                "fov_clamped": keep & survivor & stress_scene.fov_clamped(vtx, u)}
        return {"u": u, "g": g, "ref": ref, "keep": keep, "sets": sets, "density": grad_ref.density_reference(vtx, u, frame, g)}

    return vtx, at


@pytest.fixture(scope="module")
def stress_camera(oracle):
    """stress_scene.camera_vertices() and, once per camera, its upstream gradient and grad_ref's camera reference."""
    vtx = stress_scene.camera_vertices()

    @functools.lru_cache(maxsize=None)
    def at(cam):
        u = stress_scene.camera(cam)
        oracle.set_exp_mode(0)
        frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
        g = grad_image(u, steps)
        return {"u": u, "g": g, "ref": grad_ref.reference(vtx, u, frame, g, camera=True)}

    return vtx, at


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("cam", stress_scene.CAMERAS)
def test_vertex_gradient_matches_reference(gs, stress, cam, level, path):
    vtx, at = stress
    r = at(cam)
    got, _, _ = _backward(gs, vtx, r["u"], r["g"], level=level, deterministic=PATHS[path])
    _check_vertices(got, r["ref"]["grad"], r["keep"], r["sets"], (cam, level, path))


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("cam", stress_scene.CAMERAS)
def test_density_matches_reference(gs, stress, cam, level, path):
    vtx, at = stress
    r = at(cam)
    gv, got, _ = _backward(gs, vtx, r["u"], r["g"], level=level, deterministic=PATHS[path], density=True)
    _check_density(got, r["density"], r["keep"], (cam, level, path))
    assert np.array_equal(got[:, 2], r["density"]["survivor"].astype(np.float64))
    assert np.array_equal(got[:, 3].astype(np.float32).view(np.uint32), r["density"]["radii"].astype(np.float32).view(np.uint32))
    # the vertex gradient that comes with it is gsb_render_backward's
    _check_vertices(gv, r["ref"]["grad"], r["keep"], r["sets"], (cam, level, path, "density"))


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("level", [0, 1])
@pytest.mark.parametrize("cam", stress_scene.CAMERAS)
def test_camera_gradient_matches_reference(gs, stress_camera, cam, level, path):
    vtx, at = stress_camera
    r = at(cam)
    assert not r["ref"]["exclude"].any()
    want = np.zeros(40)
    want[gs.UBO_FLOAT_WORDS] = r["ref"]["grad_ubo"]
    _, _, got = _backward(gs, vtx, r["u"], r["g"], level=level, deterministic=PATHS[path], camera=True)
    got = got.astype(np.float64)
    assert np.isfinite(got).all()
    rels = {name: rel(got[idx], want[idx]) for name, idx in CAMERA_GROUPS.items()}
    print((cam, level, path), "camera gradient relative error:", {k: f"{v:.3g}" for k, v in rels.items()})
    for name, r_ in rels.items():
        assert r_ <= 1e-3, (cam, level, path, name, r_)
    assert not got[DEAD].any()


@pytest.mark.parametrize("cam", stress_scene.CAMERAS)
def test_fast_mode_close_to_exact(gs, stress, cam):
    vtx, at = stress
    r = at(cam)
    ge, de, _ = _backward(gs, vtx, r["u"], r["g"], mode=0, density=True)
    gf, df, _ = _backward(gs, vtx, r["u"], r["g"], mode=1, density=True)
    keep = r["keep"]
    gf, ge, df, de = (a.astype(np.float64) for a in (gf, ge, df, de))
    for name, cols in GROUPS.items():
        err = rel(gf[keep, cols], ge[keep, cols])
        assert err <= 1e-3, (cam, name, err)
    for c in (0, 1):
        assert rel(df[keep, c], de[keep, c]) <= 1e-3, (cam, c)


@pytest.fixture(scope="module")
def garden_band(gs, oracle):
    """bench.py's garden stand-in (5.8 M Gaussians, 3200 x 1400), its first camera, and an upstream gradient that is a seeded
    normal on BAND_ROWS tile rows in the middle of the frame and zero elsewhere (and on the step-probed pixels), with the
    references over the oracle's lists of that band -- which are the full frame's lists of its tiles."""
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    import bench

    wl = bench.WORKLOADS["garden-standin"]
    vtx = bench.make_scene(gs, wl)
    u = bench.cameras(gs, wl)[0]
    r0 = (u.height + 15) // 16 // 2
    rows = (r0, r0 + BAND_ROWS)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u, rows=rows)
    g = np.zeros((u.height, u.width, 4), np.float32)
    y0, y1 = rows[0] * 16, min(u.height, rows[1] * 16)
    g[y0:y1] = np.random.default_rng(11).standard_normal((y1 - y0, u.width, 4))
    g[steps] = 0.0
    ref = grad_ref.reference(vtx, u, frame, g)
    dens = grad_ref.density_reference(vtx, u, frame, g)
    used = np.zeros(vtx.shape[0], bool)
    used[np.unique(frame["vals"])] = True
    print("garden band: tile rows", rows, "instances", frame["m"], "Gaussians in the band", int(used.sum()),
          "with a gradient", int((np.abs(ref["grad"]).sum(1) > 0).sum()))
    return {"vtx": vtx, "u": u, "g": g, "ref": ref, "density": dens, "used": used}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("level", [0, 1])
def test_full_size_band_matches_reference(gs, garden_band, level, path):
    b = garden_band
    gv, dens, _ = _backward(gs, b["vtx"], b["u"], b["g"], level=level, deterministic=PATHS[path], density=True)
    used, ref = b["used"], b["ref"]
    # outside the band's lists the upstream gradient is zero: nothing at all
    assert not gv[~used].any() and not dens[~used, :2].any()
    keep = used & ~ref["exclude"]
    assert (np.abs(ref["grad"][keep]).sum(1) > 0).sum() > 1000
    _check_vertices(gv, ref["grad"], keep, {}, ("garden band", level, path))
    _check_density(dens, b["density"], keep, ("garden band", level, path))
