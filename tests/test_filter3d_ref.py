"""tests/filter3d_ref.py on the CPU: the fp32 restatement of gsb_filter3d_variance agrees with Mip-Splatting's own float64
compute_3D_filter from the poses; the float64 filtered activation and its chain rule equal autograd; the filtered Adam step
extends adam_ref's and reduces to it at zero variance; apply_filter_3d is the reference's activation; and records filtered
by the reference keep every survivor's 2D footprint above the filter's bound in the oracle's frames."""
import math

import numpy as np
import pytest
import torch

import adam_ref
import edge_scene
import filter3d_ref as fr
import scenes
from adam_ref import GROUPS

LR = [1.6e-4, 5e-3, 5e-2, 1e-3, 2.5e-3, 1.25e-4]


def look_at_poses(k, seed=0, radius=(3.0, 12.0)):
    """k poses (pos, quat wxyz, fov, W, H) on a jittered orbit around the origin, each looking roughly at it, of mixed sizes
    and fields of view."""
    rng = np.random.default_rng(seed)
    poses = []
    for _ in range(k):
        a = rng.uniform(-math.pi, math.pi)
        r = rng.uniform(*radius)
        pos = [r * math.sin(a), rng.uniform(-1.5, 1.5), r * math.cos(a)]
        yaw = a + rng.uniform(-0.3, 0.3)
        q = scenes.quat_axis_angle([0, 1, 0], math.degrees(yaw))
        tilt = scenes.quat_axis_angle([1, 0, 0], rng.uniform(-10, 10))
        w1, x1, y1, z1 = (float(c) for c in q)
        w2, x2, y2, z2 = (float(c) for c in tilt)
        qq = np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                       w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], np.float32)
        W, H = int(rng.integers(16, 1601)), int(rng.integers(16, 1201))
        poses.append((pos, qq, float(rng.uniform(30, 90)), W, H))
    return poses


def uniforms(gs, poses):
    return [gs.uniforms_from_camera(p, q, fov, 0.1, 1000.0, W, H) for p, q, fov, W, H in poses]


def cloud(n, seed, half=4.0):
    """Points around and far beyond the cameras: many are behind or beside some of them."""
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.uniform(-half, half, (n // 2, 3)), rng.normal(0, 3 * half, (n - n // 2, 3))]).astype(np.float32)


def _compare(gs, xyz, poses):
    keep = ~fr.borderline(xyz, poses)
    pts = xyz[keep]
    got = fr.variance_f32(pts, uniforms(gs, poses))
    want = fr.variance_mip64(pts, poses)
    assert got.dtype == np.float32
    err = np.abs(got - want) / np.maximum(want, 1e-30)
    assert float(err.max()) <= 2e-5, float(err.max())
    return int(keep.sum()), float(err.max())


@pytest.mark.parametrize("k", [1, 2, 7, 64, 65, 1000])
def test_fp32_restatement_matches_mip_splatting(gs, k):
    xyz = cloud(4000, seed=k)
    kept, err = _compare(gs, xyz, look_at_poses(k, seed=k))
    print(f"k = {k}: {kept} points compared, worst relative error {err:.2e}")
    # a point near any camera's margin is left out: with 1000 cameras most are
    assert kept > (xyz.shape[0] // 2 if k < 1000 else 50)


def test_c1_and_edge_cameras_match_mip_splatting(gs):
    _, vtx, _ = scenes.c1()
    _compare(gs, vtx[:, 0:3], [scenes.CAMERAS[c] for c in scenes.CAMERAS])
    xyz = edge_scene.vertices()[0][:, 0:3]
    _compare(gs, xyz, [edge_scene.CAMERA_POSES[c] for c in edge_scene.CAMERAS])


def test_unseen_rows_and_no_row_seen(gs):
    poses = [([0, 0, 5], [1, 0, 0, 0], 45.0, 64, 48)]
    cams = uniforms(gs, poses)
    xyz = np.array([[0, 0, 0], [0, 0, -3], [0, 0, 9], [100, 0, 0], [np.nan, 0, 0]], np.float32)  # seen, seen, behind, beside, NaN
    d, seen = fr.depth_f32(xyz, cams)
    assert seen.tolist() == [True, True, False, False, False]
    var = fr.variance_f32(xyz, cams)
    assert np.array_equal(var[2:], np.full(3, var[1], np.float32)) and var[1] > var[0]
    assert not fr.variance_f32(xyz[2:], cams).any()
    np.testing.assert_allclose(var[:2], fr.variance_mip64(xyz, poses)[:2], rtol=1e-6)


def _params(n=37, seed=0):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn((n, 60), generator=g, dtype=torch.float64)
    p[:, 4:7] = p[:, 4:7] * 2.0 - 4.0
    p[:, 8:12] += torch.tensor([2.0, 0, 0, 0], dtype=torch.float64)
    var = torch.rand(n, generator=g, dtype=torch.float64) * torch.exp(2 * p[:, 4:7]).mean(1) * 3
    return p, var, g


def test_chain_rule_equals_autograd():
    p, var, g = _params()
    gv = torch.randn((p.shape[0], 60), generator=g, dtype=torch.float64)
    x = p.clone().requires_grad_()
    (fr.activate(x, var) * gv).sum().backward()
    got = fr.chain(p, gv, var)
    for name, cols in GROUPS.items():
        err = float((got[:, cols] - x.grad[:, cols]).abs().max() / x.grad[:, cols].abs().max())
        assert err <= 1e-12, (name, err)
    assert torch.autograd.gradcheck(lambda t: fr.activate(t, var[:5])[:, 4:8], (p[:5].clone().requires_grad_(),))


def test_apply_filter_3d_is_the_reference_activation(gs):
    p, var, _ = _params()
    got = gs.apply_filter_3d(adam_ref.activate(p), var)
    want = fr.activate(p, var)
    assert float((got - want).abs().max()) <= 1e-15
    x = adam_ref.activate(p).requires_grad_()
    assert torch.autograd.gradcheck(lambda t: gs.apply_filter_3d(t, var[:4]), (x[:4].detach().clone().requires_grad_(),))


def test_zero_variance_reduces_to_adam_ref(gs):
    p, _, g = _params()
    zero = torch.zeros(p.shape[0], dtype=torch.float64)
    gv = torch.randn((p.shape[0], 60), generator=g, dtype=torch.float64)
    m, v = torch.randn(p.shape, generator=g, dtype=torch.float64) * 1e-3, torch.rand(p.shape, generator=g, dtype=torch.float64) * 1e-6
    cfg = gs.adam_config(LR, step=3)
    for a, b in zip(fr.step(p, m, v, gv, cfg, zero), adam_ref.step(p, m, v, gv, cfg)):
        assert float((a - b).abs().max()) <= 1e-15
    assert torch.equal(fr.activate(p, zero)[:, 7], adam_ref.activate(p)[:, 7])


def test_filtered_step_extends_adam_ref(gs):
    """Outside the scale and opacity columns the filtered step is adam_ref's; the moved rows follow the filtered chain rule."""
    p, var, g = _params()
    gv = torch.randn((p.shape[0], 60), generator=g, dtype=torch.float64)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    cfg = gs.adam_config(LR, step=1)
    rows = torch.arange(p.shape[0]) % 3 != 0
    P, M, V, X = fr.step(p, m, v, gv, cfg, var, rows)
    P0, M0, V0, X0 = adam_ref.step(p, m, v, gv, cfg, rows)
    other = [c for c in range(60) if c not in range(4, 8)]
    for a, b in ((P, P0), (M, M0), (V, V0), (X, X0)):
        assert torch.equal(a[:, other], b[:, other])
    assert torch.equal(P[~rows], p[~rows])
    grad = fr.chain(p, gv, var)
    assert torch.allclose(M[rows][:, 4:8], (1 - cfg.beta1) * grad[rows][:, 4:8], rtol=1e-14, atol=0)  # m = lerp(0, g, 1 - beta1)
    assert torch.allclose(X[:, 4:8], fr.activate(P, var)[:, 4:8])


def _footprints(gs, oracle, vtx, names, cams):
    """Every camera's seen survivors of the records filtered by the reference satisfy the bound."""
    var = fr.variance_f32(vtx[:, 0:3], cams)
    d, seen = fr.depth_f32(vtx[:, 0:3], cams)
    d = np.where(seen, d, d[seen].max())
    f = fr.focal_f32(cams)
    filt = fr.activate(torch.from_numpy(gs.raw_parameters(torch.from_numpy(vtx).double()).numpy()), torch.from_numpy(var))
    rec = filt.numpy().astype(np.float32)
    rec[:, 8:12] = vtx[:, 8:12]
    checked = 0
    for name, u in zip(names, cams):
        attr, _ = oracle.preprocess(rec, oracle.cov3d(rec), u)
        _, seen_c = fr.depth_f32(vtx[:, 0:3], [u])
        live = (attr["color_radii"][:, 3] > 0) & seen_c
        if not live.any():
            continue
        slack, lam_max, bound = fr.footprint_slack(attr["conic_opacity"][live][:, 0:3], attr["depth"][live], d[live], f, u)
        tol = 1e-4 * bound + 1e-5 * (lam_max + 0.3)
        assert bool((slack >= -tol).all()), (name, float((slack + tol).min()))
        checked += int(live.sum())
    return checked


def test_footprint_bound_c1_and_edge(gs, oracle):
    _, vtx, _ = scenes.c1()
    names = list(scenes.CAMERAS)
    assert _footprints(gs, oracle, vtx, names, [scenes.camera(c) for c in names]) > 1000
    ev = edge_scene.vertices()[0]
    names = list(edge_scene.CAMERAS)
    assert _footprints(gs, oracle, ev, names, [edge_scene.camera(c) for c in names]) > 100
