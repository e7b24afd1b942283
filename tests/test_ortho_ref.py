"""The orthographic camera's closed forms (tests/ortho_ref.py, the kernels' formulas) against autograd of the float64 map,
gradcheck of the float64 preprocess, the translation identity, the colour's independence of the position, the fp32 colour
restatement against float64, a pinhole pulled back to infinity converging to the orthographic map, and the lens helpers.
CPU only."""
import numpy as np
import pytest
import torch

import ortho_ref
import scenes

CAMS = {"square": (300.0, 300.0, 319.5, 239.5), "anisotropic": (412.5, 287.25, 301.0, 250.5),
        "off_centre": (150.0, 175.0, -40.25, 610.75)}


def _points(n, seed):
    rng = np.random.default_rng(seed)
    return np.c_[rng.uniform(-3, 3, (n, 2)), rng.uniform(0.3, 9.0, n)]


@pytest.mark.parametrize("name", sorted(CAMS))
def test_closed_forms_match_autograd(name):
    cam = CAMS[name]
    t = _points(64, 3)
    rng = np.random.default_rng(4)
    dJ, duv, df = rng.normal(size=(64, 2, 3)), rng.normal(size=(64, 2)), rng.normal(size=64)
    L0 = torch.tensor(ortho_ref.lens_values(cam)[:4])
    for p, w, g, h, want_t, want_l in zip(torch.tensor(t), torch.tensor(dJ), torch.tensor(duv), torch.tensor(df),
                                          ortho_ref.grad_t(cam, duv, df), ortho_ref.lens_grad(t, dJ, duv)):
        J = torch.func.jacrev(lambda q: ortho_ref.project(q[None], cam)[0])(p)
        assert np.abs(J.numpy() - ortho_ref.jacobian(cam)).max() <= 1e-12

        def phi(q, L):
            c = (L[0], L[1], L[2], L[3])
            jac = torch.func.jacrev(lambda s: ortho_ref.project(s[None], c)[0])(q)
            return (jac * w).sum() + (ortho_ref.project(q[None], c)[0] * g).sum() + h * q[2]

        a, b = torch.func.grad(phi, argnums=(0, 1))(p, L0)
        assert np.abs(a.numpy() - want_t).max() <= 1e-12 * max(1.0, np.abs(want_t).max())
        assert np.abs(b.numpy() - want_l).max() <= 1e-12 * max(1.0, np.abs(want_l).max())


def _rows(n=6, seed=0):
    vtx = scenes.c1(n=2000, seed=seed)[1]
    u = scenes.camera("c1")
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    t = (V @ np.c_[vtx[:, :3], np.ones(len(vtx))].T)[2]
    return vtx[t > 0.5][:n].astype(np.float64), u


def test_gradcheck_vertex_view_and_lens_leaves():
    rows, u = _rows()
    cl = ortho_ref.leaves(u, CAMS["anisotropic"])
    rng = np.random.default_rng(1)
    w = [torch.tensor(rng.normal(size=s)) for s in ((len(rows), 2), (len(rows), 3), (len(rows), 3), (len(rows),))]

    def f(v, view, lens):
        out = ortho_ref.pre({**cl, "view_mat": view, "lens": lens}, antialiased=True)(v, u)
        uv, conic, op, col, _, z = out
        return (uv * w[0]).sum() + (conic * w[1]).sum() + (col * w[2]).sum() + (op * w[3]).sum() + z.sum()

    v = torch.tensor(rows, requires_grad=True)
    view = cl["view_mat"].detach().clone().requires_grad_()
    lens = cl["lens"].detach().clone().requires_grad_()
    assert torch.autograd.gradcheck(f, (v, view, lens), eps=1e-6, atol=1e-6, rtol=1e-5)


def test_translation_identity():
    """Sum_i dL/dp_i = R^T dL/d(view column 3): the frame moves with the camera, to float64 rounding."""
    rows, u = _rows(40, 2)
    cl = ortho_ref.leaves(u, CAMS["off_centre"])
    v = torch.tensor(rows, requires_grad=True)
    uv, conic, op, col, _, z = ortho_ref.pre(cl)(v, u)
    rng = np.random.default_rng(5)
    loss = sum((a * torch.tensor(rng.normal(size=tuple(a.shape)))).sum() for a in (uv, conic, op, col, z))
    loss.backward()
    R = cl["view_mat"].detach().numpy().reshape(4, 4).T[:3, :3]
    g_trans = cl["view_mat"].grad.numpy()[12:15]
    lhs = v.grad.numpy()[:, :3].sum(0)
    assert np.abs(lhs - R.T @ g_trans).max() <= 1e-9 * max(1.0, np.abs(lhs).max())
    assert cl["camera_position"].grad is None


def test_colour_is_independent_of_position():
    rows, u = _rows(20, 3)
    v = torch.tensor(rows, requires_grad=True)
    col, _ = ortho_ref.colour(v, torch.tensor(np.asarray(list(u.view_mat), np.float64)))
    moved = rows.copy()
    moved[:, :3] += np.random.default_rng(0).normal(size=(20, 3)) * 5.0
    col2, _ = ortho_ref.colour(torch.tensor(moved), torch.tensor(np.asarray(list(u.view_mat), np.float64)))
    assert torch.equal(col, col2)
    col.sum().backward()
    assert not v.grad[:, :3].any()


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_fp32_colour_against_float64(degree):
    rows, u = _rows(200, 4)
    got = ortho_ref.colour32(rows[:, 12:60], u.view_mat, degree).astype(np.float64)
    want, _ = ortho_ref.colour(torch.tensor(rows), torch.tensor(np.asarray(list(u.view_mat), np.float32).astype(np.float64)),
                               degree)
    assert np.abs(got - want.numpy()).max() <= 1e-6


def test_pinhole_pulled_back_converges_at_first_order():
    """A pinhole of focal f D whose centre sits D behind the camera plane: its uv and J differ from the orthographic camera
    of focal f by O(1 / D), so D times the difference stays bounded while the difference itself falls tenfold per decade."""
    t = _points(50, 6)
    f = 250.0
    errs = []
    for D in (1e2, 1e3, 1e4, 1e5):
        uv, J = ortho_ref.pinhole_pullback(t, f, D)
        uo = np.stack([f * t[:, 0], f * t[:, 1]], 1)
        errs.append(max(np.abs(uv - uo).max(), np.abs(J - ortho_ref.jacobian((f, f, 0.0, 0.0))).max()))
    errs = np.array(errs)
    assert (errs[1:] < errs[:-1] / 8).all(), errs
    assert (errs * np.array([1e2, 1e3, 1e4, 1e5])).max() <= 2.0 * f * 9.0 * 3.0, errs


def test_pinhole_pulled_back_conic_converges():
    rows, u = _rows(30, 7)
    cam = (200.0, 200.0, 0.0, 0.0)
    v = torch.tensor(rows)
    V = torch.tensor(np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T.copy())
    t = ortho_ref.view_positions(v, V).numpy()
    conic_o = ortho_ref.pre(ortho_ref.leaves(u, cam))(v, u)[1].detach()
    s, q = rows[:, 4:7], rows[:, 8:12]
    Sig = []
    for si, qi in zip(s, q):
        w, x, y, z = qi
        R = np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y + 2 * z * w, 2 * x * z - 2 * y * w],
                      [2 * x * y - 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z + 2 * x * w],
                      [2 * x * z + 2 * y * w, 2 * y * z - 2 * x * w, 1 - 2 * x * x - 2 * y * y]])
        M = si[:, None] * R
        Sig.append(M.T @ M)
    Sig = np.array(Sig)
    errs = []
    for D in (1e3, 1e4, 1e5):
        _, J = ortho_ref.pinhole_pullback(t, cam[0], D)
        T = J @ V.numpy()[:3, :3]
        cov = T @ Sig @ T.transpose(0, 2, 1)
        a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
        det = a * c - b * b
        conic = np.stack([c / det, -b / det, a / det], 1)
        errs.append(np.abs(conic - conic_o.numpy()).max() / np.abs(conic_o.numpy()).max())
    assert errs[1] < errs[0] / 8 and errs[2] < errs[1] / 8, errs


def test_lens_tensor_round_trip(gs):
    cam = gs.ortho_camera(412.5, 287.25, -3.125, 250.5)
    assert cam.kind == gs.CAMERA_ORTHO and list(cam.k) == [0.0] * 4 and cam.max_theta == 0.0
    w = gs.lens_tensor(cam)
    assert w.shape == (8,) and not w[4:].any()
    back = gs.lens_camera(w, 0.0, gs.CAMERA_ORTHO)
    assert bytes(back) == bytes(cam)
    with pytest.raises(ValueError):
        gs.lens_camera(w, 0.0, 7)
