"""The density-control statistics' float64 reference (grad_ref.density_reference) and gs_b200.densify_and_prune.  CPU only.

density_reference takes grad_ref's blend with per-(pixel, entry) offsets as leaves; summed over pixels its uv gradient must
be grad_ref's own, and its absolute gradient can only be larger (triangle inequality).  densify_and_prune is checked on a
hand-built statistics table: which rows clone, split and prune, the source index, and the children's geometry."""
import numpy as np
import pytest
import torch

import grad_ref
import scenes
from backward_util import grad_image


def _grad_ref_uv(vtx, u, frame, g):
    """dL/d uv (n, 2) through grad_ref's own tile blend, uv as one float64 leaf (the loop of grad_ref.reference)."""
    v_all, used, local = grad_ref.survivors(vtx, frame)
    with torch.no_grad():
        uv, conic, op, col, _ = grad_ref.preprocess(torch.tensor(v_all[used].astype(np.float64)), u)
    uv = uv.clone().requires_grad_()
    gimg = torch.tensor(np.asarray(g, np.float64)[..., :3])
    for tl in grad_ref.tiles(u, frame, local):
        rgb = grad_ref.blend_tile(uv[tl.idx], conic[tl.idx], op[tl.idx], col[tl.idx], tl.fx, tl.fy)[0]
        (rgb * gimg[tl.py, tl.px]).sum().backward()
    out = np.zeros((v_all.shape[0], 2))
    out[used] = uv.grad.numpy()
    return out


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_per_pixel_leaves_sum_to_grad_ref(oracle, cam):
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    g = grad_image(u, steps)
    ref = grad_ref.density_reference(vtx, u, frame, g)
    want = _grad_ref_uv(vtx, u, frame, g)
    assert np.abs(want).max() > 0
    err = np.abs(ref["duv"] - want).max()
    assert err <= 1e-12 * np.abs(want).max(), (cam, err)
    # triangle inequality, per Gaussian: |sum_p a_p| <= sum_p |a_p| per component, so the norms are ordered too
    d = ref["density"]
    assert (d[:, 1] >= d[:, 0] * (1 - 1e-12)).all()
    assert (d[:, 1] > d[:, 0] * 1.01).any()  # opposite signs cancel for some Gaussians
    # the view count is the survivor set, and a survivor always has a radius >= 1 pixel
    assert (d[:, 2] == ref["survivor"]).all() and (ref["radii"][ref["survivor"]] >= 1).all()
    assert not d[~ref["survivor"]].any()


def _table():
    """Eight activated records with chosen scale / opacity and their statistics.  grad_threshold 0.5, scene_extent 10:
    clone / split at max scale 0.1, world-size prune at 1.0."""
    gen = torch.Generator().manual_seed(11)
    n = 8
    v = torch.randn((n, 60), generator=gen)
    v[:, 3] = 1.0
    q = torch.randn((n, 4), generator=gen)
    v[:, 8:12] = q / q.norm(dim=1, keepdim=True)
    v[:, 4:7] = torch.tensor([0.05, 0.5, 0.05, 0.05, 0.05, 0.05, 2.0, 3.2])[:, None] * torch.tensor([1.0, 0.7, 0.4])
    v[:, 7] = torch.tensor([0.5, 0.5, 0.001, 0.5, 0.5, 0.5, 0.5, 0.5])
    d = torch.tensor([  # grad, absgrad, views, max radius
        [3.0, 3.0, 3, 4],     # 0: hot and small -> clone
        [2.0, 2.5, 2, 9],     # 1: hot and large -> split
        [0.1, 0.1, 1, 2],     # 2: opacity 0.001 -> pruned
        [0.2, 0.4, 2, 3],     # 3: cold -> kept
        [3.0, 8.0, 10, 5],    # 4: avg 0.3 -> kept; avg absgrad 0.8 -> clone with use_absgrad
        [0.0, 0.0, 1, 50],    # 5: cold, 50 px -> pruned by max_screen_size
        [0.0, 0.0, 0, 0],     # 6: never seen, scale 2.0 > 1.0 -> pruned by the world-size rule
        [1.2, 1.2, 2, 7],     # 7: hot and large -> split; children 2.0 > 1.0 -> pruned by the world-size rule
    ], dtype=torch.float32)
    return v, d


def _kw(**extra):
    return {"grad_threshold": 0.5, "scene_extent": 10.0, **extra}


def test_densify_and_prune_counts_and_source(gs):
    v, d = _table()
    out, src = gs.densify_and_prune(v, d, generator=torch.Generator().manual_seed(5), **_kw())
    assert src.dtype == torch.int64
    # kept rows, clones, first children, second children; row 2 pruned
    assert src.tolist() == [0, 3, 4, 5, 6, 0, 1, 7, 1, 7]
    assert out.shape == (10, 60)
    assert torch.equal(out[:6], v[[0, 3, 4, 5, 6, 0]])  # kept and cloned rows are copied as they are
    out, src = gs.densify_and_prune(v, d, generator=torch.Generator().manual_seed(5), **_kw(max_screen_size=20))
    assert src.tolist() == [0, 3, 4, 0, 1, 1]
    out, src = gs.densify_and_prune(v, d, generator=torch.Generator().manual_seed(5), **_kw(use_absgrad=True))
    assert src.tolist() == [0, 3, 4, 5, 6, 0, 4, 1, 7, 1, 7]
    out, src = gs.densify_and_prune(v, d, **_kw(min_opacity=0.0, grad_threshold=100.0))
    assert src.tolist() == list(range(8)) and torch.equal(out, v)  # nothing to do


def test_densify_and_prune_children(gs):
    from scipy.spatial.transform import Rotation

    v, d = _table()
    out, src = gs.densify_and_prune(v, d, generator=torch.Generator().manual_seed(5), **_kw())
    eps = torch.randn((4, 3), generator=torch.Generator().manual_seed(5))  # rows 1, 7 (first children), 1, 7 (second)
    children = out[6:]
    assert src[6:].tolist() == [1, 7, 1, 7]
    for j, parent in enumerate([1, 7, 1, 7]):
        p = v[parent].double()
        R = Rotation.from_quat(p[[9, 10, 11, 8]].numpy()).as_matrix()  # scipy: scalar last
        want = p[0:3].numpy() + R @ (p[4:7].numpy() * eps[j].double().numpy())
        assert np.allclose(children[j, 0:3].double().numpy(), want, rtol=0, atol=1e-5), (j, children[j, 0:3], want)
        assert torch.equal(children[j, 4:7], v[parent, 4:7] / 1.6)
        assert torch.equal(children[j, 7:], v[parent, 7:])  # opacity, rotation, SH copied
    assert (out[:, 3] == 1.0).all()  # position.w
    assert not torch.equal(children[0, 0:3], children[2, 0:3])  # the two children of one parent differ
