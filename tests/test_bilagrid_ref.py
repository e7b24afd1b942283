"""The float64 bilateral-grid reference (tests/bilagrid_ref.py) against F.grid_sample in float64, gradcheck of its hand-derived
VJP, and bilateral_grid_tv / identity_bilateral_grids against explicit loops.  CPU only."""
import numpy as np
import pytest
import torch

import bilagrid_ref as br

CASES = [((5, 3), (2, 2, 2)), ((17, 31), (16, 16, 8)), ((23, 9), (5, 9, 3)), ((40, 33), (64, 64, 16))]


@pytest.mark.parametrize("size,shape", CASES, ids=[f"{w}x{h}-{'x'.join(map(str, s))}" for (w, h), s in CASES])
@pytest.mark.parametrize("spread", [0.05, 1.0], ids=["near", "far"])
def test_reference_equals_grid_sample(size, shape, spread):
    w, h = size
    img = br.random_image(w, h, seed=w * h)
    gray = br._slice(img, br.random_grid(shape, 0.0, 0))["gray"]
    assert (gray < 0).any() and (gray > 1).any() and ((gray > 0) & (gray < 1)).any()
    grid = br.random_grid(shape, spread, seed=7)
    g_out = np.random.default_rng(3).normal(size=(h, w, 4))
    ref = br.forward(img, grid)
    d_img, d_grid = br.vjp(img, grid, g_out)
    ti = torch.tensor(img, dtype=torch.float64, requires_grad=True)
    tg = torch.tensor(grid, requires_grad=True)
    out = br.torch_path(ti, tg)
    assert np.abs(out.detach().numpy() - ref).max() <= 1e-12
    (out[..., :3] * torch.tensor(g_out[..., :3])).sum().backward()
    assert np.abs(tg.grad.numpy() - d_grid).max() <= 1e-12 * max(1.0, np.abs(d_grid).max())
    assert np.abs(ti.grad.numpy()[..., :3] - d_img[..., :3]).max() <= 1e-12 * max(1.0, np.abs(d_img).max())
    assert np.all(d_img[..., 3] == 0)


class _Ref(torch.autograd.Function):
    @staticmethod
    def forward(fctx, image, grid):
        fctx.save_for_backward(image, grid)
        return torch.from_numpy(br.forward(image.numpy(), grid.numpy()))

    @staticmethod
    def backward(fctx, g):
        image, grid = fctx.saved_tensors
        di, dg = br.vjp(image.numpy(), grid.numpy(), g.numpy())
        di[..., 3] = g.numpy()[..., 3]  # A is copied
        return torch.from_numpy(di), torch.from_numpy(dg)


def test_gradcheck():
    img = br.random_image(6, 5, seed=11).astype(np.float64)
    L = 4
    # keep the luma away from z node planes (the slice's kinks), so finite differences see one linear piece
    for _ in range(100):
        near = br.node_distance(img, L) < 1e-3
        if not near.any():
            break
        img[near] = br.random_image(1, int(near.sum()), seed=int(near.sum()) + 99).reshape(-1, 4)
    assert not (br.node_distance(img, L) < 1e-3).any()
    grid = br.random_grid((3, 4, L), 0.5, seed=2)
    ti = torch.tensor(img, requires_grad=True)
    tg = torch.tensor(grid, requires_grad=True)
    assert torch.autograd.gradcheck(_Ref.apply, (ti, tg), eps=1e-6, atol=1e-8)


def test_identity_returns_the_image():
    img = br.random_image(9, 7, seed=5)
    out = br.forward(img, br.random_grid((4, 3, 5), 0.0, 0))
    assert np.abs(out - img.astype(np.float64)).max() <= 1e-15


def test_tv_equals_explicit_loop(gs):
    grids = torch.from_numpy(np.random.default_rng(4).normal(size=(3, 12, 4, 3, 5)))
    n, K, L, Y, X = grids.shape
    g = grids.numpy()
    total = 0.0
    for axis, (dl, dy, dx) in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1))):
        s, cnt = 0.0, 0
        for i in range(n):
            for k in range(K):
                for l in range(L - dl):
                    for y in range(Y - dy):
                        for x in range(X - dx):
                            s += (g[i, k, l + dl, y + dy, x + dx] - g[i, k, l, y, x]) ** 2
                            cnt += 1
        total += s / cnt
    assert abs(float(gs.bilateral_grid_tv(grids)) - total) <= 1e-12 * total
    assert float(gs.bilateral_grid_tv(grids[1])) == pytest.approx(float(gs.bilateral_grid_tv(grids[1:2])), rel=1e-15)


def test_identity_grids(gs):
    g = gs.identity_bilateral_grids(2, shape=(5, 4, 3))
    assert g.shape == (2, 12, 3, 4, 5) and g.dtype == torch.float32
    eye = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32).reshape(12)
    assert np.array_equal(g.numpy(), np.broadcast_to(eye[None, :, None, None, None], g.shape))
    assert float(gs.bilateral_grid_tv(g)) == 0.0
