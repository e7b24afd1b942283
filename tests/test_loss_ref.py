"""The float64 loss reference (tests/loss_ref.py) on the CPU: its SSIM map equals an independent scipy computation, its
autograd gradient passes gradcheck, identical images give SSIM 1, L1 0 and a zero gradient, and the hand-derived gather form
of the gradient that gsb_image_loss implements equals autograd's."""
import numpy as np
import pytest
import torch

import loss_ref


def _pair(seed, h, w, flat=False):
    rng = np.random.default_rng(seed)
    x, y = rng.uniform(0, 1, (3, h, w)), rng.uniform(0, 1, (3, h, w))
    if flat:  # large constant regions (sigma exactly 0 inside them) next to noise
        x[:, : h // 2] = 0.25
        y[:, : h // 2] = 0.75
        x[:, :, : w // 3] = 1.0
    return x, y


@pytest.mark.parametrize("h, w, flat", [(2, 3, False), (11, 11, False), (23, 31, False), (24, 40, True)])
def test_ssim_map_matches_scipy(h, w, flat):
    x, y = _pair(1, h, w, flat)
    got = loss_ref.ssim_map(torch.from_numpy(x), torch.from_numpy(y)).numpy()
    want = loss_ref.ssim_map_scipy(x, y)
    assert np.abs(got - want).max() <= 1e-12


def test_window_is_the_normalised_gaussian():
    g = loss_ref.gauss1d()
    assert g.shape == (11,) and abs(g.sum() - 1) <= 1e-15 and np.array_equal(g, g[::-1])
    assert np.isclose(g[5] / g[6], np.exp(1 / 4.5))


def test_gradcheck():
    x, y = _pair(2, 7, 9)
    xt = torch.from_numpy(x).requires_grad_()
    yt = torch.from_numpy(y)
    assert torch.autograd.gradcheck(lambda t: loss_ref.loss_terms(t, yt, 0.2)["loss"], (xt,), eps=1e-6, atol=1e-8)


def test_identical_images():
    x, _ = _pair(3, 12, 17)
    img = np.zeros((12, 17, 4), np.float32)
    img[..., :3] = x.transpose(1, 2, 0)
    r = loss_ref.reference(img, img, 0.2)
    assert abs(r["ssim"] - 1) <= 1e-12 and r["l1"] == 0 and r["mse"] == 0 and abs(r["loss"]) <= 1e-12
    assert np.abs(r["grad"]).max() <= 1e-12


@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("h, w, flat", [(1, 1, False), (2, 3, False), (16, 16, False), (33, 17, True)])
def test_gather_form_equals_autograd(h, w, flat, lam):
    x, y = _pair(4, h, w, flat)
    xt = torch.from_numpy(x).requires_grad_()
    (want,) = torch.autograd.grad(loss_ref.loss_terms(xt, torch.from_numpy(y), lam)["loss"], xt)
    want = want.numpy()
    got = loss_ref.gather_gradient(x, y, lam)
    assert np.abs(got - want).max() <= 1e-12 * max(np.abs(want).max(), 1e-30)
