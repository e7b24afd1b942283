"""The numpy model of gsb_image_loss's arithmetic (tests/loss_model.py) meets the GPU tests' tolerances against the float64
reference on the inputs of tests/test_gpu_loss_regimes.py that need no renderer, so the precision of the kernels' design
is checked without a GPU; the GPU file pins the kernels to the model."""
import pytest

import loss_model
import loss_ref
from test_gpu_loss_regimes import (FLAT_NOISE, FLAT_PAIRS, GEOMETRY, LAM, STRIPS, check, flat_case, mixed_case,
                                   out_of_range_case)


def _check_model(x, y, what, lam=LAM):
    m = loss_model.model(x, y, lam)
    return check([m["loss"], m["l1"], m["ssim"], m["mse"]], m["grad"], loss_ref.reference(x, y, lam), what)


@pytest.mark.parametrize("where", ["frame", "region"])
@pytest.mark.parametrize("noise", FLAT_NOISE, ids=["exact", "noise1e-3", "noise1e-4"])
@pytest.mark.parametrize("pair", FLAT_PAIRS, ids=[f"{a}_vs_{b}" for a, b in FLAT_PAIRS])
def test_flat_regions(pair, noise, where):
    _check_model(*flat_case(*pair, noise, where), (pair, noise, where))


@pytest.mark.parametrize("kind", ["wide", "near_flat_1.8", "flat_1.8_in_wide"])
def test_out_of_range_values(kind):
    for lam in (0.2, 1.0):
        _check_model(*out_of_range_case(kind), (kind, lam), lam)


def test_sizes_and_strips():
    for w in GEOMETRY:
        for h in GEOMETRY:
            _check_model(*mixed_case(w, h, seed=w * 100 + h), (w, h))
    for n in STRIPS:
        for w, h in ((n, 1), (1, n)):
            _check_model(*mixed_case(w, h, seed=n), (w, h))
