"""The float64 restatement behind the backward tests (tests/grad_ref.py) computes the function the product renders: its
image equals the oracle's (mode 0, libm expf) within 1e-4 per channel.  CPU only.

The comparison skips the pixels oracle.render_frame_probed flags: there `alpha < 1/255` or `T' < 1e-4` sits within 0.2 % of
its threshold, so fp32 and float64 may take the other side of the step (a jump of up to alpha * T * colour).  The backward
tests zero the upstream gradient on the same pixels."""
import numpy as np
import pytest

import grad_ref
import scenes


@pytest.mark.parametrize("cam", ["c1", "odd_size", "inside"])
def test_grad_ref_image_matches_oracle(oracle, cam):
    _, vtx, _ = scenes.c1()
    u = scenes.camera(cam)
    oracle.set_exp_mode(0)
    frame, steps = oracle.render_frame_probed(vtx, oracle.cov3d(vtx), u)
    assert frame["m"] > 0
    assert steps.mean() < 0.05  # the step pixels are a small minority
    ref = grad_ref.reference(vtx, u, frame)["image"]
    err = np.abs(ref - frame["rgba"][..., :3].astype(np.float64)).max(-1)
    assert err[~steps].max() <= 1e-4, (cam, float(err[~steps].max()))
