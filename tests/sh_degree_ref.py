"""Float64 reference of gsb_set_sh_degree, layered on tests/grad_ref.py (which stays as it is): preprocess.comp:73-108's
colour summed over the (d + 1)^2 coefficients of bands <= d only, restated here from the view direction, while uv, conic and
opacity are grad_ref's.  The coefficients of higher bands take no part, so their gradient is 0.  Test infrastructure only."""
from __future__ import annotations

from unittest import mock

import numpy as np
import torch

import grad_ref
from grad_ref import SH_C0, SH_C1, SH_C2, SH_C3

_plain_preprocess = grad_ref.preprocess


def sh_colour(v: torch.Tensor, cam_pos: torch.Tensor, degree: int):
    """The colour (k, 3) with only red clamped at 0, and the unclamped red (k,), of the rows of v at `degree`."""
    nk = (degree + 1) ** 2
    sh = v[:, 12:12 + 3 * nk].reshape(-1, nk, 3)
    d = v[:, 0:3] - cam_pos
    d = d / torch.sqrt((d * d).sum(1, keepdim=True))
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, zz = x * x, y * y, z * z
    basis = [torch.full_like(x, SH_C0)]
    if degree >= 1:
        basis += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if degree >= 2:
        basis += [SH_C2[0] * x * y, SH_C2[1] * y * z, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * z * x, SH_C2[4] * (xx - yy)]
    if degree >= 3:
        basis += [SH_C3[0] * (3 * xx - yy) * y, SH_C3[1] * x * y * z, SH_C3[2] * (4 * zz - xx - yy) * y,
                  SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * (xx - yy) * z,
                  SH_C3[6] * x * (xx - 3 * yy)]
    col = (torch.stack(basis, -1)[:, :, None] * sh).sum(1) + 0.5
    red = col[:, 0]
    return torch.stack([torch.where(red < 0, torch.zeros_like(red), red), col[:, 1], col[:, 2]], -1), red


def preprocess(v: torch.Tensor, u, cam=None, sh_degree=3):
    """grad_ref.preprocess with the colour of degree sh_degree (0..3)."""
    uv, conic, op, _, _ = _plain_preprocess(v, u, cam)
    if cam is None:
        cam_pos = torch.tensor(np.asarray(list(u.camera_position)[:3], np.float64))
    else:
        cam_pos = cam["camera_position"][:3]
    col, red = sh_colour(v, cam_pos, sh_degree)
    return uv, conic, op, col, red


def reference(vertices, u, frame, grad_image=None, camera=False, sh_degree=3):
    """grad_ref.reference of a frame at degree sh_degree: the image, dL/dvertices (the columns of higher bands 0), the
    exclusions and, with camera=True, dL/d(the UBO's float fields)."""
    with mock.patch.object(grad_ref, "preprocess", lambda v, u, cam=None: preprocess(v, u, cam, sh_degree)):
        return grad_ref.reference(vertices, u, frame, grad_image, camera)
