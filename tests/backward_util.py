"""Shared pieces of the backward tests: the upstream gradient, the error measure, the recorded frame, the error-code check
and the parameter groups the gradients are compared by.  Test infrastructure only."""
import numpy as np
import pytest

# column groups of the 60-float vertex record
GROUPS = {"position": slice(0, 3), "scale": slice(4, 7), "opacity": slice(7, 8), "rotation": slice(8, 12),
          "sh_dc": slice(12, 15), "sh_rest": slice(15, 60)}
# gsb_uniforms word groups of the camera gradient (the struct as 40 4-byte words; proj_mat at 4, view_mat at 20, column-major)
CAMERA_GROUPS = {
    "camera_position": [0, 1, 2],
    "view_3x3": [20 + c * 4 + r for c in range(3) for r in range(3)],
    "view_translation": [32, 33, 34],
    "proj_013x3": [4 + c * 4 + k for c in range(3) for k in (0, 1, 3)],
    "proj_translation": [16, 17, 19],
    "tan_fov": [38, 39],
}
# the words that can be non-zero; the others (camera_position.w, proj row 2, view row 3, width, height) are always zero
LIVE = sorted(sum(CAMERA_GROUPS.values(), []))
DEAD = np.setdiff1d(np.arange(40), LIVE)


def grad_image(u, steps=None, seed=7):
    """A seeded standard-normal upstream gradient (H, W, 4) float32, zero on the pixels `steps` (H, W) when given."""
    g = np.random.default_rng(seed).standard_normal((u.height, u.width, 4)).astype(np.float32)
    if steps is not None:
        g[steps] = 0.0
    return g


def rel(a, b):
    """||a - b|| / ||b||; torch tensors are compared in float64 on the host."""
    if hasattr(a, "cpu"):
        a, b = a.double().cpu().numpy(), b.double().cpu().numpy()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def render(ctx, u, level=0, mode=0):
    """A recorded frame of u at tile-cull `level` in `mode`: the frame the next backward call differentiates."""
    ctx.set_mode(mode)
    ctx.set_tile_cull(level)
    ctx.set_backward(True)
    ctx.render(u)


def expect(gs, ctx, code, fn, prefix=""):
    """fn() raises GsbError `code` and leaves a last-error message on ctx that starts with `prefix` (the entry's name)."""
    with pytest.raises(gs.GsbError) as ei:
        fn()
    assert ei.value.code == code
    msg = gs.lib.gsb_last_error(ctx.h).decode()
    assert msg != "" and msg.startswith(prefix)


def translation_identity(grad_pos_sum, grad_pos_abs, u, g_ubo):
    """Moving every Gaussian by delta equals t_view += V3 delta, t_proj += P3 delta, campos -= delta, so
    sum_i dL/dp_i = V3^T g(view_mat[12..14]) + P3^T g(proj_mat[12, 13, 15]) - g(camera_position).  g_ubo: the 38 float fields.
    Returns the residual and, per component, the sum of the absolute values of every term."""
    P = np.asarray(list(u.proj_mat), np.float64).reshape(4, 4).T
    V = np.asarray(list(u.view_mat), np.float64).reshape(4, 4).T
    g_c, g_p, g_v = g_ubo[0:3], g_ubo[4:20], g_ubo[20:36]
    rows = [0, 1, 3]
    tv = V[:3, :3].T * g_v[12:15][None, :]  # tv[k, r] = V[r, k] g(t_view[r])
    tp = P[rows, :3].T * g_p[[12, 13, 15]][None, :]
    rhs = tv.sum(1) + tp.sum(1) - g_c
    scale = grad_pos_abs + np.abs(tv).sum(1) + np.abs(tp).sum(1) + np.abs(g_c)
    return grad_pos_sum - rhs, scale
