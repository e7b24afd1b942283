"""A numpy model of gsb_image_loss's arithmetic (csrc/gsb_loss.cu, DESIGN.md section 11): the window passes and every
per-pixel term in float64, the gather terms A, B, C rounded to float32 where the kernel stores them, the gradient
gathered in float64 and rounded to float32 once.  Only the order of the float64 sums differs from the kernels', so the
model lets the precision of the kernels be checked against tests/loss_ref.py without a GPU, and the kernels be pinned to it
on one.  Test infrastructure only."""
import numpy as np
import scipy.ndimage

from loss_ref import C1, C2, as_chw, gauss1d


def _blur(a):
    """The zero-padded separable correlation of each (H, W) plane of a (3, H, W) float64 array with the window: the
    horizontal pass, then the vertical one, as the kernels run them."""
    g = gauss1d()
    h = scipy.ndimage.correlate1d(a, g, axis=2, mode="constant", cval=0.0)
    return scipy.ndimage.correlate1d(h, g, axis=1, mode="constant", cval=0.0)


def gather_terms(x, y):
    """(S, A, B, C) of (3, H, W) float64 arrays of float32 values: S in float64, A, B, C as the float32 values the forward
    kernel stores, with A taken relative to the pixel's own values, A = dS/dmu_x - 2 (mu_x - x) B - (mu_y - y) C."""
    ux, uy = _blur(x), _blur(y)
    vx = _blur(x * x) - ux * ux
    vy = _blur(y * y) - uy * uy
    cxy = _blur(x * y) - ux * uy
    a1, a2 = 2 * ux * uy + C1, 2 * cxy + C2
    b1, b2 = ux * ux + uy * uy + C1, vx + vy + C2
    r1, r2 = 1 / b1, 1 / b2
    s = a1 * a2 * (r1 * r2)
    dmx = 2 * uy * a2 * (r1 * r2) - 2 * ux * s * r1
    B = -s * r2
    C = 2 * a1 * (r1 * r2)
    A = dmx - 2 * (ux - x) * B - (uy - y) * C
    f32 = [t.astype(np.float32).astype(np.float64) for t in (A, B, C)]
    return (s, *f32)


def model(image, target, lam, grad=True):
    """The kernels' loss terms {"loss", "l1", "ssim", "mse"} of an (H, W, 4) float32 frame against an (H, W, 4) float32 or
    uint8 target and, with grad, the gradient as an (H, W, 4) float64 array of float32 values with A = 0."""
    lam = float(np.float32(lam))
    x = as_chw(image).numpy()
    y = as_chw(target).numpy()
    n = x.size
    d = (x.astype(np.float32) - y.astype(np.float32)).astype(np.float64)
    s, A, B, C = gather_terms(x, y)
    l1, mse, ssim = np.abs(d).sum() / n, (d * d).sum() / n, s.sum() / n
    out = {"loss": (1 - lam) * l1 + lam * (1 - ssim), "l1": l1, "ssim": ssim, "mse": mse}
    if grad:
        g = _blur(A) + 2 * (x * _blur(B) - _blur(x * B)) + (y * _blur(C) - _blur(y * C))
        v = ((1 - lam) / n * np.sign(x - y) - lam / n * g).astype(np.float32)
        h = np.zeros(x.shape[1:] + (4,), np.float64)
        h[..., :3] = v.transpose(1, 2, 0)
        out["grad"] = h
    return out
