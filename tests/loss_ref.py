"""Float64 restatement of the photometric loss of 3DGS training, the Inria `loss_utils` pair l1_loss / ssim (Kerbl et al.
2023): loss = (1 - lambda) L1 + lambda (1 - SSIM) over the RGB channels, SSIM with an 11 x 11 Gaussian window (sigma 1.5)
applied as F.conv2d(..., padding=5, groups=3), C1 = 0.01^2, C2 = 0.03^2.  gsb_image_loss is checked against it.

`reference` runs in float64 torch with the gradient from autograd, on the CPU or, for large frames, on a CUDA device.
`ssim_map_scipy` and `gather_gradient` restate the SSIM map and the hand-derived gather form of the gradient the kernels
implement in float64 numpy / scipy, independently of torch.  Test infrastructure only."""
import numpy as np
import scipy.ndimage
import torch
import torch.nn.functional as F

C1, C2 = 0.01 ** 2, 0.03 ** 2
RADIUS, SIGMA = 5, 1.5


def gauss1d():
    i = np.arange(2 * RADIUS + 1, dtype=np.float64)
    g = np.exp(-(i - RADIUS) ** 2 / (2 * SIGMA ** 2))
    return g / g.sum()


def window2d():
    g = gauss1d()
    return np.outer(g, g)


def as_chw(a, device="cpu"):
    """(3, H, W) float64 of the RGB channels of an (H, W, 4) float32 or uint8 frame (numpy or torch); uint8 is read as
    float32(v) / 255 in float32, as the kernels read an RGBA8 target."""
    t = torch.as_tensor(a).to(device)
    if t.dtype == torch.uint8:
        t = t.to(torch.float32) / 255.0
    return t[..., :3].to(torch.float64).permute(2, 0, 1).contiguous()


def ssim_map(x, y):
    """The SSIM map of (3, H, W) float64 tensors x and y, as loss_utils._ssim computes it."""
    w = torch.from_numpy(window2d()).to(x.device)[None, None].expand(3, 1, -1, -1).contiguous()

    def blur(t):
        return F.conv2d(t[None], w, padding=RADIUS, groups=3)[0]

    mu_x, mu_y = blur(x), blur(y)
    sxx = blur(x * x) - mu_x * mu_x
    syy = blur(y * y) - mu_y * mu_y
    sxy = blur(x * y) - mu_x * mu_y
    return ((2 * mu_x * mu_y + C1) * (2 * sxy + C2)) / ((mu_x * mu_x + mu_y * mu_y + C1) * (sxx + syy + C2))


def loss_terms(x, y, lam):
    """{"loss", "l1", "ssim", "mse"} of (3, H, W) float64 tensors (0-d tensors, differentiable in x)."""
    d = x - y
    l1, mse, ssim = d.abs().mean(), (d * d).mean(), ssim_map(x, y).mean()
    return {"loss": (1 - lam) * l1 + lam * (1 - ssim), "l1": l1, "ssim": ssim, "mse": mse}


def reference(image, target, lam, device="cpu", grad=True):
    """The loss terms of an (H, W, 4) frame against an (H, W, 4) float32 or uint8 target as floats, and with grad the
    gradient d loss / d image as an (H, W, 4) float64 numpy array with A = 0.  lam is used as the float32 value the C ABI
    receives."""
    lam = float(np.float32(lam))
    x = as_chw(image, device).requires_grad_(grad)
    y = as_chw(target, device)
    t = loss_terms(x, y, lam)
    out = {k: float(v.detach()) for k, v in t.items()}
    if grad:
        (g,) = torch.autograd.grad(t["loss"], x)
        h = np.zeros(tuple(x.shape[1:]) + (4,), np.float64)
        h[..., :3] = g.permute(1, 2, 0).cpu().numpy()
        out["grad"] = h
    return out


def _correlate(a):
    """Zero-padded correlation of each (H, W) plane of a (3, H, W) array with the 2D window."""
    w = window2d()
    return np.stack([scipy.ndimage.correlate(p, w, mode="constant", cval=0.0) for p in a])


def ssim_map_scipy(x, y):
    """The SSIM map of (3, H, W) float64 numpy arrays through scipy.ndimage.correlate."""
    mu_x, mu_y = _correlate(x), _correlate(y)
    sxx = _correlate(x * x) - mu_x ** 2
    syy = _correlate(y * y) - mu_y ** 2
    sxy = _correlate(x * y) - mu_x * mu_y
    return ((2 * mu_x * mu_y + C1) * (2 * sxy + C2)) / ((mu_x ** 2 + mu_y ** 2 + C1) * (sxx + syy + C2))


def gather_gradient(x, y, lam):
    """d loss / d x of (3, H, W) float64 numpy arrays in the gather form the kernels implement:
    (1 - lam) / N sign(x - y) - lam / N (w * A + 2 x (w * B) + y (w * C)), with per output pixel B = dS / d sigma_x^2,
    C = dS / d sigma_xy and A = dS / d mu_x - 2 mu_x B - mu_y C (w * = the zero-padded correlation with the window)."""
    mu_x, mu_y = _correlate(x), _correlate(y)
    sxx = _correlate(x * x) - mu_x ** 2
    syy = _correlate(y * y) - mu_y ** 2
    sxy = _correlate(x * y) - mu_x * mu_y
    a1, a2 = 2 * mu_x * mu_y + C1, 2 * sxy + C2
    b1, b2 = mu_x ** 2 + mu_y ** 2 + C1, sxx + syy + C2
    s = a1 * a2 / (b1 * b2)
    d_mu = 2 * mu_y * a2 / (b1 * b2) - 2 * mu_x * s / b1
    B = -s / b2
    C = 2 * a1 / (b1 * b2)
    A = d_mu - 2 * mu_x * B - mu_y * C
    g = _correlate(A) + 2 * x * _correlate(B) + y * _correlate(C)
    n = x.size
    return (1 - lam) / n * np.sign(x - y) - lam / n * g
