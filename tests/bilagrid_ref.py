"""Float64 reference of the bilateral-grid colour correction (gsb_bilagrid_apply / gsb_bilagrid_backward, DESIGN.md section 17):
an explicit trilinear slice-and-apply in numpy and its hand-derived VJP.  `torch_path` is the same map through F.grid_sample
(bilinear, align_corners=True, border padding) plus the affine product, in any dtype, for cross-checks and for the
torch baseline of tools/bench_bilagrid.py."""
import numpy as np

LUMA = np.array([0.299, 0.587, 0.114])


def _axis(n, g):
    """Cell index and fraction of pixel coordinates 0 .. n - 1 on a grid axis of g nodes."""
    i = (np.arange(n) + 0.5) / n * (g - 1)
    i0 = np.minimum(np.floor(i), g - 2).astype(np.int64)
    return i0, i - i0


def _slice(image, grid):
    """Per pixel: corner indices, weights and the sliced A (H, W, 12), in float64."""
    image = np.asarray(image, np.float64)
    grid = np.asarray(grid, np.float64)
    _, L, Y, X = grid.shape
    H, W = image.shape[:2]
    x0, fx = _axis(W, X)
    y0, fy = _axis(H, Y)
    gray = (LUMA[0] * image[..., 0] + LUMA[1] * image[..., 1]) + LUMA[2] * image[..., 2]
    iz = np.clip(gray, 0.0, 1.0) * (L - 1)
    z0 = np.minimum(np.floor(iz), L - 2).astype(np.int64)
    fz = iz - z0
    X0, FX = np.broadcast_to(x0[None, :], (H, W)), np.broadcast_to(fx[None, :], (H, W))
    Y0, FY = np.broadcast_to(y0[:, None], (H, W)), np.broadcast_to(fy[:, None], (H, W))
    corners = []  # (dz, dy, dx, weight, d weight / d iz)
    for dz in (0, 1):
        wz, dwz = (1 - fz, -1.0) if dz == 0 else (fz, 1.0)
        for dy in (0, 1):
            wy = 1 - FY if dy == 0 else FY
            for dx in (0, 1):
                wx = 1 - FX if dx == 0 else FX
                corners.append((dz, dy, dx, wz * wy * wx, dwz * wy * wx))
    A = np.zeros((H, W, 12))
    dA = np.zeros((H, W, 12))  # d A / d iz
    for dz, dy, dx, w, dw in corners:
        node = grid[:, z0 + dz, Y0 + dy, X0 + dx]  # (12, H, W)
        A += (w * node).transpose(1, 2, 0)
        dA += (dw * node).transpose(1, 2, 0)
    inside = (gray > 0) & (gray < 1)
    return dict(A=A, dA=dA, corners=corners, x0=X0, y0=Y0, z0=z0, inside=inside, iz=iz, gray=gray)


def _inputs(image):
    image = np.asarray(image, np.float64)
    return np.concatenate([image[..., :3], np.ones(image.shape[:2] + (1,))], axis=-1)  # (r, g, b, 1)


def forward(image, grid):
    """out (H, W, 4) float64: out_c = sum_j A_cj in_j, A copied."""
    s = _slice(image, grid)
    v = _inputs(image)
    out = np.empty(np.shape(image), np.float64)
    for c in range(3):
        out[..., c] = (s["A"][..., 4 * c:4 * c + 4] * v).sum(-1)
    out[..., 3] = np.asarray(image, np.float64)[..., 3]
    return out


def vjp(image, grid, grad_out):
    """(d image (H, W, 4) with A = 0, d grid (12, L, Y, X)) of sum(grad_out[..., :3] * out[..., :3]), in float64."""
    grid = np.asarray(grid, np.float64)
    _, L, Y, X = grid.shape
    s = _slice(image, grid)
    v = _inputs(image)
    g = np.asarray(grad_out, np.float64)[..., :3]
    A, dA = s["A"], s["dA"]
    d_image = np.zeros(np.shape(image), np.float64)
    for j in range(3):
        d_image[..., j] = sum(A[..., 4 * c + j] * g[..., c] for c in range(3))
    t = sum(g[..., c] * (dA[..., 4 * c:4 * c + 4] * v).sum(-1) for c in range(3)) * (L - 1)
    t = np.where(s["inside"], t, 0.0)
    for j in range(3):
        d_image[..., j] += LUMA[j] * t
    q = np.einsum("hwc,hwj->hwcj", g, v).reshape(g.shape[:2] + (12,))  # q[4 c + j] = g_c in_j
    d_grid = np.zeros_like(grid)
    for dz, dy, dx, w, _ in s["corners"]:
        idx = (s["z0"] + dz, s["y0"] + dy, s["x0"] + dx)
        for k in range(12):
            np.add.at(d_grid[k], idx, w * q[..., k])
    return d_image, d_grid


def node_distance(image, L):
    """Per pixel, the distance of its luma to the nearest z node plane or clamp, in units of gray (for per-value bounds)."""
    s_gray = (LUMA[0] * np.asarray(image, np.float64)[..., 0] + LUMA[1] * np.asarray(image, np.float64)[..., 1]) \
        + LUMA[2] * np.asarray(image, np.float64)[..., 2]
    planes = np.arange(L) / (L - 1)
    return np.abs(s_gray[..., None] - planes).min(-1)


def torch_path(image, grid, coords32=False):
    """The same correction through F.grid_sample (trilinear, align_corners=True, border padding) and the affine product,
    in the dtype and on the device of the inputs: image (H, W, 4), grid (12, L, Y, X).  Differentiable in both.

    coords32=True samples at the definition's fp32 coordinates ix, iy and iz = clamp(gray, 0, 1) (L - 1), each step an fp32
    IEEE operation, carried exactly in the inputs' dtype; d/d gray is the inputs' own.  In float64 this is the reference of
    the kernels: one ulp of ix moves a far-from-identity 64-node grid's output by up to 3e-5."""
    import torch
    import torch.nn.functional as F

    H, W = image.shape[:2]
    _, L, Y, X = grid.shape
    dev, dt = image.device, image.dtype
    rgb = image[..., :3]
    gray = (0.299 * rgb[..., 0] + 0.587 * rgb[..., 1]) + 0.114 * rgb[..., 2]
    z = gray * 2 - 1
    if coords32:
        f = torch.float32

        def axis(n, g):  # in numpy: torch on CUDA divides by a scalar through its reciprocal, not as IEEE division
            i = (np.arange(n, dtype=np.float32) + np.float32(0.5)) / np.float32(n) * np.float32(g - 1)
            return torch.from_numpy(i).to(dev).to(dt) / (g - 1) * 2 - 1

        xs, ys = axis(W, X), axis(H, Y)
        r = image.detach()[..., :3].to(f)
        iz = ((0.299 * r[..., 0] + 0.587 * r[..., 1]) + 0.114 * r[..., 2]).clamp(0.0, 1.0) * (L - 1)
        z = z + (iz.to(dt) / (L - 1) * 2 - 1 - z).detach()
    else:
        xs = (torch.arange(W, device=dev, dtype=dt) + 0.5) / W * 2 - 1
        ys = (torch.arange(H, device=dev, dtype=dt) + 0.5) / H * 2 - 1
    coords = torch.stack([xs[None, :].expand(H, W), ys[:, None].expand(H, W), z], dim=-1)
    A = F.grid_sample(grid[None], coords[None, None], mode="bilinear", padding_mode="border", align_corners=True)
    A = A[0, :, 0].permute(1, 2, 0).reshape(H, W, 3, 4)  # (H, W, 12) -> rows c, columns j
    out = (A[..., :3] * rgb[..., None, :]).sum(-1) + A[..., 3]
    return torch.cat([out, image[..., 3:]], dim=-1)


def random_grid(shape, spread, seed):
    """A (12, L, Y, X) float64 grid: identity plus uniform noise of half-width `spread` (X, Y, L = shape)."""
    X, Y, L = shape
    rng = np.random.default_rng(seed)
    g = rng.uniform(-spread, spread, (12, L, Y, X))
    for c in range(3):
        g[4 * c + c] += 1.0
    return g


def random_image(w, h, seed, lo=-0.3, hi=1.3):
    """(H, W, 4) float32 image: a per-pixel level uniform in [lo, hi] plus per-channel noise of 0.1, so the luma falls below 0,
    inside [0, 1] and above 1."""
    rng = np.random.default_rng(seed)
    level = rng.uniform(lo, hi, (h, w, 1))
    img = level + rng.uniform(-0.1, 0.1, (h, w, 4))
    if w * h >= 3:  # at least one pixel of each kind
        img.reshape(-1, 4)[:3, :3] = np.array([[-0.2], [0.5], [1.2]])
    return img.astype(np.float32)
