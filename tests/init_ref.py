"""Reference of gsb_init_from_points' scale column (include/gs_b200.h, DESIGN.md section 13) in numpy fp32, and the point
clouds its tests and tools/bench_init.py run on.

D of row i is the mean of the m = min(3, n - 1) smallest d = (dx*dx + dy*dy) + dz*dz (dx = x_j - x_i, one fp32 operation
each) over the rows j != i, summed in ascending order; the scale is sqrt(max(D, 1e-7)).  `d_ref` takes the candidate
neighbours of a float64 cKDTree query with k = min(n, 16), excluding the row itself by index, and computes d for them in
fp32.  Its premise -- no point outside the k candidates can be among the m smallest -- is checked per row: the k-th
candidate's float64 squared distance must exceed the m-th fp32 value by a relative 1e-5 (an fp32 d is within a few ulp of
the float64 one); rows that fail it are queried again with k doubled, up to k = n.  `d_brute` is the all-pairs
computation the reference is tested against."""
import numpy as np

FLOOR = np.float32(1e-7)


def sq_dist(a, b):
    """d of every pair, fp32, one IEEE operation at a time in the header's order (numpy never contracts to FMA)."""
    dx, dy, dz = (b[..., k] - a[..., k] for k in range(3))
    return (dx * dx + dy * dy) + dz * dz


def mean_smallest(d_sorted, m):
    """((d_1 + d_2) + d_3) / 3 over the m smallest, fp32, ascending; 0 for m = 0."""
    if m == 0:
        return np.zeros(d_sorted.shape[0], np.float32)
    acc = d_sorted[:, 0].copy()
    for k in range(1, m):
        acc = acc + d_sorted[:, k]
    return acc / np.float32(m)


def scale_from_d(D):
    return np.sqrt(np.maximum(D.astype(np.float32), FLOOR))


def d_brute(xyz, rows=None):
    """D of `rows` (default all) against every other row, all pairs in fp32."""
    xyz = np.ascontiguousarray(xyz, np.float32)
    n = xyz.shape[0]
    rows = np.arange(n) if rows is None else np.asarray(rows)
    m = min(3, n - 1)
    out = np.empty(rows.shape[0], np.float32)
    for s in range(0, rows.shape[0], 256):
        r = rows[s:s + 256]
        d = sq_dist(xyz[r][:, None, :], xyz[None, :, :])
        d[np.arange(r.shape[0]), r] = np.inf  # not itself, by index
        out[s:s + 256] = mean_smallest(np.sort(d, 1), m)
    return out


def d_ref(xyz, rows=None, tree=None, k0=16):
    """D of `rows` (default all) from cKDTree candidates, premise checked and k enlarged where it fails."""
    from scipy.spatial import cKDTree

    xyz = np.ascontiguousarray(xyz, np.float32)
    n = xyz.shape[0]
    rows = np.arange(n) if rows is None else np.asarray(rows)
    m = min(3, n - 1)
    if m == 0:
        return np.zeros(rows.shape[0], np.float32)
    x64 = xyz.astype(np.float64)
    tree = cKDTree(x64) if tree is None else tree
    out = np.empty(rows.shape[0], np.float32)
    todo = np.arange(rows.shape[0])
    k = min(n, k0)
    while todo.size:
        r = rows[todo]
        dist, idx = tree.query(x64[r], k=k, workers=-1)
        dist, idx = dist.reshape(r.shape[0], k), idx.reshape(r.shape[0], k)
        d = sq_dist(xyz[r][:, None, :], xyz[idx])
        d[idx == r[:, None]] = np.inf  # not itself, by index
        ds = np.sort(d, 1)
        ok = np.full(r.shape[0], k == n) | (dist[:, -1] ** 2 > ds[:, m - 1].astype(np.float64) * (1 + 1e-5))
        out[todo[ok]] = mean_smallest(ds[ok], m)
        todo = todo[~ok]
        k = min(n, 2 * k)
    return out


# ---------------------------------------------------------------- point clouds (seeded)
def uniform(n, seed=0, half=1.0):
    return np.random.default_rng(seed).uniform(-half, half, (n, 3)).astype(np.float32)


def heavy_tailed(n, seed=0, dup_clusters=True):
    """95 % in a 1 m cube, 5 % spread over a 10 km cube; with dup_clusters, 2 % of the rows are copies of other rows in
    clusters of 2 to 40 identical points."""
    rng = np.random.default_rng(seed)
    far = n // 20
    xyz = np.concatenate([rng.uniform(-0.5, 0.5, (n - far, 3)), rng.uniform(-5000.0, 5000.0, (far, 3))]).astype(np.float32)
    if dup_clusters:
        budget = n // 50
        while budget > 0:
            size = int(rng.integers(2, 41))
            src = int(rng.integers(0, n))
            dst = rng.integers(0, n, size - 1)
            xyz[dst] = xyz[src]
            budget -= size
    return xyz[rng.permutation(n)]


def planar(n, seed=0):
    """A tilted 20 m x 20 m plane: z = 0.3 x - 0.2 y + 1, rounded to fp32."""
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-10.0, 10.0, (n, 2))
    return np.column_stack([xy, 0.3 * xy[:, 0] - 0.2 * xy[:, 1] + 1.0]).astype(np.float32)


def collinear(n, seed=0):
    rng = np.random.default_rng(seed)
    t = rng.uniform(-3.0, 3.0, n)
    return np.column_stack([t, 2.0 * t + 1.0, -0.5 * t]).astype(np.float32)


def lattice(side=12):
    """An integer lattice: every point has 6 neighbours at the same distance (massive ties)."""
    g = np.arange(side, dtype=np.float32)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


def duplicates(n, sizes=(2, 3, 4, 40), seed=0):
    """Uniform points with one cluster of identical points of each size."""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-1.0, 1.0, (n, 3)).astype(np.float32)
    at = 0
    for s in sizes:
        xyz[at:at + s] = xyz[at]
        at += s
    return xyz[rng.permutation(n)]


def offset_grid(n, seed=0):
    """Coordinates near 1e4 at 1e-2 spacing: d is dominated by the rounding of x_j - x_i."""
    rng = np.random.default_rng(seed)
    return (1e4 + 1e-2 * rng.integers(0, 40, (n, 3))).astype(np.float32)


SMALL_CLOUDS = {
    "uniform": lambda: uniform(3000, 1),
    "heavy_tailed": lambda: heavy_tailed(3000, 2),
    "duplicates": lambda: duplicates(2000, seed=3),
    "lattice": lambda: lattice(12),
    "planar": lambda: planar(2500, 4),
    "collinear": lambda: collinear(2000, 5),
    "offset_1e4": lambda: offset_grid(2000, 6),
    "n1": lambda: uniform(1, 7),
    "n2": lambda: uniform(2, 8),
    "n3": lambda: uniform(3, 9),
    "n4": lambda: uniform(4, 10),
}

# the 1 M clouds tools/bench_init.py times (the garden stand-in's positions come from bench.py's own scene)
BENCH_CLOUDS = {
    "heavy_tailed_1m": lambda: heavy_tailed(1_000_000, 11),
    "planar_1m": lambda: planar(1_000_000, 12),
}
