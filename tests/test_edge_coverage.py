"""The edge scene of the forward and backward parity tests (tests/edge_scene.py) reaches every regime it is there for, so
that a later edit to the scene cannot quietly drop one: measured with the oracle's lists and float64 arithmetic only."""
import functools

import numpy as np
import pytest

import edge_scene
import gs_b200 as gs

EMIT_BIG = 128   # k_emit / k_emit_coarse: Gaussians covering more tiles (blocks) than this are expanded by the whole block
EC_CHUNK = 1024  # survivors per k_emit_coarse chunk
EC_MAXBIG = 32   # block-expanded Gaussians per k_emit_coarse chunk
EMIT_WIN = 4096  # instances a chunk stages in shared memory per window

# the least each count may be: about half of what the scene gives (measured values in the comments)
MIN_COUNTS = {
    # adjacent equal-key entries of different colours (80 110), duplicate pairs sharing a list (200 of 200), needles with
    # A C / det >= 1e4 and a tile of max alpha < 1/255 (136; 83 of them with AABBs of <= 128 tiles), survivors over 128 tiles
    # (254), Gaussians of chunk 0 over 128 coarse blocks at shift 2 (75) and shift 1 (133), chunk 0's shift-2 entries
    # (26 768), survivors whose pixel radius is +inf (k_project's mid * mid overflows) and whose tile-AABB conversion
    # therefore saturates on +-inf (6; none saturates on a finite argument)
    "axis": {"tie_pairs": 40_000, "dup_shared": 100, "needle_cull": 68, "needle_cull_small": 40, "over_128_tiles": 125,
             "chunk0_big_s2": 37, "chunk0_big_s1": 66, "chunk0_entries_s2": 13_000, "saturated_inf_radius": 3},
    # (0 ties of different colours: only duplicates tie here), (200, 17)
    "rotated_odd": {"dup_shared": 100, "over_128_tiles": 8},
    # (1 584, 6)
    "near_plane": {"tie_pairs": 800, "saturated_inf_radius": 3},
}


@functools.lru_cache(maxsize=None)
def frame(cam):
    import oracle

    vtx, masks, pairs = edge_scene.vertices()
    oracle.set_exp_mode(1)
    try:
        f = oracle.render_frame(vtx, oracle.cov3d(vtx), edge_scene.camera(cam))
    finally:
        oracle.set_exp_mode(0)
    return vtx, masks, pairs, f


def max_alpha_per_tile(a, tiles_x, x0, y0, x1, y1):
    """float64 max over each tile (tx, ty) of tiles [x0, x1) x [y0, y1) of opacity * exp(power), power as render.comp:66,
    for one oracle attr record a: an (y1 - y0, x1 - x0) array."""
    co = a["conic_opacity"].astype(np.float64)
    xs = np.arange(x0 * 16, x1 * 16, dtype=np.float64)
    ys = np.arange(y0 * 16, y1 * 16, dtype=np.float64)
    dx = a["uv"][0] - xs[None, :]
    dy = a["uv"][1] - ys[:, None]
    power = -0.5 * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy
    al = co[3] * np.exp(np.minimum(power, 0.0))
    return al.reshape(y1 - y0, 16, x1 - x0, 16).max(axis=(1, 3))


def saturates(attr, u):
    """Gaussians whose tile-AABB float -> int conversion (k_project, the oracle's f2i_trunc) saturates, in their fp32 order."""
    uv = attr["uv"].astype(np.float32)
    r = attr["color_radii"][:, 3].astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        args = [(uv[:, 0] - r) / np.float32(16), (uv[:, 1] - r) / np.float32(16),
                (((uv[:, 0] + r) + np.float32(16)) - np.float32(1)) / np.float32(16),
                (((uv[:, 1] + r) + np.float32(16)) - np.float32(1)) / np.float32(16)]
    return np.any([np.abs(a) >= np.float32(2.0 ** 31) for a in args], axis=0)


def coverage(cam):
    vtx, masks, pairs, f = frame(cam)
    u = edge_scene.camera(cam)
    n = vtx.shape[0]
    attr, tiles_n = f["attr"], f["tiles"]
    tiles_x = (u.width + 15) // 16
    keys, vals = f["keys"], f["vals"]
    surv = tiles_n > 0
    c = {}
    # adjacent list entries with equal keys (tile and depth bits) and different colours: the image depends on the tie order
    same = keys[1:] == keys[:-1]
    col = attr["color_radii"][:, :3]
    c["tie_pairs"] = int((same & (col[vals[1:]] != col[vals[:-1]]).any(1)).sum())
    # duplicate pairs that share a tile list
    pid = np.full((2, n), -1)
    pid[0, pairs[:, 0]] = np.arange(len(pairs))
    pid[1, pairs[:, 1]] = np.arange(len(pairs))
    t = (keys >> np.uint64(32)).astype(np.int64)
    sides = []
    for s in (0, 1):
        p = pid[s][vals]
        sides.append(np.unique(t[p >= 0] * len(pairs) + p[p >= 0]))
    c["dup_shared"] = int(np.unique(np.intersect1d(sides[0], sides[1]) % len(pairs)).size)
    # needles with A C / det >= 1e4 (float64 of the fp32 conic) that have an AABB tile of float64 max alpha < 1/255, and the
    # ones among them whose AABB is small enough (<= EMIT_BIG tiles) for k_emit's level 1 row spans
    co = attr["conic_opacity"].astype(np.float64)
    det = co[:, 0] * co[:, 2] - co[:, 1] ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        aniso = np.where(det > 0, co[:, 0] * co[:, 2] / det, 0.0)
    cand = np.nonzero(masks["needle"] & surv & (aniso >= 1e4))[0]
    culled = 0
    culled_small = 0
    for i in cand:
        x0, y0, x1, y1 = (int(v) for v in attr["aabb"][i])
        if (max_alpha_per_tile(attr[i], tiles_x, x0, y0, x1, y1) < 1.0 / 255.0).any():
            culled += 1
            culled_small += int(tiles_n[i] <= EMIT_BIG)
    c["needle_cull"] = culled
    c["needle_cull_small"] = culled_small
    c["over_128_tiles"] = int((tiles_n > EMIT_BIG).sum())
    # k_emit_coarse's first chunk of the depth order: Gaussians with more than EMIT_BIG coarse blocks, and its entries
    vis = np.nonzero(surv)[0]
    order = vis[np.argsort(attr["depth"][vis].view(np.uint32), kind="stable")]
    a = attr["aabb"].astype(np.int64)

    def blocks(s):
        return (((a[:, 2] - 1) >> s) - (a[:, 0] >> s) + 1) * (((a[:, 3] - 1) >> s) - (a[:, 1] >> s) + 1) * surv

    chunk0 = order[:EC_CHUNK]
    c["chunk0_big_s2"] = int((blocks(2)[chunk0] > EMIT_BIG).sum())
    c["chunk0_big_s1"] = int((blocks(1)[chunk0] > EMIT_BIG).sum())
    c["chunk0_entries_s2"] = int(blocks(2)[chunk0].sum())
    sat = saturates(attr, u) & surv
    inf_radius = np.isposinf(attr["color_radii"][:, 3])
    c["saturated_inf_radius"] = int((sat & inf_radius).sum())
    c["saturated_finite"] = int((sat & ~inf_radius).sum())  # reported only: out of fp32's reach with a footprint in the frame
    return c


@pytest.mark.parametrize("cam", edge_scene.CAMERAS)
def test_edge_scene_reaches_every_regime(cam):
    counts = coverage(cam)
    print(cam, counts)
    for name, least in MIN_COUNTS[cam].items():
        assert counts[name] >= least, (cam, name, counts[name], least)
    if cam == "axis":
        assert counts["chunk0_big_s2"] > EC_MAXBIG and counts["chunk0_big_s1"] > EC_MAXBIG
        assert counts["chunk0_entries_s2"] > EMIT_WIN


def test_duplicates_straddle_every_shard_boundary():
    vtx, _, pairs = edge_scene.vertices()
    n = vtx.shape[0]
    lo, hi = pairs.min(1), pairs.max(1)
    counts = {}
    for w in (2, 3, 8):
        for r in range(1, w):
            b = gs.shard_slice(n, r, w)[0]
            counts[(w, r)] = int(((lo < b) & (hi >= b)).sum())
    print("pairs straddling each boundary", counts)  # 43-100 per boundary
    assert min(counts.values()) >= 20


def test_near_plane_rows():
    """The near rows' fates: at the near_plane camera view depth prev(0.2f) and 0.2f are culled, next(0.2f) survives; at the
    axis camera the grid neighbour below 0.2f is culled and the one above survives."""
    import oracle

    vtx, masks, _ = edge_scene.vertices()
    fates = {}
    for name, x, y, z, _ in edge_scene.near_depths():
        cam = name.split("/")[0]
        row = np.nonzero(masks["near"] & (vtx[:, 0] == x) & (vtx[:, 1] == y) & (vtx[:, 2] == z))[0]
        assert row.size == 1, name
        _, tiles = oracle.preprocess(vtx[row], oracle.cov3d(vtx[row]), edge_scene.camera(cam))
        fates[name] = bool(tiles[0] > 0)
    print(fates)
    assert fates == {"near_plane/below": False, "near_plane/at": False, "near_plane/above": True,
                     "axis/below": False, "axis/above": True}


def test_opacity_edge_fates():
    """Each opacity-edge row is centred exactly on a pixel of the axis camera, where power is 0 and alpha = min(0.99,
    opacity): the blend's `alpha < 1/255` skip and the 0.99 clamp are decided at equality.  Pinned on the oracle's frame by
    rendering the tile row of those pixels again with the row's opacity set to 0: the pixel changes iff the row is blended
    there.  Opacity 0 and the float below 1/255 are skipped; 1/255 itself and everything above are kept; 0.99 and the float
    above it are clamped to 0.99.  (The CUDA frame equals the oracle's bit for bit at levels 0, 1 and 2.)"""
    import oracle

    vtx, masks, _, f = frame("axis")
    u = edge_scene.camera("axis")
    rows = (520 // 16, 520 // 16 + 1)
    cov = oracle.cov3d(vtx)
    kept, clamped = [], []
    for op in edge_scene.OPACITY_EDGES:
        i = int(np.nonzero(masks["opacity"] & (vtx[:, 7] == np.float32(op)))[0][0])
        a = f["attr"][i]
        px, py = (int(c) for c in a["uv"])
        assert (a["uv"] == np.float32([px, py])).all() and py == 520 and f["tiles"][i] > 0, (op, a["uv"])
        al = min(np.float32(0.99), np.float32(a["conic_opacity"][3]) * np.float32(oracle.exp_shared(-0.0)))
        clamped.append(bool(np.float32(a["conic_opacity"][3]) > al))
        off = vtx.copy()
        off[i, 7] = 0.0
        oracle.set_exp_mode(1)
        try:
            ref = oracle.render_frame(off, cov, u, rows)["rgba"]
        finally:
            oracle.set_exp_mode(0)
        kept.append(bool((ref[py, px] != f["rgba"][py, px]).any()))  # the oracle returns the whole frame's rows
    print(list(zip(edge_scene.OPACITY_EDGES, kept, clamped)))
    assert kept == [False, False, True, True, True, True, True, True]
    assert clamped == [False] * 6 + [False, True]  # 0.99f * 1 == 0.99f: min() returns it either way
    assert al == np.float32(0.99)


@pytest.mark.parametrize("cam", edge_scene.BACKWARD_CAMERAS)
def test_duplicate_gradients_are_distinguishable(cam):
    """The two copies of a duplicate sit at one depth; the one later in index order is blended behind the other, so for the
    pairs of edge_scene.backward_case their float64 gradients differ by more than the backward tests' per-Gaussian tolerance,
    and a swapped order fails that check.  At the axis camera this holds for every such pair (99; smallest 1.86 x the
    tolerance); at rotated_odd for 128 of 131 (smallest 0.50 x), so there at least 95 % are required."""
    from test_gpu_backward_regimes import RTOL, _atol

    b = edge_scene.backward_case(cam)
    ref, pairs = b["ref"]["grad"], b["pairs"]
    atol = _atol(ref, b["keep"], slice(0, 60))
    ra, rb = ref[pairs[:, 0]], ref[pairs[:, 1]]
    sep = np.linalg.norm(ra - rb, axis=1) / (RTOL * np.maximum(np.linalg.norm(ra, axis=1), np.linalg.norm(rb, axis=1)) + atol)
    print(cam, "duplicate pairs checked", len(pairs), "separated", int((sep > 1).sum()), "smallest separation / tolerance",
          float(sep.min()))
    assert len(pairs) >= 50
    if cam == "axis":
        assert (sep > 1.0).all()
    else:
        assert (sep > 1.0).mean() >= 0.95
