"""The oracle (oracle/gs_oracle.c) against the reference renderer's own compute shaders, run on the CPU stage by stage.

The oracle is a restatement of the reference's shaders; every bit-exact CUDA test inherits its reading of them.  Here the
shader source itself, translated to C++ by oracle/glsl_to_cpp.py onto oracle/glsl_shim.hpp and dispatched as the
reference's Renderer.cpp records it (oracle/ref_driver.cpp, built into oracle/_ref/ by `python __graft_entry__.py build`),
is compared with the oracle bit for bit:
  - stage by stage, the same inputs into both sides: precomp_cov3d / gso_cov3d, preprocess / gso_preprocess,
    prefix_sum / gso_scan_inclusive, preprocess_sort / gso_emit_keys, hist + sort x 8 / gso_sort,
    tile_boundary / gso_tile_ranges, render / gso_blend (both exp modes);
  - whole frames at exp modes 0 and 1 on c1 at every camera of scenes.CAMERAS, the edge scene, the scale scene, the
    anti-aliasing tests' subpixel scene and both golden fixtures.
Only the arithmetic GLSL leaves to the implementation follows the oracle's choice (glsl_shim.hpp's header, DESIGN.md
"Parity with the reference's shaders"); the rest is the shaders' own code.
"""
from __future__ import annotations

import ctypes as C
import functools
import sys
from pathlib import Path

import numpy as np
import pytest

import edge_scene
import scale_scene
import scenes

GOLD_DIR = Path(__file__).parent / "golden"


@pytest.fixture(scope="module")
def ref():
    import ref_shaders

    try:
        ref_shaders.load()
    except (RuntimeError, OSError) as e:  # a missing reference build is a failure, not a skip
        pytest.fail(str(e), pytrace=False)
    return ref_shaders


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def same(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


# ------------------------------------------------------------------------------------------------------------- scenes
def _axis_640(gs):
    """edge_scene's axis pose at 640 x 360: the plane's exact depth ties need only the pose, not the frame size."""
    pos, q, fov, _, _ = edge_scene.CAMERA_POSES["axis"]
    return gs.uniforms_from_camera(pos, q, fov, 0.1, 1000.0, 640, 360)


@functools.lru_cache(maxsize=None)
def scene_vertices(scene):
    if scene == "c1":
        return scenes.c1()[1]
    if scene == "edge":
        return edge_scene.vertices()[0]
    if scene == "scale":
        return scale_scene.vertices()[0]
    if scene == "subpixel":
        from test_gpu_antialias import subpixel_scene

        return subpixel_scene()
    raise KeyError(scene)


def case(name):
    """'scene/camera' -> (vertices, uniforms)"""
    import gs_b200 as gs

    scene, cam = name.split("/")
    if scene == "golden":
        sys.path.insert(0, str(GOLD_DIR))
        from test_golden import load

        _, vtx, u = load(gs, cam)
        return vtx, u
    vtx = scene_vertices(scene)
    if cam == "axis640":
        return vtx, _axis_640(gs)
    if scene in ("c1", "subpixel"):
        return vtx, scenes.camera(cam)
    return vtx, edge_scene.camera(cam)


FRAME_CASES = ([f"c1/{c}" for c in scenes.CAMERAS] + ["edge/axis640", "edge/rotated_odd", "edge/near_plane",
               "scale/axis640", "scale/rotated_odd", "subpixel/c1", "golden/c1_small", "golden/c1_odd"])
STAGE_CASES = ["c1/c1", "c1/inside", "c1/odd_size", "c1/tiny", "c1/away", "edge/axis640", "edge/near_plane",
               "scale/rotated_odd", "subpixel/c1"]


def oracle_frame(oracle, vtx, u, mode):
    oracle.set_exp_mode(mode)
    try:
        return oracle.render_frame(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)


def check_attr(ra, rt, oa, ot, where):
    """Every field of the survivors; of the culled rows only color_radii.w and tiles, which the shader writes before
    its first early return (the rest of a culled row is whatever the buffer held)."""
    assert np.array_equal(rt, ot), where
    live = ot > 0
    for field in oa.dtype.names:
        assert same(ra[field][live], oa[field][live]), (where, field)
    assert not ra["color_radii"][~live, 3].any() and not oa["color_radii"][~live, 3].any(), where


# ------------------------------------------------------------------------------------------------------- stage by stage
@pytest.mark.parametrize("scene", ["c1", "edge", "scale", "subpixel"])
def test_cov3d(ref, oracle, scene):
    vtx = scene_vertices(scene)
    for factor in (1.0, 0.75):
        assert same(ref.cov3d(vtx, factor), oracle.cov3d(vtx, factor)), (scene, factor)


@pytest.mark.parametrize("name", STAGE_CASES)
def test_stages(ref, oracle, name):
    """Each stage fed the oracle's output of the stage before, on both sides."""
    vtx, u = case(name)
    cov = oracle.cov3d(vtx)
    of = oracle_frame(oracle, vtx, u, 0)
    ra, rt = ref.preprocess(vtx, cov, u)
    check_attr(ra, rt, of["attr"], of["tiles"], name)
    rs, rm = ref.scan(of["tiles"])
    assert np.array_equal(rs, of["scan"]) and rm == of["m"], name
    rk, rv = ref.emit_keys(of["attr"], of["scan"], of["tiles_x"], of["m"])
    assert np.array_equal(rk, of["keys_unsorted"]) and np.array_equal(rv, of["vals_unsorted"]), name
    sk, sv = ref.sort_pairs(of["keys_unsorted"], of["vals_unsorted"])
    assert np.array_equal(sk, of["keys"]) and np.array_equal(sv, of["vals"]), name
    T = of["tiles_x"] * of["tiles_y"]
    assert np.array_equal(ref.tile_ranges(of["keys"], T), of["ranges"]), name
    for mode in (0, 1):
        ref.set_exp_mode(mode)
        try:
            img = ref.blend(of["attr"], of["vals"], of["ranges"], u.width, u.height)
        finally:
            ref.set_exp_mode(0)
        want = of["rgba"] if mode == 0 else oracle_frame(oracle, vtx, u, 1)["rgba"]
        assert same(img, want), (name, mode)


def _view_depth(vtx, u):
    """p_view.z as preprocess.comp computes it (view_mat * position, one rounding per product and per sum)."""
    m = np.frombuffer(bytes(u), np.float32)[20:36].reshape(4, 4)  # view_mat[column][row]
    p = vtx[:, 0:4]
    s = m[0, 2] * p[:, 0]
    for k in (1, 2, 3):
        s = (s + m[k, 2] * p[:, k]).astype(np.float32)
    return s


def test_preprocess_early_return_writes(ref, oracle):
    """Which fields preprocess.comp writes before each early return, seen on a buffer filled with a sentinel:
      view depth <= 0.2          color_radii.w = 0 and tiles = 0 only;
      det(cov2d) <= 0            the same;
      no tile in the AABB        also conic_opacity (written before the tile count is known);
      survivor                   every field.
    The oracle zeroes culled rows instead; nothing downstream reads them (preprocess_sort skips color_radii.w == 0)."""
    rows, us = [], []
    for name in ("c1/inside", "c1/away", "edge/near_plane", "scale/rotated_odd", "c1/odd_size"):
        vtx, u = case(name)
        rows.append(vtx)
        us.append(u)
    seen = set()
    for vtx, u in zip(rows, us):
        cov = oracle.cov3d(vtx)
        sentinel = np.frombuffer(b"\xa5" * (64 * len(vtx)), oracle.ATTR_DTYPE).copy()
        ra, rt = ref.preprocess(vtx, cov, u, attr=sentinel, tiles=np.full(len(vtx), 0xA5A5A5A5, np.uint32))
        oa, ot = oracle.preprocess(vtx, cov, u)
        check_attr(ra, rt, oa, ot, "sentinel")
        culled = ot == 0
        depth_cut = _view_depth(vtx, u) <= np.float32(0.2)
        for i in np.nonzero(culled)[0]:
            written = tuple(f for f in oracle.ATTR_DTYPE.names if f != "color_radii"
                            and not same(ra[f][i], sentinel[f][i]))
            assert same(ra["color_radii"][i, :3], sentinel["color_radii"][i, :3]), i
            path = "depth" if depth_cut[i] else ("det" if written == () else "tiles")
            expected = ("conic_opacity",) if path == "tiles" else ()
            assert written == expected, (i, path, written)
            seen.add(path)
        assert not depth_cut[~culled].any()
    assert {"depth", "tiles"} <= seen, seen  # both reached; det <= 0 needs a degenerate cov2d no scene has


@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 511, 512, 513, 1000, 4097, 65535, 65536, 65537, 100_003])
def test_scan(ref, oracle, n):
    """Across workgroup (256) and pass (powers of two) boundaries, with zeros and with uint32 wraparound."""
    rng = np.random.default_rng(n)
    tiles = rng.integers(0, 40, n).astype(np.uint32) * (rng.random(n) < 0.6)
    for t in (tiles, tiles | np.uint32(0x40000000)):
        t = np.ascontiguousarray(t, np.uint32)
        rs, total = ref.scan(t)
        os_ = np.zeros(n, np.uint32)
        oracle.lib.gso_scan_inclusive.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        oracle.lib.gso_scan_inclusive.restype = C.c_uint64
        om = oracle.lib.gso_scan_inclusive(t.ctypes.data, n, os_.ctypes.data)
        assert np.array_equal(rs, os_) and total == om, n


@pytest.mark.parametrize("m", [1, 2, 255, 256, 257, 8191, 8192, 8193, 100_003])
def test_sort_random(ref, oracle, m):
    """Random 64-bit keys: across block (256) and workgroup (32 blocks) boundaries."""
    rng = np.random.default_rng(m * 7 + 1)
    keys = rng.integers(0, 2**63, size=m, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=m, dtype=np.uint64)
    vals = np.arange(m, dtype=np.uint32)
    rk, rv = ref.sort_pairs(keys, vals)
    ok, ov = oracle.sort_pairs(keys, vals)
    assert np.array_equal(rk, ok) and np.array_equal(rv, ov)


def test_sort_is_stable_on_heavy_ties(ref, oracle):
    """The reference's radix sort keeps input order among equal keys: test_gpu_sort's heavy-duplicate set (5 tiles x 3
    depths), a constant key, presorted and reversed keys.  Ties of (tile, depth) decide the blend order of the edge scene's
    plane and duplicates; test_stages and test_frame cover its own keys."""
    rng = np.random.default_rng(7)
    m = 300_000
    ties = (rng.integers(0, 5, size=m, dtype=np.uint64) << np.uint64(32)) | rng.integers(0, 3, size=m, dtype=np.uint64)
    k = 50_000
    for keys in (ties, np.full(k, 0x1234_5678_9ABC, np.uint64), np.arange(k, dtype=np.uint64) * 977,
                 (np.arange(k, dtype=np.uint64)[::-1] * 31).copy()):
        vals = np.arange(keys.size, dtype=np.uint32)
        rk, rv = ref.sort_pairs(keys, vals)
        order = np.argsort(keys, kind="stable")
        assert np.array_equal(rk, keys[order]) and np.array_equal(rv, vals[order])
        ok, ov = oracle.sort_pairs(keys, vals)
        assert np.array_equal(rk, ok) and np.array_equal(rv, ov)


def test_tile_ranges(ref, oracle):
    """Empty tiles, the first and the last tile, a single instance, one tile holding everything, and no instance."""
    oracle.lib.gso_tile_ranges.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
    oracle.lib.gso_tile_ranges.restype = None

    def oranges(keys, T):
        out = np.empty(2 * T, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint64)
        oracle.lib.gso_tile_ranges(keys.ctypes.data, keys.size, T, out.ctypes.data)
        return out.reshape(-1, 2)

    rng = np.random.default_rng(3)
    T = 1200
    tiles = np.sort(np.concatenate([[0, 0, T - 1], rng.choice(np.arange(1, T - 1), 300), [T - 1] * 5])).astype(np.uint64)
    sets = {"spread": tiles, "first_only": np.zeros(7, np.uint64), "last_only": np.full(3, T - 1, np.uint64),
            "single": np.array([517], np.uint64), "middle": np.full(2000, 600, np.uint64), "none": np.zeros(0, np.uint64)}
    for what, t in sets.items():
        keys = (t << np.uint64(32)) | rng.integers(0, 2**32, t.size, dtype=np.uint64)
        keys = np.sort(keys)
        assert np.array_equal(ref.tile_ranges(keys, T), oranges(keys, T)), what


# -------------------------------------------------------------------------------------------------------- whole frames
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", FRAME_CASES)
def test_frame(ref, oracle, name, mode):
    vtx, u = case(name)
    of = oracle_frame(oracle, vtx, u, mode)
    ref.set_exp_mode(mode)
    try:
        rf = ref.render_frame(vtx, u)
    finally:
        ref.set_exp_mode(0)
    assert rf["m"] == of["m"], name
    check_attr(rf["attr"], rf["tiles"], of["attr"], of["tiles"], name)
    for k in ("scan", "keys_unsorted", "vals_unsorted", "keys", "vals", "ranges", "rgba"):
        assert same(rf[k], of[k]), (name, mode, k)
