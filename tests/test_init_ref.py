"""CPU side of gsb_init_from_points: the cKDTree reference of D (tests/init_ref.py) equals the all-pairs fp32 brute force
bit for bit on every small cloud; ply_records is the exact inverse of the PLY loader's column layout; load_points_ply reads
the point-cloud PLY of Inria's storePly bit for bit and refuses every other format."""
import numpy as np
import pytest

import init_ref
from init_ref import SMALL_CLOUDS


@pytest.mark.parametrize("name", list(SMALL_CLOUDS))
def test_reference_equals_brute_force(name):
    xyz = SMALL_CLOUDS[name]()
    ref, brute = init_ref.d_ref(xyz), init_ref.d_brute(xyz)
    assert np.array_equal(ref.view(np.uint32), brute.view(np.uint32))
    s = init_ref.scale_from_d(ref)
    assert s.dtype == np.float32 and bool((s >= np.sqrt(np.float32(1e-7))).all())


def test_reference_covers_ties_and_duplicates():
    """The premise check has to enlarge k: inside the 40-point cluster every candidate of k = 16 and 32 is at distance 0."""
    xyz = init_ref.duplicates(500, sizes=(40,), seed=1)
    d = init_ref.d_ref(xyz)
    assert int((d == 0).sum()) == 40
    lat = init_ref.d_ref(init_ref.lattice(6))
    assert bool((lat == 1.0).all())  # even a corner point has three neighbours at distance 1


def test_reference_small_n():
    assert init_ref.d_ref(init_ref.uniform(1)).tolist() == [0.0]
    two = init_ref.uniform(2, 3)
    d = init_ref.sq_dist(two[0], two[1])
    assert init_ref.d_ref(two).tolist() == [d, d]


def _params_from_ply(rec):
    """Raw parameters in the record's column layout from 62-float PLY records, by SURVEY Appendix A0: sh[0..2] = f_dc and
    sh[3 j + c] = f_rest[15 c + j - 1]; column 3 = 1."""
    p = np.empty((rec.shape[0], 60), np.float32)
    p[:, 0:3] = rec[:, 0:3]
    p[:, 3] = 1.0
    p[:, 4:7] = rec[:, 55:58]
    p[:, 7] = rec[:, 54]
    p[:, 8:12] = rec[:, 58:62]
    p[:, 12:15] = rec[:, 6:9]
    for j in range(1, 16):
        for c in range(3):
            p[:, 12 + 3 * j + c] = rec[:, 9 + 15 * c + j - 1]
    return p


def test_ply_records_inverts_the_loader_layout(gs):
    rec = gs.synth_records(5, 4000)
    params = _params_from_ply(rec)
    out = gs.ply_records(params)
    want = rec.copy()
    want[:, 3:6] = 0.0
    assert out.dtype == np.float32 and out.shape == (4000, 62)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32))
    # the host loader's activation reads the same values from both
    assert np.array_equal(gs.activate_records(out).view(np.uint32), gs.activate_records(rec).view(np.uint32))
    import torch

    assert np.array_equal(gs.ply_records(torch.from_numpy(params)).view(np.uint32), out.view(np.uint32))


def _store_ply(path, xyz, rgb, coord="f4", normals=True):
    """The layout of Inria's storePly: x, y, z, nx, ny, nz, red, green, blue, binary little-endian."""
    fields = [("x", coord), ("y", coord), ("z", coord)]
    if normals:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    dt = np.dtype([(k, "<" + t.lstrip("<")) for k, t in fields])
    a = np.zeros(xyz.shape[0], dt)
    for k, name in enumerate("xyz"):
        a[name] = xyz[:, k]
    for k, name in enumerate(("red", "green", "blue")):
        a[name] = rgb[:, k]
    if normals:
        a["nx"] = 0.25
    ptype = {"f4": "float", "f8": "double"}[coord]
    names = {"f4": "float", "f8": "double", "u1": "uchar"}
    head = "ply\nformat binary_little_endian 1.0\ncomment storePly layout\n" + f"element vertex {xyz.shape[0]}\n"
    head += "".join(f"property {names[t.lstrip('<')] if k not in 'xyz' else ptype} {k}\n" for k, t in fields)
    head += "end_header\n"
    path.write_bytes(head.encode() + a.tobytes())


@pytest.mark.parametrize("coord", ["f4", "f8"], ids=["float", "double"])
def test_load_points_ply_reads_store_ply(gs, tmp_path, coord):
    rng = np.random.default_rng(0)
    xyz = rng.normal(0, 3, (1000, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (1000, 3)).astype(np.uint8)
    path = tmp_path / "points3D.ply"
    _store_ply(path, xyz, rgb, coord)
    got_xyz, got_rgb = gs.load_points_ply(path)
    assert got_xyz.dtype == np.float32 and got_rgb.dtype == np.float32
    assert np.array_equal(got_xyz.view(np.uint32), xyz.view(np.uint32))
    want_rgb = rgb.astype(np.float32) / np.float32(255)
    assert np.array_equal(got_rgb.view(np.uint32), want_rgb.view(np.uint32))
    _store_ply(path, xyz, rgb, coord, normals=False)
    assert np.array_equal(gs.load_points_ply(path)[0].view(np.uint32), xyz.view(np.uint32))


def _header(body_lines, fmt="binary_little_endian", n=2):
    return ("ply\nformat " + fmt + " 1.0\n" + f"element vertex {n}\n" + "".join(l + "\n" for l in body_lines) +
            "end_header\n").encode()


GOOD = ["property float x", "property float y", "property float z", "property uchar red", "property uchar green",
        "property uchar blue"]


def test_load_points_ply_refuses_other_formats(gs, tmp_path):
    path = tmp_path / "p.ply"
    rec = bytes(15 * 2)
    path.write_bytes(_header(GOOD) + rec)
    assert gs.load_points_ply(path)[0].shape == (2, 3)  # the good layout itself
    bad = {
        "ascii": _header(GOOD, fmt="ascii") + b"0 0 0 0 0 0\n0 0 0 0 0 0\n",
        "big-endian": _header(GOOD, fmt="binary_big_endian") + rec,
        "list": _header(GOOD + ["property list uchar int vertex_indices"]) + rec,
        "face element": _header(GOOD) .replace(b"end_header", b"element face 0\nproperty list uchar int vertex_indices\nend_header") + rec,
        "missing red": _header([l for l in GOOD if "red" not in l]) + rec,
        "missing z": _header([l for l in GOOD if " z" not in l]) + rec,
        "int coordinate": _header([l.replace("float x", "int x") for l in GOOD]) + rec,
        "float colour": _header([l.replace("uchar red", "float red") for l in GOOD]) + rec,
        "truncated": _header(GOOD) + rec[:-1],
        "not a ply": b"hello\n",
    }
    for what, data in bad.items():
        path.write_bytes(data)
        with pytest.raises(ValueError):
            gs.load_points_ply(path)
        print("refused:", what)
