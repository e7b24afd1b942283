"""(1) The C++ headless viewer (apps/viewer/main.cpp's flags without a window) end to end on a small PLY.
(2) Frame sharding over real GPUs: one process per GPU through gsb_create_sharded / gsb_render_sharded (skipped on a
one-GPU box; tests/test_gpu_shard.py covers the protocol on one GPU), and one process driving all GPUs through gsb_group_*
(two ranks on cuda:0 on a one-GPU box); the frame every rank ends up with must be bit-identical to the single-GPU frame."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import scenes

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def test_headless_viewer_cli(gs, oracle, tmp_path):
    exe = ROOT / "3dgs.cpp_b200" / "gs_viewer_headless"
    assert exe.exists(), "run __graft_entry__.build()"
    rec = gs.synth_records(42, 10_000)
    ply = tmp_path / "c1.ply"
    gs.write_ply(ply, rec)
    out = tmp_path / "frame.ppm"
    r = subprocess.run([str(exe), "-w", "640", "-h", "480", "--frames", "3", "--camera", "0,0,5", "--out", str(out), str(ply)],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    info = json.loads(r.stdout.strip().splitlines()[-1])
    vtx = gs.activate_records(rec)
    u = gs.uniforms_from_camera([0, 0, 5], [1, 0, 0, 0], 45.0, 0.1, 1000.0, 640, 480)
    oracle.set_exp_mode(1)
    try:
        ref = oracle.render_frame(vtx, oracle.cov3d(vtx), u)
    finally:
        oracle.set_exp_mode(0)
    assert info["gaussians"] == 10_000 and info["instances"] == ref["m"] and info["frame_ms"] > 0
    data = out.read_bytes()
    head = b"P6\n640 480\n255\n"
    assert data.startswith(head)
    rgb = np.frombuffer(data[len(head):], np.uint8).reshape(480, 640, 3)
    assert np.array_equal(rgb, oracle.pack_unorm8(ref["rgba"])[..., :3])
    assert info["load_ms"] > 0 and info["read_activate_ms"] > 0 and info["upload_ms"] > 0
    # float dump (PFM, rows bottom to top) with coarse bins on: the unquantised blend, bit for bit
    pfm = tmp_path / "frame.pfm"
    r = subprocess.run([str(exe), "-w", "640", "-h", "480", "--camera", "0,0,5", "--cull", "2", "--float-out", str(pfm), str(ply)],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    blob = pfm.read_bytes()
    head_f = b"PF\n640 480\n-1.0\n"
    assert blob.startswith(head_f)
    img = np.frombuffer(blob[len(head_f):], "<f4").reshape(480, 640, 3)[::-1]
    assert np.array_equal(img, ref["rgba"][..., :3])
    assert json.loads(r.stdout.strip().splitlines()[-1])["instances_aabb"] == ref["m"]
    # camera path: one JSON line per pose, pose 0 = the camera above, pose 1 looks from further away
    poses = tmp_path / "poses.txt"
    poses.write_text("# x y z qw qx qy qz [fov]\n0 0 5 1 0 0 0\n0 0 7 1 0 0 0 60\n")
    r = subprocess.run([str(exe), "-w", "640", "-h", "480", "--camera-path", str(poses), str(ply)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    lines = [json.loads(l) for l in r.stdout.strip().splitlines()]
    assert [l["pose"] for l in lines] == [0, 1] and lines[0]["instances"] == ref["m"]
    u2 = gs.uniforms_from_camera([0, 0, 7], [1, 0, 0, 0], 60.0, 0.1, 1000.0, 640, 480)
    assert lines[1]["instances"] == oracle.render_frame(vtx, oracle.cov3d(vtx), u2)["m"]
    # missing file: logged, non-zero exit (the reference catches at top level, main.cpp:94-105)
    r = subprocess.run([str(exe), "/nonexistent.ply"], capture_output=True, text=True)
    assert r.returncode != 0 and "File does not exist" in r.stderr


WORKER = r'''
# one process per GPU through the product's own ABI: gsb_create_sharded (NCCL bootstrap + cudaIpc windows), scene sharded by
# Gaussian index, gsb_render_sharded (peer-memory routing + peer-store blend); torch.distributed only carries the 128-byte id
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.path.join(os.environ["GS_ROOT"], "3dgs.cpp_b200", "python")); sys.path.insert(0, os.path.join(os.environ["GS_ROOT"], "tests"))
import gs_b200 as g, scenes
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("gloo")
box = [g.shard_unique_id() if rank == 0 else None]
dist.broadcast_object_list(box, src=0)
ctx = g.ShardedContext(rank, rank, world, box[0])
_, vtx, _ = scenes.c1()
first, count = g.shard_slice(vtx.shape[0], rank, world)
ctx.upload_slice(vtx[first:first + count], vtx.shape[0])
ok = True
single = g.Context(rank); single.upload(vtx)
for cam in ("odd_size", "c1", "inside", "c1"):
    u = scenes.camera(cam)
    for fmt in (g.FORMAT_RGBA32F, g.FORMAT_BGRA8):
        got = ctx.render_sharded(u, fmt)                 # every rank receives the whole frame
        ok = ok and np.array_equal(got, single.render(u, fmt))
flags = [None] * world
dist.all_gather_object(flags, bool(ok))
if rank == 0:
    print("MULTI_OK" if all(flags) else f"MULTI_MISMATCH {flags}")
ctx.close(); single.close()
dist.destroy_process_group()
'''


def _gpus():
    torch = pytest.importorskip("torch")
    return torch.cuda.device_count()


@pytest.mark.parametrize("gather", ["peer", "nccl"])
def test_two_gpu_sharded_frame_equals_single_gpu(gs, tmp_path, gather):
    if _gpus() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, GS_ROOT=str(ROOT), GSB_SHARD_GATHER=gather)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29533", str(script)], capture_output=True, text=True, timeout=300, env=env)
    assert "MULTI_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_in_process_group_over_all_gpus(gs, ctx):
    n = _gpus()
    # a group needs two ranks; on a one-GPU machine both ranks share cuda:0 (a group may list a device more than once)
    devices = list(range(min(n, 8))) if n >= 2 else [0, 0]
    _, vtx, _ = scenes.c1()
    ctx.upload(vtx)
    grp = gs.Group(devices)
    try:
        grp.upload(vtx)
        for cam in ("c1", "odd_size", "wide"):
            u = scenes.camera(cam)
            assert np.array_equal(grp.render(u, gs.FORMAT_RGBA32F), ctx.render(u, gs.FORMAT_RGBA32F)), cam
    finally:
        grp.close()
