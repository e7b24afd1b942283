#!/usr/bin/env python
"""Times the fisheye camera gradient (gsb_render_backward_fisheye, DESIGN.md section 22) on bench.py's workload and poses,
on one GPU at tile-cull level 1, atomic and deterministic.  Two fisheyes over the pinhole's frame: fisheye_k0 (fx, fy the
pinhole's focal, k = 0, max_theta 175 deg) and fisheye180 (an equidistant 180 degree lens, focal W / pi).  Device-event
times of one backward call after each recorded frame:
  vertices        gsb_render_backward of the fisheye frame (the vertex-only path);
  camera_lens     gsb_render_backward_fisheye with grad_vertices, grad_uniforms and grad_lens;
  camera_only     the same without grad_vertices (a frozen scene: pose and lens only);
  pinhole_camera  gsb_render_backward_camera of the pinhole frame, as an anchor.
Prints one JSON line with the card name and its power limit.  Writes nothing.

usage: python tools/bench_fisheye_camera.py [--steps K] [--warmup W] [--rounds R] [--workload NAME]"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402  (workloads, scene generator, camera orbit)
import gs_b200 as g  # noqa: E402
from bench_backward import power_limit_w  # noqa: E402
from bench_fisheye import lenses  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workload", default="garden-standin", choices=sorted(bench.WORKLOADS))
    args = ap.parse_args()
    steps, warmup = max(1, args.steps), max(1, args.warmup)
    wl = bench.WORKLOADS[args.workload]
    W, H = wl["w"], wl["h"]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cams = bench.cameras(g, wl)
    lens = lenses(cams[0])
    vtx = torch.from_numpy(bench.make_scene(g, wl)).to(dev)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    s = g._torch_stream_arg(stream)
    fb = torch.zeros((H, W, 4), dtype=torch.uint8, device=dev)
    gi = torch.randn((H, W, 4), generator=torch.Generator(device=dev).manual_seed(0), device=dev, dtype=torch.float32)
    gv = torch.empty_like(vtx)
    gu = torch.empty(40, dtype=torch.float32, device=dev)
    gl = torch.empty(10, dtype=torch.float32, device=dev)

    ctx = g.Context(0)
    ctx.set_tile_cull(1)
    ctx.upload(vtx)
    peak_m = 0
    for cam in lens.values():  # size the arena over every camera and pose
        ctx.set_camera_model(cam)
        for i in range(bench.NUM_CAMERAS):
            ctx.render_into(cams[i], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            peak_m = max(peak_m, ctx.stats().num_instances)
    ctx.reserve(int(peak_m * 1.3) + 65536)
    ctx.set_timers(False)
    ctx.set_backward(True)

    calls = {
        "vertices": lambda: ctx._backward(vtx.data_ptr(), gi.data_ptr(), gv.data_ptr(), s),
        "camera_lens": lambda: ctx._backward_fisheye(vtx.data_ptr(), gi.data_ptr(), gv.data_ptr(), s, grad_uniforms_ptr=gu.data_ptr(),
                                                     grad_lens_ptr=gl.data_ptr()),
        "camera_only": lambda: ctx._backward_fisheye(vtx.data_ptr(), gi.data_ptr(), None, s, grad_uniforms_ptr=gu.data_ptr(),
                                                     grad_lens_ptr=gl.data_ptr()),
        "pinhole_camera": lambda: ctx._backward(vtx.data_ptr(), gi.data_ptr(), gv.data_ptr(), s, grad_uniforms_ptr=gu.data_ptr()),
    }

    def timed(cam, call):
        ctx.set_camera_model(cam)
        times = []
        for i in range(warmup + steps):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            call()
            e1.record(stream)
            e1.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
        return float(np.mean(times))

    rounds = []
    for _ in range(max(1, args.rounds)):  # the variants alternated, so all see the same card state
        r = {}
        for det in (False, True):
            ctx.set_backward_deterministic(det)
            mode = "deterministic" if det else "atomic"
            r[mode] = {"pinhole_camera": timed(None, calls["pinhole_camera"])}
            for lname in ("fisheye_k0", "fisheye180"):
                for cname in ("vertices", "camera_lens", "camera_only"):
                    r[mode][f"{lname}/{cname}"] = timed(lens[lname], calls[cname])
        rounds.append(r)
    ctx.close()
    mean = {m: {k: float(np.mean([r[m][k] for r in rounds])) for k in rounds[0][m]} for m in rounds[0]}
    print(json.dumps({
        "metric": "fisheye180_camera_lens_backward_ms", "value": mean["atomic"]["fisheye180/camera_lens"], "unit": "ms",
        "higher_is_better": False, "steps": steps, "warmup": warmup,
        "config": {**bench.bench_config(args.workload, wl), "tile_cull": 1, "blend_mode": "exact"},
        "mean": mean, "rounds": rounds,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "CUDA events on one stream around one backward call after each recorded frame",
    }))


if __name__ == "__main__":
    main()
