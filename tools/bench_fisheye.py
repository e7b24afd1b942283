#!/usr/bin/env python
"""Times the fisheye camera model (gsb_set_camera_model, DESIGN.md section 19) against the pinhole frame on bench.py's
workload and poses, on one GPU at tile-cull level 1.  Three cameras per pose:
  pinhole     the UBO's camera (bench.py's frame);
  fisheye_k0  a fisheye whose fx and fy equal the pinhole's focal, k = 0, the pinhole's principal point (max_theta 175 deg);
  fisheye180  an equidistant 180 degree lens over the frame's width (focal W / pi), k = 0, max_theta 90 degrees.
Device-event times of (a) the frame (BGRA8, K back-to-back frames over the orbit), (b) gsb_render_backward of a recorded
whole frame with a seeded upstream gradient, (c) k_project alone (the context's own per-stage timer, GSB timers on), the
three cameras alternated over --rounds rounds in one process; N_v and M of each at every pose.  Prints one JSON line with
the card name and its power limit.  Writes nothing.

usage: python tools/bench_fisheye.py [--steps K] [--warmup W] [--rounds R] [--workload NAME]"""
import argparse
import json
import math
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


def lenses(u):
    W, H = u.width, u.height
    f = W / (2.0 * u.tan_fovx)
    return {
        "pinhole": None,
        "fisheye_k0": g.fisheye_camera(f, H / (2.0 * u.tan_fovy), (W - 1) / 2.0, (H - 1) / 2.0, max_theta=math.radians(175.0)),
        "fisheye180": g.fisheye_camera(W / math.pi, W / math.pi, (W - 1) / 2.0, (H - 1) / 2.0, max_theta=math.radians(90.0)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workload", default="garden-standin", choices=sorted(bench.WORKLOADS))
    args = ap.parse_args()
    steps, warmup = max(1, args.steps), max(1, args.warmup)
    wl = bench.WORKLOADS[args.workload]
    W, H = wl["w"], wl["h"]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cams = bench.cameras(g, wl)
    lens = lenses(cams[0])
    vtx_dev = torch.from_numpy(bench.make_scene(g, wl)).to(dev)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    fb = torch.zeros((H, W, 4), dtype=torch.uint8, device=dev)
    grad_img = torch.randn((H, W, 4), generator=torch.Generator(device=dev).manual_seed(0), device=dev, dtype=torch.float32)
    grad_vtx = torch.empty_like(vtx_dev)

    ctx = g.Context(0)
    ctx.set_tile_cull(1)
    ctx.upload(vtx_dev)
    peak_m, counts = 0, {}
    for name, cam in lens.items():  # size the arena over every camera; N_v, M and k_project's time per pose
        ctx.set_camera_model(cam)
        counts[name] = []
        for i in range(bench.NUM_CAMERAS):
            ctx.render_into(cams[i], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            st = ctx.stats()
            peak_m = max(peak_m, st.num_instances)
            counts[name].append({"num_visible": int(st.num_visible), "num_instances": int(st.num_instances)})
    ctx.reserve(int(peak_m * 1.3) + 65536)

    def project_ms(cam):  # timers on: k_project between the context's own events
        ctx.set_camera_model(cam)
        ctx.set_timers(True)
        ctx.set_backward(False)
        t = []
        for i in range(warmup + steps):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            if i >= warmup:
                t.append(ctx.stats().preprocess_ms)
        return float(np.mean(t))

    def frame_ms(cam):
        ctx.set_camera_model(cam)
        ctx.set_timers(False)
        ctx.set_backward(False)
        for i in range(warmup):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream, sync=False)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(steps):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream, sync=False)
        e1.record(stream)
        torch.cuda.synchronize()
        ctx.stats()  # raises if a frame overflowed the arena
        return e0.elapsed_time(e1) / steps

    def backward_ms(cam):
        ctx.set_camera_model(cam)
        ctx.set_timers(False)
        ctx.set_backward(True)
        times = []
        for i in range(warmup + steps):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ctx.render_backward(vtx_dev.data_ptr(), grad_img.data_ptr(), grad_vtx.data_ptr(), stream=stream)
            e1.record(stream)
            e1.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
        ctx.set_backward(False)
        return float(np.mean(times))

    rounds = []
    for _ in range(max(1, args.rounds)):  # the cameras alternated, so all see the same card state
        r = {"project_ms": {}, "frame_ms": {}, "backward_ms": {}}
        for name, cam in lens.items():
            r["project_ms"][name] = project_ms(cam)
            r["frame_ms"][name] = frame_ms(cam)
            r["backward_ms"][name] = backward_ms(cam)
        rounds.append(r)
    ctx.close()
    mean = {k: {n: float(np.mean([r[k][n] for r in rounds])) for n in lens} for k in rounds[0]}
    print(json.dumps({
        "metric": "fisheye180_frame_ms", "value": mean["frame_ms"]["fisheye180"], "unit": "ms", "higher_is_better": False,
        "steps": steps, "warmup": warmup,
        "config": {**bench.bench_config(args.workload, wl), "tile_cull": 1, "blend_mode": "exact", "output": "BGRA8"},
        "mean": mean, "rounds": rounds, "counts": counts,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "CUDA events on one stream; frames back to back; the backward timed alone after each recorded frame; "
               "k_project from the context's stage timers in separate timed frames",
    }))


if __name__ == "__main__":
    main()
