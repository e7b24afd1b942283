#!/usr/bin/env python
"""Times the background colour (gsb_set_background, DESIGN.md section 15) against the default black frame on bench.py's
workloads, on one GPU at tile-cull level 1, EXACT: device-event times of (a) the frame (BGRA8, K back-to-back frames over the
camera orbit), (b) gsb_render_backward of a recorded whole frame with a seeded upstream gradient, each over black and over
(0.25, 0.5, 0.75), alternated over --rounds rounds in one process, and (c) gsb_background_gradient alone.  Prints one JSON
line with the card name and its power limit.  Writes nothing.

usage: python tools/bench_background.py [--steps K] [--warmup W] [--rounds R] [--workload NAME]"""
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

BG = (0.25, 0.5, 0.75)


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
    vtx_dev = torch.from_numpy(bench.make_scene(g, wl)).to(dev)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    fb = torch.zeros((H, W, 4), dtype=torch.uint8, device=dev)
    grad_img = torch.randn((H, W, 4), generator=torch.Generator(device=dev).manual_seed(0), device=dev, dtype=torch.float32)
    grad_vtx = torch.empty_like(vtx_dev)

    ctx = g.Context(0)
    ctx.set_tile_cull(1)
    ctx.set_mode(g.MODE_EXACT)
    ctx.upload(vtx_dev)
    peak_m = 0
    for i in range(bench.NUM_CAMERAS):  # size the instance arena (regrow path) like bench.py
        ctx.render_into(cams[i], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
        peak_m = max(peak_m, ctx.stats().num_instances)
    ctx.reserve(int(peak_m * 1.3) + 65536)
    ctx.set_timers(False)

    def frame_ms(bg):
        ctx.set_background(bg)
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

    def backward_ms(bg, what="backward"):
        ctx.set_background(bg)
        ctx.set_backward(True)
        times = []
        for i in range(warmup + steps):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            if what == "backward":
                ctx.render_backward(vtx_dev.data_ptr(), grad_img.data_ptr(), grad_vtx.data_ptr(), stream=stream)
            else:
                ctx.background_gradient(grad_img, stream)
            e1.record(stream)
            e1.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
        return float(np.mean(times))

    rounds = []
    for _ in range(max(1, args.rounds)):  # default and background alternated, so both see the same card state
        rounds.append({
            "frame_ms": {"black": frame_ms(None), "background": frame_ms(BG)},
            "backward_ms": {"black": backward_ms(None), "background": backward_ms(BG)},
            "background_gradient_ms": backward_ms(BG, "gradient"),
        })
    ctx.close()
    print(json.dumps({
        "metric": "background_frame_ms", "value": float(np.mean([r["frame_ms"]["background"] for r in rounds])), "unit": "ms",
        "higher_is_better": False, "steps": steps, "warmup": warmup,
        "config": {**bench.bench_config(args.workload, wl), "tile_cull": 1, "blend_mode": "exact", "output": "BGRA8",
                   "background": BG},
        "rounds": rounds,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "CUDA events on one stream; frames back to back; the backward and gsb_background_gradient timed alone after "
               "each recorded frame",
    }))


if __name__ == "__main__":
    main()
