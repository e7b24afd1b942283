#!/usr/bin/env python
"""Times the reverse mode (DESIGN.md section 10) on bench.py's workloads: on one GPU at tile-cull level 1, device-event times
of (a) the plain forward, (b) the recording forward (gsb_set_backward on) and (c) gsb_render_backward of a recorded whole
frame with a seeded upstream gradient (RGBA32F layout), then gsb_render_backward_camera of such a frame (d) with both
outputs and (e) with the camera gradient only (grad_vertices = NULL), then gsb_render_backward_density with the outputs of
(d) and of (e) plus the density statistics.  Prints one JSON line with the card name and its power limit.  Writes nothing.

usage: python tools/bench_backward.py [--steps K] [--warmup W] [--workload NAME] [--mode exact|fast]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))
import bench  # noqa: E402  (workloads, scene generator, camera orbit)
import gs_b200 as g  # noqa: E402


def power_limit_w(index):
    """The board power limit in W as nvidia-smi reports it (a read-only query), or None."""
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip())
    except (OSError, ValueError, subprocess.TimeoutExpired):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workload", default="garden-standin", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--mode", default="exact", choices=["exact", "fast"])
    args = ap.parse_args()
    steps, warmup = max(1, args.steps), max(1, args.warmup)
    wl = bench.WORKLOADS[args.workload]
    W, H = wl["w"], wl["h"]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = g.Context(0)
    ctx.set_mode(g.MODE_EXACT if args.mode == "exact" else g.MODE_FAST)
    ctx.set_tile_cull(1)
    cams = bench.cameras(g, wl)
    vtx = bench.make_scene(g, wl)
    ctx.upload(vtx)
    vtx_dev = torch.from_numpy(vtx).to(dev)
    del vtx
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    fb = torch.zeros((H, W, 4), dtype=torch.uint8, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    grad_img = torch.randn((H, W, 4), generator=gen, device=dev, dtype=torch.float32)
    grad_vtx = torch.empty_like(vtx_dev)
    peak_m = 0
    for i in range(bench.NUM_CAMERAS):  # size the instance arena (regrow path) like bench.py
        ctx.render_into(cams[i], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
        peak_m = max(peak_m, ctx.stats().num_instances)
    ctx.reserve(int(peak_m * 1.3) + 65536)
    ctx.set_timers(False)

    def forward_ms(record):
        ctx.set_backward(record)
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

    plain = forward_ms(False)
    recording = forward_ms(True)

    def backward_ms(grad_vertices_ptr, grad_uniforms_ptr=None, density_ptr=None):
        times = []
        for i in range(warmup + steps):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)  # a recorded whole frame
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ctx.render_backward(vtx_dev.data_ptr(), grad_img.data_ptr(), grad_vertices_ptr, stream=stream,
                                grad_uniforms_ptr=grad_uniforms_ptr, density_ptr=density_ptr)
            e1.record(stream)
            e1.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
        return times

    grad_ubo = torch.empty(40, dtype=torch.float32, device=dev)  # a whole gsb_uniforms
    back = backward_ms(grad_vtx.data_ptr())
    back_cam = backward_ms(grad_vtx.data_ptr(), grad_ubo.data_ptr())  # gsb_render_backward_camera, scene and camera
    back_cam_only = backward_ms(None, grad_ubo.data_ptr())  # a frozen scene: the camera only
    density = torch.zeros((vtx_dev.shape[0], 4), dtype=torch.float32, device=dev)  # accumulated into across the calls
    # gsb_render_backward_density with the same outputs as the two camera arms, plus the density statistics
    back_dens = backward_ms(grad_vtx.data_ptr(), grad_ubo.data_ptr(), density.data_ptr())
    back_dens_cam_only = backward_ms(None, grad_ubo.data_ptr(), density.data_ptr())
    ctx.set_backward(False)
    ctx.close()
    print(json.dumps({
        "metric": "backward_ms", "value": float(np.mean(back)), "unit": "ms", "higher_is_better": False, "steps": steps,
        "warmup": warmup, "config": {**bench.bench_config(args.workload, wl), "tile_cull": 1, "blend_mode": args.mode,
                                     "output": "BGRA8 (forward); upstream gradient RGBA32F"},
        "forward_plain_ms": plain, "forward_recording_ms": recording,
        "recording_overhead": recording / plain - 1.0 if plain > 0 else None,
        "backward_ms": float(np.mean(back)), "backward_ms_median": float(np.median(back)),
        "camera_backward_ms": float(np.mean(back_cam)), "camera_only_backward_ms": float(np.mean(back_cam_only)),
        "density_backward_ms": float(np.mean(back_dens)), "density_camera_only_backward_ms": float(np.mean(back_dens_cam_only)),
        "gpu":torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "CUDA events on one stream: K back-to-back forwards per arm; the backward timed alone after each recorded frame",
    }))


if __name__ == "__main__":
    main()
