#!/usr/bin/env python
"""Times the depth and alpha outputs (gsb_render_depth, gsb_render_backward_depth, DESIGN.md section 20) against the
colour-only entries on bench.py's workload and poses, on one GPU, in one process:
  blend       k_blend of a plain frame (gsb_render) against a depth frame (gsb_render_depth), RGBA32F into device memory,
              from the context's own stage timers (render_ms; frame_ms for the whole frame), at tile-cull level 1 with the
              backward state recorded and at level 2 without it;
  backward    gsb_render_backward_density against gsb_render_backward_depth of the same recorded depth frame, with seeded
              upstream gradients (colour, and (D, A) for the depth entry), atomic and deterministic, timed alone with CUDA
              events after each frame.
The variants are alternated over --rounds rounds.  Prints one JSON line with the card name and its power limit.  Writes
nothing.

usage: python tools/bench_depth.py [--steps K] [--warmup W] [--rounds R] [--workload NAME]"""
import argparse
import ctypes as C
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
    sarg = g._torch_stream_arg(stream)
    img = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    da = torch.zeros((H, W, 2), dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    grad_img = torch.randn((H, W, 4), generator=gen, device=dev, dtype=torch.float32)
    grad_da = torch.randn((H, W, 2), generator=gen, device=dev, dtype=torch.float32)
    grad_vtx = torch.empty_like(vtx_dev)
    density = torch.zeros((vtx_dev.shape[0], 4), dtype=torch.float32, device=dev)

    ctx = g.Context(0)
    ctx.upload(vtx_dev)

    def frame(u, depth):
        if depth:
            ctx._ck(g.lib.gsb_render_depth(ctx.h, C.byref(u), 0, g.ALL_ROWS, img.data_ptr(), 0, g.MEM_DEVICE, g.FORMAT_RGBA32F,
                                           da.data_ptr(), 0, sarg))
        else:
            ctx._ck(g.lib.gsb_render(ctx.h, C.byref(u), 0, g.ALL_ROWS, img.data_ptr(), 0, g.MEM_DEVICE, g.FORMAT_RGBA32F, sarg))

    peak_m = 0
    for level in (1, 2):  # size the arena over every pose and level
        ctx.set_tile_cull(level)
        for i in range(bench.NUM_CAMERAS):
            frame(cams[i], False)
            peak_m = max(peak_m, ctx.stats().num_instances)
    ctx.reserve(int(peak_m * 1.3) + 65536)

    def blend_ms(level, record, depth):
        ctx.set_tile_cull(level)
        ctx.set_backward(record)
        ctx.set_timers(True)
        render, whole = [], []
        for i in range(warmup + steps):
            frame(cams[i % bench.NUM_CAMERAS], depth)
            st = ctx.stats()
            if i >= warmup:
                render.append(st.render_ms)
                whole.append(st.frame_ms)
        return float(np.mean(render)), float(np.mean(whole))

    def backward_ms(depth, deterministic):
        ctx.set_tile_cull(1)
        ctx.set_backward(True)
        ctx.set_timers(False)
        ctx.set_backward_deterministic(deterministic)
        times = []
        for i in range(warmup + steps):
            frame(cams[i % bench.NUM_CAMERAS], True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            if depth:
                ctx._ck(g.lib.gsb_render_backward_depth(ctx.h, vtx_dev.data_ptr(), grad_img.data_ptr(), 0, grad_da.data_ptr(), 0,
                                                        grad_vtx.data_ptr(), None, density.data_ptr(), sarg))
            else:
                ctx._ck(g.lib.gsb_render_backward_density(ctx.h, vtx_dev.data_ptr(), grad_img.data_ptr(), 0, grad_vtx.data_ptr(),
                                                          None, density.data_ptr(), sarg))
            e1.record(stream)
            e1.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
        ctx.set_backward_deterministic(False)
        return float(np.mean(times))

    blend_cases = {"level1_recorded": (1, True), "level2_plain": (2, False)}
    rounds = []
    for _ in range(max(1, args.rounds)):  # the variants alternated, so all see the same card state
        r = {"blend_ms": {}, "frame_ms": {}, "backward_ms": {}}
        for name, (level, record) in blend_cases.items():
            for depth in (False, True):
                key = f"{name}_{'depth' if depth else 'plain'}"
                r["blend_ms"][key], r["frame_ms"][key] = blend_ms(level, record, depth)
        for det in (False, True):
            for depth in (False, True):
                key = f"{'deterministic' if det else 'atomic'}_{'depth' if depth else 'density'}"
                r["backward_ms"][key] = backward_ms(depth, det)
        rounds.append(r)
    ctx.close()
    mean = {k: {n: float(np.mean([r[k][n] for r in rounds])) for n in rounds[0][k]} for k in rounds[0]}
    print(json.dumps({
        "metric": "level1_recorded_depth_blend_ms", "value": mean["blend_ms"]["level1_recorded_depth"], "unit": "ms",
        "higher_is_better": False, "steps": steps, "warmup": warmup,
        "config": {**bench.bench_config(args.workload, wl), "blend_mode": "exact", "output": "RGBA32F + (D, A) float2"},
        "mean": mean, "rounds": rounds,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "k_blend and the whole frame from the context's stage timers (CUDA events); each backward call timed alone "
               "with CUDA events on one stream after its recorded depth frame",
    }))


if __name__ == "__main__":
    main()
