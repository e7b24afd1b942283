#!/usr/bin/env python
"""Times the rendered feature maps (gsb_render_features, gsb_render_backward_features, DESIGN.md section 21) on bench.py's
workload and poses, on one GPU, in one process, at tile-cull level 1 with the backward state recorded:
  anchors     k_blend of the same frames (the context's render_ms) and gsb_render_backward_density of the recorded frame;
  forward     gsb_render_features after each frame, at C in --channels (default 3, 16, 32, 64);
  backward    gsb_render_backward_features with seeded image and feature-map gradients at the same C, atomic and
              deterministic.
Every call is timed alone with CUDA events on one stream after its frame.  The variants are alternated over --rounds rounds.
Prints one JSON line with the card name and its power limit.  Writes nothing.

usage: python tools/bench_features.py [--steps K] [--warmup W] [--rounds R] [--channels 3,16,32,64] [--workload NAME]"""
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
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--channels", default="3,16,32,64")
    ap.add_argument("--workload", default="garden-standin", choices=sorted(bench.WORKLOADS))
    args = ap.parse_args()
    steps, warmup = max(1, args.steps), max(1, args.warmup)
    channels = [int(c) for c in args.channels.split(",")]
    wl = bench.WORKLOADS[args.workload]
    W, H = wl["w"], wl["h"]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cams = bench.cameras(g, wl)
    vtx_dev = torch.from_numpy(bench.make_scene(g, wl)).to(dev)
    n = vtx_dev.shape[0]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    sarg = g._torch_stream_arg(stream)
    img = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    grad_img = torch.randn((H, W, 4), generator=gen, device=dev, dtype=torch.float32)
    feats = {c: torch.rand((n, c), generator=gen, device=dev, dtype=torch.float32) for c in channels}
    fmaps = {c: torch.empty((H, W, c), dtype=torch.float32, device=dev) for c in channels}
    grad_fm = {c: torch.randn((H, W, c), generator=gen, device=dev, dtype=torch.float32) for c in channels}
    grad_f = {c: torch.empty((n, c), dtype=torch.float32, device=dev) for c in channels}
    grad_vtx = torch.empty_like(vtx_dev)
    density = torch.zeros((n, 4), dtype=torch.float32, device=dev)

    ctx = g.Context(0)
    ctx.upload(vtx_dev)
    ctx.set_tile_cull(1)
    ctx.set_backward(True)

    def frame(u):
        ctx._ck(g.lib.gsb_render(ctx.h, C.byref(u), 0, g.ALL_ROWS, img.data_ptr(), 0, g.MEM_DEVICE, g.FORMAT_RGBA32F, sarg))

    peak_m = 0
    for i in range(bench.NUM_CAMERAS):  # size the arena over every pose
        frame(cams[i])
        peak_m = max(peak_m, ctx.stats().num_instances)
    ctx.reserve(int(peak_m * 1.3) + 65536)

    def timed(call, deterministic=False, stats=False):
        """Mean ms of `call` after each frame of the orbit; with stats, the frames' render_ms instead."""
        ctx.set_backward_deterministic(deterministic)
        ctx.set_timers(stats)
        times = []
        for i in range(warmup + steps):
            frame(cams[i % bench.NUM_CAMERAS])
            if stats:
                t = ctx.stats().render_ms
            else:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                call()
                e1.record(stream)
                e1.synchronize()
                t = e0.elapsed_time(e1)
            if i >= warmup:
                times.append(t)
        ctx.set_backward_deterministic(False)
        return float(np.mean(times))

    def density_backward():
        ctx._ck(g.lib.gsb_render_backward_density(ctx.h, vtx_dev.data_ptr(), grad_img.data_ptr(), 0, grad_vtx.data_ptr(), None,
                                                  density.data_ptr(), sarg))

    def forward(c):
        return lambda: ctx._ck(g.lib.gsb_render_features(ctx.h, feats[c].data_ptr(), c, fmaps[c].data_ptr(), 0, sarg))

    def backward(c):
        return lambda: ctx._ck(g.lib.gsb_render_backward_features(
            ctx.h, vtx_dev.data_ptr(), grad_img.data_ptr(), 0, None, 0, feats[c].data_ptr(), c, grad_fm[c].data_ptr(), 0,
            grad_vtx.data_ptr(), None, grad_f[c].data_ptr(), density.data_ptr(), sarg))

    rounds = []
    for _ in range(max(1, args.rounds)):  # the variants alternated, so all see the same card state
        r = {"blend_ms": timed(None, stats=True), "backward_ms": {}, "forward_ms": {}}
        for det in (False, True):
            tag = "deterministic" if det else "atomic"
            r["backward_ms"][f"{tag}_density"] = timed(density_backward, det)
            for c in channels:
                r["backward_ms"][f"{tag}_features_c{c}"] = timed(backward(c), det)
        for c in channels:
            r["forward_ms"][f"c{c}"] = timed(forward(c))
        rounds.append(r)
    ctx.close()
    mean = {"blend_ms": float(np.mean([r["blend_ms"] for r in rounds]))}
    for k in ("forward_ms", "backward_ms"):
        mean[k] = {name: float(np.mean([r[k][name] for r in rounds])) for name in rounds[0][k]}
    key = f"c{16 if 16 in channels else channels[0]}"
    print(json.dumps({
        "metric": f"features_forward_{key}_ms", "value": mean["forward_ms"][key], "unit": "ms", "higher_is_better": False,
        "steps": steps, "warmup": warmup,
        "config": {**bench.bench_config(args.workload, wl), "blend_mode": "exact", "tile_cull": 1, "channels": channels},
        "mean": mean, "rounds": rounds,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "k_blend from the context's stage timers (CUDA events); each feature and backward call timed alone with CUDA "
               "events on one stream after its recorded frame; the backward entries include the density statistics",
    }))


if __name__ == "__main__":
    main()
