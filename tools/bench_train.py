#!/usr/bin/env python
"""Times one whole training step on bench.py's garden stand-in (5.8 M Gaussians, 3200x1400; DESIGN.md section 12):
  torch     render_torch + image_loss_torch + autograd through torch's activations + torch.optim.Adam(fused=True)
  dense     SceneAdam(selective=False): render, gsb_image_loss, gsb_render_backward + gsb_adam_step
  selective SceneAdam(selective=True)
each from the same raw parameters against a seeded uniform target, cycling bench.py's cameras; a step's time is a host clock
around the step ending in a device synchronise, median (and min, max) over --steps steps after --warmup steps.  Also times
gsb_adam_step alone with CUDA events (dense: back to back; selective: after a fresh frame each time) with its bytes from the
shapes -- 2152 B per updated row: params and both moments read and written (3 x 480 B), grad_vertices read and vertices
written (2 x 240 B), the scene words stored (232 B) -- and its bandwidth against the 3.35 TB/s data-sheet bound.  Prints one
JSON line with the card name and power limit.  Writes nothing.

usage: python tools/bench_train.py [--steps K] [--warmup W]"""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402  (the workload and its cameras)
import gs_b200 as g  # noqa: E402
from bench_loss import HBM_TBS, power_limit_w  # noqa: E402

LR = [1.6e-4, 5e-3, 5e-2, 1e-3, 2.5e-3, 1.25e-4]  # Inria's position, scaling, opacity, rotation, f_dc, f_rest (f_dc / 20)
GROUP_COLS = [slice(0, 3), slice(4, 7), slice(7, 8), slice(8, 12), slice(12, 15), slice(15, 60)]
ROW_BYTES = 3 * 2 * 240 + 2 * 240 + 232
LAMBDA = 0.2


def timed_steps(step, cams, steps, warmup):
    """Per-step seconds of `step(u)` over steps, after warmup, each ended by a device synchronise."""
    times = []
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        step(cams[i % len(cams)])
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(time.perf_counter() - t0)
    return times


def summary(times):
    ms = [t * 1e3 for t in times]
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms)}


def torch_path(ctx, vertices, target, cams, steps, warmup):
    raw = g.raw_parameters(vertices)
    leaves = [raw[:, c].clone().contiguous().requires_grad_() for c in GROUP_COLS]
    col3 = vertices[:, 3:4]
    opt = torch.optim.Adam([{"params": [t], "lr": lr} for t, lr in zip(leaves, LR)], eps=1e-15, fused=True)

    def step(u):
        opt.zero_grad()
        pos, ls, lo, q, dc, rest = leaves
        v = torch.cat([pos, col3, ls.exp(), torch.sigmoid(lo), q / q.norm(dim=1, keepdim=True), dc, rest], 1)
        g.image_loss_torch(ctx, g.render_torch(ctx, v, u), target, LAMBDA).backward()
        opt.step()

    return timed_steps(step, cams, steps, warmup)


def scene_adam_path(ctx, vertices, target, cams, steps, warmup, selective):
    opt = g.SceneAdam(ctx, vertices, LR, selective=selective)
    grad = torch.empty_like(target)

    def step(u):
        ctx.image_loss(opt.render(u), target, LAMBDA, grad_image=grad)
        opt.step(grad)

    times = timed_steps(step, cams, steps, warmup)
    # the step alone
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    alone, visible = [], []
    for i in range(warmup + steps):
        opt.render(cams[i % len(cams)])
        if selective:
            visible.append(ctx.stats().num_visible)
        opt.steps += 1
        cfg = g.adam_config(LR, eps=1e-15, step=opt.steps, selective=selective)
        start.record()
        ctx.adam_step(opt.params, opt.exp_avg, opt.exp_avg_sq, opt.grad, opt.vertices, cfg)
        end.record()
        end.synchronize()
        if i >= warmup:
            alone.append(start.elapsed_time(end))
    rows = statistics.median(visible[warmup:]) if selective else vertices.shape[0]
    ms = statistics.median(alone)
    nbytes = ROW_BYTES * rows
    return times, {"median_ms": ms, "min_ms": min(alone), "max_ms": max(alone), "rows": int(rows), "bytes": int(nbytes),
                   "tb_per_s": nbytes / (ms * 1e-3) / 1e12, "hbm_fraction": nbytes / (ms * 1e-3) / 1e12 / HBM_TBS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train: no CUDA device")
    wl = bench.WORKLOADS["garden-standin"]
    cams = bench.cameras(g, wl)
    vertices = torch.from_numpy(bench.make_scene(g, wl)).cuda()
    target = torch.rand((wl["h"], wl["w"], 4), generator=torch.Generator(device="cuda").manual_seed(0), device="cuda")
    out = {"workload": "garden-standin", "n_gaussians": wl["n"], "width": wl["w"], "height": wl["h"],
           "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(0), "steps": args.steps,
           "warmup": args.warmup, "row_bytes": ROW_BYTES}
    ctx = g.Context(0)
    try:
        ctx.set_tile_cull(1)
        ctx.set_timers(False)
        out["torch_step"] = summary(torch_path(ctx, vertices, target, cams, args.steps, args.warmup))
        torch.cuda.empty_cache()
        for name, sel in (("dense", False), ("selective", True)):
            times, alone = scene_adam_path(ctx, vertices, target, cams, args.steps, args.warmup, sel)
            out[f"{name}_step"] = summary(times)
            out[f"{name}_adam_step_alone"] = alone
            torch.cuda.empty_cache()
    finally:
        ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
