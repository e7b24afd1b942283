#!/usr/bin/env python
"""Times Mip-Splatting's 3D smoothing filter on bench.py's garden stand-in (5.8 M Gaussians, 3200x1400; DESIGN.md
section 18), and runs the zoom-in experiment:
  variance   gsb_filter3d_variance at k = 8, 64 and 512 orbit cameras, a host clock around each call (it returns once the
             variances are written), with the (Gaussian, camera) pairs per second
  adam       the plain and the filtered dense and selective Adam step (gsb_adam_step vs gsb_adam_step_filter3d), alternated
             call by call, CUDA events around each; bytes from the shapes: 4 x 240 B read (params, moments, gradient),
             3 x 240 B written (params, moments), 240 B of records and 232 B of scene words written per updated row, + 4 B
             of variance for the filtered step (+ 16 B of survivor record per row, selective)
  zoom       the same fine-texture synthetic target (c1's cloud at a third of its scales) trained from the same start at
             160x120 in the anti-aliased mode, with and without the filter, then rendered at 640x480: PSNR against the
             640x480 target at the training poses
medians (and min, max) over --steps calls after --warmup.  Prints one JSON line with the card name and power limit.
Writes nothing.

usage: python tools/bench_filter3d.py [--steps K] [--warmup W] [--zoom-steps Z]"""
import argparse
import json
import math
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
from bench_train import LR, summary  # noqa: E402

ROW_BYTES = 4 * 240 + 3 * 240 + 240 + 232
SELECTIVE_ROW_BYTES = 16


def orbit(wl, k):
    """k cameras on a full orbit around the scene centre at bench.py's distance, each looking at it."""
    cams = []
    for i in range(k):
        a = 2 * math.pi * i / k
        d = wl["cam"][2]
        pos = (d * math.sin(a), wl["cam"][1], d * math.cos(a))
        cams.append(g.uniforms_from_camera(pos, (math.cos(a / 2), 0.0, math.sin(a / 2), 0.0), wl["fov"], 0.1, 1000.0,
                                           wl["w"], wl["h"]))
    return cams


def stats(ms):
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms)}


def bench_variance(ctx, v, wl, steps, warmup):
    out = {}
    for k in (8, 64, 512):
        cams = orbit(wl, k)
        ms = []
        for i in range(warmup + steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.filter3d_variance(v, cams)
            if i >= warmup:
                ms.append((time.perf_counter() - t0) * 1e3)
        s = stats(ms)
        s["pairs_per_s"] = v.shape[0] * k / (s["median_ms"] * 1e-3)
        out[f"k{k}"] = s
    return out


def bench_adam(ctx, vertices, cams, var, steps, warmup):
    """Plain vs filtered, dense and selective, alternated call by call on the same arrays (the values drift; the work does
    not depend on them)."""
    n = vertices.shape[0]
    p = g.raw_parameters(vertices)
    m, s = torch.zeros_like(vertices), torch.zeros_like(vertices)
    grad = torch.randn(vertices.shape, generator=torch.Generator(device="cuda").manual_seed(0), device="cuda") * 1e-6
    v = vertices.clone()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {}
    for selective in (False, True):
        times = {"plain": [], "filtered": []}
        nv = n
        for i in range(warmup + steps):
            for name, variance in (("plain", None), ("filtered", var)):
                if selective:
                    ctx.set_backward(True)
                    ctx.render(cams[i % len(cams)])
                    nv = ctx.stats().num_visible
                cfg = g.adam_config(LR, step=i + 1, selective=selective)
                start.record()
                ctx.adam_step(p, m, s, grad, v, cfg, variance=variance)
                end.record()
                end.synchronize()
                if i >= warmup:
                    times[name].append(start.elapsed_time(end))
        mode = "selective" if selective else "dense"
        for name, ms in times.items():
            rows = nv if selective else n
            nbytes = rows * (ROW_BYTES + (4 if name == "filtered" else 0) + (SELECTIVE_ROW_BYTES if selective else 0))
            st = stats(ms)
            st.update({"rows": rows, "bytes": nbytes, "tb_per_s": nbytes / (st["median_ms"] * 1e-3) / 1e12,
                       "hbm_fraction": nbytes / (st["median_ms"] * 1e-3) / 1e12 / HBM_TBS})
            out[f"{mode}_{name}"] = st
    return out


def zoom_experiment(zoom_steps):
    """PSNR at 640x480 of a scene trained at 160x120, with and without the 3D filter (both in the anti-aliased mode)."""
    rec = g.synth_records(42, 10_000)
    target = torch.from_numpy(g.activate_records(rec)).cuda()
    target[:, 4:7] /= 3.0
    poses = [([0, 0, 5], [1, 0, 0, 0]), ([0.6, 0.1, 5.2], [0.99863, 0, 0.05234, 0]), ([-0.5, -0.3, 4.8], [0.99905, -0.04362, 0, 0]),
             ([0.3, 0.4, 5.1], [0.99966, 0.02618, 0.0, 0.0])]
    low = [g.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 160, 120) for p, q in poses]
    high = [g.uniforms_from_camera(p, q, 45.0, 0.1, 1000.0, 640, 480) for p, q in poses]
    out = {"zoom_steps": zoom_steps}
    for name, filtered in (("without_filter", False), ("with_filter", True)):
        ctx = g.Context(0)
        try:
            ctx.set_antialiased(True)
            ctx.set_backward(True)
            with torch.no_grad():
                t_low = [g.render_torch(ctx, target, u).clone() for u in low]
                t_high = [g.render_torch(ctx, target, u).clone() for u in high]
            start = target[::2].clone()
            start[:, 4:7] *= 2.0
            opt = g.SceneAdam(ctx, start, [1e-3, 5e-3, 5e-2, 1e-3, 1e-2, 5e-4], selective=False,
                              filter_cameras=low if filtered else None)
            grad = torch.empty((120, 160, 4), dtype=torch.float32, device="cuda")
            for it in range(zoom_steps):
                k = it % len(low)
                ctx.image_loss(opt.render(low[k]), t_low[k], 0.2, grad_image=grad)
                opt.step(grad)
                if filtered and it % 100 == 99:
                    opt.update_filter_3d()
            out[name] = {"psnr_160x120": statistics.mean(g.image_metrics(ctx, opt.render(u), t)["psnr"] for u, t in zip(low, t_low)),
                         "psnr_640x480": statistics.mean(g.image_metrics(ctx, opt.render(u), t)["psnr"] for u, t in zip(high, t_high))}
        finally:
            ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--zoom-steps", type=int, default=1500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_filter3d: no CUDA device")
    wl = bench.WORKLOADS["garden-standin"]
    vertices = torch.from_numpy(bench.make_scene(g, wl)).cuda()
    out = {"workload": "garden-standin", "n_gaussians": vertices.shape[0], "width": wl["w"], "height": wl["h"],
           "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(0), "steps": args.steps, "warmup": args.warmup}
    ctx = g.Context(0)
    try:
        ctx.set_tile_cull(1)
        ctx.set_timers(False)
        ctx.upload(vertices)
        out["variance"] = bench_variance(ctx, vertices, wl, args.steps, args.warmup)
        var = ctx.filter3d_variance(vertices, bench.cameras(g, wl))
        out["adam"] = bench_adam(ctx, vertices, bench.cameras(g, wl), var, args.steps, args.warmup)
    finally:
        ctx.close()
    torch.cuda.empty_cache()
    out["zoom"] = zoom_experiment(args.zoom_steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
