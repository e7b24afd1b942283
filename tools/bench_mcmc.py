#!/usr/bin/env python
"""Times 3DGS-MCMC's scene updates on bench.py's garden stand-in (5.8 M Gaussians, 3200x1400; DESIGN.md section 16):
  noise      gsb_mcmc_noise over every row, CUDA events around each call, with its bytes from the shapes -- 100 B per row:
             params' position float4 read and written (2 x 16 B), the scene's position + opacity read and written
             (2 x 16 B), Sigma read (16 + 8 B), the record's position written (12 B) -- and the bandwidth that makes
  relocate   gsb_mcmc_relocate of 5 % of the rows onto sources drawn by opacity (mcmc_sample) from the rest, CUDA events
             around each call (it returns once the rows are written: counting pass, check, host read of the flag, writes)
  step       a whole SceneAdam step (dense Adam), render + gsb_image_loss + backward + gsb_adam_step, against the same step
             with opacity_reg = scale_reg = 0.01 and inject_noise(); a host clock around the step ending in a device
             synchronise, cycling bench.py's cameras, tile-cull level 1, timers off
medians (and min, max) over --steps calls after --warmup.  Prints one JSON line with the card name and power limit.
Writes nothing.

usage: python tools/bench_mcmc.py [--steps K] [--warmup W]"""
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
from bench_train import LR, summary  # noqa: E402

NOISE_ROW_BYTES = 2 * 16 + 2 * 16 + 16 + 8 + 12
LAMBDA = 0.2


def event_times(fn, steps, warmup):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for i in range(warmup + steps):
        start.record()
        fn(i)
        end.record()
        end.synchronize()
        if i >= warmup:
            out.append(start.elapsed_time(end))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mcmc: no CUDA device")
    wl = bench.WORKLOADS["garden-standin"]
    cams = bench.cameras(g, wl)
    vertices = torch.from_numpy(bench.make_scene(g, wl)).cuda()
    n = vertices.shape[0]
    target = torch.rand((wl["h"], wl["w"], 4), generator=torch.Generator(device="cuda").manual_seed(0), device="cuda")
    out = {"workload": "garden-standin", "n_gaussians": n, "width": wl["w"], "height": wl["h"],
           "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(0), "steps": args.steps, "warmup": args.warmup}
    ctx = g.Context(0)
    try:
        ctx.set_tile_cull(1)
        ctx.set_timers(False)
        # ---- the entries alone
        ctx.upload(vertices)
        v = vertices.clone()
        p = g.raw_parameters(v)
        m, s = torch.zeros_like(v), torch.zeros_like(v)
        ms = event_times(lambda i: ctx.mcmc_noise(p, v, 80.0, 1, i), args.steps, args.warmup)
        med = statistics.median(ms)
        nbytes = NOISE_ROW_BYTES * n
        out["noise"] = {"median_ms": med, "min_ms": min(ms), "max_ms": max(ms), "row_bytes": NOISE_ROW_BYTES, "bytes": nbytes,
                        "tb_per_s": nbytes / (med * 1e-3) / 1e12, "hbm_fraction": nbytes / (med * 1e-3) / 1e12 / HBM_TBS}
        gen = torch.Generator().manual_seed(0)
        k = n // 20
        dst = torch.randperm(n, generator=gen)[:k]
        w = v[:, 7].clone()
        w[dst.cuda()] = 0.0
        src = g.mcmc_sample(w, k, gen).to(torch.int32)
        dst = dst.to(torch.int32).cuda()
        ms = event_times(lambda i: ctx.mcmc_relocate(p, m, s, v, dst, src), args.steps, args.warmup)
        out["relocate"] = {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "k": k,
                           "sources": int(torch.unique(src).numel())}
        del p, m, s, v
        torch.cuda.empty_cache()
        # ---- whole steps
        for name, mcmc in (("step_plain", False), ("step_mcmc", True)):
            opt = g.SceneAdam(ctx, vertices, LR, selective=False)
            grad = torch.empty_like(target)
            times = []
            for i in range(args.warmup + args.steps):
                t0 = time.perf_counter()
                ctx.image_loss(opt.render(cams[i % len(cams)]), target, LAMBDA, grad_image=grad)
                if mcmc:
                    opt.step(grad, opacity_reg=0.01, scale_reg=0.01)
                    opt.inject_noise()
                else:
                    opt.step(grad)
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times.append(time.perf_counter() - t0)
            out[name] = summary(times)
            del opt
            torch.cuda.empty_cache()
    finally:
        ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
