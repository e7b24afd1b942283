#!/usr/bin/env python
"""Times gsb_init_from_points (DESIGN.md section 13) on three clouds:
  garden        the 5.8 M positions of bench.py's garden stand-in (uniform in its box)
  heavy_tailed  1 M points: 95 % in a 1 m cube, 5 % over a 10 km cube, 2 % of the rows in clusters of 2-40 duplicates
  planar        1 M points on a tilted 20 m x 20 m plane
(tests/init_ref.py's generators).  A call's time is CUDA events around it on torch's current stream, median (and min, max)
over --calls calls after --warmup calls.  The CPU baseline is scipy's cKDTree build + query (k = 4, workers=-1) on the same
host, median of --cpu-reps runs.  The same run checks that both give the same D: the GPU's scale column against
sqrt(max(D, 1e-7)) with D from that tree (tests/init_ref.py's d_ref: the fp32 formula over the tree's candidates, k enlarged
until no other point can be among the three smallest), word for word on every row.  Prints one JSON line per cloud, then
one with the card's name and power limit.  Writes nothing.

usage: python tools/bench_init.py [--calls K] [--warmup W] [--cpu-reps R]"""
import argparse
import json
import os
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))
import bench  # noqa: E402  (the garden stand-in)
import gs_b200 as g  # noqa: E402
import init_ref  # noqa: E402
from bench_loss import power_limit_w  # noqa: E402


def clouds():
    yield "garden", np.ascontiguousarray(bench.make_scene(g, bench.WORKLOADS["garden-standin"])[:, 0:3])
    yield "heavy_tailed", init_ref.BENCH_CLOUDS["heavy_tailed_1m"]()
    yield "planar", init_ref.BENCH_CLOUDS["planar_1m"]()


def gpu_times(ctx, xyz, rgb, calls, warmup):
    ms = []
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(warmup + calls):
        start.record()
        out = ctx.init_from_points(xyz, rgb)
        end.record()
        end.synchronize()
        if i >= warmup:
            ms.append(start.elapsed_time(end))
    return ms, out


def cpu_baseline(xyz, reps):
    """cKDTree build + query (k = 4) on all host threads: seconds per run and the last tree."""
    from scipy.spatial import cKDTree

    x64 = xyz.astype(np.float64)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        tree = cKDTree(x64)
        tree.query(x64, k=4, workers=-1)
        times.append(time.perf_counter() - t0)
    return times, tree


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-reps", type=int, default=3)
    args = ap.parse_args()
    ctx = g.Context(0)
    for name, xyz in clouds():
        n = xyz.shape[0]
        rgb = np.random.default_rng(0).uniform(0, 1, (n, 3)).astype(np.float32)
        ms, out = gpu_times(ctx, torch.from_numpy(xyz).cuda(), torch.from_numpy(rgb).cuda(), args.calls, args.warmup)
        scale = out[:, 4].cpu().numpy()
        cpu_s, tree = cpu_baseline(xyz, args.cpu_reps)
        want = init_ref.scale_from_d(init_ref.d_ref(xyz, tree=tree))
        mismatches = int((scale.view(np.uint32) != want.view(np.uint32)).sum())
        med, cpu_med = statistics.median(ms), statistics.median(cpu_s)
        print(json.dumps({"cloud": name, "n": n, "gpu_median_ms": med, "gpu_min_ms": min(ms), "gpu_max_ms": max(ms),
                          "gpu_points_per_s": n / (med * 1e-3), "ckdtree_k4_median_s": cpu_med,
                          "ckdtree_points_per_s": n / cpu_med, "speedup": cpu_med / (med * 1e-3), "cpu_threads": os.cpu_count(),
                          "rows_compared": n, "scale_mismatches": mismatches}), flush=True)
    ctx.close()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(0)}))


if __name__ == "__main__":
    main()
