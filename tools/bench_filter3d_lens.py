#!/usr/bin/env python
"""Times gsb_filter3d_variance_lens, the 3D smoothing filter from cameras with their own lenses, on bench.py's garden stand-in
(5.8 M Gaussians, 3200x1400; DESIGN.md section 24), against gsb_filter3d_variance on the same cameras: k = 8, 64 and 512
orbit cameras (tools/bench_filter3d.py's), each as
  pinhole    the existing entry (no lenses)
  lens-pin   the new entry with every camera PINHOLE (its words equal the existing entry's here, which is checked)
  phone      the new entry through an OpenCV phone lens at the pinhole's focal
  fish180    the new entry through a 180 deg fisheye whose rim touches the frame's shorter edge
alternated call by call, a host clock around each call (it returns once the variances are written).  Medians (and min,
max) over --steps calls after --warmup, with the (Gaussian, camera) pairs per second.  Prints one JSON line with the card
name and power limit.  Writes nothing.

usage: python tools/bench_filter3d_lens.py [--steps K] [--warmup W]"""
import argparse
import json
import math
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))
sys.path.insert(0, str(ROOT / "tools"))
import bench  # noqa: E402  (the workload)
import gs_b200 as g  # noqa: E402
from bench_filter3d import orbit, stats  # noqa: E402
from bench_loss import power_limit_w  # noqa: E402

PHONE = (-0.12, 0.03, 0.0008, -0.0006)


def lenses(u):
    fx = u.width / (2.0 * float(u.tan_fovx))
    cx, cy = u.width / 2.0 - 0.5, u.height / 2.0 - 0.5
    rim = math.pi / 2
    return {"lens-pin": g.CameraModel(), "phone": g.opencv_camera(fx, fx, cx, cy, PHONE),
            "fish180": g.fisheye_camera(min(u.width, u.height) / 2.0 / rim, min(u.width, u.height) / 2.0 / rim, cx, cy,
                                        (0.0, 0.0, 0.0, 0.0), rim)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    wl = bench.WORKLOADS["garden-standin"]
    ctx = g.Context(0)
    v = torch.from_numpy(bench.make_scene(g, wl)).cuda()
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(0), "n": v.shape[0]}
    for k in (8, 64, 512):
        cams = orbit(wl, k)
        models = lenses(cams[0])
        runs = {"pinhole": lambda: ctx.filter3d_variance(v, cams)}
        for name, m in models.items():
            runs[name] = (lambda m=m: ctx.filter3d_variance(v, cams, m))
        assert torch.equal(runs["pinhole"]().view(torch.int32), runs["lens-pin"]().view(torch.int32))
        ms = {name: [] for name in runs}
        for i in range(args.warmup + args.steps):
            for name, fn in runs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                if i >= args.warmup:
                    ms[name].append((time.perf_counter() - t0) * 1e3)
        res = {}
        for name, t in ms.items():
            s = stats(t)
            s["pairs_per_s"] = v.shape[0] * k / (s["median_ms"] * 1e-3)
            res[name] = s
        out[f"k{k}"] = res
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
