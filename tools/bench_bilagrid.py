#!/usr/bin/env python
"""Times the bilateral-grid colour correction (gsb_bilagrid_apply / gsb_bilagrid_backward, DESIGN.md section 17) at bench.py's
three workload frame sizes and the default 16 x 16 x 8 grid, against the same map in float32 torch (F.grid_sample, trilinear,
align_corners=True, border padding, plus the affine product; forward, and forward + autograd backward).  Device-event times
over --steps calls after --warmup, medians over --rounds rounds alternated in one process; the bytes each call moves, from the
shapes, and their share of the 3.35 TB/s HBM3 data-sheet bound.  The image is seeded noise whose luma covers all z-cells (the
most z-levels per warp the backward can meet).  Prints one JSON line with the card name and its power limit.  Writes nothing.

usage: python tools/bench_bilagrid.py [--steps K] [--warmup W] [--rounds R]"""
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
sys.path.insert(0, str(ROOT / "tests"))
import bench  # noqa: E402  (workload frame sizes)
import bilagrid_ref  # noqa: E402  (the torch path)
import gs_b200 as g  # noqa: E402
from bench_backward import power_limit_w  # noqa: E402

WORKLOADS = ["garden-standin", "bicycle-standin", "truck-standin"]
SHAPE = (16, 16, 8)  # X, Y, L
HBM_TBS = 3.35


def blocks(w, h, shape):
    """The backward's block count: cells of the frame along each axis, cut into 32 x 32 pixel blocks."""
    X, Y, _ = shape
    n = []
    for size, nodes, step in ((w, X, 32), (h, Y, 32)):
        i = (np.arange(size, dtype=np.float32) + np.float32(0.5)) / np.float32(size) * np.float32(nodes - 1)
        cell = np.minimum(np.floor(i), nodes - 2).astype(np.int64)
        longest = np.bincount(cell, minlength=nodes - 1).max()
        n.append((nodes - 1) * -(-longest // step))
    return int(n[0] * n[1])


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    steps, warmup = max(1, args.steps), max(1, args.warmup)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = g.Context(0)
    X, Y, L = SHAPE
    grid_words = 12 * L * Y * X
    results = {}
    for name in WORKLOADS:
        W, H = bench.WORKLOADS[name]["w"], bench.WORKLOADS[name]["h"]
        img = torch.from_numpy(bilagrid_ref.random_image(W, H, seed=0, lo=-0.1, hi=1.1)).to(dev)
        grid = torch.from_numpy(bilagrid_ref.random_grid(SHAPE, 0.1, seed=1).astype(np.float32)).to(dev)
        go = torch.randn((H, W, 4), generator=torch.Generator(device=dev).manual_seed(0), device=dev)
        out, gi, gg = torch.empty_like(img), torch.empty_like(img), torch.empty_like(grid)
        ti, tg = img.clone().requires_grad_(), grid.clone().requires_grad_()

        def torch_fwd():
            with torch.no_grad():
                bilagrid_ref.torch_path(img, grid)

        def torch_fwd_bwd():
            ti.grad = tg.grad = None
            bilagrid_ref.torch_path(ti, tg).backward(go)

        def ours_fwd():
            ctx.bilagrid_apply(img, grid, out)

        def ours_bwd():
            ctx.bilagrid_backward(img, grid, go, gi, gg)

        def ours_fwd_bwd():
            ours_fwd()
            ours_bwd()

        rounds = []
        for _ in range(max(1, args.rounds)):
            rounds.append({"apply_ms": timed(ours_fwd, steps, warmup), "backward_ms": timed(ours_bwd, steps, warmup),
                           "fused_pair_ms": timed(ours_fwd_bwd, steps, warmup),
                           "torch_forward_ms": timed(torch_fwd, steps, warmup),
                           "torch_forward_backward_ms": timed(torch_fwd_bwd, steps, warmup)})
        med = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
        px = W * H
        nb = blocks(W, H, SHAPE)
        # apply: image in, out; each block stages its 4 L 12 grid words.  backward: image and grad_out in, grad_image out, the
        # staged words, a partial row of 48 L fp64 per block written and read back, the grid gradient written.
        bytes_apply = 32 * px + nb * 48 * L * 4
        bytes_backward = 48 * px + nb * 48 * L * 4 + 2 * nb * 48 * L * 8 + grid_words * 4
        results[name] = {
            "width": W, "height": H, **med,
            "speedup_pair_vs_torch": med["torch_forward_backward_ms"] / med["fused_pair_ms"],
            "bytes_apply": bytes_apply, "bytes_backward": bytes_backward,
            "apply_share_of_hbm": bytes_apply / (med["apply_ms"] * 1e-3) / (HBM_TBS * 1e12),
            "backward_share_of_hbm": bytes_backward / (med["backward_ms"] * 1e-3) / (HBM_TBS * 1e12),
            "rounds": rounds,
        }
    ctx.close()
    garden = results["garden-standin"]
    print(json.dumps({
        "metric": "bilagrid_pair_ms", "value": garden["fused_pair_ms"], "unit": "ms", "higher_is_better": False,
        "steps": steps, "warmup": warmup, "grid": {"x": X, "y": Y, "l": L}, "results": results,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "CUDA events on torch's current stream around back-to-back calls; medians over rounds; bytes from the shapes",
    }))


if __name__ == "__main__":
    main()
