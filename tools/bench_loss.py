#!/usr/bin/env python
"""Times gsb_image_loss (DESIGN.md section 11) at the frame sizes of bench.py's workloads against the same loss written in
float32 torch (F.conv2d forward, autograd backward), on seeded uniform images: device-event times of the fused call with the
gradient, the fused call without it (metrics only) and the torch loss with its gradient.  Prints one JSON line with the
card name and power limit, the bytes each fused call moves (from the shapes) and the bandwidth it reaches against the
3.35 TB/s data-sheet bound, and the largest deviation between the two implementations.  Writes nothing.

usage: python tools/bench_loss.py [--steps K] [--warmup W] [--lambda L]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))
import bench  # noqa: E402  (workload frame sizes)
import gs_b200 as g  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet
SIZES = ["garden-standin", "bicycle-standin", "truck-standin"]


def power_limit_w(index):
    """The board power limit in W as nvidia-smi reports it (a read-only query), or None."""
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip())
    except (OSError, ValueError, subprocess.TimeoutExpired):
        return None


def torch_loss(x, y, lam, win):
    """The Inria l1_loss / ssim pair on the RGB channels of (H, W, 4) float32 tensors, in float32 torch."""
    X = x[..., :3].permute(2, 0, 1)[None]
    Y = y[..., :3].permute(2, 0, 1)[None]

    def blur(t):
        return F.conv2d(t, win, padding=5, groups=3)

    mu_x, mu_y = blur(X), blur(Y)
    sxx = blur(X * X) - mu_x * mu_x
    syy = blur(Y * Y) - mu_y * mu_y
    sxy = blur(X * Y) - mu_x * mu_y
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    ssim = (((2 * mu_x * mu_y + c1) * (2 * sxy + c2)) / ((mu_x * mu_x + mu_y * mu_y + c1) * (sxx + syy + c2))).mean()
    return (1 - lam) * (X - Y).abs().mean() + lam * (1 - ssim)


def timed(fn, steps, warmup, stream):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--lambda", dest="lam", type=float, default=0.2)
    args = ap.parse_args()
    steps, warmup, lam = max(1, args.steps), max(1, args.warmup), args.lam
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    ctx = g.Context(0)
    i = np.arange(11, dtype=np.float64)
    g1 = np.exp(-(i - 5) ** 2 / 4.5)
    g1 /= g1.sum()
    win = torch.from_numpy(np.outer(g1, g1)).to(dev, torch.float32)[None, None].expand(3, 1, 11, 11).contiguous()
    rows = []
    for name in SIZES:
        W, H = bench.WORKLOADS[name]["w"], bench.WORKLOADS[name]["h"]
        gen = torch.Generator(device=dev).manual_seed(0)
        x = torch.rand((H, W, 4), generator=gen, device=dev)
        y = torch.rand((H, W, 4), generator=gen, device=dev)
        grad = torch.empty_like(x)
        xt = x.clone().requires_grad_()

        def fused():
            ctx.image_loss(x, y, lam, grad)

        def fused_metrics():
            ctx.image_loss(x, y, lam)

        def reference():
            (gt,) = torch.autograd.grad(torch_loss(xt, y, lam, win), xt)
            return gt

        t_fused = timed(fused, steps, warmup, stream)
        t_metrics = timed(fused_metrics, steps, warmup, stream)
        t_torch = timed(reference, steps, warmup, stream)
        res = ctx.image_loss(x, y, lam, grad)
        ref_loss = torch_loss(xt, y, lam, win)
        (ref_grad,) = torch.autograd.grad(ref_loss, xt)
        torch.cuda.synchronize()
        px = W * H
        # the fused call's traffic by design: forward reads image and target (16 B each) and, with a gradient, writes the
        # 9 gather terms (36 B); the backward reads them, the image and the target, and writes the gradient (16 B).  Halo
        # re-reads (hits in L2) are not counted.
        bytes_grad, bytes_metrics = px * (32 + 36 + 36 + 32 + 16), px * 32
        rows.append({
            "workload": name, "width": W, "height": H,
            "fused_ms": t_fused, "fused_metrics_only_ms": t_metrics, "torch_fp32_ms": t_torch,
            "speedup": t_torch / t_fused,
            "fused_bytes": bytes_grad, "fused_metrics_only_bytes": bytes_metrics,
            "fused_tbs": bytes_grad / (t_fused * 1e-3) / 1e12, "fused_metrics_only_tbs": bytes_metrics / (t_metrics * 1e-3) / 1e12,
            "fused_share_of_hbm": bytes_grad / (t_fused * 1e-3) / 1e12 / HBM_TBS,
            "fused_metrics_only_share_of_hbm": bytes_metrics / (t_metrics * 1e-3) / 1e12 / HBM_TBS,
            "max_loss_dev": abs(float(res[0]) - float(ref_loss.detach())),
            "max_grad_dev_rel": float((grad[..., :3] - ref_grad[..., :3]).abs().max() / ref_grad[..., :3].abs().max()),
        })
    ctx.close()
    print(json.dumps({
        "metric": "image_loss_ms", "value": rows[0]["fused_ms"], "unit": "ms", "higher_is_better": False, "steps": steps,
        "warmup": warmup, "lambda_dssim": lam, "sizes": rows,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0), "hbm_datasheet_tbs": HBM_TBS,
        "how": "CUDA events on torch's current stream, K back-to-back calls per arm after W warm-up calls; torch arm = float32 "
               "loss (F.conv2d, groups=3) and torch.autograd.grad of it, on the same (H, W, 4) tensors",
    }))


if __name__ == "__main__":
    main()
