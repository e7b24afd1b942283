#!/usr/bin/env python
"""Times the spherical-harmonics degree (gsb_set_sh_degree, DESIGN.md section 25) at degrees 0-3 on bench.py's workload and
poses, on one GPU at tile-cull level 1.  Per degree, device-event times of (a) k_project alone (the context's own stage
timer, GSB timers on) with its algorithmic bytes 40 N + gather(d) N_v + 72 N_v (gather = 16, 48, 112, 192 B of fp32 SH per
survivor) over the time, against the H100 SXM's 3.35 TB/s; (b) the frame (BGRA8, K back-to-back frames over the orbit);
(c) gsb_render_backward of a recorded whole frame with a seeded upstream gradient; (d) one SceneAdam step (render excluded:
gsb_render_backward + gsb_adam_step), dense and selective.  The degrees are alternated over --rounds rounds in one process.
Prints one JSON line with the card name and its power limit.  Writes nothing.

usage: python tools/bench_sh_degree.py [--steps K] [--warmup W] [--rounds R] [--workload NAME]"""
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
import bench  # noqa: E402  (workloads, scene generator, camera orbit)
import gs_b200 as g  # noqa: E402
from bench_backward import power_limit_w  # noqa: E402

DEGREES = (0, 1, 2, 3)
GATHER_BYTES = {0: 16, 1: 48, 2: 112, 3: 192}  # whole float4 words holding the live coefficients
HBM_BYTES_PER_S = 3.35e12
LR = [1.6e-3, 5e-3, 5e-2, 1e-3, 2.5e-3, 1.25e-4]


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
    n = vtx_dev.shape[0]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    fb = torch.zeros((H, W, 4), dtype=torch.uint8, device=dev)
    grad_img = torch.randn((H, W, 4), generator=torch.Generator(device=dev).manual_seed(0), device=dev, dtype=torch.float32)
    grad_vtx = torch.empty_like(vtx_dev)

    ctx = g.Context(0)
    ctx.set_tile_cull(1)
    ctx.upload(vtx_dev)
    peak_m, nv = 0, []
    for i in range(bench.NUM_CAMERAS):  # size the arena; N_v per pose (the degree does not change the survivors)
        ctx.render_into(cams[i], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
        st = ctx.stats()
        peak_m = max(peak_m, st.num_instances)
        nv.append(int(st.num_visible))
    ctx.reserve(int(peak_m * 1.3) + 65536)

    def project(d):  # timers on: k_project between the context's own events, and its bytes over that time
        ctx.set_sh_degree(d)
        ctx.set_timers(True)
        ctx.set_backward(False)
        t, rate = [], []
        for i in range(warmup + steps):
            c = i % bench.NUM_CAMERAS
            ctx.render_into(cams[c], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            if i >= warmup:
                ms = ctx.stats().preprocess_ms
                t.append(ms)
                rate.append((40 * n + (GATHER_BYTES[d] + 72) * nv[c]) / (ms * 1e-3))
        return float(np.mean(t)), float(np.mean(rate))

    def frame_ms(d):
        ctx.set_sh_degree(d)
        ctx.set_timers(False)
        ctx.set_backward(False)
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

    def backward_ms(d):
        ctx.set_sh_degree(d)
        ctx.set_timers(False)
        ctx.set_backward(True)
        times = []
        for i in range(warmup + steps):
            ctx.render_into(cams[i % bench.NUM_CAMERAS], fb.data_ptr(), g.FORMAT_BGRA8, stream=stream)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ctx.render_backward(vtx_dev.data_ptr(), grad_img.data_ptr(), grad_vtx.data_ptr(), stream=stream)
            e1.record(stream)
            e1.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
        ctx.set_backward(False)
        return float(np.mean(times))

    rounds = []
    for _ in range(max(1, args.rounds)):  # the degrees alternated, so all see the same card state
        r = {"project_ms": {}, "project_tb_s": {}, "project_hbm_fraction": {}, "frame_ms": {}, "backward_ms": {}}
        for d in DEGREES:
            ms, rate = project(d)
            r["project_ms"][d], r["project_tb_s"][d] = ms, rate / 1e12
            r["project_hbm_fraction"][d] = rate / HBM_BYTES_PER_S
            r["frame_ms"][d] = frame_ms(d)
            r["backward_ms"][d] = backward_ms(d)
        rounds.append(r)
    ctx.close()

    # one SceneAdam step (gsb_render_backward + gsb_adam_step) per degree, dense and selective, on a context of its own
    adam = {}
    tctx = g.Context(0)
    tctx.set_tile_cull(1)
    for selective in (False, True):
        opt = g.SceneAdam(tctx, vtx_dev, LR, selective=selective)
        key = "selective" if selective else "dense"
        adam[key] = {}
        for _ in range(max(1, args.rounds)):
            for d in DEGREES:
                opt.sh_degree = d
                times = []
                for i in range(warmup + steps):
                    opt.render(cams[i % bench.NUM_CAMERAS])
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    opt.step(grad_img)
                    e1.record(stream)
                    e1.synchronize()
                    if i >= warmup:
                        times.append(e0.elapsed_time(e1))
                adam[key].setdefault(d, []).append(float(np.mean(times)))
        adam[key] = {d: float(np.mean(v)) for d, v in adam[key].items()}
        del opt
    tctx.close()

    mean = {k: {d: float(np.mean([r[k][d] for r in rounds])) for d in DEGREES} for k in rounds[0]}
    print(json.dumps({
        "metric": "sh_degree0_frame_ms", "value": mean["frame_ms"][0], "unit": "ms", "higher_is_better": False,
        "steps": steps, "warmup": warmup,
        "config": {**bench.bench_config(args.workload, wl), "tile_cull": 1, "blend_mode": "exact", "output": "BGRA8"},
        "mean": mean, "adam_step_ms": adam, "rounds": rounds, "num_visible": nv, "n": n,
        "gpu": torch.cuda.get_device_properties(dev).name, "power_limit_w": power_limit_w(0),
        "how": "CUDA events on one stream; frames back to back; the backward and the Adam step timed alone after each "
               "recorded frame; k_project from the context's stage timers in separate timed frames",
    }))


if __name__ == "__main__":
    main()
