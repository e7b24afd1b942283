#!/usr/bin/env python
"""Second half of the reference-harness patch kit (patches/reference_offscreen.patch, SURVEY 8f row 3).

On a Vulkan-capable GPU, the patched reference prints one JSON line and writes a float32 RGBA dump:

    GS_BENCH_FRAMES=200 GS_BENCH_WARMUP=20 GS_BENCH_CAMERA="0,0,5,1,0,0,0,45" GS_BENCH_DUMP=ref.f32 \
        ./vulkan_splatting_viewer -w 3200 -h 1400 --no-gui -i scene.ply > ref.json

This script renders the same .ply / camera / size through libgsb200 (C ABI, GSB_MODE_EXACT, instance culling off so that
`instances` is comparable) and reports: per-channel L-infinity of the two float images (north_star tolerance 1e-4),
the two `instances` counts, and frames/s of both (the >= 2x target of BASELINE.json).  Needs a GPU; nothing here reads
/root/reference.

usage: tools/compare_reference_dump.py scene.ply ref.json ref.f32
"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "3dgs.cpp_b200" / "python"))


def main():
    ply, ref_json, ref_dump = sys.argv[1:4]
    import gs_b200 as g

    ref = json.loads(Path(ref_json).read_text().strip().splitlines()[-1])
    W, H = int(ref["width"]), int(ref["height"])
    cam = [float(x) for x in (sys.argv[4] if len(sys.argv) > 4 else "0,0,0,1,0,0,0,45").split(",")]
    cam += [45.0] * (8 - len(cam))
    img_ref = np.fromfile(ref_dump, np.float32).reshape(H, W, 4)

    vtx = g.activate_records(g.load_ply(ply))
    ctx = g.Context(0)
    ctx.set_mode(g.MODE_EXACT)
    ctx.set_tile_cull(False)  # M then equals the reference's `instances`
    ctx.upload(vtx)
    # the reference's Renderer::camera defaults: nearPlane 0.1, farPlane 1000 (Renderer.h:78-84)
    u = g.uniforms_from_camera(cam[0:3], cam[3:7], cam[7], 0.1, 1000.0, W, H)
    img = ctx.render(u, g.FORMAT_RGBA32F)
    st = ctx.stats()
    linf = float(np.abs(img[..., :3] - img_ref[..., :3]).max())
    ctx.set_tile_cull(True)
    ctx.set_timers(False)
    import time
    for _ in range(20):
        ctx.render(u, g.FORMAT_RGBA32F)
    t0 = time.perf_counter()
    n = int(ref.get("frames", 200))
    for _ in range(n):
        ctx.render(u, g.FORMAT_RGBA32F)
    fps = n / (time.perf_counter() - t0)
    out = {"linf_rgb": linf, "within_1e-4": linf <= 1e-4, "alpha_all_one": bool((img_ref[..., 3] == 1.0).all()),
           "instances_b200": int(st.num_instances), "instances_reference": ref.get("instances_last"),
           "fps_b200_blocking_render": fps, "fps_reference_gpu_stages": ref.get("fps_gpu_stages"),
           "fps_reference_wall": ref.get("fps_wall"),
           "speedup_vs_reference_gpu_stages": fps / ref["fps_gpu_stages"] if ref.get("fps_gpu_stages") else None}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
