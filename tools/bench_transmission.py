"""Measure the materials' transmission (RenderConfig.transmission in the light sampling mode, DESIGN.md section 12).

It reports:
  - S-1M's blob grid with every other blob glass (roughness 0.05 and 0.3, IOR 1.5) at 1920 x 1080, 16 and 64 spp, max_bounce 2 and 8:
    ms, Mrays/s, rays by kind, and the four kernel classes' times (a separate profile = 1 render)
  - the cost of the flag on a scene without glass: bench.py's C3 scene in mode 4 with and without the flag, alternated
and the card's name and power limit.  Prints one JSON line.  bench.py itself is unchanged.

    python tools/bench_transmission.py [--spps 16,64] [--bounces 2,8] [--reps 3]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads of the benchmark)
from bench_adaptive import gpu_card  # noqa: E402

W, H = 1920, 1080


def timed(torch, sc, cfg, fb, stream, warm=True):
    if warm:   # the first call at a new batch shape sizes the scratch; the first light sampling call builds the light table
        sc.render_device(cfg, fb, stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    sc.render_device(cfg, fb, stream)
    ev1.record(stream)
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spps", default="16,64")
    ap.add_argument("--bounces", default="2,8")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_transmission.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api
    from tests import transmission_scenes as ts
    stream = torch.cuda.current_stream()
    fb = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    out = {"metric": "transmission: glass S-1M and the flag's cost on C3", "gpu": gpu_card(0), "image": [W, H]}

    tris, nodes, eye, cam = ts.grid_glass(15, 13, 4)
    sc = api.Scene(tris, nodes)
    rows = {}
    try:
        for mb in [int(x) for x in args.bounces.split(",") if x]:
            for spp in [int(x) for x in args.spps.split(",") if x]:
                cfg = api.RenderConfig(width=W, height=H, spp=spp, max_bounce=mb, mode=api.MODE_DISNEY_LIGHTS, eye=tuple(eye),
                                       camera_rotate=tuple(cam), env_color=(0.2, 0.25, 0.3), transmission=True)
                ms = timed(torch, sc, cfg, fb, stream)
                c = sc.counters()
                cfg.profile = 1
                sc.render_device(cfg, fb, stream)
                torch.cuda.synchronize()
                kt = sc.kernel_times()
                rows["bounces %d, %d spp" % (mb, spp)] = {
                    "ms": ms, "mrays_per_s": c.rays / (ms * 1e3), "rays": {"primary": int(c.primary_rays), "bounce": int(c.bounce_rays),
                                                                          "shadow": int(c.shadow_rays)},
                    "kernel_ms_profiled": {k: v[0] for k, v in kt.items()}}
    finally:
        sc.close()
    out["s1m_glass"] = rows

    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image=None, scaling="auto")
    wl = bench.build_workload("c3", device_cache=True)
    w, h, _ = bench.image_for(run_args, wl, 1)
    runner = bench.Runner(run_args, wl, 0, 1, 0, w, h)
    try:
        base = runner.cfg(0, 16).__dict__
        arms = {"mode4": api.RenderConfig(**{**base, "mode": api.MODE_DISNEY_LIGHTS}),
                "mode4_flag": api.RenderConfig(**{**base, "mode": api.MODE_DISNEY_LIGHTS, "transmission": True})}
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, cfg in arms.items():
                times[k].append(timed(torch, runner.scene, cfg, runner.d_fb, runner.stream))
        out["c3_flag_cost"] = {"image": [w, h], "spp": 16, "ms": times}
    finally:
        runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
