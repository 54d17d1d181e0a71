"""Measure the thin-lens camera (RenderConfig.lens_radius / EZRT_PARAM_THIN_LENS, DESIGN.md section 13).

For bench.py's C3, C4 and C2 views at their own image sizes, 16 spp: the pinhole (flag off) and the lens at R = 1e-4, 0.02 and 0.1
of the scene's extent (its bounding-box diagonal), focused at the distance of the scene's centre.  Per case:
  - ms (CUDA events, a warm render, median of --reps) and Mrays/s, deferred rays;
  - per-kernel time of one render through torch.profiler (as tools/bench_camera.py);
  - camera-pass node visits per camera ray: a max_bounce = 0 render with profile = 2.
The tiny radius gives what the unfused bounce 0 (k_generate<true> + the per-ray bounce kernel) costs against the fused pinhole
camera pass.  Prints one JSON line with the card's name and power limit.

    python tools/bench_lens.py [--workloads c3,c4,c2] [--reps 3] [--radii 1e-4,0.02,0.1]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (the workloads and the per-workload runner of the benchmark)
from bench_adaptive import gpu_card  # noqa: E402
from bench_camera import kernel_base  # noqa: E402

RADII = (1e-4, 0.02, 0.1)


def timed(torch, runner, cfg):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(runner.stream)
    runner.scene.render_device(cfg, runner.d_fb, runner.stream)
    ev1.record(runner.stream)
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1)


def kernels(torch, runner, cfg):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        runner.scene.render_device(cfg, runner.d_fb, runner.stream)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA" or not e.name:
            continue
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        out[kernel_base(e.name)] = round(out.get(kernel_base(e.name), 0.0) + us / 1e3, 3)
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c4,c2")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--radii", default=",".join("%g" % r for r in RADII), help="lens radii as fractions of the scene's extent")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lens.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image=None, scaling="auto")
    out = {"metric": "thin-lens camera: 16 spp renders of bench.py's views", "gpu": gpu_card(0), "workloads": {}}
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H, _ = bench.image_for(run_args, wl, 1)
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            base = runner.cfg(0, 16).__dict__
            p = runner.scene.tris[:, :9].reshape(-1, 3)
            lo, hi = p.min(0), p.max(0)
            extent = float(np.linalg.norm(hi - lo))
            c2 = np.asarray(base["camera_rotate"], np.float64)[8:11]   # the focus distance is a depth along -column 2
            focus = float(np.dot((lo + hi) / 2 - np.asarray(base["eye"], np.float64), -c2 / np.linalg.norm(c2)))
            cases = {"pinhole": api.RenderConfig(**base)}
            for r in [float(x) for x in args.radii.split(",") if x]:
                cases["R=%g" % r] = api.RenderConfig(**{**base, "lens_radius": r * extent, "focus_distance": focus})
            rows = {}
            for k, cfg in cases.items():
                timed(torch, runner, cfg)   # warm: scratch sized, modules loaded
                ms = sorted(timed(torch, runner, cfg) for _ in range(args.reps))
                c = runner.scene.counters()
                kt = kernels(torch, runner, cfg)
                cam = api.RenderConfig(**{**cfg.__dict__, "max_bounce": 0, "profile": 2})
                runner.scene.render_device(cam, runner.d_fb, runner.stream)
                torch.cuda.synchronize()
                cc = runner.scene.counters()
                rows[k] = {"ms": [round(x, 3) for x in ms], "mrays_per_s": round(c.rays / (ms[len(ms) // 2] * 1e3), 1),
                           "rays": int(c.rays), "deferred_rays": int(c.deferred_rays), "kernel_ms": kt,
                           "camera_node_visits_per_ray": round(cc.node_visits / max(1, cc.primary_rays), 2),
                           "camera_deferred_rays": int(cc.deferred_rays)}
            out["workloads"][name] = {"image": [W, H], "extent": round(extent, 4), "focus_distance": round(focus, 4), "cases": rows}
        finally:
            runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
