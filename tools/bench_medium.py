"""Measure the homogeneous medium (RenderConfig.medium / EZRT_PARAM_MEDIUM, DESIGN.md section 14).

For bench.py's C3 and C4 views at 1920x1080, 16 spp, 2 and 8 bounces, in the light sampling mode: plain mode 4, and a box over the
scene's bounds with vertical optical depth 0.5 and 2 (sigma_t = depth / the box's height; albedo 0.8, g = 0.3).  Per case: ms over
warm renders (median of --reps), Mrays/s, primary / bounce / shadow rays and the per-kernel time of one render (torch.profiler).
Then the cost of the MEDIUM kernels alone: a flagged render whose box touches nothing against plain mode 4, alternated --reps times
in this one process.  Prints one JSON line with the card's name and power limit, read before and after.

    python tools/bench_medium.py [--workloads c3,c4] [--reps 3] [--depths 0.5,2] [--bounces 2,8]
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
from bench_lens import kernels, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c4")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--depths", default="0.5,2")
    ap.add_argument("--bounces", default="2,8")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_medium.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image="1920x1080", scaling="auto")
    out = {"metric": "homogeneous medium: 16 spp renders of bench.py's views at 1920x1080", "gpu": gpu_card(0), "workloads": {}}
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H = 1920, 1080
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        try:
            p = runner.scene.tris[:, :9].reshape(-1, 3)
            lo, hi = p.min(0).astype(np.float64), p.max(0).astype(np.float64)
            height = float(hi[1] - lo[1])
            rows = {}
            for nb in [int(x) for x in args.bounces.split(",") if x]:
                base = {**runner.cfg(0, 16).__dict__, "mode": api.MODE_DISNEY_LIGHTS, "max_bounce": nb}
                cases = {"mode4": (api.RenderConfig(**base), None)}
                for depth in [float(x) for x in args.depths.split(",") if x]:
                    cases["depth=%g" % depth] = (api.RenderConfig(**{**base, "medium": True}),
                                                 dict(sigma_t=depth / height, albedo=(0.8, 0.8, 0.8), g=0.3, box_min=tuple(lo), box_max=tuple(hi)))
                for k, (cfg, fog) in cases.items():
                    runner.scene.set_medium(**fog) if fog else runner.scene.set_medium(None)
                    timed(torch, runner, cfg)
                    ms = sorted(timed(torch, runner, cfg) for _ in range(args.reps))
                    c = runner.scene.counters()
                    rows["bounces=%d %s" % (nb, k)] = {"ms": [round(x, 3) for x in ms], "mrays_per_s": round(c.rays / (ms[len(ms) // 2] * 1e3), 1),
                                                       "primary_rays": int(c.primary_rays), "bounce_rays": int(c.bounce_rays),
                                                       "shadow_rays": int(c.shadow_rays), "kernel_ms": kernels(torch, runner, cfg)}
                # the MEDIUM kernels alone: a box no segment meets, alternated with plain mode 4
                far = hi + 10.0 * (hi - lo) + 1.0
                runner.scene.set_medium(sigma_t=1.0, albedo=(0.8, 0.8, 0.8), g=0.3, box_min=tuple(far), box_max=tuple(far + 1.0))
                plain, flagged = api.RenderConfig(**base), api.RenderConfig(**{**base, "medium": True})
                timed(torch, runner, flagged)
                alt = {"mode4": [], "untouched box": []}
                for _ in range(args.reps):
                    alt["mode4"].append(round(timed(torch, runner, plain), 3))
                    alt["untouched box"].append(round(timed(torch, runner, flagged), 3))
                rows["bounces=%d alternated" % nb] = alt
                runner.scene.set_medium(None)
            out["workloads"][name] = {"image": [W, H], "box": [list(lo), list(hi)], "cases": rows}
        finally:
            runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
