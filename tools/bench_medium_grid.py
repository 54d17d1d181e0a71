"""Measure the heterogeneous medium (RenderConfig.medium_grid / EZRT_PARAM_MEDIUM_GRID, DESIGN.md section 20).

For bench.py's C3 and C4 views at 1920x1080, 16 spp, 2 and 8 bounces, in the light sampling mode, over a box holding the scene's
bounds (albedo 0.8, g = 0.3): plain mode 4; the homogeneous medium at vertical optical depth 0.5 and 2; a constant grid of ones at
the same depths (delta and ratio tracking's cost over the analytic flight); scenes.smoke_grid at 128^3 and 256^3 with sigma_t set so
that the mean vertical depth (sigma_t * mean density * box height) is 0.5 and 2.  Per case: ms over warm renders (median of --reps),
Mrays/s, primary / bounce / shadow rays and the per-kernel time of one render (torch.profiler).  Then the cost of the GRID kernels
alone: a box that no segment meets, rendered homogeneous and with the grid, alternated with plain mode 4 --reps times in this one
process.  Prints one JSON
line with the card's name and power limit, read before and after.

    python tools/bench_medium_grid.py [--workloads c3,c4] [--reps 3] [--depths 0.5,2] [--bounces 2,8] [--plumes 128,256]
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
    ap.add_argument("--plumes", default="128,256")
    args = ap.parse_args()
    bench.quiet_stdout()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_medium_grid.py: no CUDA device -- the product has no CPU path")
    torch.cuda.set_device(0)
    from ezrt_b200 import api, scenes
    run_args = argparse.Namespace(traverse="accel", pipeline="wavefront", frames_per_batch=0, spp_per_step=16, image="1920x1080", scaling="auto")
    out = {"metric": "heterogeneous medium: 16 spp renders of bench.py's views at 1920x1080", "gpu": gpu_card(0), "workloads": {}}
    depths = [float(x) for x in args.depths.split(",") if x]
    plumes = {n: scenes.smoke_grid(n, 0) for n in [int(x) for x in args.plumes.split(",") if x]}
    ones = np.ones((2, 2, 2), np.float32)
    for name in [x for x in args.workloads.split(",") if x]:
        wl = bench.build_workload(name, device_cache=True)
        W, H = 1920, 1080
        runner = bench.Runner(run_args, wl, 0, 1, 0, W, H)
        sc = runner.scene
        try:
            p = sc.tris[:, :9].reshape(-1, 3)
            lo, hi = p.min(0).astype(np.float64), p.max(0).astype(np.float64)
            height = float(hi[1] - lo[1])
            box = dict(albedo=(0.8, 0.8, 0.8), g=0.3, box_min=tuple(lo), box_max=tuple(hi))
            rows = {}
            for nb in [int(x) for x in args.bounces.split(",") if x]:
                base = {**runner.cfg(0, 16).__dict__, "mode": api.MODE_DISNEY_LIGHTS, "max_bounce": nb}
                plain = api.RenderConfig(**base)
                homo = api.RenderConfig(**{**base, "medium": True})
                grid = api.RenderConfig(**{**base, "medium": True, "medium_grid": True})
                cases = {"mode4": (plain, None, None)}
                for depth in depths:
                    cases["homogeneous depth=%g" % depth] = (homo, depth / height, None)
                    cases["constant grid depth=%g" % depth] = (grid, depth / height, ones)
                    for n, g in plumes.items():
                        cases["plume %d^3 depth=%g" % (n, depth)] = (grid, depth / (height * float(g.mean())), g)
                for k, (cfg, sigma_t, g) in cases.items():
                    sc.set_medium(sigma_t=sigma_t, **box) if sigma_t else sc.set_medium(None)
                    sc.set_medium_grid(g)
                    timed(torch, runner, cfg)
                    ms = sorted(timed(torch, runner, cfg) for _ in range(args.reps))
                    c = sc.counters()
                    rows["bounces=%d %s" % (nb, k)] = {"ms": [round(x, 3) for x in ms], "mrays_per_s": round(c.rays / (ms[len(ms) // 2] * 1e3), 1),
                                                       "primary_rays": int(c.primary_rays), "bounce_rays": int(c.bounce_rays),
                                                       "shadow_rays": int(c.shadow_rays), "kernel_ms": kernels(torch, runner, cfg)}
                # the MEDIUM and the MEDIUM + GRID kernels alone: a box no segment meets, rendered homogeneous and with the grid, alternated
                # with plain mode 4 (grid - homogeneous is the GRID kernels' own cost)
                far = hi + 10.0 * (hi - lo) + 1.0
                sc.set_medium(sigma_t=1.0, albedo=(0.8, 0.8, 0.8), g=0.3, box_min=tuple(far), box_max=tuple(far + 1.0))
                sc.set_medium_grid(ones)
                timed(torch, runner, homo)
                timed(torch, runner, grid)
                alt = {"mode4": [], "untouched box, homogeneous": [], "untouched box, grid": []}
                for _ in range(args.reps):
                    alt["mode4"].append(round(timed(torch, runner, plain), 3))
                    alt["untouched box, homogeneous"].append(round(timed(torch, runner, homo), 3))
                    alt["untouched box, grid"].append(round(timed(torch, runner, grid), 3))
                rows["bounces=%d alternated" % nb] = alt
                sc.set_medium(None)
                sc.set_medium_grid(None)
            out["workloads"][name] = {"image": [W, H], "box": [list(lo), list(hi)], "cases": rows}
        finally:
            runner.close()
    out["gpu_after"] = gpu_card(0)
    bench.emit(out)


if __name__ == "__main__":
    main()
